// TSDF volumes (omnidata_b200/volume.py TSDFVolume): posed depth frames fused into a dense truncated signed-distance
// grid, depth rendered back from it by raycasting, and a triangle mesh extracted by marching tetrahedra.  Definitions
// in DESIGN.md §3 "TSDF volumes" and include/omnidata_b200.h; oracle/volume_oracle.py restates them in float64 (the
// coloured raycast: oracle/color_volume_oracle.py).
//
//   tsdf_integrate_kernel  one thread per grid point, looping over up to kFramesPerLaunch frames in order; the poses
//                          travel by value in the kernel parameters, so a call needs no device copy of them
//   tsdf_raycast_kernel    one thread per pixel: box entry, fixed-step march, first + to - crossing of valid samples
//   mesh_count_kernel      one thread per point: the 7-bit mask of its edges carrying a vertex and the triangle count of
//                          the cell it is the lowest corner of; per-block totals
//   mesh_scan_kernel       one CTA: exclusive scan of the block totals, and the two grand totals
//   mesh_base_kernel       per block: each point's first vertex id (block base + local scan of the mask popcounts)
//   mesh_emit_kernel       per block: vertices of each point's edges, triangles of each point's cell
//
// The projection, the ray march and the vertex placement are written with explicit round-to-nearest fp64 operations and
// the running means with explicit fp32 operations (no contraction into FMAs), so that the oracle reproduces them
// operation by operation.  Integer scans only and no atomics: every output is bit-reproducible, and a grid point's
// result does not depend on how its frames were split into calls.  Built without fast-math.
#include <cmath>
#include <string>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kVolThreads = 256;
constexpr int kFramesPerLaunch = 16;          // 16 x 12 doubles of poses in the kernel parameters (1.5 KB of 4 KB)

struct VolGrid {
  int nx, ny, nz;
  double ox, oy, oz, voxel;
};
struct VolCam {
  double fx, fy, cx, cy;
};
struct VolPoses {                             // per frame: R row-major (9), then t (3), of camera-to-world
  double m[kFramesPerLaunch][12];
};

// Kuhn split: tetrahedron q of a cell has corners v0 = 0, v1 = e_a, v2 = e_a + e_b, v3 = (1, 1, 1) for the q-th
// permutation (a, b, c) of the axes, as 3-bit corner codes (bit 0 x, bit 1 y, bit 2 z).  kTetOdd: the permutation is
// odd, so the tetrahedron (v0, v1, v2, v3) is negatively oriented and every triangle's winding is reversed.
__constant__ unsigned char kTetCorner[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7},
                                               {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ unsigned char kTetOdd[6] = {0, 1, 1, 0, 0, 1};
// tetrahedron edges (a, b), a < b
__constant__ unsigned char kTetEdge[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
// Marching tetrahedra for a positively oriented tetrahedron, by the 4-bit mask of corners with F < 0: up to two
// triangles as edge indices, wound so that the normal points from F < 0 towards F > 0.  -1: no triangle.
__constant__ signed char kTetTri[16][2][3] = {
    {{-1, -1, -1}, {-1, -1, -1}}, {{0, 1, 2}, {-1, -1, -1}}, {{0, 4, 3}, {-1, -1, -1}}, {{1, 2, 4}, {1, 4, 3}},
    {{1, 3, 5}, {-1, -1, -1}},    {{0, 5, 2}, {0, 3, 5}},    {{0, 4, 5}, {0, 5, 1}},    {{2, 4, 5}, {-1, -1, -1}},
    {{2, 5, 4}, {-1, -1, -1}},    {{0, 1, 5}, {0, 5, 4}},    {{0, 5, 3}, {0, 2, 5}},    {{1, 5, 3}, {-1, -1, -1}},
    {{1, 3, 4}, {1, 4, 2}},       {{0, 3, 4}, {-1, -1, -1}}, {{0, 2, 1}, {-1, -1, -1}}, {{-1, -1, -1}, {-1, -1, -1}}};

ODB_DEVINL int tet_triangles(int inside) { return (inside == 0 || inside == 15) ? 0 : (__popc(inside) == 2 ? 2 : 1); }

// ---------------------------------------------------------------------------------------------------- integrate
__global__ void __launch_bounds__(kVolThreads) tsdf_integrate_kernel(float* __restrict__ F, float* __restrict__ W,
                                                                     float* __restrict__ C,
                                                                     const float* __restrict__ depth,
                                                                     const float* __restrict__ rgb, int h, int w,
                                                                     int frames, VolGrid G, VolCam K, double trunc,
                                                                     VolPoses P) {
  const long long n = (long long)G.nx * G.ny * G.nz;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int i = (int)(p % G.nx), j = (int)((p / G.nx) % G.ny), k = (int)(p / ((long long)G.nx * G.ny));
  const double X = __dadd_rn(G.ox, __dmul_rn(G.voxel, (double)i));
  const double Y = __dadd_rn(G.oy, __dmul_rn(G.voxel, (double)j));
  const double Z = __dadd_rn(G.oz, __dmul_rn(G.voxel, (double)k));
  const long long plane = (long long)h * w;
  float f = F[p], wt = W[p];
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (C) {
    c0 = C[p];
    c1 = C[n + p];
    c2 = C[2 * n + p];
  }
  bool seen = false;
  for (int fr = 0; fr < frames; ++fr) {
    const double* m = P.m[fr];
    const double dx = __dsub_rn(X, m[9]), dy = __dsub_rn(Y, m[10]), dz = __dsub_rn(Z, m[11]);
    // Xc = R^T (X - t)
    const double zc = __dadd_rn(__dadd_rn(__dmul_rn(m[2], dx), __dmul_rn(m[5], dy)), __dmul_rn(m[8], dz));
    if (!(zc > 0.0)) continue;
    const double xc = __dadd_rn(__dadd_rn(__dmul_rn(m[0], dx), __dmul_rn(m[3], dy)), __dmul_rn(m[6], dz));
    const double yc = __dadd_rn(__dadd_rn(__dmul_rn(m[1], dx), __dmul_rn(m[4], dy)), __dmul_rn(m[7], dz));
    const double u = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fx, xc), zc), K.cx), 0.5));
    const double v = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fy, yc), zc), K.cy), 0.5));
    if (!(u >= 0.0 && u <= (double)(w - 1) && v >= 0.0 && v <= (double)(h - 1))) continue;
    const long long off = (long long)v * w + (long long)u;
    const float d = depth[fr * plane + off];
    if (!(isfinite(d) && d > 0.f)) continue;
    const double eta = __dsub_rn((double)d, zc);
    if (eta < -trunc) continue;
    const float fo = (float)fmin(1.0, __ddiv_rn(eta, trunc));
    const float w1 = __fadd_rn(wt, 1.f);
    f = __fdiv_rn(__fadd_rn(__fmul_rn(f, wt), fo), w1);
    if (C) {
      const float* px = rgb + 3 * fr * plane + off;
      c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, wt), px[0]), w1);
      c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, wt), px[plane]), w1);
      c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, wt), px[2 * plane]), w1);
    }
    wt = w1;
    seen = true;
  }
  if (seen) {
    F[p] = f;
    W[p] = wt;
    if (C) {
      C[p] = c0;
      C[n + p] = c1;
      C[2 * n + p] = c2;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- raycast
struct RaySampler {
  const float *F, *W;
  const float* C;                                 // colour planes [3][n] (the coloured raycast only)
  VolGrid G;
  double lo[3];
  // the trilinear cell of world point o + t d: its lowest corner's index and the fractions
  ODB_DEVINL long long locate(const double o[3], const double d[3], double t, double fr[3]) const {
    const int n[3] = {G.nx, G.ny, G.nz};
    int c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double g = __ddiv_rn(__dsub_rn(__dadd_rn(o[a], __dmul_rn(t, d[a])), lo[a]), G.voxel);
      const double fl = fmin(fmax(floor(g), 0.0), (double)(n[a] - 2));
      c[a] = (int)fl;
      fr[a] = fmin(fmax(__dsub_rn(g, fl), 0.0), 1.0);
    }
    return c[0] + c[1] * (long long)G.nx + c[2] * (long long)G.nx * G.ny;
  }
  // trilinear interpolation of plane V over the cell at base: the (y, z) corner pairs, x first, then y, then z
  ODB_DEVINL double trilinear(const float* V, long long base, const double fr[3]) const {
    const long long sy = G.nx, sz = (long long)G.nx * G.ny;
    double cv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const long long e = base + (q & 1) * sy + (q >> 1) * sz;
      cv[q] = lerp_rn((double)V[e], (double)V[e + 1], fr[0]);
    }
    return lerp_rn(lerp_rn(cv[0], cv[1], fr[1]), lerp_rn(cv[2], cv[3], fr[1]), fr[2]);
  }
  // trilinear F at world point o + t d; false when a corner has W = 0
  ODB_DEVINL bool sample(const double o[3], const double d[3], double t, double& val) const {
    double fr[3];
    const long long base = locate(o, d, t, fr);
    const long long sy = G.nx, sz = (long long)G.nx * G.ny;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const long long e = base + (q & 1) * sy + (q >> 1) * sz;
      if (!(W[e] > 0.f && W[e + 1] > 0.f)) return false;
    }
    val = trilinear(F, base, fr);
    return true;
  }
  // trilinear colour channel a at o + t d (a sample already found valid: every corner has W > 0)
  ODB_DEVINL double color(const double o[3], const double d[3], double t, int a) const {
    double fr[3];
    const long long base = locate(o, d, t, fr);
    return trilinear(C + a * ((long long)G.nx * G.ny * G.nz), base, fr);
  }
};

// kColor: also rgb [3][h][w], the colour at the hit (NaN where nothing is hit), looked up once the hit is found, so the
// march and the depth are the depth-only kernel's operation for operation
template <bool kColor>
__global__ void __launch_bounds__(128) tsdf_raycast_kernel(RaySampler S, VolCam K, VolPoses P, int h, int w,
                                                           double step, float* __restrict__ out,
                                                           float* __restrict__ rgb) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const double* m = P.m[0];
  const double rx = __ddiv_rn(__dsub_rn((double)x, K.cx), K.fx), ry = __ddiv_rn(__dsub_rn((double)y, K.cy), K.fy);
  const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry)), 1.0));
  const double ux = __ddiv_rn(rx, nrm), uy = __ddiv_rn(ry, nrm), uz = __ddiv_rn(1.0, nrm);
  double d[3], o[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    d[a] = __dadd_rn(__dadd_rn(__dmul_rn(m[3 * a], ux), __dmul_rn(m[3 * a + 1], uy)), __dmul_rn(m[3 * a + 2], uz));
    o[a] = m[9 + a];
  }
  const int n[3] = {S.G.nx, S.G.ny, S.G.nz};
  double t0 = 0.0, t1 = INFINITY;
  bool miss = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = S.lo[a], hi = __dadd_rn(lo, __dmul_rn(S.G.voxel, (double)(n[a] - 1)));
    if (d[a] == 0.0) {
      miss |= o[a] < lo || o[a] > hi;
    } else {
      const double ta = __ddiv_rn(__dsub_rn(lo, o[a]), d[a]), tb = __ddiv_rn(__dsub_rn(hi, o[a]), d[a]);
      t0 = fmax(t0, fmin(ta, tb));
      t1 = fmin(t1, fmax(ta, tb));
    }
  }
  float z = 0.f;
  bool hit = false;
  double t_lo = 0.0, t_hi = 0.0, frac = 0.0;
  if (!miss && t0 <= t1) {
    bool prev_ok = false;
    double prev = 0.0, tp = t0;
    for (long long s = 0;; ++s) {
      const double t = __dadd_rn(t0, __dmul_rn((double)s, step));
      if (!(t <= t1)) break;
      double val;
      const bool ok = S.sample(o, d, t, val);
      if (ok && prev_ok && prev > 0.0 && val <= 0.0) {
        frac = __ddiv_rn(prev, __dsub_rn(prev, val));
        const double th = __dadd_rn(tp, __dmul_rn(step, frac));
        z = (float)__dmul_rn(th, uz);
        hit = true;
        t_lo = tp;
        t_hi = t;
        break;
      }
      prev_ok = ok;
      prev = val;
      tp = t;
    }
  }
  const long long px = (long long)y * w + x, plane = (long long)h * w;
  out[px] = z;
  if constexpr (kColor) {
#pragma unroll 1
    for (int a = 0; a < 3; ++a)
      rgb[a * plane + px] = hit ? (float)lerp_rn(S.color(o, d, t_lo, a), S.color(o, d, t_hi, a), frac) : NAN;
  }
}

// ---------------------------------------------------------------------------------------------------- mesh
struct MeshWs {                 // odb_tsdf_mesh_workspace_bytes
  long long* base;              // [2][blocks]: exclusive vertex / face base of each block
  int* vbase;                   // [n]: first vertex id of each point
  int* blk;                     // [2][blocks]: vertex / face count of each block
  unsigned char *mask, *ntri;   // [n]
};

static long long mesh_blocks(long long n) { return (n + kVolThreads - 1) / kVolThreads; }

static MeshWs mesh_ws(void* workspace, long long n) {
  const long long nb = mesh_blocks(n);
  MeshWs M;
  M.base = static_cast<long long*>(workspace);
  M.vbase = reinterpret_cast<int*>(M.base + 2 * nb);
  M.blk = M.vbase + n;
  M.mask = reinterpret_cast<unsigned char*>(M.blk + 2 * nb);
  M.ntri = M.mask + n;
  return M;
}

ODB_DEVINL long long corner_offset(int code, const VolGrid& G) {
  return (code & 1) + ((code >> 1) & 1) * (long long)G.nx + ((code >> 2) & 1) * (long long)G.nx * G.ny;
}

// exclusive scan of v over the CTA (kVolThreads threads); total = the CTA's sum
ODB_DEVINL int block_exclusive_scan(int v, int& total) {
  __shared__ int warp_sum[kVolThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += t;
  }
  if (lane == 31) warp_sum[wid] = s;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int q = 0; q < kVolThreads / 32; ++q) {
    const int t = warp_sum[q];
    before += q < wid ? t : 0;
    total += t;
  }
  __syncthreads();
  return before + s - v;
}

// the 8 corners of the cell at point (i, j, k), W = 0 outside the grid
ODB_DEVINL void load_corners(const float* F, const float* W, const VolGrid& G, long long p, int i, int j, int k,
                             float f[8], float wt[8]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const bool in = i + (c & 1) < G.nx && j + ((c >> 1) & 1) < G.ny && k + ((c >> 2) & 1) < G.nz;
    const long long q = p + corner_offset(c, G);
    f[c] = in ? F[q] : 0.f;
    wt[c] = in ? W[q] : 0.f;
  }
}

ODB_DEVINL int edge_mask(const float f[8], const float wt[8]) {
  int mask = 0;
  if (wt[0] > 0.f) {
#pragma unroll
    for (int c = 1; c < 8; ++c)
      if (wt[c] > 0.f && ((f[0] < 0.f) != (f[c] < 0.f))) mask |= 1 << (c - 1);
  }
  return mask;
}

// corner bit masks of a cell: bit c of obs when W > 0, of neg when F < 0 (registers, no local-memory indexing below)
ODB_DEVINL void corner_bits(const float f[8], const float wt[8], int& obs, int& neg) {
  obs = neg = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    obs |= (wt[c] > 0.f ? 1 : 0) << c;
    neg |= (f[c] < 0.f ? 1 : 0) << c;
  }
}

// inside mask of tetrahedron q (bit v: corner v has F < 0), or -1 when a corner has W = 0
ODB_DEVINL int tet_inside(int q, int obs, int neg) {
  int m = 0;
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const int c = kTetCorner[q][v];
    if (!((obs >> c) & 1)) return -1;
    m |= ((neg >> c) & 1) << v;
  }
  return m;
}

ODB_DEVINL bool is_cell(const VolGrid& G, int i, int j, int k) { return i < G.nx - 1 && j < G.ny - 1 && k < G.nz - 1; }

__global__ void __launch_bounds__(kVolThreads) mesh_count_kernel(const float* __restrict__ F,
                                                                 const float* __restrict__ W, VolGrid G, MeshWs M) {
  const long long n = (long long)G.nx * G.ny * G.nz, nb = gridDim.x;
  const long long p = (long long)blockIdx.x * kVolThreads + threadIdx.x;
  int mask = 0, tris = 0;
  if (p < n) {
    const int i = (int)(p % G.nx), j = (int)((p / G.nx) % G.ny), k = (int)(p / ((long long)G.nx * G.ny));
    float f[8], wt[8];
    load_corners(F, W, G, p, i, j, k, f, wt);
    mask = edge_mask(f, wt);
    int obs, neg;
    corner_bits(f, wt, obs, neg);
    if (is_cell(G, i, j, k))
      for (int q = 0; q < 6; ++q) {
        const int m = tet_inside(q, obs, neg);
        if (m >= 0) tris += tet_triangles(m);
      }
    M.mask[p] = (unsigned char)mask;
    M.ntri[p] = (unsigned char)tris;
  }
  int tv, tf;
  block_exclusive_scan(__popc(mask), tv);
  block_exclusive_scan(tris, tf);
  if (threadIdx.x == 0) {
    M.blk[blockIdx.x] = tv;
    M.blk[nb + blockIdx.x] = tf;
  }
}

// one CTA of 1024 threads: each scans a contiguous run of block totals
__global__ void __launch_bounds__(1024) mesh_scan_kernel(MeshWs M, long long nb, long long* __restrict__ counts) {
  __shared__ long long run[2][1024];
  const long long per = (nb + 1023) / 1024, b0 = min(nb, threadIdx.x * per), b1 = min(nb, b0 + per);
  for (int s = 0; s < 2; ++s) {
    long long sum = 0;
    for (long long b = b0; b < b1; ++b) sum += M.blk[s * nb + b];
    run[s][threadIdx.x] = sum;
  }
  __syncthreads();
  if (threadIdx.x < 2) {                          // 1024 run totals, serially: exclusive prefix and grand total
    long long acc = 0;
    for (int t = 0; t < 1024; ++t) {
      const long long v = run[threadIdx.x][t];
      run[threadIdx.x][t] = acc;
      acc += v;
    }
    counts[threadIdx.x] = acc;
  }
  __syncthreads();
  for (int s = 0; s < 2; ++s) {
    long long acc = run[s][threadIdx.x];
    for (long long b = b0; b < b1; ++b) {
      M.base[s * nb + b] = acc;
      acc += M.blk[s * nb + b];
    }
  }
}

__global__ void __launch_bounds__(kVolThreads) mesh_base_kernel(VolGrid G, MeshWs M) {
  const long long n = (long long)G.nx * G.ny * G.nz;
  const long long p = (long long)blockIdx.x * kVolThreads + threadIdx.x;
  const int c = p < n ? __popc(M.mask[p]) : 0;
  int total;
  const int local = block_exclusive_scan(c, total);
  if (p < n) M.vbase[p] = (int)(M.base[blockIdx.x] + local);
}

__global__ void __launch_bounds__(kVolThreads) mesh_emit_kernel(const float* __restrict__ F,
                                                                const float* __restrict__ W,
                                                                const float* __restrict__ C, VolGrid G, MeshWs M,
                                                                float* __restrict__ verts, int* __restrict__ faces,
                                                                float* __restrict__ colors) {
  const long long n = (long long)G.nx * G.ny * G.nz, nb = gridDim.x;
  const long long p = (long long)blockIdx.x * kVolThreads + threadIdx.x;
  const int tris = p < n ? M.ntri[p] : 0;
  int total;
  const long long fbase = M.base[nb + blockIdx.x] + block_exclusive_scan(tris, total);
  if (p >= n) return;
  const int mask = M.mask[p];
  if (mask == 0 && tris == 0) return;
  const int i = (int)(p % G.nx), j = (int)((p / G.nx) % G.ny), k = (int)(p / ((long long)G.nx * G.ny));
  float f[8], wt[8];
  load_corners(F, W, G, p, i, j, k, f, wt);
  long long vid = M.vbase[p];
#pragma unroll
  for (int c = 1; c < 8; ++c) {
    if (!((mask >> (c - 1)) & 1)) continue;
    const long long q = p + corner_offset(c, G);
    const double fp = f[0], s = __ddiv_rn(fp, __dsub_rn(fp, (double)f[c]));
    const double g[3] = {__dadd_rn((double)i, (c & 1) ? s : 0.0), __dadd_rn((double)j, ((c >> 1) & 1) ? s : 0.0),
                         __dadd_rn((double)k, ((c >> 2) & 1) ? s : 0.0)};
    const double org[3] = {G.ox, G.oy, G.oz};
#pragma unroll
    for (int a = 0; a < 3; ++a) verts[3 * vid + a] = (float)__dadd_rn(org[a], __dmul_rn(G.voxel, g[a]));
    if (C && colors) {
#pragma unroll
      for (int a = 0; a < 3; ++a) colors[3 * vid + a] = (float)lerp_rn((double)C[a * n + p], (double)C[a * n + q], s);
    }
    ++vid;
  }
  if (tris == 0) return;
  int obs, neg;
  corner_bits(f, wt, obs, neg);
  long long fo = fbase;
  for (int q = 0; q < 6; ++q) {
    const int m = tet_inside(q, obs, neg);
    if (m < 0) continue;
    for (int t = 0; t < 2; ++t) {
      if (kTetTri[m][t][0] < 0) break;
      int id[3];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const int edge = kTetTri[m][t][e];
        const int ca = kTetCorner[q][kTetEdge[edge][0]], cb = kTetCorner[q][kTetEdge[edge][1]];
        const long long owner = p + corner_offset(ca, G);
        const int dir = (ca ^ cb) - 1;            // cb's corner bits contain ca's
        id[e] = M.vbase[owner] + __popc(M.mask[owner] & ((1 << dir) - 1));
      }
      const int odd = kTetOdd[q];
      faces[3 * fo] = id[0];
      faces[3 * fo + 1] = id[odd ? 2 : 1];
      faces[3 * fo + 2] = id[odd ? 1 : 2];
      ++fo;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- host
static bool grid_ok(int32_t nx, int32_t ny, int32_t nz, double ox, double oy, double oz, double voxel, VolGrid& G) {
  for (int32_t d : {nx, ny, nz})
    if (d < 2 || d > ODB_TSDF_MAX_DIM) return false;
  if ((int64_t)nx * ny * nz > ODB_TSDF_MAX_POINTS) return false;
  if (!(std::isfinite(ox) && std::isfinite(oy) && std::isfinite(oz) && std::isfinite(voxel) && voxel > 0.0))
    return false;
  G.nx = nx; G.ny = ny; G.nz = nz;
  G.ox = ox; G.oy = oy; G.oz = oz;
  G.voxel = voxel;
  return true;
}

static bool cam_ok(double fx, double fy, double cx, double cy, VolCam& K) {
  if (!(std::isfinite(fx) && fx > 0.0 && std::isfinite(fy) && fy > 0.0 && std::isfinite(cx) && std::isfinite(cy)))
    return false;
  K.fx = fx; K.fy = fy; K.cx = cx; K.cy = cy;
  return true;
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_tsdf_mesh_workspace_bytes(int32_t nx, int32_t ny, int32_t nz) {
  VolGrid G;
  if (!grid_ok(nx, ny, nz, 0.0, 0.0, 0.0, 1.0, G)) return -1;
  const long long n = (long long)nx * ny * nz, nb = mesh_blocks(n);
  return 2 * nb * 8 + n * 4 + 2 * nb * 4 + 2 * n;
}

extern "C" int odb_tsdf_integrate(float* tsdf, float* weight, float* color, int32_t nx, int32_t ny, int32_t nz,
                                  double ox, double oy, double oz, double voxel, double trunc, const float* depth,
                                  const float* rgb, int32_t b, int32_t h, int32_t w, double fx, double fy, double cx,
                                  double cy, const double* cam_to_world, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  VolGrid G;
  VolCam K;
  if (!tsdf || !weight || !depth || !cam_to_world || (color == nullptr) != (rgb == nullptr) ||
      !grid_ok(nx, ny, nz, ox, oy, oz, voxel, G) || !(std::isfinite(trunc) && trunc > 0.0) || !planes_ok(b, h, w) ||
      !cam_ok(fx, fy, cx, cy, K) || !aligned(tsdf, 4) || !aligned(weight, 4) || !aligned(color, 4) ||
      !aligned(depth, 4) || !aligned(rgb, 4))
    return fail(ODB_ERR_INVALID, "tsdf_integrate: bad argument");
  double tmp[12];
  for (int32_t f = 0; f < b; ++f)
    if (!pose_ok(cam_to_world + 16 * (int64_t)f, tmp))
      return fail(ODB_ERR_INVALID, "tsdf_integrate: a pose is not a finite rigid camera-to-world matrix");
  const long long n = (long long)nx * ny * nz, plane = (long long)h * w;
  const unsigned blocks = (unsigned)((n + kVolThreads - 1) / kVolThreads);
  for (int32_t f0 = 0; f0 < b; f0 += kFramesPerLaunch) {
    const int frames = b - f0 < kFramesPerLaunch ? b - f0 : kFramesPerLaunch;
    VolPoses P;
    for (int f = 0; f < frames; ++f) pose_ok(cam_to_world + 16 * (int64_t)(f0 + f), P.m[f]);
    tsdf_integrate_kernel<<<blocks, kVolThreads, 0, stream>>>(tsdf, weight, color, depth + f0 * plane,
                                                              rgb ? rgb + 3 * f0 * plane : nullptr, h, w, frames, G, K,
                                                              trunc, P);
    count_launch();
  }
  return check_launch("tsdf_integrate");
}

// odb_tsdf_raycast (color, rgb NULL) and odb_tsdf_raycast_color
static int tsdf_raycast(const char* name, const float* tsdf, const float* weight, const float* color, int32_t nx,
                        int32_t ny, int32_t nz, double ox, double oy, double oz, double voxel,
                        const double* cam_to_world, int32_t h, int32_t w, double fx, double fy, double cx, double cy,
                        double step, float* out, float* rgb, cudaStream_t stream) {
  VolGrid G;
  VolCam K;
  VolPoses P;
  if (!tsdf || !weight || !out || !cam_to_world || (color == nullptr) != (rgb == nullptr) ||
      !grid_ok(nx, ny, nz, ox, oy, oz, voxel, G) || !planes_ok(1, h, w) || !cam_ok(fx, fy, cx, cy, K) ||
      !(std::isfinite(step) && step >= voxel / 64.0 && step <= voxel) || !aligned(tsdf, 4) || !aligned(weight, 4) ||
      !aligned(out, 4) || !aligned(color, 4) || !aligned(rgb, 4))
    return fail(ODB_ERR_INVALID, (std::string(name) + ": bad argument").c_str());
  if (!pose_ok(cam_to_world, P.m[0]))
    return fail(ODB_ERR_INVALID, (std::string(name) + ": the pose is not a finite rigid camera-to-world matrix").c_str());
  RaySampler S;
  S.F = tsdf;
  S.W = weight;
  S.C = color;
  S.G = G;
  S.lo[0] = ox; S.lo[1] = oy; S.lo[2] = oz;
  const dim3 grid((w + 127) / 128, h);
  if (color)
    tsdf_raycast_kernel<true><<<grid, 128, 0, stream>>>(S, K, P, h, w, step, out, rgb);
  else
    tsdf_raycast_kernel<false><<<grid, 128, 0, stream>>>(S, K, P, h, w, step, out, nullptr);
  count_launch();
  return check_launch(name);
}

extern "C" int odb_tsdf_raycast(const float* tsdf, const float* weight, int32_t nx, int32_t ny, int32_t nz, double ox,
                                double oy, double oz, double voxel, const double* cam_to_world, int32_t h, int32_t w,
                                double fx, double fy, double cx, double cy, double step, float* out, void* stream_) {
  return tsdf_raycast("tsdf_raycast", tsdf, weight, nullptr, nx, ny, nz, ox, oy, oz, voxel, cam_to_world, h, w, fx, fy,
                      cx, cy, step, out, nullptr, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_tsdf_raycast_color(const float* tsdf, const float* weight, const float* color, int32_t nx,
                                      int32_t ny, int32_t nz, double ox, double oy, double oz, double voxel,
                                      const double* cam_to_world, int32_t h, int32_t w, double fx, double fy,
                                      double cx, double cy, double step, float* out, float* rgb, void* stream_) {
  if (!color || !rgb) return fail(ODB_ERR_INVALID, "tsdf_raycast_color: bad argument");
  return tsdf_raycast("tsdf_raycast_color", tsdf, weight, color, nx, ny, nz, ox, oy, oz, voxel, cam_to_world, h, w, fx,
                      fy, cx, cy, step, out, rgb, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_tsdf_mesh_count(const float* tsdf, const float* weight, int32_t nx, int32_t ny, int32_t nz,
                                   void* workspace, int64_t* counts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  VolGrid G;
  if (!tsdf || !weight || !workspace || !counts || !grid_ok(nx, ny, nz, 0.0, 0.0, 0.0, 1.0, G) ||
      !aligned(tsdf, 4) || !aligned(weight, 4) || !aligned(workspace, 8) || !aligned(counts, 8))
    return fail(ODB_ERR_INVALID, "tsdf_mesh_count: bad argument");
  const long long n = (long long)nx * ny * nz, nb = mesh_blocks(n);
  const MeshWs M = mesh_ws(workspace, n);
  mesh_count_kernel<<<(unsigned)nb, kVolThreads, 0, stream>>>(tsdf, weight, G, M);
  count_launch();
  mesh_scan_kernel<<<1, 1024, 0, stream>>>(M, nb, reinterpret_cast<long long*>(counts));
  count_launch();
  mesh_base_kernel<<<(unsigned)nb, kVolThreads, 0, stream>>>(G, M);
  count_launch();
  return check_launch("tsdf_mesh_count");
}

extern "C" int odb_tsdf_mesh_emit(const float* tsdf, const float* weight, const float* color, int32_t nx, int32_t ny,
                                  int32_t nz, double ox, double oy, double oz, double voxel, const void* workspace,
                                  float* vertices, int32_t* faces, float* colors, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  VolGrid G;
  if (!tsdf || !weight || !workspace || (color == nullptr) != (colors == nullptr) ||
      !grid_ok(nx, ny, nz, ox, oy, oz, voxel, G) || !aligned(tsdf, 4) || !aligned(weight, 4) ||
      !aligned(color, 4) || !aligned(workspace, 8) || !aligned(vertices, 4) || !aligned(faces, 4) ||
      !aligned(colors, 4))
    return fail(ODB_ERR_INVALID, "tsdf_mesh_emit: bad argument");
  const long long n = (long long)nx * ny * nz, nb = mesh_blocks(n);
  const MeshWs M = mesh_ws(const_cast<void*>(workspace), n);
  mesh_emit_kernel<<<(unsigned)nb, kVolThreads, 0, stream>>>(tsdf, weight, color, G, M, vertices, faces, colors);
  count_launch();
  return check_launch("tsdf_mesh_emit");
}
