// Sparse metric alignment (omnidata_b200/sparse.py SparseDepthAligner): a relative depth prediction a is mapped to
// metres by smooth scale and shift fields S, T fitted to sparse measured depths (LiDAR, SfM points).  Definition in
// DESIGN.md §3 "Sparse metric alignment" and include/omnidata_b200.h; oracle/sparse_oracle.py restates it in float64.
//
// The fields are the bilinear resize (align_corners=False) of a gy x gx grid of nodes (s_i, t_i).  Along an axis of
// length L with g nodes, pixel x sits at u = ((x + 0.5) g) / L - 0.5; the node centres u = 0 .. g - 1 cut the axis into
// g + 1 regions (region 0: u < 0, region r: r - 1 <= u < r, region g: u >= g - 1), and inside a region the same nodes
// (max(r - 1, 0), min(r, g - 1)) are active with weights (1 - f, f), f = clamp(u, 0, g - 1) - floor(...).  So a region
// of the image has the same <= 4 active nodes everywhere, and the normal equations of the fit are sums of per-region
// moments.
//
//   sparse_moments_kernel  per chunk of a region (fixed chunks: the partition depends on h, w and the grid only): the
//                          fp64 moments of the points, with the IRLS weights of the previous nodes formed inline
//   sparse_reduce_kernel   per region: its chunks' moments in a fixed order (ordered_sum8)
//   sparse_solve_kernel    per image: status rules, band assembly (data term + smoothness), band_cholesky_solve
//                          (fp64.cuh), nodes out
//   sparse_record_kernel   per image: RMS relative residual of the final fit
//   sparse_apply_kernel    per pixel: S, T interpolated in fp64, depth_hat (fp64.cuh), rounded to fp32 once
//
// The points are not compacted into a list: a pass over the map reads 8-9 bytes per pixel, and compacting would itself
// read the map once and need a count (a host synchronisation or a worst-case buffer) before the list can be walked.
// Without floating-point atomics and with fixed partitions the results are bit-reproducible and independent of the
// batch.  Built without fast-math: the interpolation and the apply are written with explicit round-to-nearest
// operations so that the oracle reproduces them operation by operation.
#include <cmath>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kSparseThreads = 256;
constexpr int kChunkPixels = 4096;          // pixels of one moments chunk, at most
constexpr int kMomStride = 48;              // doubles per chunk / region moments
// moments of a region: 10 node pairs (c <= d of its 4 local nodes) x (S w pc pd a^2, S w pc pd a, S w pc pd), then per
// local node (S w pc a y, S w pc y), then (n, S a, S a^2, #non-finite a, S w, S w a, S w a^2, #(w < 1), S r^2)
constexpr int kQRhs = 30, kQN = 38, kQRes = 46, kQ = 47;

struct SparseGeom {
  int h, w, gy, gx;
  int cw, ch, ncx, ncy;                     // chunk width / height, chunks per region along x / y
};

// u = ((x + 0.5) g) / L - 0.5, every operation rounded to nearest
ODB_DEVINL double node_coord(int x, int g, int L) {
  return __dsub_rn(__ddiv_rn(__dmul_rn((double)x + 0.5, (double)g), (double)L), 0.5);
}
// the first node i0 and the fraction f of position x: u clamped to [0, g - 1], i0 = floor(u), f = u - i0 (exact)
ODB_DEVINL void node_lerp(int x, int g, int L, int& i0, double& f) {
  const double u = fmin(fmax(node_coord(x, g, L), 0.0), (double)(g - 1));
  const double fl = floor(u);
  i0 = (int)fl;
  f = u - fl;
}
// first pixel of region r (0 .. g + 1: L) along an axis: region r >= 1 starts at the first x with u(x) >= r - 1
ODB_DEVINL int region_start(int r, int g, int L) {
  if (r == 0) return 0;
  if (r > g) return L;
  const long long num = (long long)(2 * r - 1) * L - g;          // ((r - 1/2) L / g - 1/2) * 2g >= 0 as g <= L
  int x = (int)min((long long)L, (num + 2LL * g - 1) / (2LL * g));
  while (x > 0 && node_coord(x - 1, g, L) >= r - 1) --x;
  while (x < L && node_coord(x, g, L) < r - 1) ++x;
  return x;
}
// S (c = 0) or T (c = 1) at a pixel: (1 - fy) ((1 - fx) n00 + fx n01) + fy ((1 - fx) n10 + fx n11), nodes [gy][gx][2]
ODB_DEVINL double field_at(const double* nodes, int gy, int gx, int iy0, int ix0, double fy, double fx, int c) {
  const int iy1 = min(iy0 + 1, gy - 1), ix1 = min(ix0 + 1, gx - 1);
  const double* r0 = nodes + (long long)iy0 * gx * 2;
  const double* r1 = nodes + (long long)iy1 * gx * 2;
  const double ex = __dsub_rn(1.0, fx), ey = __dsub_rn(1.0, fy);
  const double top = __dadd_rn(__dmul_rn(ex, r0[ix0 * 2 + c]), __dmul_rn(fx, r0[ix1 * 2 + c]));
  const double bot = __dadd_rn(__dmul_rn(ex, r1[ix0 * 2 + c]), __dmul_rn(fx, r1[ix1 * 2 + c]));
  return __dadd_rn(__dmul_rn(ey, top), __dmul_rn(fy, bot));
}
// z = S a + T
ODB_DEVINL double affine_at(const double* nodes, int gy, int gx, int iy0, int ix0, double fy, double fx, double a) {
  const double s = field_at(nodes, gy, gx, iy0, ix0, fy, fx, 0), t = field_at(nodes, gy, gx, iy0, ix0, fy, fx, 1);
  return __dadd_rn(__dmul_rn(s, a), t);
}

// Chunk blockIdx.x of image blockIdx.y: region (ry, rx) = chunk / (ncy ncx), then a ch x cw rectangle of it.
// part[b][chunk][kMomStride] = the region moments over the chunk's points; prev (nullable) = the previous fit's nodes
// [b][gy][gx][2]: with it, r = (z - y) / y and, where delta > 0, w = min(1, delta / |r|); without, w = 1.
__global__ void __launch_bounds__(kSparseThreads) sparse_moments_kernel(const float* __restrict__ pred,
                                                                        const float* __restrict__ sparse,
                                                                        const void* mask, int mask_kind, SparseGeom G,
                                                                        int disparity, double min_depth,
                                                                        double max_depth,
                                                                        const double* __restrict__ prev, double delta,
                                                                        double* __restrict__ part) {
  __shared__ double warp_part[kSparseThreads / 32][kQ];
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int per_region = G.ncy * G.ncx;
  const int region = chunk / per_region, k = chunk - region * per_region;
  const int ry = region / (G.gx + 1), rx = region - ry * (G.gx + 1);
  const int cy = k / G.ncx, cx = k - cy * G.ncx;
  const int y0 = region_start(ry, G.gy, G.h) + cy * G.ch, y1 = min(y0 + G.ch, region_start(ry + 1, G.gy, G.h));
  const int x0 = region_start(rx, G.gx, G.w) + cx * G.cw, x1 = min(x0 + G.cw, region_start(rx + 1, G.gx, G.w));
  const int rh = max(y1 - y0, 0), rw = max(x1 - x0, 0);
  const long long base = (long long)b * G.h * G.w;
  const double* pn = prev != nullptr ? prev + (long long)b * G.gy * G.gx * 2 : nullptr;
  double acc[kQ];
#pragma unroll
  for (int q = 0; q < kQ; ++q) acc[q] = 0.0;
  for (int e = threadIdx.x; e < rh * rw; e += kSparseThreads) {
    const int y = y0 + e / rw, x = x0 + e % rw;
    const long long i = base + (long long)y * G.w + x;
    if (!mask_valid(mask, mask_kind, i)) continue;
    const double g = sparse[i];
    if (!depth_valid(g, min_depth, max_depth)) continue;
    const double a = pred[i];
    const double yv = disparity ? __drcp_rn(g) : g;
    int iy0, ix0;
    double fy, fx;
    node_lerp(y, G.gy, G.h, iy0, fy);
    node_lerp(x, G.gx, G.w, ix0, fx);
    double w = 1.0;
    if (pn != nullptr) {
      const double r = __ddiv_rn(__dsub_rn(affine_at(pn, G.gy, G.gx, iy0, ix0, fy, fx, a), yv), yv);
      acc[kQRes] += r * r;
      if (delta > 0.0) {
        w = fmin(1.0, __ddiv_rn(delta, fabs(r)));
        acc[kQN + 7] += w < 1.0 ? 1.0 : 0.0;
      }
    }
    const double phi[4] = {(1.0 - fy) * (1.0 - fx), (1.0 - fy) * fx, fy * (1.0 - fx), fy * fx};
    const double aa = a * a;
    int q = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const double wc = w * phi[c];
#pragma unroll
      for (int d = c; d < 4; ++d, q += 3) {
        const double v = wc * phi[d];
        acc[q] += v * aa;
        acc[q + 1] += v * a;
        acc[q + 2] += v;
      }
      acc[kQRhs + 2 * c] += wc * a * yv;
      acc[kQRhs + 2 * c + 1] += wc * yv;
    }
    acc[kQN] += 1.0;
    acc[kQN + 1] += a;
    acc[kQN + 2] += aa;
    acc[kQN + 3] += isfinite(a) ? 0.0 : 1.0;
    acc[kQN + 4] += w;
    acc[kQN + 5] += w * a;
    acc[kQN + 6] += w * aa;
  }
  // fixed-order block reduction: butterfly within each warp, then the warps in order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < kQ; ++q) {
    double v = acc[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) warp_part[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < kQ) {
    double s = 0.0;
#pragma unroll
    for (int v = 0; v < kSparseThreads / 32; ++v) s += warp_part[v][threadIdx.x];
    part[((long long)b * gridDim.x + chunk) * kMomStride + threadIdx.x] = s;
  }
}

// out[b][region][q] = sum over the region's chunks of part[b][chunk][q] in a fixed order.  grid (regions, b)
__global__ void __launch_bounds__(kSparseThreads) sparse_reduce_kernel(const double* __restrict__ part,
                                                                       int per_region, double* __restrict__ out) {
  const int region = blockIdx.x, b = blockIdx.y;
  const long long r = (long long)b * gridDim.x + region;
  const double* p = part + r * per_region * kMomStride;
  const int col = threadIdx.x & 31;
  for (int q0 = 0; q0 < kQ; q0 += 32) {
    const int q = q0 + col;
    const double s = ordered_sum8(per_region, q < kQ, [&](int c) { return p[(long long)c * kMomStride + q]; });
    if (threadIdx.x < 32 && q < kQ) out[r * kMomStride + q] = s;
    __syncthreads();
  }
}

// band half-bandwidth + 1 of the interleaved (s_k, t_k) system: bilinear weights couple nodes k and k + gx + 1
__host__ __device__ inline int sparse_band_width(int gy, int gx) { return gy > 1 ? 2 * gx + 4 : 4; }

// One CTA per image.  Status: n < 2 -> 1, a non-finite prediction on V -> 3, global weighted det <= 0 -> 2; the
// nodes are then NaN.  Otherwise the normal equations of
//   E = S_V w (S a + T - y)^2 + (smooth / n_e) S_{i~j} S_V ((s_i - s_j) a + (t_i - t_j))^2
// with unknowns (s_0, t_0, s_1, t_1, ...): node k assembles rows 2k and 2k + 1 of the lower band (band[r * w + q] =
// A[r][r - q]) from the <= 4 regions around it, in shared memory when it fits, else in the image's slice of
// `workspace`.  records[b] = (n, status, -, fraction with w < 1, 0, 0, 0, 0); the residual is sparse_record_kernel's.
__global__ void __launch_bounds__(kSparseThreads, 1) sparse_solve_kernel(const double* __restrict__ moments, int gy,
                                                                      int gx, double smooth, int band_in_smem,
                                                                      double* workspace, double* __restrict__ nodes,
                                                                      double* __restrict__ records) {
  extern __shared__ double sm[];
  __shared__ double s_tot[8];
  __shared__ int s_status;
  const int b = blockIdx.x;
  const int K = gy * gx, n = 2 * K, w = sparse_band_width(gy, gx), R = (gy + 1) * (gx + 1);
  const double* M = moments + (long long)b * R * kMomStride;
  const int col = threadIdx.x & 31;
  // image totals (n, S a, S a^2, #non-finite, S w, S w a, S w a^2, #(w < 1)), regions in a fixed order
  const double tot = ordered_sum8(R, col < 8, [&](int r) { return M[(long long)r * kMomStride + kQN + col]; });
  if (threadIdx.x < 8) s_tot[threadIdx.x] = tot;
  __syncthreads();
  if (threadIdx.x == 0) {
    const double np = s_tot[0], det = s_tot[6] * s_tot[4] - s_tot[5] * s_tot[5];
    const int status = np < 2.0 ? 1 : s_tot[3] > 0.0 ? 3 : det > 0.0 ? 0 : 2;
    double* rec = records + (long long)b * ODB_SPARSE_RECORD;
    rec[0] = np;
    rec[1] = status;
    rec[3] = np > 0.0 ? s_tot[7] / np : 0.0;
    for (int q = 4; q < ODB_SPARSE_RECORD; ++q) rec[q] = 0.0;
    s_status = status;
  }
  __syncthreads();
  double* out = nodes + (long long)b * n;
  if (s_status != 0) {
    for (int e = threadIdx.x; e < n; e += blockDim.x) out[e] = NAN;
    return;
  }
  const int edges = gy * (gx - 1) + (gy - 1) * gx;
  const double lam = edges > 0 ? smooth / edges : 0.0;
  const double g00 = lam * s_tot[2], g01 = lam * s_tot[1], g11 = lam * s_tot[0];
  double* rhs = sm;
  double* band = band_in_smem ? sm + n : workspace + (long long)b * n * w;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    double* rs = band + (long long)(2 * k) * w;
    double* rt = rs + w;
    for (int q = 0; q < w; ++q) rs[q] = rt[q] = 0.0;
    const int iy = k / gx, ix = k - iy * gx;
    double bs = 0.0, bt = 0.0;
    for (int ry = iy; ry <= iy + 1; ++ry) {
      for (int rx = ix; rx <= ix + 1; ++rx) {
        const double* m = M + (long long)(ry * (gx + 1) + rx) * kMomStride;
        const int ylo = max(ry - 1, 0), yhi = min(ry, gy - 1), xlo = max(rx - 1, 0), xhi = min(rx, gx - 1);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (((c >> 1) ? yhi : ylo) * gx + ((c & 1) ? xhi : xlo) != k) continue;
          bs += m[kQRhs + 2 * c];
          bt += m[kQRhs + 2 * c + 1];
#pragma unroll
          for (int d = 0; d < 4; ++d) {
            const int l = ((d >> 1) ? yhi : ylo) * gx + ((d & 1) ? xhi : xlo);
            if (l > k) continue;
            const int lo = min(c, d), hi = max(c, d);
            const double* pm = m + 3 * (lo * 4 - lo * (lo - 1) / 2 + hi - lo);    // pair index of (lo, hi)
            if (l == k) {
              rs[0] += pm[0];
              rt[1] += pm[1];
              rt[0] += pm[2];
            } else {
              const int o = 2 * (k - l);
              rs[o] += pm[0];
              rs[o - 1] += pm[1];
              rt[o + 1] += pm[1];
              rt[o] += pm[2];
            }
          }
        }
      }
    }
    const int deg = (ix > 0) + (ix < gx - 1) + (iy > 0) + (iy < gy - 1);
    rs[0] += deg * g00;
    rt[1] += deg * g01;
    rt[0] += deg * g11;
    for (int side = 0; side < 2; ++side) {            // the left, then the upper neighbour l < k
      if (side == 0 ? ix == 0 : iy == 0) continue;
      const int o = side == 0 ? 2 : 2 * gx;
      rs[o] -= g00;
      rs[o - 1] -= g01;
      rt[o + 1] -= g01;
      rt[o] -= g11;
    }
    rhs[2 * k] = bs;
    rhs[2 * k + 1] = bt;
  }
  __syncthreads();
  band_cholesky_solve(band, rhs, n, w);
  for (int e = threadIdx.x; e < n; e += blockDim.x) out[e] = rhs[e];
}

// records[b][2] = sqrt(S_V r^2 / n) of the final fit (NaN unless status 0).  grid (b)
__global__ void __launch_bounds__(kSparseThreads) sparse_record_kernel(const double* __restrict__ moments, int regions,
                                                                       double* __restrict__ records) {
  const int b = blockIdx.x;
  const double* M = moments + (long long)b * regions * kMomStride;
  const double s = ordered_sum8(regions, (threadIdx.x & 31) == 0,
                                [&](int r) { return M[(long long)r * kMomStride + kQRes]; });
  if (threadIdx.x == 0) {
    double* rec = records + (long long)b * ODB_SPARSE_RECORD;
    rec[2] = rec[1] == 0.0 ? sqrt(s / rec[0]) : NAN;
  }
}

// d = depth_hat(a, S, T) rounded to fp32 once; NaN where a is not finite or the nodes are NaN.  Each thread writes 4
// consecutive pixels of a row (16-byte accesses when `vec`).  grid (ceil(ceil(w / 4) / 256), h, b)
__global__ void __launch_bounds__(kSparseThreads) sparse_apply_kernel(const float* __restrict__ pred,
                                                                      const double* __restrict__ nodes, int h, int w,
                                                                      int gy, int gx, int disparity, double min_depth,
                                                                      double max_depth, int vec,
                                                                      float* __restrict__ out) {
  const int x0 = (blockIdx.x * kSparseThreads + threadIdx.x) * 4, y = blockIdx.y, b = blockIdx.z;
  if (x0 >= w) return;
  const long long row = ((long long)b * h + y) * w;
  const double* nb = nodes + (long long)b * gy * gx * 2;
  int iy0;
  double fy;
  node_lerp(y, gy, h, iy0, fy);
  float a[4], d[4];
  if (vec) {
    const float4 v = *reinterpret_cast<const float4*>(pred + row + x0);
    a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
  } else {
    for (int j = 0; j < 4; ++j) a[j] = x0 + j < w ? pred[row + x0 + j] : 0.0f;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int ix0;
    double fx;
    node_lerp(min(x0 + j, w - 1), gx, w, ix0, fx);
    const double s = field_at(nb, gy, gx, iy0, ix0, fy, fx, 0), t = field_at(nb, gy, gx, iy0, ix0, fy, fx, 1);
    const double v = depth_hat((double)a[j], s, t, disparity, min_depth, max_depth);
    d[j] = isfinite(a[j]) && !isnan(s) && !isnan(t) ? (float)v : NAN;
  }
  if (vec) {
    *reinterpret_cast<float4*>(out + row + x0) = make_float4(d[0], d[1], d[2], d[3]);
  } else {
    for (int j = 0; j < 4; ++j)
      if (x0 + j < w) out[row + x0 + j] = d[j];
  }
}

// The chunks of a region: the extent of a region is at most L / g + 2 pixels along an axis (L / 2 + 2 for g = 1)
static int region_cover(int g, int L) { return min(L, (g > 1 ? L / g : L / 2) + 2); }

static SparseGeom sparse_geom(int h, int w, int gy, int gx) {
  SparseGeom G;
  G.h = h; G.w = w; G.gy = gy; G.gx = gx;
  const int cov_y = region_cover(gy, h), cov_x = region_cover(gx, w);
  G.cw = min(cov_x, kChunkPixels);
  G.ch = min(cov_y, max(1, kChunkPixels / G.cw));
  G.ncx = (cov_x + G.cw - 1) / G.cw;
  G.ncy = (cov_y + G.ch - 1) / G.ch;
  return G;
}

static bool sparse_shape_ok(int32_t b, int32_t h, int32_t w, int32_t gy, int32_t gx) {
  return planes_ok(b, h, w) && gy >= 1 && gx >= 1 && gy <= h && gx <= w && gy * gx <= ODB_SPARSE_MAX_NODES;
}

static bool sparse_range_ok(int32_t space, double min_depth, double max_depth) {
  const bool disparity = space == ODB_SPACE_DISPARITY;
  return (space == ODB_SPACE_DEPTH || disparity) && std::isfinite(min_depth) && min_depth >= 0.0 &&
         !std::isnan(max_depth) && max_depth > min_depth && (!disparity || std::isfinite(max_depth));
}

static size_t sparse_smem_bytes(int gy, int gx) {
  const size_t n = 2 * (size_t)gy * gx;
  return (n + n * sparse_band_width(gy, gx)) * sizeof(double);
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_sparse_align_workspace_bytes(int32_t b, int32_t h, int32_t w, int32_t grid_y, int32_t grid_x) {
  if (!sparse_shape_ok(b, h, w, grid_y, grid_x)) return -1;
  const SparseGeom G = sparse_geom(h, w, grid_y, grid_x);
  const int64_t regions = (int64_t)(grid_y + 1) * (grid_x + 1);
  const int64_t chunks = regions * G.ncy * G.ncx;
  const int64_t n = 2 * (int64_t)grid_y * grid_x;
  const int64_t band = sparse_smem_bytes(grid_y, grid_x) <= kBandSmemMax ? 0 : n * sparse_band_width(grid_y, grid_x);
  return (int64_t)b * ((chunks + regions) * kMomStride + band) * (int64_t)sizeof(double);
}

extern "C" int odb_sparse_align_fit(const float* pred, const float* sparse, const void* mask, int32_t mask_dtype,
                                    int32_t b, int32_t h, int32_t w, int32_t grid_y, int32_t grid_x, int32_t space,
                                    double min_depth, double max_depth, double smooth, double robust,
                                    int32_t iterations, void* workspace, double* nodes, double* records,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool irls = robust != 0.0;
  if (!pred || !sparse || !workspace || !nodes || !records || !sparse_shape_ok(b, h, w, grid_y, grid_x) ||
      !metric_mask_ok(mask, mask_dtype) || !aligned(pred, 4) || !aligned(sparse, 4) || !aligned(workspace, 8) ||
      !aligned(nodes, 8) || !aligned(records, 8) || !sparse_range_ok(space, min_depth, max_depth) ||
      !std::isfinite(smooth) || smooth < 0.0 || (grid_y * grid_x > 1 && !(smooth > 0.0)) || !std::isfinite(robust) ||
      robust < 0.0 || (irls ? iterations < 2 || iterations > 32 : iterations != 1))
    return fail(ODB_ERR_INVALID, "sparse_align_fit: bad argument");
  const SparseGeom G = sparse_geom(h, w, grid_y, grid_x);
  const int regions = (grid_y + 1) * (grid_x + 1), per_region = G.ncy * G.ncx, chunks = regions * per_region;
  double* part = static_cast<double*>(workspace);
  double* mom = part + (long long)b * chunks * kMomStride;
  double* band_ws = mom + (long long)b * regions * kMomStride;
  const size_t n = 2 * (size_t)grid_y * grid_x;
  const bool in_smem = sparse_smem_bytes(grid_y, grid_x) <= kBandSmemMax;
  const size_t smem = in_smem ? sparse_smem_bytes(grid_y, grid_x) : n * sizeof(double);
  static bool configured[kMaxDevices] = {};
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(sparse_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kBandSmemMax);
    if (e != cudaSuccess) return fail_cuda(e, "sparse_align_fit: cudaFuncSetAttribute");
    configured[dev] = true;
  }
  const int disp = space == ODB_SPACE_DISPARITY ? 1 : 0;
  // iterations solves, then the residual pass of the final nodes
  for (int it = 0; it <= iterations; ++it) {
    const bool last = it == iterations;
    sparse_moments_kernel<<<dim3(chunks, b), kSparseThreads, 0, stream>>>(
        pred, sparse, mask, mask_dtype, G, disp, min_depth, max_depth, it > 0 ? nodes : nullptr, last ? 0.0 : robust,
        part);
    count_launch();
    sparse_reduce_kernel<<<dim3(regions, b), kSparseThreads, 0, stream>>>(part, per_region, mom);
    count_launch();
    if (last) {
      sparse_record_kernel<<<b, kSparseThreads, 0, stream>>>(mom, regions, records);
    } else {
      sparse_solve_kernel<<<b, kSparseThreads, smem, stream>>>(mom, grid_y, grid_x, smooth, in_smem ? 1 : 0, band_ws,
                                                               nodes, records);
    }
    count_launch();
  }
  return check_launch("sparse_align_fit");
}

extern "C" int odb_sparse_align_apply(const float* pred, const double* nodes, int32_t b, int32_t h, int32_t w,
                                      int32_t grid_y, int32_t grid_x, int32_t space, double min_depth,
                                      double max_depth, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!pred || !nodes || !out || !sparse_shape_ok(b, h, w, grid_y, grid_x) || !aligned(pred, 4) ||
      !aligned(nodes, 8) || !aligned(out, 4) || !sparse_range_ok(space, min_depth, max_depth))
    return fail(ODB_ERR_INVALID, "sparse_align_apply: bad argument");
  const int vec = w % 4 == 0 && aligned(pred, 16) && aligned(out, 16) ? 1 : 0;
  const int quads = (w + 3) / 4;
  sparse_apply_kernel<<<dim3((quads + kSparseThreads - 1) / kSparseThreads, h, b), kSparseThreads, 0, stream>>>(
      pred, nodes, h, w, grid_y, grid_x, space == ODB_SPACE_DISPARITY ? 1 : 0, min_depth, max_depth, vec, out);
  count_launch();
  return check_launch("sparse_align_apply");
}
