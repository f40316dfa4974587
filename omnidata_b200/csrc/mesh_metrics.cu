// Mesh metrics (omnidata_b200/mesh.py, omnidata_b200/metrics.py MeshMetrics): surface sampling of triangle meshes,
// exact nearest neighbours between point sets, frustum culling and the accuracy / completion / F-score of a
// reconstructed mesh against a ground-truth mesh.  Definitions in DESIGN.md §3 "Mesh metrics" and
// include/omnidata_b200.h; oracle/mesh_oracle.py restates them in float64.
//
//   sample_count_kernel   one thread per face: area, sample count floor(A rho + xi), bad-index / non-finite flags
//   scan_*_kernel         integer exclusive scan (tile sums, one CTA over the tiles, tile-local scan)
//   sample_emit_kernel    one thread per sample: binary search of the face offsets, then the sample's position
//   nn_box_kernel         bounding box of the reference set by integer atomicMin / atomicMax on order-preserving keys
//   nn_count_kernel / nn_scatter_kernel   a uniform grid over the box: per-cell counts (integer atomics), scan, scatter
//   nn_query_kernel       one thread per query: Chebyshev rings of cells until no unexamined cell can hold a point as
//                         near as the best one
//   frustum_kernel        one thread per point, the cameras' poses read from device memory
//   compact_scatter_kernel   order-preserving compaction after a scan of the mask
//   mm_slab_kernel / mm_fold_kernel   per-slab fp64 sums and counts of the distances, metrics.cu's ordered slab
//                         reduction, one thread folding the scene's record into the state
//
// Explicit round-to-nearest fp64 operations (no contraction) wherever the oracle reproduces a result bit for bit.
// Integer atomics only (the box, the grid's counts and the scatter, whose order within a cell no output depends on);
// no floating-point atomics.  Built without fast-math.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "select.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {
namespace {

constexpr int kT = 256;                       // threads of the elementwise and scan kernels
constexpr int kItems = 8;                     // items per thread of a scan tile
constexpr int kTile = kT * kItems;
constexpr long long kMaxSampleCount = 1ll << 31;   // a face's count is clamped here before the scan (no overflow)

// ---------------------------------------------------------------------------------------------------- scan
template <typename T>
ODB_DEVINL T block_scan_excl(T v, T& total) {
  __shared__ T warp_tot[kT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += t;
  }
  if (lane == 31) warp_tot[wid] = s;
  __syncthreads();
  T before = 0;
  total = 0;
#pragma unroll
  for (int q = 0; q < kT / 32; ++q) {
    const T t = warp_tot[q];
    before += q < wid ? t : 0;
    total += t;
  }
  __syncthreads();
  return before + s - v;
}

// the value an input adds to the scan: itself, or for a uint8 mask 1 where it is nonzero (a mask may hold 255)
template <typename T, typename In>
ODB_DEVINL T scan_value(In v) {
  return (T)v;
}
template <>
ODB_DEVINL long long scan_value<long long, unsigned char>(unsigned char v) {
  return v != 0 ? 1 : 0;
}

// tile_sum[tile] = the sum of the tile's kTile inputs
template <typename In, typename T>
__global__ void __launch_bounds__(kT) scan_tile_kernel(const In* __restrict__ in, long long n, T* __restrict__ tile_sum) {
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems;
  T s = 0;
#pragma unroll
  for (int k = 0; k < kItems; ++k)
    if (base + k < n) s += scan_value<T>(in[base + k]);
  T total;
  block_scan_excl(s, total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// one CTA of 1024 threads: tile_sum becomes its exclusive scan in place, total[0] the grand total
template <typename T>
__global__ void __launch_bounds__(1024) scan_top_kernel(T* __restrict__ tile_sum, long long tiles,
                                                        T* __restrict__ total) {
  __shared__ T run[1024];
  const long long per = (tiles + 1023) / 1024, b0 = min(tiles, threadIdx.x * per), b1 = min(tiles, b0 + per);
  T sum = 0;
  for (long long b = b0; b < b1; ++b) sum += tile_sum[b];
  run[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    T acc = 0;
    for (int t = 0; t < 1024; ++t) {
      const T v = run[t];
      run[t] = acc;
      acc += v;
    }
    total[0] = acc;
  }
  __syncthreads();
  T acc = run[threadIdx.x];
  for (long long b = b0; b < b1; ++b) {
    const T v = tile_sum[b];
    tile_sum[b] = acc;
    acc += v;
  }
}

// out[i] = tile_base[tile] + the exclusive scan of the tile's inputs before i
template <typename In, typename T>
__global__ void __launch_bounds__(kT) scan_apply_kernel(const In* __restrict__ in, long long n,
                                                        const T* __restrict__ tile_base, T* __restrict__ out) {
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems;
  T v[kItems];
  T s = 0;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    v[k] = base + k < n ? scan_value<T>(in[base + k]) : (T)0;
    s += v[k];
  }
  T total;
  T acc = tile_base[blockIdx.x] + block_scan_excl(s, total);
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    if (base + k < n) out[base + k] = acc;
    acc += v[k];
  }
}

long long scan_tiles(long long n) { return (n + kTile - 1) / kTile; }

// out[0..n) = the exclusive scan of in, total[0] = the sum (device); tiles: scan_tiles(n) entries of scratch
template <typename In, typename T>
void exclusive_scan(const In* in, long long n, T* tiles, T* out, T* total, cudaStream_t stream) {
  const long long nt = scan_tiles(n);
  if (nt) {
    scan_tile_kernel<In, T><<<(unsigned)nt, kT, 0, stream>>>(in, n, tiles);
    count_launch();
  }
  scan_top_kernel<T><<<1, 1024, 0, stream>>>(tiles, nt, total);
  count_launch();
  if (nt) {
    scan_apply_kernel<In, T><<<(unsigned)nt, kT, 0, stream>>>(in, n, tiles, out);
    count_launch();
  }
}

// ---------------------------------------------------------------------------------------------------- sampling
__host__ __device__ inline unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the uniform draw j of face t: (splitmix64(splitmix64(key ^ t) ^ j) >> 11) 2^-53, key = splitmix64(splitmix64(seed)
// ^ stream); j = 0 for the count's xi, 2k + 1 and 2k + 2 for sample k's r1, r2
ODB_DEVINL double draw(unsigned long long key, unsigned long long t, unsigned long long j) {
  return (double)(splitmix64(splitmix64(key ^ t) ^ j) >> 11) * 0x1p-53;
}

struct Tri {
  double a[3], b[3], c[3];
};

ODB_DEVINL Tri load_tri(const float* V, int i0, int i1, int i2) {
  Tri T;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    T.a[q] = V[3ll * i0 + q];
    T.b[q] = V[3ll * i1 + q];
    T.c[q] = V[3ll * i2 + q];
  }
  return T;
}

__global__ void __launch_bounds__(kT) sample_count_kernel(const float* __restrict__ V, long long nv,
                                                          const int* __restrict__ F, long long nf, double rho,
                                                          unsigned long long key, long long* __restrict__ cnt,
                                                          unsigned long long* __restrict__ flags) {
  const long long t = (long long)blockIdx.x * kT + threadIdx.x;
  if (t >= nf) return;
  const int i0 = F[3 * t], i1 = F[3 * t + 1], i2 = F[3 * t + 2];
  if (i0 < 0 || i1 < 0 || i2 < 0 || i0 >= nv || i1 >= nv || i2 >= nv) {
    atomicOr(flags, 1ull);
    cnt[t] = 0;
    return;
  }
  const Tri T = load_tri(V, i0, i1, i2);
  bool finite = true;
#pragma unroll
  for (int q = 0; q < 3; ++q) finite = finite && isfinite(T.a[q]) && isfinite(T.b[q]) && isfinite(T.c[q]);
  if (!finite) {
    atomicOr(flags, 2ull);
    cnt[t] = 0;
    return;
  }
  double e1[3], e2[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    e1[q] = __dsub_rn(T.b[q], T.a[q]);
    e2[q] = __dsub_rn(T.c[q], T.a[q]);
  }
  const double cx = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
  const double cy = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
  const double cz = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
  const double area =
      __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))));
  const double x = floor(__dadd_rn(__dmul_rn(area, rho), draw(key, (unsigned long long)t, 0ull)));
  cnt[t] = x < (double)kMaxSampleCount ? (long long)x : kMaxSampleCount;     // NaN (inf - inf) too
}

__global__ void __launch_bounds__(kT) sample_emit_kernel(const float* __restrict__ V, const int* __restrict__ F,
                                                         long long nf, const long long* __restrict__ off,
                                                         long long total, unsigned long long key,
                                                         float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= total) return;
  long long lo = 0, hi = nf - 1;                  // the last face whose offset is <= i (empty faces share offsets)
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  const long long t = lo, k = i - off[lo];
  const Tri T = load_tri(V, F[3 * t], F[3 * t + 1], F[3 * t + 2]);
  const double r1 = draw(key, (unsigned long long)t, 2ull * (unsigned long long)k + 1ull);
  const double r2 = draw(key, (unsigned long long)t, 2ull * (unsigned long long)k + 2ull);
  const double s = __dsqrt_rn(r1);
  const double w0 = __dsub_rn(1.0, s), w1 = __dmul_rn(s, __dsub_rn(1.0, r2)), w2 = __dmul_rn(s, r2);
#pragma unroll
  for (int q = 0; q < 3; ++q)
    out[3 * i + q] =
        (float)__dadd_rn(__dadd_rn(__dmul_rn(w0, T.a[q]), __dmul_rn(w1, T.b[q])), __dmul_rn(w2, T.c[q]));
}

// ---------------------------------------------------------------------------------------------------- nearest
// order-preserving int key of a float (-0 below +0) and its inverse
ODB_DEVINL int float_key(float x) {
  const int b = __float_as_int(x);
  return b >= 0 ? b : b ^ 0x7FFFFFFF;
}

struct Grid {
  double lo[3], hi[3], h;
  int n[3];
};

// the cell of a point along axis a: clamp(floor((p - lo) / h), 0, n - 1), the same expression for points and queries
ODB_DEVINL int cell_axis(const Grid& G, double p, int a) {
  const double g = floor(__ddiv_rn(__dsub_rn(p, G.lo[a]), G.h));
  return (int)fmin(fmax(g, 0.0), (double)(G.n[a] - 1));
}
ODB_DEVINL long long cell_of(const Grid& G, double x, double y, double z) {
  return ((long long)cell_axis(G, z, 2) * G.n[1] + cell_axis(G, y, 1)) * G.n[0] + cell_axis(G, x, 0);
}

// box[0..2] = min keys, box[3..5] = max keys of the reference set; box[6] |= 1 for a non-finite reference point, 2 for
// a non-finite query
__global__ void nn_box_init_kernel(int* __restrict__ box) {
  if (threadIdx.x < 3) {
    box[threadIdx.x] = INT_MAX;
    box[3 + threadIdx.x] = INT_MIN;
  } else if (threadIdx.x == 3) {
    box[6] = 0;
  }
}

__global__ void __launch_bounds__(kT) nn_box_kernel(const float* __restrict__ R, long long nr,
                                                    const float* __restrict__ Q, long long nq, int* __restrict__ box) {
  int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN};
  int flag = 0;
  const long long stride = (long long)gridDim.x * kT, n = nr > nq ? nr : nq;
  for (long long i = (long long)blockIdx.x * kT + threadIdx.x; i < n; i += stride) {
    if (i < nr) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float v = R[3 * i + a];
        if (!isfinite(v)) flag |= 1;
        const int k = float_key(v);
        mn[a] = min(mn[a], k);
        mx[a] = max(mx[a], k);
      }
    }
    if (i < nq) {
#pragma unroll
      for (int a = 0; a < 3; ++a)
        if (!isfinite(Q[3 * i + a])) flag |= 2;
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  flag = (int)__reduce_or_sync(0xffffffffu, (unsigned)flag);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (mn[a] != INT_MAX) atomicMin(box + a, mn[a]);
      if (mx[a] != INT_MIN) atomicMax(box + 3 + a, mx[a]);
    }
    if (flag) atomicOr(box + 6, flag);
  }
}

__global__ void __launch_bounds__(kT) nn_count_kernel(const float* __restrict__ R, long long nr, Grid G,
                                                      int* __restrict__ cnt) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= nr) return;
  atomicAdd(cnt + cell_of(G, R[3 * i], R[3 * i + 1], R[3 * i + 2]), 1);
}

// pts[start[cell] + the point's rank among its cell's arrivals] = (x, y, z, index bits); the rank depends on
// scheduling, and no output depends on it (the tie rule of nn_query_kernel)
__global__ void __launch_bounds__(kT) nn_scatter_kernel(const float* __restrict__ R, long long nr, Grid G,
                                                        const int* __restrict__ start, int* __restrict__ fill,
                                                        float4* __restrict__ pts) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= nr) return;
  const float x = R[3 * i], y = R[3 * i + 1], z = R[3 * i + 2];
  const long long c = cell_of(G, x, y, z);
  pts[start[c] + atomicAdd(fill + c, 1)] = make_float4(x, y, z, __int_as_float((int)i));
}

// The lower bound of nn_query_kernel's stopping rule along axis A: the squared distance from q to the box [lo, hi] with
// axis A's range cut at the edge of ring r (each side where cells remain), widened by the margin.  g2: q's squared
// gaps to the whole box per axis.  Each step rounded to nearest.
template <int A>
ODB_DEVINL void ring_bound(const Grid& G, const double q[3], const int c[3], int r, double margin, const double g2[3],
                           double& bound, bool& more) {
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const int j = side ? c[A] + r + 1 : c[A] - r - 1;
    if (j < 0 || j >= G.n[A]) continue;
    more = true;
    double lo = G.lo[A], hi = G.hi[A];
    if (side)
      lo = fmax(lo, __dsub_rn(__dadd_rn(G.lo[A], __dmul_rn((double)j, G.h)), margin));
    else
      hi = fmin(hi, __dadd_rn(__dadd_rn(G.lo[A], __dmul_rn((double)(j + 1), G.h)), margin));
    const double g = fmax(0.0, fmax(__dsub_rn(lo, q[A]), __dsub_rn(q[A], hi)));
    double s = 0.0;
#pragma unroll
    for (int b = 0; b < 3; ++b) s = __dadd_rn(s, b == A ? __dmul_rn(g, g) : g2[b]);
    bound = fmin(bound, s);
  }
}

__global__ void __launch_bounds__(kT) nn_query_kernel(const float* __restrict__ Q, long long nq, Grid G,
                                                      const int* __restrict__ start, const float4* __restrict__ pts,
                                                      double* __restrict__ dist, int* __restrict__ index) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= nq) return;
  const double q[3] = {(double)Q[3 * i], (double)Q[3 * i + 1], (double)Q[3 * i + 2]};
  int c[3];
  double margin[3], g2[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    c[a] = cell_axis(G, q[a], a);
    margin[a] = 0x1p-40 * (fabs(G.lo[a]) + fabs(G.hi[a]) + G.h + fabs(q[a]));
    const double g = fmax(0.0, fmax(__dsub_rn(G.lo[a], q[a]), __dsub_rn(q[a], G.hi[a])));
    g2[a] = __dmul_rn(g, g);
  }
  double best = INFINITY;
  int bi = -1;
  for (int r = 0;; ++r) {
    const int z0 = max(c[2] - r, 0), z1 = min(c[2] + r, G.n[2] - 1);
    const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, G.n[1] - 1);
    for (int z = z0; z <= z1; ++z)
      for (int y = y0; y <= y1; ++y) {
        const bool face = z == c[2] - r || z == c[2] + r || y == c[1] - r || y == c[1] + r;
        const int xs = face ? 1 : 2 * r;
        for (int x = c[0] - r; x <= c[0] + r; x += xs) {
          if (x < 0 || x >= G.n[0]) continue;
          const long long cell = ((long long)z * G.n[1] + y) * G.n[0] + x;
          const int e = start[cell + 1];
          for (int j = start[cell]; j < e; ++j) {
            const float4 p = pts[j];
            const double dx = __dsub_rn(q[0], (double)p.x), dy = __dsub_rn(q[1], (double)p.y),
                         dz = __dsub_rn(q[2], (double)p.z);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            const int id = __float_as_int(p.w);
            if (d2 < best || (d2 == best && id < bi)) {
              best = d2;
              bi = id;
            }
          }
        }
      }
    // a lower bound on the squared distance to any point of an unexamined cell: such a cell lies beyond ring r along
    // some axis and side, so its points lie in the box with that axis's range cut at the ring's edge (widened by the
    // margin that covers the rounding of the cell expression and of these bounds)
    double bound = INFINITY;
    bool more = false;
    ring_bound<0>(G, q, c, r, margin[0], g2, bound, more);
    ring_bound<1>(G, q, c, r, margin[1], g2, bound, more);
    ring_bound<2>(G, q, c, r, margin[2], g2, bound, more);
    if (!more || best < __dmul_rn(bound, 1.0 - 0x1p-40)) break;
  }
  dist[i] = __dsqrt_rn(best);
  index[i] = bi;
}

__global__ void __launch_bounds__(kT) nn_empty_kernel(long long nq, double* __restrict__ dist,
                                                      int* __restrict__ index) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= nq) return;
  dist[i] = INFINITY;
  index[i] = -1;
}

// ---------------------------------------------------------------------------------------------------- culling
struct Cam {
  double fx, fy, cx, cy;
};

// mask[i] = 1 when some camera sees point i: odb_tsdf_integrate's projection and nearest-pixel rule, 0 < z <= max_depth
__global__ void __launch_bounds__(kT) frustum_kernel(const float* __restrict__ X, long long n,
                                                     const double* __restrict__ T, int frames, int h, int w, Cam K,
                                                     double max_depth, unsigned char* __restrict__ mask) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= n) return;
  const double x = X[3 * i], y = X[3 * i + 1], z = X[3 * i + 2];
  unsigned char seen = 0;
  for (int f = 0; f < frames && !seen; ++f) {
    const double* m = T + 16ll * f;
    const double dx = __dsub_rn(x, m[3]), dy = __dsub_rn(y, m[7]), dz = __dsub_rn(z, m[11]);
    const double zc = __dadd_rn(__dadd_rn(__dmul_rn(m[2], dx), __dmul_rn(m[6], dy)), __dmul_rn(m[10], dz));
    if (!(zc > 0.0 && zc <= max_depth)) continue;
    const double xc = __dadd_rn(__dadd_rn(__dmul_rn(m[0], dx), __dmul_rn(m[4], dy)), __dmul_rn(m[8], dz));
    const double yc = __dadd_rn(__dadd_rn(__dmul_rn(m[1], dx), __dmul_rn(m[5], dy)), __dmul_rn(m[9], dz));
    const double u = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fx, xc), zc), K.cx), 0.5));
    const double v = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fy, yc), zc), K.cy), 0.5));
    if (u >= 0.0 && u <= (double)(w - 1) && v >= 0.0 && v <= (double)(h - 1)) seen = 1;
  }
  mask[i] = seen;
}

__global__ void __launch_bounds__(kT) compact_scatter_kernel(const float* __restrict__ X, long long n,
                                                             const unsigned char* __restrict__ mask,
                                                             const long long* __restrict__ off,
                                                             float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kT + threadIdx.x;
  if (i >= n || !mask[i]) return;
  const long long o = off[i];
#pragma unroll
  for (int a = 0; a < 3; ++a) out[3 * o + a] = X[3 * i + a];
}

// ---------------------------------------------------------------------------------------------------- metrics
struct Thresholds {
  double t[ODB_MESH_MAX_THRESHOLDS];
};

// slab partials [slab][kPartStride] = (sum of d, #(d < t_0), ..., #(d < t_3)) over the slab's kSlab distances
__global__ void __launch_bounds__(kT) mm_slab_kernel(const double* __restrict__ d, long long n, Thresholds th, int nt,
                                                     double* __restrict__ part) {
  __shared__ double scratch[32];
  double acc[1 + ODB_MESH_MAX_THRESHOLDS] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < (int)(kSlab / kT); ++k) {
    const long long i = blockIdx.x * kSlab + k * kT + threadIdx.x;
    if (i >= n) continue;
    const double v = d[i];
    acc[0] += v;
#pragma unroll
    for (int q = 0; q < ODB_MESH_MAX_THRESHOLDS; ++q) acc[1 + q] += (q < nt && v < th.t[q]) ? 1.0 : 0.0;
  }
  double* out = part + (long long)blockIdx.x * kPartStride;
#pragma unroll
  for (int q = 0; q < 1 + ODB_MESH_MAX_THRESHOLDS; ++q) {
    const double r = block_sum_d(acc[q], scratch);
    if (threadIdx.x == 0) out[q] = r;
  }
}

// One thread: the scene's record and its fold into the state (include/omnidata_b200.h odb_mesh_metrics_update)
__global__ void mm_fold_kernel(const double* __restrict__ sp, const double* __restrict__ sg, long long np,
                               long long ng, int nt, long long culled_p, long long culled_g, double* __restrict__ rec,
                               double* __restrict__ sums, long long* __restrict__ counts) {
  if (threadIdx.x != 0) return;
  for (int q = 0; q < ODB_MESH_RECORD; ++q) rec[q] = NAN;
  rec[0] = (double)np;
  rec[1] = (double)ng;
  counts[0] += 1;
  counts[3] += np;
  counts[4] += ng;
  counts[5] += culled_p;
  counts[6] += culled_g;
  if (ng == 0) {
    counts[1] += 1;
    return;
  }
  const double dnp = (double)np, dng = (double)ng;
  for (int k = 0; k < nt; ++k) {
    const double P = np > 0 ? __ddiv_rn(sp[1 + k], dnp) : 0.0;
    const double R = __ddiv_rn(sg[1 + k], dng);
    const double s = __dadd_rn(P, R);
    const double F = s > 0.0 ? __ddiv_rn(__dmul_rn(__dmul_rn(2.0, P), R), s) : 0.0;
    rec[5 + 3 * k] = P;
    rec[6 + 3 * k] = R;
    rec[7 + 3 * k] = F;
    sums[3 + 3 * k] += P;
    sums[4 + 3 * k] += R;
    sums[5 + 3 * k] += F;
  }
  if (np == 0) {
    counts[2] += 1;
    return;
  }
  const double acc = __ddiv_rn(sp[0], dnp), comp = __ddiv_rn(sg[0], dng);
  const double ch = __dmul_rn(__dadd_rn(acc, comp), 0.5);
  rec[2] = acc;
  rec[3] = comp;
  rec[4] = ch;
  sums[0] += acc;
  sums[1] += comp;
  sums[2] += ch;
}

// ---------------------------------------------------------------------------------------------------- host
unsigned grid_1d(long long n) { return (unsigned)((n + kT - 1) / kT); }

bool points_ok(const float* p, long long n) { return n >= 0 && n <= ODB_MESH_MAX_POINTS && (n == 0 || (p && aligned(p, 4))); }

// the grid of (lo, hi, h) from a host array of 7 doubles; false unless finite, lo <= hi, h > 0 and at most
// ODB_NN_MAX_CELLS cells
bool grid_of(const double* g, Grid& G, long long& cells) {
  if (!g) return false;
  for (int q = 0; q < 7; ++q)
    if (!std::isfinite(g[q])) return false;
  if (!(g[6] > 0.0)) return false;
  cells = 1;
  for (int a = 0; a < 3; ++a) {
    if (!(g[a] <= g[3 + a])) return false;
    const double n = std::floor((g[3 + a] - g[a]) / g[6]) + 1.0;
    if (!(n <= (double)ODB_NN_MAX_CELLS)) return false;
    G.lo[a] = g[a];
    G.hi[a] = g[3 + a];
    G.n[a] = (int)n;
    cells *= G.n[a];
    if (cells > ODB_NN_MAX_CELLS) return false;
  }
  G.h = g[6];
  return true;
}

struct NnWs {
  int* start;       // [cells + 1]
  int* fill;        // [cells + 1]
  int* tiles;       // [scan_tiles(cells + 1)], then the total
  float4* pts;      // [n]
};
NnWs nn_ws(void* ws, long long n, long long cells) {
  NnWs W;
  W.pts = static_cast<float4*>(ws);
  W.start = reinterpret_cast<int*>(W.pts + n);
  W.fill = W.start + cells + 1;
  W.tiles = W.fill + cells + 1;
  return W;
}
long long nn_ws_bytes(long long n, long long cells) {
  return 16 * n + 4 * (2 * (cells + 1) + scan_tiles(cells + 1) + 1);
}

}  // namespace
}  // namespace odb

using namespace odb;

extern "C" int64_t odb_mesh_sample_workspace_bytes(int64_t faces) {
  if (faces < 0 || faces > INT_MAX) return -1;
  return 8 * (2 * faces + scan_tiles(faces));
}

static bool mesh_ok(const float* vertices, int64_t nv, const int32_t* faces, int64_t nf) {
  return nv >= 0 && nv <= INT_MAX && nf >= 0 && nf <= INT_MAX && (nv == 0 || (vertices && aligned(vertices, 4))) &&
         (nf == 0 || (faces && aligned(faces, 4)));
}

extern "C" int odb_mesh_sample_count(const float* vertices, int64_t nv, const int32_t* faces, int64_t nf,
                                     double density, int64_t seed, int64_t rng_stream, void* workspace, int64_t* info,
                                     void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!mesh_ok(vertices, nv, faces, nf) || !(std::isfinite(density) && density > 0.0) || !workspace || !info ||
      !aligned(workspace, 8) || !aligned(info, 8))
    return fail(ODB_ERR_INVALID, "mesh_sample_count: bad argument");
  long long* off = static_cast<long long*>(workspace);
  long long* cnt = off + nf;
  long long* tiles = cnt + nf;
  long long* total = reinterpret_cast<long long*>(info);
  const unsigned long long key = splitmix64(splitmix64((unsigned long long)seed) ^ (unsigned long long)rng_stream);
  cudaError_t e = cudaMemsetAsync(info, 0, 2 * sizeof(int64_t), stream);
  if (e != cudaSuccess) return fail_cuda(e, "mesh_sample_count");
  if (nf) {
    sample_count_kernel<<<grid_1d(nf), kT, 0, stream>>>(vertices, nv, faces, nf, density, key, cnt,
                                                        reinterpret_cast<unsigned long long*>(info + 1));
    count_launch();
  }
  exclusive_scan<long long, long long>(cnt, nf, tiles, off, total, stream);
  return check_launch("mesh_sample_count");
}

extern "C" int odb_mesh_sample_emit(const float* vertices, int64_t nv, const int32_t* faces, int64_t nf,
                                    int64_t seed, int64_t rng_stream, const void* workspace, int64_t total,
                                    float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!mesh_ok(vertices, nv, faces, nf) || !workspace || !aligned(workspace, 8) || total < 0 ||
      total > ODB_MESH_MAX_POINTS || (total > 0 && (nf == 0 || !out || !aligned(out, 4))))
    return fail(ODB_ERR_INVALID, "mesh_sample_emit: bad argument");
  const unsigned long long key = splitmix64(splitmix64((unsigned long long)seed) ^ (unsigned long long)rng_stream);
  if (total) {
    sample_emit_kernel<<<grid_1d(total), kT, 0, stream>>>(vertices, faces, nf,
                                                          static_cast<const long long*>(workspace), total, key, out);
    count_launch();
  }
  return check_launch("mesh_sample_emit");
}

extern "C" int odb_nn_bounds(const float* reference, int64_t n_ref, const float* query, int64_t n_query, int32_t* box,
                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!points_ok(reference, n_ref) || !points_ok(query, n_query) || !box || !aligned(box, 4))
    return fail(ODB_ERR_INVALID, "nn_bounds: bad argument");
  nn_box_init_kernel<<<1, 32, 0, stream>>>(box);
  count_launch();
  const long long n = n_ref > n_query ? n_ref : n_query;
  if (n) {
    const long long blocks = std::min<long long>(grid_1d(n), 8ll * num_sms());
    nn_box_kernel<<<(unsigned)blocks, kT, 0, stream>>>(reference, n_ref, query, n_query, box);
    count_launch();
  }
  return check_launch("nn_bounds");
}

extern "C" int64_t odb_nn_workspace_bytes(int64_t n_ref, const double* grid) {
  Grid G;
  long long cells;
  if (n_ref < 0 || n_ref > ODB_MESH_MAX_POINTS || !grid_of(grid, G, cells)) return -1;
  return nn_ws_bytes(n_ref, cells);
}

extern "C" int odb_nn_build(const float* reference, int64_t n_ref, const double* grid, void* workspace,
                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Grid G;
  long long cells;
  if (!points_ok(reference, n_ref) || !grid_of(grid, G, cells) || !workspace || !aligned(workspace, 16))
    return fail(ODB_ERR_INVALID, "nn_build: bad argument");
  const NnWs W = nn_ws(workspace, n_ref, cells);
  cudaError_t e = cudaMemsetAsync(W.fill, 0, 4 * (cells + 1), stream);
  if (e != cudaSuccess) return fail_cuda(e, "nn_build");
  if (n_ref) {
    nn_count_kernel<<<grid_1d(n_ref), kT, 0, stream>>>(reference, n_ref, G, W.fill);
    count_launch();
  }
  exclusive_scan<int, int>(W.fill, cells + 1, W.tiles, W.start, W.tiles + scan_tiles(cells + 1), stream);
  e = cudaMemsetAsync(W.fill, 0, 4 * (cells + 1), stream);
  if (e != cudaSuccess) return fail_cuda(e, "nn_build");
  if (n_ref) {
    nn_scatter_kernel<<<grid_1d(n_ref), kT, 0, stream>>>(reference, n_ref, G, W.start, W.fill, W.pts);
    count_launch();
  }
  return check_launch("nn_build");
}

extern "C" int odb_nn_query(const float* query, int64_t n_query, int64_t n_ref, const double* grid,
                            const void* workspace, double* distance, int32_t* index, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Grid G;
  long long cells;
  if (!points_ok(query, n_query) || n_ref < 0 || n_ref > ODB_MESH_MAX_POINTS ||
      (n_ref > 0 && (!grid_of(grid, G, cells) || !workspace || !aligned(workspace, 16))) ||
      (n_query > 0 && (!distance || !index || !aligned(distance, 8) || !aligned(index, 4))))
    return fail(ODB_ERR_INVALID, "nn_query: bad argument");
  if (n_query == 0) return check_launch("nn_query");
  if (n_ref == 0) {
    nn_empty_kernel<<<grid_1d(n_query), kT, 0, stream>>>(n_query, distance, index);
  } else {
    const NnWs W = nn_ws(const_cast<void*>(workspace), n_ref, cells);
    nn_query_kernel<<<grid_1d(n_query), kT, 0, stream>>>(query, n_query, G, W.start, W.pts, distance, index);
  }
  count_launch();
  return check_launch("nn_query");
}

extern "C" int odb_frustum_mask(const float* points, int64_t n, const double* cam_to_world, int32_t frames, int32_t h,
                                int32_t w, double fx, double fy, double cx, double cy, double max_depth,
                                uint8_t* mask, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!points_ok(points, n) || !cam_to_world || !aligned(cam_to_world, 8) || frames < 1 || !planes_ok(1, h, w) ||
      !(std::isfinite(fx) && fx > 0.0 && std::isfinite(fy) && fy > 0.0 && std::isfinite(cx) && std::isfinite(cy)) ||
      !(std::isfinite(max_depth) && max_depth > 0.0) || (n > 0 && !mask))
    return fail(ODB_ERR_INVALID, "frustum_mask: bad argument");
  if (n) {
    const Cam K = {fx, fy, cx, cy};
    frustum_kernel<<<grid_1d(n), kT, 0, stream>>>(points, n, cam_to_world, frames, h, w, K, max_depth, mask);
    count_launch();
  }
  return check_launch("frustum_mask");
}

extern "C" int64_t odb_compact_workspace_bytes(int64_t n) {
  if (n < 0 || n > ODB_MESH_MAX_POINTS) return -1;
  return 8 * (n + scan_tiles(n) + 1);
}

extern "C" int odb_compact_points(const float* points, const uint8_t* mask, int64_t n, void* workspace, float* out,
                                  int64_t* count, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!points_ok(points, n) || (n > 0 && (!mask || !out || !aligned(out, 4))) || !workspace ||
      !aligned(workspace, 8) || !count || !aligned(count, 8))
    return fail(ODB_ERR_INVALID, "compact_points: bad argument");
  long long* off = static_cast<long long*>(workspace);
  exclusive_scan<unsigned char, long long>(mask, n, off + n, off, reinterpret_cast<long long*>(count), stream);
  if (n) {
    compact_scatter_kernel<<<grid_1d(n), kT, 0, stream>>>(points, n, mask, off, out);
    count_launch();
  }
  return check_launch("compact_points");
}

extern "C" int64_t odb_mesh_metrics_workspace_bytes(int64_t n_pred, int64_t n_gt) {
  if (n_pred < 0 || n_gt < 0 || n_pred > ODB_MESH_MAX_POINTS || n_gt > ODB_MESH_MAX_POINTS) return -1;
  return ((n_pred + kSlab - 1) / kSlab + (n_gt + kSlab - 1) / kSlab + 2) * kPartStride * (int64_t)sizeof(double);
}

extern "C" int odb_mesh_metrics_update(const double* dist_pred, int64_t n_pred, const double* dist_gt, int64_t n_gt,
                                       const double* thresholds, int32_t n_thresholds, int64_t pred_culled,
                                       int64_t gt_culled, void* workspace, double* record, double* state_sums,
                                       int64_t* state_counts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Thresholds th = {{0.0, 0.0, 0.0, 0.0}};
  bool ok = thresholds && n_thresholds >= 1 && n_thresholds <= ODB_MESH_MAX_THRESHOLDS;
  for (int k = 0; ok && k < n_thresholds; ++k) {
    th.t[k] = thresholds[k];
    ok = std::isfinite(th.t[k]) && th.t[k] > 0.0;
  }
  if (!ok || n_pred < 0 || n_gt < 0 || n_pred > ODB_MESH_MAX_POINTS || n_gt > ODB_MESH_MAX_POINTS ||
      (n_pred > 0 && (!dist_pred || !aligned(dist_pred, 8))) || (n_gt > 0 && (!dist_gt || !aligned(dist_gt, 8))) ||
      pred_culled < 0 || gt_culled < 0 || !workspace || !record || !state_sums || !state_counts ||
      !aligned(workspace, 8) || !aligned(record, 8) || !aligned(state_sums, 8) || !aligned(state_counts, 8))
    return fail(ODB_ERR_INVALID, "mesh_metrics_update: bad argument");
  const int sp = (int)((n_pred + kSlab - 1) / kSlab), sg = (int)((n_gt + kSlab - 1) / kSlab);
  double* part = static_cast<double*>(workspace);
  double* rows = part + (long long)(sp + sg) * kPartStride;
  if (sp) {
    mm_slab_kernel<<<sp, kT, 0, stream>>>(dist_pred, n_pred, th, n_thresholds, part);
    count_launch();
  }
  if (sg) {
    mm_slab_kernel<<<sg, kT, 0, stream>>>(dist_gt, n_gt, th, n_thresholds, part + (long long)sp * kPartStride);
    count_launch();
  }
  launch_slab_reduce(part, 1, sp, 1 + ODB_MESH_MAX_THRESHOLDS, 0u, 0u, rows, stream);
  launch_slab_reduce(part + (long long)sp * kPartStride, 1, sg, 1 + ODB_MESH_MAX_THRESHOLDS, 0u, 0u,
                     rows + kPartStride, stream);
  mm_fold_kernel<<<1, 32, 0, stream>>>(rows, rows + kPartStride, n_pred, n_gt, n_thresholds, pred_culled, gt_culled,
                                       record, state_sums, reinterpret_cast<long long*>(state_counts));
  count_launch();
  return check_launch("mesh_metrics_update");
}
