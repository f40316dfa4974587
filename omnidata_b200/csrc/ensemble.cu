// Test-time ensembling of depth and surface-normal predictions (omnidata_b200/ensemble.py EnsemblePredictor): K
// predictions of one image (input sizes x horizontal mirror) are put in one frame and merged per pixel.  Definitions in
// DESIGN.md §3 "Test-time ensembles"; oracle/ensemble_oracle.py restates them in float64.
//
// Members are fp32 [K][B][C][H][W], each as its predictor returned it resized to H x W, still mirrored where bit k of
// `flips` is set: every kernel reads member k at column W - 1 - x for output column x (gather form), so no pass is spent
// on un-mirroring.  Member 0 is the reference frame.
//
//   depth:  ensemble_gram_kernel (fixed 4 096-pixel slabs) -> ensemble_gram_reduce_kernel (per image, fixed order)
//           -> ensemble_align_solve_kernel (one CTA per image: fp64 Cholesky of the 2 (K - 1) normal equations,
//              band_cholesky_solve at full band width)
//           -> ensemble_merge_depth_kernel<N> (per pixel: d_k = s_k a_k + t_k, median and MAD by a sorting network)
//   normal: ensemble_merge_normal_kernel (per pixel: normalised mean of the decoded, un-mirrored members)
//
// No floating-point atomics; the slab partition depends on H x W only, so every result is independent of the batch and
// repeat runs give the same bits.  Built without fast-math: the merges (and angle_deg, fp64.cuh) are written with
// explicit round-to-nearest fp64 operations so that the float64 oracle reproduces them operation by operation.
#include <cmath>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kEnsThreads = 256;
constexpr int kEnsSlabIters = kSlab / kEnsThreads;
constexpr int kEnsMaxK = ODB_ENSEMBLE_MAX_MEMBERS;
constexpr double kEnsKappa = 1e-6;

// Gram sums of the augmented member vector v = (a_0, ..., a_{K-1}, 1) over the pixels where all members are finite:
// the packed upper triangle of v^T v, (i, j) with i <= j <= K at tri(i, j); G(K, K) = n, G(k, K) = S a_k.
__host__ __device__ inline int gram_size(int k) { return (k + 1) * (k + 2) / 2; }
__host__ __device__ inline int tri(int i, int j, int k) { return i * (k + 1) - i * (i - 1) / 2 + (j - i); }

ODB_DEVINL long long member_index(long long plane, int y, int x, int W, bool flipped) {
  return plane + (long long)y * W + (flipped ? W - 1 - x : x);
}

// Slab partials part[b][slab][gram_size(K)].  Each 256-pixel step stages the K un-mirrored values of every pixel (zeros
// and a 0 in the ones-row where any member is not finite) in shared memory; thread (q, r) then adds the products of
// entry q over the pixels r, r + R, ... (R = 256 / gram_size replicas), and the R partials of q are added in replica
// order at the end.  Each member value is read from HBM once.  grid (slabs, B)
__global__ void __launch_bounds__(kEnsThreads) ensemble_gram_kernel(const float* __restrict__ members, int K, int flips,
                                                                    int B, int H, int W, double* __restrict__ part) {
  __shared__ float vals[kEnsMaxK + 1][kEnsThreads + 1];
  __shared__ double red[kEnsThreads];
  const int b = blockIdx.y, nq = gram_size(K), R = kEnsThreads / nq;
  const long long hw = (long long)H * W;
  const int q = threadIdx.x % nq, r = threadIdx.x / nq;
  int qi = 0, qj = 0;                                       // (i, j) of entry q
  for (int i = 0, e = 0; i <= K; ++i)
    for (int j = i; j <= K; ++j, ++e)
      if (e == q) qi = i, qj = j;
  double acc0 = 0.0, acc1 = 0.0;                            // two chains, added at the end in a fixed order
  for (int it = 0; it < kEnsSlabIters; ++it) {
    const long long i = blockIdx.x * kSlab + it * kEnsThreads + threadIdx.x;
    bool valid = i < hw;
    const int y = valid ? (int)(i / W) : 0, x = valid ? (int)(i - (long long)y * W) : 0;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      const float v = valid ? __ldg(members + member_index(((long long)k * B + b) * hw, y, x, W, (flips >> k) & 1)) : 0.0f;
      vals[k][threadIdx.x] = v;
      valid = valid && isfinite(v);
    }
    if (!valid)                                             // this thread's own column: no barrier needed
      for (int k = 0; k < K; ++k) vals[k][threadIdx.x] = 0.0f;
    vals[K][threadIdx.x] = valid ? 1.0f : 0.0f;
    __syncthreads();
    if (r < R) {
      int p = r;
      for (; p + R < kEnsThreads; p += 2 * R) {
        acc0 = fma((double)vals[qi][p], (double)vals[qj][p], acc0);
        acc1 = fma((double)vals[qi][p + R], (double)vals[qj][p + R], acc1);
      }
      if (p < kEnsThreads) acc0 = fma((double)vals[qi][p], (double)vals[qj][p], acc0);
    }
    __syncthreads();
  }
  red[threadIdx.x] = acc0 + acc1;
  __syncthreads();
  if (threadIdx.x < nq) {
    double s = 0.0;
    for (int rr = 0; rr < R; ++rr) s += red[rr * nq + threadIdx.x];
    part[((long long)b * gridDim.x + blockIdx.x) * nq + threadIdx.x] = s;
  }
}

// gram[b][q] = the sum over the image's slabs of part[b][slab][q], by ordered_sum8 (fixed order).  grid (ceil(nq / 32), B)
__global__ void __launch_bounds__(256) ensemble_gram_reduce_kernel(const double* __restrict__ part, int slabs, int nq,
                                                                   double* __restrict__ gram) {
  const int b = blockIdx.y, q = blockIdx.x * 32 + (threadIdx.x & 31);
  const double* p = part + (long long)b * slabs * nq;
  const double s = ordered_sum8(slabs, q < nq, [&](int sl) { return p[(long long)sl * nq + q]; });
  if (threadIdx.x < 32 && q < nq) gram[(long long)b * nq + q] = s;
}

// One CTA per image.  Unknowns x = (s_1, t_1, ..., s_{K-1}, t_{K-1}), s_0 = 1, t_0 = 0.  With c_km = K [k = m] - 1,
// G_km = S a_k a_m, S_k = S a_k, n = |V| and kn = kappa n, the gradient of E set to zero reads, for m >= 1:
//   s_m: sum_{k>=1} c_km (G_km s_k + S_m t_k) + kn s_m = kn + G_0m
//   t_m: sum_{k>=1} c_km (S_k s_k + n t_k)   + kn t_m = S_0
// (E = K sum_k |d_k|^2 - |sum_k d_k|^2 + kappa n sum_{k>=1} ((s_k - 1)^2 + t_k^2), d_k = s_k a_k + t_k).  The lower
// triangle is assembled as a band of full width M (band_cholesky_solve, fp64.cuh).  scale_shift[b][k] = (s_k, t_k).
__global__ void __launch_bounds__(kEnsThreads) ensemble_align_solve_kernel(const double* __restrict__ gram, int K,
                                                                           double* __restrict__ scale_shift) {
  constexpr int kM = 2 * (kEnsMaxK - 1);
  __shared__ double band[kM * kM];
  __shared__ double rhs[kM];
  const int b = blockIdx.x, M = 2 * (K - 1), nq = gram_size(K);
  const double* G = gram + (long long)b * nq;
  const double n = G[tri(K, K, K)], kn = kEnsKappa * n;
  for (int e = threadIdx.x; e < M * M; e += blockDim.x) {
    const int row = e / M, col = e - row * M, m = row / 2 + 1, k = col / 2 + 1;
    if (col > row) continue;
    const double c = (k == m ? (double)K : 0.0) - 1.0, ridge = (k == m && (row & 1) == (col & 1)) ? kn : 0.0;
    double g;
    if ((row & 1) == 0) g = (col & 1) == 0 ? G[tri(min(k, m), max(k, m), K)] : G[tri(m, K, K)];
    else g = (col & 1) == 0 ? G[tri(k, K, K)] : n;
    band[row * M + (row - col)] = c * g + ridge;
  }
  for (int row = threadIdx.x; row < M; row += blockDim.x)
    rhs[row] = (row & 1) == 0 ? kn + G[tri(0, row / 2 + 1, K)] : G[tri(0, K, K)];
  __syncthreads();
  band_cholesky_solve(band, rhs, M, M);
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    double* st = scale_shift + ((long long)b * K + k) * 2;
    st[0] = k == 0 ? 1.0 : rhs[2 * (k - 1)];
    st[1] = k == 0 ? 0.0 : rhs[2 * (k - 1) + 1];
  }
}

// Ascending bitonic sorting network over N (a power of two) registers; fully unrolled, so every index is static.
template <int N>
ODB_DEVINL void sort_network(float (&v)[N]) {
  constexpr int kLog = N == 2 ? 1 : N == 4 ? 2 : N == 8 ? 3 : 4;
  static_assert(N == 1 << kLog, "N must be 2, 4, 8 or 16");
#pragma unroll
  for (int lk = 1; lk <= kLog; ++lk) {
#pragma unroll
    for (int lj = lk - 1; lj >= 0; --lj) {
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const int k = 1 << lk, l = i ^ (1 << lj);
        if (l > i) {
          const float a = v[i], c = v[l];
          const bool up = (i & k) == 0;
          v[i] = up ? fminf(a, c) : fmaxf(a, c);
          v[l] = up ? fmaxf(a, c) : fminf(a, c);
        }
      }
    }
  }
}

// the median of v[0..K-1] after sorting (v[K..N-1] = +inf): the middle value, or the fp32 mean of the two middle values
template <int N>
ODB_DEVINL float median_of(float (&v)[N], int K) {
  sort_network<N>(v);
  // v ascending, so v[r] = max_{i <= r} v[i]: maxima instead of a pick at a run-time index, which the compiler would
  // turn into an indexed load from a local-memory copy of v
  float lo = -INFINITY, hi = -INFINITY;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    lo = fmaxf(lo, i <= (K - 1) / 2 ? v[i] : -INFINITY);
    hi = fmaxf(hi, i <= K / 2 ? v[i] : -INFINITY);
  }
  return (K & 1) ? lo : __fmul_rn(__fadd_rn(lo, hi), 0.5f);
}

// Loads the 4 values of member k at output columns x0..x0+3 of row y (un-mirrored): one 16-byte load when `vec`
// (W % 4 == 0 and 16-byte aligned planes: a mirrored quad is also an aligned quad, reversed), else scalar loads with
// columns past W read as column W - 1.
ODB_DEVINL float4 load_quad(const float* __restrict__ plane, int y, int x0, int W, bool flipped, bool vec) {
  const float* row = plane + (long long)y * W;
  if (vec) {
    if (!flipped) return __ldg(reinterpret_cast<const float4*>(row + x0));
    const float4 q = __ldg(reinterpret_cast<const float4*>(row + (W - 4 - x0)));
    return make_float4(q.w, q.z, q.y, q.x);
  }
  float e[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int x = min(x0 + u, W - 1);
    e[u] = __ldg(row + (flipped ? W - 1 - x : x));
  }
  return make_float4(e[0], e[1], e[2], e[3]);
}

ODB_DEVINL float quad_get(const float4& q, int u) { return u == 0 ? q.x : u == 1 ? q.y : u == 2 ? q.z : q.w; }
ODB_DEVINL void quad_set(float4& q, int u, float v) {
  if (u == 0) q.x = v; else if (u == 1) q.y = v; else if (u == 2) q.z = v; else q.w = v;
}
ODB_DEVINL void store_quad(float* __restrict__ row, int x0, int W, bool vec, const float4& q) {
  if (vec) {
    *reinterpret_cast<float4*>(row + x0) = q;
    return;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (x0 + u < W) row[x0 + u] = quad_get(q, u);
}

// Depth merge, one thread per 4 consecutive pixels of a row.  Where all K members are finite: d_k = fp32(s_k a_k + t_k)
// (fp64, round-to-nearest, one rounding to fp32), out = median_k d_k, spread = median_k |d_k - out| (fp32); elsewhere
// out = member 0, spread = NaN.  N = the power of two >= K; pads are +inf.  grid (ceil(H ceil(W / 4) / 256), B)
template <int N>
__global__ void __launch_bounds__(kEnsThreads) ensemble_merge_depth_kernel(const float* __restrict__ members,
                                                                           const double* __restrict__ scale_shift,
                                                                           int K, int flips, int B, int H, int W,
                                                                           int vec, float* __restrict__ out,
                                                                           float* __restrict__ spread) {
  __shared__ double st[2 * kEnsMaxK];
  const int b = blockIdx.y;
  for (int e = threadIdx.x; e < 2 * K; e += blockDim.x) st[e] = scale_shift[(long long)b * 2 * K + e];
  __syncthreads();
  const int Q = (W + 3) / 4;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)H * Q) return;
  const int y = (int)(e / Q), x0 = (int)(e - (long long)y * Q) * 4;
  const long long hw = (long long)H * W;
  float4 a[N];                                              // all members' quads are loaded before any is used
#pragma unroll
  for (int k = 0; k < N; ++k)
    if (k < K) a[k] = load_quad(members + ((long long)k * B + b) * hw, y, x0, W, (flips >> k) & 1, vec != 0);
  float4 o, sp;
#pragma unroll 1
  for (int u = 0; u < 4; ++u) {
    float d[N];
    bool valid = true;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      d[k] = INFINITY;
      if (k < K) {
        const float v = quad_get(a[k], u);
        valid = valid && isfinite(v);
        d[k] = (float)__dadd_rn(__dmul_rn(st[2 * k], (double)v), st[2 * k + 1]);
      }
    }
    float m = quad_get(a[0], u), dev = NAN;
    if (valid) {
      m = median_of<N>(d, K);
#pragma unroll
      for (int k = 0; k < N; ++k) d[k] = k < K ? fabsf(__fsub_rn(d[k], m)) : INFINITY;
      dev = median_of<N>(d, K);
    }
    quad_set(o, u, m);
    quad_set(sp, u, dev);
  }
  store_quad(out + (long long)b * hw + (long long)y * W, x0, W, vec != 0, o);
  if (spread != nullptr) store_quad(spread + (long long)b * hw + (long long)y * W, x0, W, vec != 0, sp);
}

ODB_DEVINL double clamp01(float v) { return (double)fminf(fmaxf(v, 0.0f), 1.0f); }     // a NaN component clamps to 0
ODB_DEVINL double decode(float v) { return __dsub_rn(__dmul_rn(2.0, clamp01(v)), 1.0); }

// Normal merge, one thread per 4 consecutive pixels of a row.  Member k decoded as n_k = 2 clamp(c, 0, 1) - 1, x
// negated where mirrored; m = (S_k n_k) / K; out = (m / |m| + 1) / 2 in fp64, rounded once to fp32, or member 0's
// clamped value where |m| <= 1e-6.  spread = (S_k theta_k) / K in degrees, theta_k = atan2(|n_k x o|, n_k . o) with
// o = 2 out - 1 (a second pass over the members, only when spread is wanted).  grid (ceil(H ceil(W / 4) / 256), B)
__global__ void __launch_bounds__(kEnsThreads) ensemble_merge_normal_kernel(const float* __restrict__ members, int K,
                                                                            int flips, int B, int H, int W, int vec,
                                                                            float* __restrict__ out,
                                                                            float* __restrict__ spread) {
  const int Q = (W + 3) / 4;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)H * Q) return;
  const int b = blockIdx.y, y = (int)(e / Q), x0 = (int)(e - (long long)y * Q) * 4;
  const long long hw = (long long)H * W;
  double m[4][3] = {};
  float4 c0[3];
  for (int k = 0; k < K; ++k) {
    const bool fl = (flips >> k) & 1;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4 a = load_quad(members + (((long long)k * B + b) * 3 + c) * hw, y, x0, W, fl, vec != 0);
      if (k == 0) c0[c] = a;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double n = decode(quad_get(a, u));
        m[u][c] = __dadd_rn(m[u][c], (c == 0 && fl) ? -n : n);
      }
    }
  }
  double o[4][3];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    double v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __ddiv_rn(m[u][c], (double)K);
    const double norm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])),
                                             __dmul_rn(v[2], v[2])));
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float r = norm <= 1e-6 ? (float)clamp01(quad_get(c0[c], u))
                                   : (float)__dmul_rn(__dadd_rn(__ddiv_rn(v[c], norm), 1.0), 0.5);
      quad_set(c0[c], u, r);                                 // c0 now holds the output
      o[u][c] = __dsub_rn(__dmul_rn(2.0, (double)r), 1.0);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) store_quad(out + ((long long)b * 3 + c) * hw + (long long)y * W, x0, W, vec != 0, c0[c]);
  if (spread == nullptr) return;
  double th[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < K; ++k) {
    const bool fl = (flips >> k) & 1;
    double n[4][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4 a = load_quad(members + (((long long)k * B + b) * 3 + c) * hw, y, x0, W, fl, vec != 0);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double v = decode(quad_get(a, u));
        n[u][c] = (c == 0 && fl) ? -v : v;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) th[u] = __dadd_rn(th[u], angle_deg(n[u], o[u]));
  }
  float4 sp;
#pragma unroll
  for (int u = 0; u < 4; ++u) quad_set(sp, u, (float)__ddiv_rn(th[u], (double)K));
  store_quad(spread + (long long)b * hw + (long long)y * W, x0, W, vec != 0, sp);
}

static bool ens_geometry_ok(int32_t k, int32_t b, int32_t h, int32_t w) {
  return k >= 1 && k <= kEnsMaxK && planes_ok(b, h, w);
}
static bool ens_flips_ok(int32_t k, int32_t flips) { return flips >= 0 && (flips >> k) == 0 && (flips & 1) == 0; }
// 16-byte accesses: rows of a multiple of 4 floats and 16-byte aligned buffers
static bool ens_vec(int32_t w, const void* members, const void* out, const void* spread) {
  return w % 4 == 0 && aligned(members, 16) && aligned(out, 16) && (!spread || aligned(spread, 16));
}
static dim3 merge_grid(int32_t b, int32_t h, int32_t w) {
  const long long quads = (long long)h * ((w + 3) / 4);
  return dim3((unsigned)((quads + kEnsThreads - 1) / kEnsThreads), b);
}

template <int N>
static void launch_merge_depth(const float* members, const double* st, int32_t k, int32_t flips, int32_t b, int32_t h,
                               int32_t w, int vec, float* out, float* spread, cudaStream_t stream) {
  ensemble_merge_depth_kernel<N><<<merge_grid(b, h, w), kEnsThreads, 0, stream>>>(members, st, k, flips, b, h, w, vec,
                                                                                  out, spread);
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_ensemble_gram_workspace_bytes(int32_t k, int32_t b, int32_t h, int32_t w) {
  if (!ens_geometry_ok(k, b, h, w)) return -1;
  return (int64_t)b * slab_count(h, w) * gram_size(k) * (int64_t)sizeof(double);
}

extern "C" int odb_ensemble_gram(const float* members, int32_t k, int32_t flips, int32_t b, int32_t h, int32_t w,
                                 void* workspace, double* gram, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!members || !workspace || !gram || !ens_geometry_ok(k, b, h, w) || !ens_flips_ok(k, flips) ||
      !aligned(members, 4) || !aligned(workspace, 8) || !aligned(gram, 8))
    return fail(ODB_ERR_INVALID, "ensemble_gram: bad argument");
  const int slabs = slab_count(h, w), nq = gram_size(k);
  double* part = static_cast<double*>(workspace);
  ensemble_gram_kernel<<<dim3(slabs, b), kEnsThreads, 0, stream>>>(members, k, flips, b, h, w, part);
  count_launch();
  ensemble_gram_reduce_kernel<<<dim3((nq + 31) / 32, b), 256, 0, stream>>>(part, slabs, nq, gram);
  count_launch();
  return check_launch("ensemble_gram");
}

extern "C" int odb_ensemble_align_solve(const double* gram, int32_t k, int32_t b, double* scale_shift, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!gram || !scale_shift || !ens_geometry_ok(k, b, 1, 1) || !aligned(gram, 8) || !aligned(scale_shift, 8))
    return fail(ODB_ERR_INVALID, "ensemble_align_solve: bad argument");
  ensemble_align_solve_kernel<<<b, kEnsThreads, 0, stream>>>(gram, k, scale_shift);
  count_launch();
  return check_launch("ensemble_align_solve");
}

extern "C" int odb_ensemble_merge_depth(const float* members, const double* scale_shift, int32_t k, int32_t flips,
                                        int32_t b, int32_t h, int32_t w, float* out, float* spread, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!members || !scale_shift || !out || !ens_geometry_ok(k, b, h, w) || !ens_flips_ok(k, flips) ||
      !aligned(members, 4) || !aligned(out, 4) || !aligned(spread, 4) || !aligned(scale_shift, 8))
    return fail(ODB_ERR_INVALID, "ensemble_merge_depth: bad argument");
  const int vec = ens_vec(w, members, out, spread) ? 1 : 0;
  if (k <= 2) launch_merge_depth<2>(members, scale_shift, k, flips, b, h, w, vec, out, spread, stream);
  else if (k <= 4) launch_merge_depth<4>(members, scale_shift, k, flips, b, h, w, vec, out, spread, stream);
  else if (k <= 8) launch_merge_depth<8>(members, scale_shift, k, flips, b, h, w, vec, out, spread, stream);
  else launch_merge_depth<16>(members, scale_shift, k, flips, b, h, w, vec, out, spread, stream);
  count_launch();
  return check_launch("ensemble_merge_depth");
}

extern "C" int odb_ensemble_merge_normal(const float* members, int32_t k, int32_t flips, int32_t b, int32_t h, int32_t w,
                                         float* out, float* spread, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!members || !out || !ens_geometry_ok(k, b, h, w) || !ens_flips_ok(k, flips) || !aligned(members, 4) ||
      !aligned(out, 4) || !aligned(spread, 4))
    return fail(ODB_ERR_INVALID, "ensemble_merge_normal: bad argument");
  const int vec = ens_vec(w, members, out, spread) ? 1 : 0;
  ensemble_merge_normal_kernel<<<merge_grid(b, h, w), kEnsThreads, 0, stream>>>(members, k, flips, b, h, w, vec, out,
                                                                                spread);
  count_launch();
  return check_launch("ensemble_merge_normal");
}
