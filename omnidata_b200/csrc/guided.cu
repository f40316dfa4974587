// Guided upsampling of a low-resolution prediction (omnidata_b200/guided.py GuidedPredictor): the fast guided filter
// (He & Sun 2015).  Definitions in DESIGN.md §3 "Guided upsampling"; oracle/guided_oracle.py restates them in float64.
//
// Inputs: guide g fp32 [b][3][h][w] (the image as the predictor received it), prediction p fp32 [b][C][h][w],
// full-resolution image x fp32 [b][3][H][W].  Window W_i = the pixels within Chebyshev distance r of i, clipped at the
// border; n_i = |W_i|; mean_W(f)_i = (S_{j in W_i} f_j) / n_i, the sum taken down each column (top to bottom), then
// along the row (left to right).
//
//   coefficients (fp64; four launches, thread per low-resolution pixel):
//     guided_box_v_products_kernel  column sums of the 9 + 4C products (g_k, g_k g_l for k <= l, p_c, g_k p_c)
//     guided_solve_kernel           row sums -> means; Sigma = mean(g g^T) - mu mu^T, v_c = mean(g p_c) - mu m_c;
//                                   a_c = (Sigma + eps I)^-1 v_c by a 3x3 Cholesky, b_c = m_c - a_c . mu
//     guided_box_v_kernel           column sums of the 4C planes (a_c0, a_c1, a_c2, b_c)
//     guided_box_h_mean_kernel      row sums -> means, rounded once to fp32: coef [b][4C][h][w], plane 4c + k
//   apply (fp32, one launch): guided_apply_kernel<C>.  coef resampled to H x W with ops.resize_bilinear's tables and
//   arithmetic (horizontal pass, fp32 FMAs in tap order, rounded to fp32, then the vertical pass), and
//     q_c = fma(A_c2, x_2, fma(A_c1, x_1, fma(A_c0, x_0, B_c)))
//   per output pixel.  The resampled coefficients live in registers and shared memory only.
//
// No floating-point atomics and a fixed summation order: results are bit-reproducible and independent of the batch.
// Built without fast-math.  A NaN or inf reaches every output whose windows or resampling taps touch it.
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kGuidedThreads = 128;      // coefficient kernels: one thread per pixel, 128 along a row
constexpr int kApplyQuads = 32;          // apply CTA: 32 column quads (128 columns) x 8 output rows
constexpr int kApplyRows = 8;
constexpr int kApplyStage = 16;          // source rows staged per pass (a band of 8 rows upsampled needs <= 6)

__host__ __device__ inline int guided_products(int c) { return 9 + 4 * c; }

// the clipped window [lo, hi] of index i along an axis of length n
ODB_DEVINL void window(int i, int r, int n, int& lo, int& hi) {
  lo = max(i - r, 0);
  hi = min(i + r, n - 1);
}

// Column sums of the products: ws[b][q][y][x] = S_{y' in [y-r, y+r]} prod_q(y', x), q in the order
// g0 g1 g2 | g0g0 g0g1 g0g2 g1g1 g1g2 g2g2 | p_0..p_{C-1} | g0p_c g1p_c g2p_c for c = 0..C-1.  Products of two fp32
// values are exact in fp64.  grid (ceil(w / 128), h, b)
template <int C>
__global__ void __launch_bounds__(kGuidedThreads) guided_box_v_products_kernel(const float* __restrict__ guide,
                                                                               const float* __restrict__ pred, int h,
                                                                               int w, int r, double* __restrict__ ws) {
  constexpr int NP = 9 + 4 * C;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const long long hw = (long long)h * w;
  const float* g = guide + (long long)b * 3 * hw + x;
  const float* p = pred + (long long)b * C * hw + x;
  double s[NP];
#pragma unroll
  for (int q = 0; q < NP; ++q) s[q] = 0.0;
  int lo, hi;
  window(y, r, h, lo, hi);
  for (int yy = lo; yy <= hi; ++yy) {
    const long long o = (long long)yy * w;
    const double g0 = __ldg(g + o), g1 = __ldg(g + hw + o), g2 = __ldg(g + 2 * hw + o);
    s[0] += g0; s[1] += g1; s[2] += g2;
    s[3] += g0 * g0; s[4] += g0 * g1; s[5] += g0 * g2; s[6] += g1 * g1; s[7] += g1 * g2; s[8] += g2 * g2;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const double pc = __ldg(p + c * hw + o);
      s[9 + c] += pc;
      s[9 + C + 3 * c] += g0 * pc;
      s[10 + C + 3 * c] += g1 * pc;
      s[11 + C + 3 * c] += g2 * pc;
    }
  }
  double* out = ws + (long long)b * NP * hw + (long long)y * w + x;
#pragma unroll
  for (int q = 0; q < NP; ++q) out[q * hw] = s[q];
}

// Row sums of the column sums -> window means, then the local linear model per pixel: a_c = (Sigma + eps I)^-1 v_c
// (Cholesky L L^T of the 3x3, forward and back substitution), b_c = m_c - a_c . mu.  coefs[b][4c + k][y][x] =
// a_ck (k < 3), b_c (k = 3).  grid (ceil(w / 128), h, b)
template <int C>
__global__ void __launch_bounds__(kGuidedThreads) guided_solve_kernel(const double* __restrict__ ws, int h, int w,
                                                                      int r, double eps,
                                                                      double* __restrict__ coefs) {
  constexpr int NP = 9 + 4 * C;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const long long hw = (long long)h * w;
  const double* src = ws + (long long)b * NP * hw + (long long)y * w;
  int ylo, yhi, xlo, xhi;
  window(y, r, h, ylo, yhi);
  window(x, r, w, xlo, xhi);
  const double n = (double)(yhi - ylo + 1) * (double)(xhi - xlo + 1);
  double m[NP];
#pragma unroll
  for (int q = 0; q < NP; ++q) {
    double s = 0.0;
    for (int xx = xlo; xx <= xhi; ++xx) s += src[q * hw + xx];
    m[q] = s / n;
  }
  const double mu0 = m[0], mu1 = m[1], mu2 = m[2];
  // A = Sigma + eps I, lower triangle
  const double a00 = m[3] - mu0 * mu0 + eps, a10 = m[4] - mu1 * mu0, a20 = m[5] - mu2 * mu0;
  const double a11 = m[6] - mu1 * mu1 + eps, a21 = m[7] - mu2 * mu1, a22 = m[8] - mu2 * mu2 + eps;
  const double l00 = sqrt(a00), l10 = a10 / l00, l20 = a20 / l00;
  const double l11 = sqrt(a11 - l10 * l10), l21 = (a21 - l20 * l10) / l11;
  const double l22 = sqrt(a22 - l20 * l20 - l21 * l21);
  double* out = coefs + (long long)b * 4 * C * hw + (long long)y * w + x;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const double mc = m[9 + c];
    const double v0 = m[9 + C + 3 * c] - mu0 * mc, v1 = m[10 + C + 3 * c] - mu1 * mc, v2 = m[11 + C + 3 * c] - mu2 * mc;
    const double z0 = v0 / l00, z1 = (v1 - l10 * z0) / l11, z2 = (v2 - l20 * z0 - l21 * z1) / l22;   // L z = v
    const double c2 = z2 / l22, c1 = (z1 - l21 * c2) / l11, c0 = (z0 - l10 * c1 - l20 * c2) / l00;  // L^T a = z
    out[(4 * c + 0) * hw] = c0;
    out[(4 * c + 1) * hw] = c1;
    out[(4 * c + 2) * hw] = c2;
    out[(4 * c + 3) * hw] = mc - (c0 * mu0 + c1 * mu1 + c2 * mu2);
  }
}

// Column sums of `planes` fp64 planes per image.  grid (ceil(w / 128), h, b)
__global__ void __launch_bounds__(kGuidedThreads) guided_box_v_kernel(const double* __restrict__ in, int planes, int h,
                                                                      int w, int r, double* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const long long hw = (long long)h * w;
  int lo, hi;
  window(y, r, h, lo, hi);
  for (int q = 0; q < planes; ++q) {
    const double* src = in + ((long long)b * planes + q) * hw + x;
    double s = 0.0;
    for (int yy = lo; yy <= hi; ++yy) s += src[(long long)yy * w];
    out[((long long)b * planes + q) * hw + (long long)y * w + x] = s;
  }
}

// Row sums of the column sums -> window means, rounded once to fp32.  grid (ceil(w / 128), h, b)
__global__ void __launch_bounds__(kGuidedThreads) guided_box_h_mean_kernel(const double* __restrict__ in, int planes,
                                                                           int h, int w, int r,
                                                                           float* __restrict__ coef) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const long long hw = (long long)h * w;
  int ylo, yhi, xlo, xhi;
  window(y, r, h, ylo, yhi);
  window(x, r, w, xlo, xhi);
  const double n = (double)(yhi - ylo + 1) * (double)(xhi - xlo + 1);
  for (int q = 0; q < planes; ++q) {
    const long long row = ((long long)b * planes + q) * hw + (long long)y * w;
    double s = 0.0;
    for (int xx = xlo; xx <= xhi; ++xx) s += in[row + xx];
    coef[row + x] = (float)(s / n);
  }
}

// Loads columns x0..x0+3 of a row: one 16-byte load when `vec`, else scalar loads with columns past W read as W - 1.
ODB_DEVINL float4 load4(const float* __restrict__ row, int x0, int W, bool vec) {
  if (vec) return __ldg(reinterpret_cast<const float4*>(row + x0));
  return make_float4(__ldg(row + min(x0, W - 1)), __ldg(row + min(x0 + 1, W - 1)), __ldg(row + min(x0 + 2, W - 1)),
                     __ldg(row + min(x0 + 3, W - 1)));
}

ODB_DEVINL float comp(const float4& v, int u) { return u == 0 ? v.x : u == 1 ? v.y : u == 2 ? v.z : v.w; }

ODB_DEVINL void store4(float* __restrict__ row, int x0, int W, bool vec, const float (&v)[4]) {
  if (vec) {
    *reinterpret_cast<float4*>(row + x0) = make_float4(v[0], v[1], v[2], v[3]);
    return;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (x0 + u < W) row[x0 + u] = v[u];
}

// Fused resample + apply.  A CTA owns 8 output rows x 128 output columns; thread (ry, q) the 4 columns 4q..4q+3 of row
// Y0 + ry.  Per output channel c, the source rows [lo, hi) the band's vertical taps touch are resampled horizontally
// (the 4 planes of c, 128 columns) into shared memory, kApplyStage rows per pass, and each thread adds the vertical
// taps that fall in the pass, in tap order.  Three CTAs per SM (80 registers; without the bound ptxas caps the kernel
// at 64 registers and spills).  grid (ceil(W / 128), ceil(H / 8), b)
template <int C>
__global__ void __launch_bounds__(kApplyQuads * kApplyRows, 3) guided_apply_kernel(
    const float* __restrict__ image, const float* __restrict__ coef, int h, int w, int H, int W,
    const int32_t* __restrict__ bounds_h, const float* __restrict__ weights_h, int ksize_h,
    const int32_t* __restrict__ bounds_v, const float* __restrict__ weights_v, int ksize_v, int vec,
    float* __restrict__ out) {
  __shared__ __align__(16) float rows[kApplyStage][4][kApplyQuads * 4];
  const int q = threadIdx.x % kApplyQuads, ry = threadIdx.x / kApplyQuads, b = blockIdx.z;
  const int Y0 = blockIdx.y * kApplyRows, Y = Y0 + ry, X0 = blockIdx.x * kApplyQuads * 4, x0 = X0 + 4 * q;
  const bool live = Y < H && x0 < W;
  const long long hw = (long long)h * w, HW = (long long)H * W;
  const int Ylast = min(Y0 + kApplyRows, H) - 1;
  const int lo = max(__ldg(bounds_v + 2 * Y0), 0);
  const int hi = min(__ldg(bounds_v + 2 * Ylast) + __ldg(bounds_v + 2 * Ylast + 1), h);
  const int ymin = Y < H ? __ldg(bounds_v + 2 * Y) : 0, ycnt = live ? __ldg(bounds_v + 2 * Y + 1) : 0;
  // horizontal taps of this thread's staging columns (clamped into the image)
  int xmin[4], xcnt[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int X = min(x0 + u, W - 1);
    xmin[u] = __ldg(bounds_h + 2 * X);
    xcnt[u] = __ldg(bounds_h + 2 * X + 1);
  }
#pragma unroll 1
  for (int c = 0; c < C; ++c) {
    float acc[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[k][u] = 0.0f;
    const float* cplane = coef + ((long long)b * 4 * C + 4 * c) * hw;
#pragma unroll 1
    for (int s0 = lo; s0 < hi; s0 += kApplyStage) {
      const int ns = min(kApplyStage, hi - s0);
      __syncthreads();                                      // the previous pass's rows are consumed
      for (int e = ry; e < ns * 4; e += kApplyRows) {       // (row, plane) pairs; this thread's 4 columns
        const int sr = e >> 2, k = e & 3;
        const float* src = cplane + k * hw + (long long)(s0 + sr) * w;
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int X = min(x0 + u, W - 1);
          const float* wt = weights_h + (long long)X * ksize_h;
          float a = 0.0f;
          for (int t = 0; t < xcnt[u]; ++t) a = __fmaf_rn(__ldg(wt + t), __ldg(src + xmin[u] + t), a);
          v[u] = a;
        }
        *reinterpret_cast<float4*>(&rows[sr][k][4 * q]) = make_float4(v[0], v[1], v[2], v[3]);
      }
      __syncthreads();
      const int t0 = max(s0 - ymin, 0), t1 = min(s0 + ns - ymin, ycnt);
      for (int t = t0; t < t1; ++t) {
        const float wv = __ldg(weights_v + (long long)Y * ksize_v + t);
        const int sr = ymin + t - s0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 v = *reinterpret_cast<const float4*>(&rows[sr][k][4 * q]);
          acc[k][0] = __fmaf_rn(wv, v.x, acc[k][0]);
          acc[k][1] = __fmaf_rn(wv, v.y, acc[k][1]);
          acc[k][2] = __fmaf_rn(wv, v.z, acc[k][2]);
          acc[k][3] = __fmaf_rn(wv, v.w, acc[k][3]);
        }
      }
    }
    if (live) {
      float4 xv[3];                                         // re-read per channel: L1 hits after the first
#pragma unroll
      for (int k = 0; k < 3; ++k) xv[k] = load4(image + ((long long)b * 3 + k) * HW + (long long)Y * W, x0, W, vec != 0);
      float o[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        o[u] = __fmaf_rn(acc[2][u], comp(xv[2], u), __fmaf_rn(acc[1][u], comp(xv[1], u),
                                                              __fmaf_rn(acc[0][u], comp(xv[0], u), acc[3][u])));
      store4(out + ((long long)b * C + c) * HW + (long long)Y * W, x0, W, vec != 0, o);
    }
  }
}

static bool guided_geometry_ok(int32_t b, int32_t c, int32_t h, int32_t w) {
  return (c == 1 || c == 3) && planes_ok(b, h, w);
}
static dim3 low_res_grid(int32_t b, int32_t h, int32_t w) {
  return dim3((unsigned)((w + kGuidedThreads - 1) / kGuidedThreads), h, b);
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_guided_workspace_bytes(int32_t b, int32_t c, int32_t h, int32_t w) {
  if (!guided_geometry_ok(b, c, h, w)) return -1;
  return (int64_t)b * h * w * (guided_products(c) + 4 * c) * (int64_t)sizeof(double);
}

extern "C" int odb_guided_coefficients(const float* guide, const float* pred, int32_t b, int32_t c, int32_t h,
                                       int32_t w, int32_t radius, double eps, void* workspace, float* coef,
                                       void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!guide || !pred || !workspace || !coef || !guided_geometry_ok(b, c, h, w) || radius < 1 ||
      radius > ODB_GUIDED_MAX_RADIUS || !std::isfinite(eps) || !(eps > 0.0) || !aligned(guide, 4) ||
      !aligned(pred, 4) || !aligned(coef, 4) || !aligned(workspace, 8))
    return fail(ODB_ERR_INVALID, "guided_coefficients: bad argument");
  const dim3 grid = low_res_grid(b, h, w);
  double* sums = static_cast<double*>(workspace);                     // [b][9 + 4c][h][w], later [b][4c][h][w]
  double* ab = sums + (long long)b * guided_products(c) * h * w;     // [b][4c][h][w]
  if (c == 1) {
    guided_box_v_products_kernel<1><<<grid, kGuidedThreads, 0, stream>>>(guide, pred, h, w, radius, sums);
    count_launch();
    guided_solve_kernel<1><<<grid, kGuidedThreads, 0, stream>>>(sums, h, w, radius, eps, ab);
  } else {
    guided_box_v_products_kernel<3><<<grid, kGuidedThreads, 0, stream>>>(guide, pred, h, w, radius, sums);
    count_launch();
    guided_solve_kernel<3><<<grid, kGuidedThreads, 0, stream>>>(sums, h, w, radius, eps, ab);
  }
  count_launch();
  guided_box_v_kernel<<<grid, kGuidedThreads, 0, stream>>>(ab, 4 * c, h, w, radius, sums);
  count_launch();
  guided_box_h_mean_kernel<<<grid, kGuidedThreads, 0, stream>>>(sums, 4 * c, h, w, radius, coef);
  count_launch();
  return check_launch("guided_coefficients");
}

extern "C" int odb_guided_apply(const float* image, const float* coef, int32_t b, int32_t c, int32_t h, int32_t w,
                                int32_t H, int32_t W, const int32_t* bounds_h, const float* weights_h, int32_t ksize_h,
                                const int32_t* bounds_v, const float* weights_v, int32_t ksize_v, float* out,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!image || !coef || !out || !bounds_h || !weights_h || !bounds_v || !weights_v || !guided_geometry_ok(b, c, h, w) ||
      !planes_ok(b, H, W) || ksize_h < 1 || ksize_v < 1 || !aligned(image, 4) || !aligned(coef, 4) ||
      !aligned(out, 4) || !aligned(bounds_h, 4) || !aligned(bounds_v, 4) || !aligned(weights_h, 4) ||
      !aligned(weights_v, 4))
    return fail(ODB_ERR_INVALID, "guided_apply: bad argument");
  const int vec = (W % 4 == 0 && aligned(image, 16) && aligned(out, 16)) ? 1 : 0;
  const dim3 grid((unsigned)((W + 4 * kApplyQuads - 1) / (4 * kApplyQuads)),
                  (unsigned)((H + kApplyRows - 1) / kApplyRows), b);
  if (c == 1)
    guided_apply_kernel<1><<<grid, kApplyQuads * kApplyRows, 0, stream>>>(image, coef, h, w, H, W, bounds_h, weights_h,
                                                                          ksize_h, bounds_v, weights_v, ksize_v, vec,
                                                                          out);
  else
    guided_apply_kernel<3><<<grid, kApplyQuads * kApplyRows, 0, stream>>>(image, coef, h, w, H, W, bounds_h, weights_h,
                                                                          ksize_h, bounds_v, weights_v, ksize_v, vec,
                                                                          out);
  count_launch();
  return check_launch("guided_apply");
}
