// Backward kernels of the DPT-Hybrid train step (train_depth.py:183-190 training_step -> loss.backward()): everything
// that is not a tensor-core contraction.  What autograd derives for the reference modules (timm Block / GroupNormAct /
// StdConv2dSame / MaxPool2dSame, modules/midas/blocks.py Interpolate + ResidualConvUnit_custom, dpt_depth.py head) is
// written out by hand here; parity is tested against torch.autograd of the reference arithmetic.
//   storage type T: bf16 (production) or fp32 (correctness mode) for activations and activation gradients;
//   statistics, affine parameters, parameter gradients, the ViT residual stream and its gradient: fp32.
// Every reduction has a fixed summation order (no floating-point atomics): bit-reproducible gradients.
#include "common.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

ODB_DEVINL void ld8(const bf16* p, float* v) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
ODB_DEVINL void ld8(const float* p, float* v) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
ODB_DEVINL void st8(bf16* p, const float* v) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]); u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
ODB_DEVINL void st8(float* p, const float* v) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
ODB_DEVINL float ldf(const bf16* p) { return __bfloat162float(*p); }
ODB_DEVINL float ldf(const float* p) { return *p; }
ODB_DEVINL void stf(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
ODB_DEVINL void stf(float* p, float v) { *p = v; }
ODB_DEVINL float2 ld2(const bf16* p) { return unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p)); }
ODB_DEVINL float2 ld2(const float* p) { return *reinterpret_cast<const float2*>(p); }
ODB_DEVINL void st2(bf16* p, float2 v) { *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v.x, v.y); }
ODB_DEVINL void st2(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }
ODB_DEVINL void st4(bf16* p, float4 v) { *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w)); }
ODB_DEVINL void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

static unsigned grid_for(long long items, int block = 256, int per_sm = 16) {
  long long blocks = (items + block - 1) / block;
  const long long cap = (long long)num_sms() * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

// ------------------------------------------------------------------------------------------ out = a + b * [m > 0]
template <typename T>
__global__ void __launch_bounds__(256) mask_add_kernel(const T* __restrict__ a, const T* __restrict__ b,
                                                       const T* __restrict__ m, T* __restrict__ out, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float vb[8], va[8], vm[8];
    ld8(b + i * 8, vb);
    if (m != nullptr) {
      ld8(m + i * 8, vm);
#pragma unroll
      for (int j = 0; j < 8; ++j) vb[j] = vm[j] > 0.f ? vb[j] : 0.f;
    }
    if (a != nullptr) {
      ld8(a + i * 8, va);
#pragma unroll
      for (int j = 0; j < 8; ++j) vb[j] += va[j];
    }
    st8(out + i * 8, vb);
  }
}

// ------------------------------------------------------------------------------------------ exact-erf GELU
ODB_DEVINL float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
ODB_DEVINL float gelu_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * expf(-0.5f * x * x);
  return cdf + x * pdf;
}
template <typename T>
__global__ void __launch_bounds__(256) gelu_fwd_kernel(const T* __restrict__ u, T* __restrict__ y, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float v[8];
    ld8(u + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = gelu_exact(v[j]);
    st8(y + i * 8, v);
  }
}
template <typename T>
__global__ void __launch_bounds__(256) gelu_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ u,
                                                       T* __restrict__ du, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float v[8], g[8];
    ld8(u + i * 8, v);
    ld8(dy + i * 8, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= gelu_grad(v[j]);
    st8(du + i * 8, g);
  }
}

// ------------------------------------------------------------------------------------------ column sums (bias grads)
// out[bt][n] = sum over rows_per_batch rows of x[bt][row][n]; stage 1: slab partials, stage 2: ordered fp64 combination.
// x rows may be strided (row_stride elements).
constexpr int kColsumMaxSlabs = 512;
constexpr int kColsumTargetBlocks = 148 * 8;
// row slabs per batch: enough blocks to fill the chip, at least 64 rows (two per row lane) per slab
static int colsum_slabs(long long batches, long long rows_per_batch, long long n) {
  const long long col_blocks = (n + 63) / 64;
  long long want = (kColsumTargetBlocks + col_blocks * batches - 1) / (col_blocks * batches);
  const long long by_rows = rows_per_batch / 64;
  if (want > by_rows) want = by_rows;
  if (want > kColsumMaxSlabs) want = kColsumMaxSlabs;
  if (want < 1) want = 1;
  return (int)want;
}
template <typename T>
__global__ void __launch_bounds__(256) colsum_partial_kernel(const T* __restrict__ x, float* __restrict__ partial,
                                                             long long rows_per_batch, int n, long long row_stride,
                                                             long long batch_stride, int slabs) {
  // block: 8 column octets (64 columns = one 128-byte bf16 segment per row) x 32 row lanes;
  // grid (ceil(n / 64), slabs, batches); four independent row loads in flight per thread
  const int oct = threadIdx.x & 7, lane_r = threadIdx.x >> 3;
  const int c0 = (blockIdx.x * 8 + oct) * 8;
  const int slab = blockIdx.y, bt = blockIdx.z;
  const long long per = (rows_per_batch + slabs - 1) / slabs;
  const long long r0 = slab * per, r1 = min(rows_per_batch, r0 + per);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < n) {
    const T* base = x + bt * batch_stride + c0;
    for (long long r = r0 + lane_r; r < r1; r += 128) {
      float v[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r + 32 * u < r1) ld8(base + (r + 32 * u) * row_stride, v[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r + 32 * u < r1) {
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += v[u][j];
        }
    }
  }
  __shared__ float s[32][64];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[lane_r][oct * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64 && blockIdx.x * 64 + threadIdx.x < n) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 32; ++q) t += s[q][threadIdx.x];
    partial[((long long)bt * slabs + slab) * n + blockIdx.x * 64 + threadIdx.x] = t;
  }
}
// out[bt][c] (+)= sum over `parts` partial rows (ordered_sum8); grid (ceil(n / 32), batches)
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                              int parts, long long n, int accumulate) {
  const long long bt = blockIdx.y;
  const long long c = (long long)blockIdx.x * 32 + (threadIdx.x & 31);
  const float* src = partial + bt * parts * n + c;
  double t = ordered_sum8(parts, c < n, [&](int p) { return __ldg(src + (long long)p * n); });
  if (threadIdx.x < 32 && c < n) {
    if (accumulate) t += (double)out[bt * n + c];
    out[bt * n + c] = (float)t;
  }
}

// ------------------------------------------------------------------------------------------ LayerNorm backward
// y = (x - mean) * rstd * g + b over the last dim.  Per row:  dx = rstd * (dy*g - mean(dy*g) - xhat * mean(dy*g*xhat)).
// ds_out = ds_in + dx (the residual-stream gradient, fp32) and optionally a T copy of it (the next GEMM operand).
// dgamma / dbeta and (optionally) the column sums of ds_out (the bias gradient of the linear layer whose output gradient
// ds_out is): each block accumulates its rows in registers and writes one partial row [3][cols].
// One warp per row, the next row's loads are issued before the current row is reduced (one block per SM, 8 warps).
template <typename T> struct Raw8;
template <> struct Raw8<bf16> {
  uint4 u;
  ODB_DEVINL void load(const bf16* p) { u = *reinterpret_cast<const uint4*>(p); }
  ODB_DEVINL void get(float* v) const {
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
};
template <> struct Raw8<float> {
  float4 a, b;
  ODB_DEVINL void load(const float* p) { a = reinterpret_cast<const float4*>(p)[0]; b = reinterpret_cast<const float4*>(p)[1]; }
  ODB_DEVINL void get(float* v) const { v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w; }
};
template <int VPL, typename T>
__global__ void __launch_bounds__(256, 1) layernorm_bwd_kernel(const T* __restrict__ dy, const float* __restrict__ x,
                                                               const float* __restrict__ gamma, const float* __restrict__ ds_in,
                                                               float* __restrict__ ds_out, T* __restrict__ ds_copy,
                                                               float* __restrict__ partial, long long rows, float eps,
                                                               int want_params, int want_colsum) {
  constexpr int COLS = VPL * 256;
  __shared__ float sh[8][COLS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float g[VPL][8], dg[VPL][8], db[VPL][8], dc[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    ld8(gamma + (i * 32 + lane) * 8, g[i]);
#pragma unroll
    for (int j = 0; j < 8; ++j) { dg[i][j] = 0.f; db[i][j] = 0.f; dc[i][j] = 0.f; }
  }
  const long long stride = (long long)gridDim.x * 8;
  long long row = (long long)blockIdx.x * 8 + warp;
  Raw8<float> xr[VPL], xn[VPL];
  Raw8<T> dr[VPL], dn[VPL];
  if (row < rows) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      xr[i].load(x + row * COLS + (i * 32 + lane) * 8);
      dr[i].load(dy + row * COLS + (i * 32 + lane) * 8);
    }
  }
  while (row < rows) {
    const long long next = row + stride;
    if (next < rows) {
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        xn[i].load(x + next * COLS + (i * 32 + lane) * 8);
        dn[i].load(dy + next * COLS + (i * 32 + lane) * 8);
      }
    }
    float xv[VPL][8], dv[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      xr[i].get(xv[i]);
      dr[i].get(dv[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += xv[i][j];
    }
    const float mean = warp_sum(s) * (1.0f / COLS);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / COLS) + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (xv[i][j] - mean) * rstd;
        const float dg_ = dv[i][j] * g[i][j];
        s1 += dg_;
        s2 += dg_ * xh;
        dg[i][j] += dv[i][j] * xh;
        db[i][j] += dv[i][j];
        xv[i][j] = xh;
      }
    s1 = warp_sum(s1) * (1.0f / COLS);
    s2 = warp_sum(s2) * (1.0f / COLS);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c0 = (i * 32 + lane) * 8;
      float o[8];
      if (ds_in != nullptr) ld8(ds_in + row * COLS + c0, o);
      else {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] += rstd * (dv[i][j] * g[i][j] - s1 - xv[i][j] * s2);
        dc[i][j] += o[j];
      }
      st8(ds_out + row * COLS + c0, o);
      if (ds_copy != nullptr) st8(ds_copy + row * COLS + c0, o);
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) { xr[i] = xn[i]; dr[i] = dn[i]; }
    row = next;
  }
  // block partials of dgamma / dbeta / column sums: 8 warps combined in a fixed order through shared memory (a frozen
  // norm, want_params == 0, skips the dgamma / dbeta passes; without column sums either the kernel ends here)
  const int passes = want_colsum ? 3 : 2;
  for (int pass = want_params ? 0 : 2; pass < passes; ++pass) {
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) sh[warp][(i * 32 + lane) * 8 + j] = pass == 0 ? dg[i][j] : (pass == 1 ? db[i][j] : dc[i][j]);
    __syncthreads();
    for (int c = threadIdx.x; c < COLS; c += 256) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += sh[w][c];
      partial[((long long)blockIdx.x * 3 + pass) * COLS + c] = t;
    }
    __syncthreads();
  }
}
// dgamma / dbeta / colsum (+)= ordered sum of the block partials [blocks][3][cols]; grid ceil((passes - first) * cols / 32)
// with first = 0, or 2 when dgamma / dbeta are not wanted (NULL)
__global__ void __launch_bounds__(256) ln_param_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dgamma,
                                                              float* __restrict__ dbeta, float* __restrict__ dcol, int blocks,
                                                              int cols, int accumulate) {
  const int passes = dcol != nullptr ? 3 : 2;
  const int first = dgamma != nullptr ? 0 : 2;
  const int e = (first * cols) + blockIdx.x * 32 + (threadIdx.x & 31);     // pass * cols + column
  const bool active = e < passes * cols;
  const float* src = partial + e;
  double t = ordered_sum8(blocks, active, [&](int b) { return __ldg(src + (long long)b * 3 * cols); });
  if (threadIdx.x < 32 && active) {
    const int pass = e / cols, c = e - pass * cols;
    float* dst = (pass == 0 ? dgamma : (pass == 1 ? dbeta : dcol)) + c;
    if (accumulate) t += (double)*dst;
    *dst = (float)t;
  }
}

// ------------------------------------------------------------------------------------------ GroupNorm backward
// stage 1: per (image, channel) sums of g and g*x, g = dy * [mask > 0] (the ReLU that follows the norm), fixed order.
template <typename T>
__global__ void __launch_bounds__(256) groupnorm_bwd_sums_kernel(const T* __restrict__ dy, const T* __restrict__ mask,
                                                                 const T* __restrict__ x, float* __restrict__ partial,
                                                                 int hw, int c, int pixels_per_block) {
  extern __shared__ float s_thr[];     // [2][planes * c]
  const int b = blockIdx.y, slab = blockIdx.x, slabs = gridDim.x;
  const int octets = c >> 3;
  const int oct = threadIdx.x % octets, plane = threadIdx.x / octets, planes = blockDim.x / octets;
  const int p0 = slab * pixels_per_block, p1 = min(hw, p0 + pixels_per_block);
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (plane < planes) {
    const long long base = ((long long)b * hw) * c + oct * 8;
    for (int p = p0 + plane; p < p1; p += planes) {
      float g[8], xv[8];
      ld8(dy + base + (long long)p * c, g);
      ld8(x + base + (long long)p * c, xv);
      if (mask != nullptr) {
        float m[8];
        ld8(mask + base + (long long)p * c, m);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = m[j] > 0.f ? g[j] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j] += g[j]; q[j] = fmaf(g[j], xv[j], q[j]); }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s_thr[plane * c + oct * 8 + j] = s[j];
      s_thr[planes * c + plane * c + oct * 8 + j] = q[j];
    }
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    double ts = 0.0, tq = 0.0;
    for (int pl = 0; pl < planes; ++pl) { ts += (double)s_thr[pl * c + ch]; tq += (double)s_thr[planes * c + pl * c + ch]; }
    float* dst = partial + (((long long)b * slabs + slab) * c + ch) * 2;
    dst[0] = (float)ts;
    dst[1] = (float)tq;
  }
}
// stage 2 (one block per image, 1024 threads): reduce the slabs (L = 1024 / c slab lanes per channel, each lane sums
// slabs l, l+L, ... in fp64, lanes combined in lane order), then the per-(image, channel / group) coefficients of
//   dx = A[c] * g + Bg[group] * x + Cg[group]   and this image's share of dgamma / dbeta.
__global__ void __launch_bounds__(1024) groupnorm_bwd_coef_kernel(const float* __restrict__ partial, const float* __restrict__ stats,
                                                                  const float* __restrict__ gamma, float* __restrict__ coef,
                                                                  float* __restrict__ dparam_partial, int slabs, int hw, int c,
                                                                  int groups) {
  extern __shared__ double sm[];      // [c] sum g, [c] sum g*x, [groups] s1, [groups] s2, then lane partials [L][c][2]
  const int b = blockIdx.x;
  const int cpg = c / groups;
  double* sg = sm; double* sgx = sm + c; double* s1 = sm + 2 * c; double* s2 = sm + 2 * c + groups;
  double* lp = sm + 2 * c + 2 * groups;
  const int L = max(1, (int)blockDim.x / c);
  for (int idx = threadIdx.x; idx < c * L; idx += blockDim.x) {
    const int l = idx / c, ch = idx - l * c;
    double ts = 0.0, tq = 0.0;
#pragma unroll 4
    for (int sl = l; sl < slabs; sl += L) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(partial + (((long long)b * slabs + sl) * c + ch) * 2));
      ts += (double)v.x;
      tq += (double)v.y;
    }
    lp[((long long)l * c + ch) * 2 + 0] = ts;
    lp[((long long)l * c + ch) * 2 + 1] = tq;
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    double ts = 0.0, tq = 0.0;
    for (int l = 0; l < L; ++l) { ts += lp[((long long)l * c + ch) * 2]; tq += lp[((long long)l * c + ch) * 2 + 1]; }
    sg[ch] = ts; sgx[ch] = tq;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    const double mean = stats[((long long)b * groups + g) * 2], rstd = stats[((long long)b * groups + g) * 2 + 1];
    double a1 = 0.0, a2 = 0.0;
    for (int j = 0; j < cpg; ++j) {
      const int ch = g * cpg + j;
      const double gm = gamma[ch];
      a1 += gm * sg[ch];
      a2 += gm * rstd * (sgx[ch] - mean * sg[ch]);
    }
    s1[g] = a1; s2[g] = a2;
  }
  __syncthreads();
  const double n = (double)hw * cpg;
  float* cf = coef + (long long)b * (c + 2 * groups);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    const int g = ch / cpg;
    const double mean = stats[((long long)b * groups + g) * 2], rstd = stats[((long long)b * groups + g) * 2 + 1];
    cf[ch] = (float)(rstd * gamma[ch]);
    if (dparam_partial != nullptr) {                                                                // NULL: frozen norm
      dparam_partial[((long long)b * 2 + 0) * c + ch] = (float)(rstd * (sgx[ch] - mean * sg[ch]));   // dgamma share
      dparam_partial[((long long)b * 2 + 1) * c + ch] = (float)sg[ch];                               // dbeta share
    }
  }
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    const double mean = stats[((long long)b * groups + g) * 2], rstd = stats[((long long)b * groups + g) * 2 + 1];
    cf[c + g] = (float)(-rstd * rstd * s2[g] / n);
    cf[c + groups + g] = (float)(rstd * (rstd * s2[g] * mean - s1[g]) / n);
  }
}
// stage 3: dx = A[c] * g + Bg * x + Cg
template <typename T>
__global__ void __launch_bounds__(256) groupnorm_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ mask,
                                                                  const T* __restrict__ x, const float* __restrict__ coef,
                                                                  T* __restrict__ dx, int hw, int c, int groups) {
  extern __shared__ float cs[];       // [c] A, [c] B (expanded), [c] C (expanded)
  const int b = blockIdx.y;
  const int cpg = c / groups, octets = c >> 3;
  const float* cf = coef + (long long)b * (c + 2 * groups);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    cs[ch] = cf[ch];
    cs[c + ch] = cf[c + ch / cpg];
    cs[2 * c + ch] = cf[c + groups + ch / cpg];
  }
  __syncthreads();
  const unsigned total = (unsigned)hw * (unsigned)octets;
  const long long base = ((long long)b * hw) * c;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned oct = i % (unsigned)octets;
    float g[8], xv[8], o[8];
    ld8(dy + base + (long long)i * 8, g);
    ld8(x + base + (long long)i * 8, xv);
    if (mask != nullptr) {
      float m[8];
      ld8(mask + base + (long long)i * 8, m);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = m[j] > 0.f ? g[j] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(cs[oct * 8 + j], g[j], fmaf(cs[c + oct * 8 + j], xv[j], cs[2 * c + oct * 8 + j]));
    st8(dx + base + (long long)i * 8, o);
  }
}

// ------------------------------------------------------------------------------------------ bilinear x2 backward
// adjoint of upsample2x (align_corners=True): dz[m][k] = sum over the <= 4 x 4 outputs that read source (m, k).
template <typename T>
__global__ void __launch_bounds__(256) upsample2x_bwd_kernel(const T* __restrict__ dout, T* __restrict__ dz, int h, int w, int c) {
  const int oh = 2 * h, ow = 2 * w;
  const int octets = c >> 3;
  const long long total = (long long)h * w * octets;
  const int bi = blockIdx.y;
  const float sy = (float)(h - 1) / (float)(oh - 1), sx = (float)(w - 1) / (float)(ow - 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oct = (int)(i % octets);
    const int k = (int)((i / octets) % w), m = (int)(i / ((long long)octets * w));
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int oy = max(2 * m - 2, 0); oy <= min(2 * m + 2, oh - 1); ++oy) {
      const float fy = oy * sy;
      int y0 = min((int)floorf(fy), h - 1);
      const int y1 = min(y0 + 1, h - 1);
      const float wy = fy - (float)y0;
      float cy = 0.f;
      if (y0 == m) cy += 1.f - wy;
      if (y1 == m) cy += wy;
      if (cy == 0.f) continue;
      for (int ox = max(2 * k - 2, 0); ox <= min(2 * k + 2, ow - 1); ++ox) {
        const float fx = ox * sx;
        int x0 = min((int)floorf(fx), w - 1);
        const int x1 = min(x0 + 1, w - 1);
        const float wx = fx - (float)x0;
        float cx = 0.f;
        if (x0 == k) cx += 1.f - wx;
        if (x1 == k) cx += wx;
        if (cx == 0.f) continue;
        float g[8];
        ld8(dout + (((long long)bi * oh + oy) * ow + ox) * c + oct * 8, g);
        const float wgt = cy * cx;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(wgt, g[j], acc[j]);
      }
    }
    st8(dz + (((long long)bi * h + m) * w + k) * c + oct * 8, acc);
  }
}

// ------------------------------------------------------------------------------------------ stem tail backward
// forward: t = maxpool3x3s2_same(relu(gn(s0))).  g_s0[iy][ix] = sum over the <= 4 windows containing (iy, ix) whose
// FIRST maximum (row-major scan, as torch) is this element, of dt[window]; zero where relu(gn(s0)) == 0.
template <typename T>
__global__ void __launch_bounds__(256) stem_pool_bwd_kernel(const T* __restrict__ dt, const T* __restrict__ s0,
                                                            const float* __restrict__ stats, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, T* __restrict__ g_s0, int h, int w,
                                                            int c, int groups) {
  extern __shared__ float coef[];      // [c] scale, [c] shift
  const int b = blockIdx.y;
  const int cpg = c / groups;
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    const int g = ch / cpg;
    const float mean = stats[((long long)b * groups + g) * 2], rstd = stats[((long long)b * groups + g) * 2 + 1];
    const float a = rstd * gamma[ch];
    coef[ch] = a;
    coef[c + ch] = beta[ch] - mean * a;
  }
  __syncthreads();
  const int oh = h / 2, ow = w / 2;
  const int octets = c >> 3;
  const long long total = (long long)h * w * octets;
  const T* sb = s0 + (long long)b * h * w * c;
  const T* db = dt + (long long)b * oh * ow * c;
  T* gb = g_s0 + (long long)b * h * w * c;
  // thread = (input pixel, 8 channels): 16-byte loads; the 3x3 neighbourhoods of its <= 4 windows come from L1/L2
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oct = (int)(i % octets);
    const int ix = (int)((i / octets) % w), iy = (int)(i / ((long long)octets * w));
    float a[8], sh[8], v[8], acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] = coef[oct * 8 + j]; sh[j] = coef[c + oct * 8 + j]; acc[j] = 0.f; }
    ld8(sb + ((long long)iy * w + ix) * c + oct * 8, v);
    bool any = false;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] = fmaxf(fmaf(v[j], a[j], sh[j]), 0.f); any |= v[j] > 0.f; }
    if (any) {
      for (int oy = max((iy - 1) / 2, 0); oy <= min(iy / 2, oh - 1); ++oy) {
        if (2 * oy > iy || 2 * oy + 2 < iy) continue;
        for (int ox = max((ix - 1) / 2, 0); ox <= min(ix / 2, ow - 1); ++ox) {
          if (2 * ox > ix || 2 * ox + 2 < ix) continue;
          bool is_arg[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) is_arg[j] = v[j] > 0.f;
          for (int dy = 0; dy < 3; ++dy) {
            const int yy = 2 * oy + dy;
            if (yy >= h) continue;
            for (int dx = 0; dx < 3; ++dx) {
              const int xx = 2 * ox + dx;
              if (xx >= w || (yy == iy && xx == ix)) continue;
              float u[8];
              ld8(sb + ((long long)yy * w + xx) * c + oct * 8, u);
              const bool before = (yy < iy) || (yy == iy && xx < ix);
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float uu = fmaxf(fmaf(u[j], a[j], sh[j]), 0.f);
                if (uu > v[j] || (before && uu == v[j])) is_arg[j] = false;
              }
            }
          }
          float g[8];
          ld8(db + ((long long)oy * ow + ox) * c + oct * 8, g);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += is_arg[j] ? g[j] : 0.f;
        }
      }
    }
    st8(gb + ((long long)iy * w + ix) * c + oct * 8, acc);
  }
}

// ------------------------------------------------------------------------------------------ stem input gradient
// Gradient of the 7x7 stride-2 TF-SAME stem convolution (timm StdConv2dSame(3, 64, 7, stride 2), padding (2, 3)) w.r.t.
// its fp32 NCHW input, from ds0 = the gradient w.r.t. its output [b][h/2][w/2][64] and the packed operand the forward
// used, w [64][kpad] (column (ky*7+kx)*3+c, already standardised):
//   dx[b][c][y][x] = sum over ky = y mod 2, kx = x mod 2, o < 64 of  w[o][(ky*7+kx)*3+c] * ds0[b][(y+2-ky)/2][(x+2-kx)/2][o]
// restricted to ds0 pixels inside the image.  Gather form: input quad (P, Q) = pixels (2P+py, 2Q+px) reads the 4 x 4
// ds0 pixels (P+1-i, Q+1-j), i, j < 4, through taps ky = 2i+py, kx = 2j+px (those <= 6).  Every dx element is written
// once by one thread, summed in a fixed order (o, then j, then i): bit-reproducible and independent of the batch.
// Block = 8 warps over a 16 x 32 quad tile, persistent over tiles; thread = two vertically adjacent quads (their 4 x 4
// windows share 3 rows, so 20 ds0 loads and 48 weight loads feed 294 FMAs per channel).  Shared memory: the weights
// re-laid as ws[o][i][j][py][px][c] fp32 (zero where a tap exceeds 6), staged once per block and read as warp-uniform
// float4 broadcasts; one 16-channel chunk of the ds0 tile + halo as fp32 planes [ch][19][35], where the lanes of a
// warp read consecutive columns of one row (no bank conflicts).
constexpr int kSigQH = 16, kSigQW = 32, kSigKC = 16;          // quad rows / quad columns per tile, channels per chunk
constexpr int kSigRows = kSigQH + 3, kSigCols = kSigQW + 3, kSigPlane = kSigRows * kSigCols;
constexpr int kSigWFloats = 64 * 16 * 12;
constexpr size_t kSigSmemBytes = (size_t)(kSigWFloats + kSigKC * kSigPlane) * sizeof(float);
template <typename T>
__global__ void __launch_bounds__(256, 2) stem_input_grad_kernel(const T* __restrict__ ds0, const T* __restrict__ w,
                                                                 float* __restrict__ dx, int b, int h, int wd, int kpad) {
  grid_dep_wait();
  grid_dep_launch();
  extern __shared__ float4 sig_smem[];
  float* ws = reinterpret_cast<float*>(sig_smem);
  float* st = ws + kSigWFloats;
  for (int e = threadIdx.x; e < kSigWFloats; e += blockDim.x) {
    const int c = e % 3, px = (e / 3) & 1, py = (e / 6) & 1, j = (e / 12) & 3, i = (e / 48) & 3, o = e / 192;
    const int ky = 2 * i + py, kx = 2 * j + px;
    ws[e] = (ky < 7 && kx < 7) ? ldf(w + (long long)o * kpad + (ky * 7 + kx) * 3 + c) : 0.f;
  }
  const int h2 = h / 2, w2 = wd / 2;
  const int tiles_y = (h2 + kSigQH - 1) / kSigQH, tiles_x = (w2 + kSigQW - 1) / kSigQW;
  const long long tiles = (long long)b * tiles_y * tiles_x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int tx = (int)(tile % tiles_x), ty = (int)((tile / tiles_x) % tiles_y);
    const int bi = (int)(tile / ((long long)tiles_x * tiles_y));
    const int P0 = ty * kSigQH, Q0 = tx * kSigQW;
    const T* db = ds0 + (long long)bi * h2 * w2 * 64;
    float acc[2][2][2][3];                                      // [quad][py][px][c]
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int k = 0; k < 12; ++k) (&acc[q][0][0][0])[k] = 0.f;
    for (int o0 = 0; o0 < 64; o0 += kSigKC) {
      __syncthreads();               // the previous chunk's readers (the first time: the weight staging) are done
      // ds0 pixels (P0 - 2 + r, Q0 - 2 + col), zero outside the image; thread item = (pixel, 8 channels)
      for (int e = threadIdx.x; e < kSigPlane * (kSigKC / 8); e += blockDim.x) {
        const int g = e % (kSigKC / 8), pix = e / (kSigKC / 8);
        const int r = pix / kSigCols, col = pix - r * kSigCols;
        const int oy = P0 - 2 + r, ox = Q0 - 2 + col;
        float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (oy >= 0 && oy < h2 && ox >= 0 && ox < w2) ld8(db + ((long long)oy * w2 + ox) * 64 + o0 + g * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) st[(g * 8 + k) * kSigPlane + pix] = v[k];
      }
      __syncthreads();
      for (int oc = 0; oc < kSigKC; ++oc) {
        // rows 2*warp .. 2*warp+4 of the tile: quad q, window index i reads row 2*warp + q + 3 - i
        const float* so = st + oc * kSigPlane + 2 * warp * kSigCols + lane + 3;
        const float4* wo = reinterpret_cast<const float4*>(ws + (o0 + oc) * 192);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float v[5];
#pragma unroll
          for (int r = 0; r < 5; ++r) v[r] = so[r * kSigCols - j];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 wa = wo[(i * 4 + j) * 3], wb = wo[(i * 4 + j) * 3 + 1], wc = wo[(i * 4 + j) * 3 + 2];
            const float wk[12] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w, wc.x, wc.y, wc.z, wc.w};
#pragma unroll
            for (int q = 0; q < 2; ++q)
#pragma unroll
              for (int py = 0; py < 2; ++py)
#pragma unroll
                for (int px = 0; px < 2; ++px) {
                  if (2 * i + py > 6 || 2 * j + px > 6) continue;
#pragma unroll
                  for (int c = 0; c < 3; ++c)
                    acc[q][py][px][c] = fmaf(wk[(py * 2 + px) * 3 + c], v[q + 3 - i], acc[q][py][px][c]);
                }
          }
        }
      }
    }
    const int Q = Q0 + lane;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int P = P0 + 2 * warp + q;
      if (P >= h2 || Q >= w2) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int py = 0; py < 2; ++py)
          *reinterpret_cast<float2*>(dx + (((long long)bi * 3 + c) * h + 2 * P + py) * wd + 2 * Q) =
              make_float2(acc[q][py][0][c], acc[q][py][1][c]);
    }
  }
}

// ------------------------------------------------------------------------------------------ pos-embed resize backward
// At a patch grid other than 24 x 24 the forward resizes the position-embedding grid (modules/midas/vit.py:102-116
// _resize_pos_embed: F.interpolate(mode="bilinear", align_corners=False)).  On each axis torch's upsample_bilinear2d maps
// output index j to  src = max(scale * (j + 0.5) - 0.5, 0), scale = (float)in / out;  i0 = (int)src,
// i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1 (both weights land on i0 when i1 == i0).  The adjoint:
//   dpos[iy][ix] = sum over jy, jx of  wy(iy, jy) * wx(ix, jx) * dgrid[jy][jx],   w(i, j) = l0 [i0(j) == i] + l1 [i1(j) == i].
// i0(j) and i1(j) never decrease with j, so the j that touch source index i are one range: from the first j with
// i1(j) >= i to the last j with i0(j) <= i (binary searches).  Gather form: block = one source pixel, thread = 4 channels
// (float4); each dpos element is summed over jy, then jx, in a fixed order and written once (no atomics, unlike torch's
// upsample_bilinear2d backward): bit-reproducible.
constexpr int kPosSrc = 24;                                     // the pretrained 384 x 384 / 16 grid
struct BilinearAxis {
  float scale;
  int in, out;
  ODB_DEVINL float src(int j) const {
    const float s = scale * (j + 0.5f) - 0.5f;
    return s < 0.f ? 0.f : s;
  }
  ODB_DEVINL int i0(int j) const { return (int)src(j); }
  ODB_DEVINL int i1(int j) const { const int a = i0(j); return a + (a < in - 1 ? 1 : 0); }
  ODB_DEVINL float weight(int i, int j) const {
    const float s = src(j);
    const int a = (int)s, b = a + (a < in - 1 ? 1 : 0);
    const float l1 = s - (float)a, l0 = 1.f - l1;
    return (a == i ? l0 : 0.f) + (b == i ? l1 : 0.f);
  }
  ODB_DEVINL void range(int i, int& first, int& last) const {
    int lo = 0, hi = out;
    while (lo < hi) { const int m = (lo + hi) >> 1; if (i1(m) >= i) hi = m; else lo = m + 1; }
    first = lo;
    lo = 0; hi = out;
    while (lo < hi) { const int m = (lo + hi) >> 1; if (i0(m) > i) hi = m; else lo = m + 1; }
    last = lo - 1;
  }
};
__global__ void __launch_bounds__(256) pos_embed_resize_bwd_kernel(const float* __restrict__ dgrid, float* __restrict__ dpos,
                                                                   int gh, int gw, int d4) {
  grid_dep_wait();
  grid_dep_launch();
  const int iy = blockIdx.x / kPosSrc, ix = blockIdx.x % kPosSrc;
  const BilinearAxis ay{(float)kPosSrc / gh, kPosSrc, gh}, ax{(float)kPosSrc / gw, kPosSrc, gw};
  int y0, y1, x0, x1;
  ay.range(iy, y0, y1);
  ax.range(ix, x0, x1);
  const float4* g = reinterpret_cast<const float4*>(dgrid);
  for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < d4; c += gridDim.y * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int jy = y0; jy <= y1; ++jy) {
      float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int jx = x0; jx <= x1; ++jx) {
        const float wx = ax.weight(ix, jx);
        const float4 v = __ldg(g + ((long long)jy * gw + jx) * d4 + c);
        row.x = fmaf(wx, v.x, row.x); row.y = fmaf(wx, v.y, row.y);
        row.z = fmaf(wx, v.z, row.z); row.w = fmaf(wx, v.w, row.w);
      }
      const float wy = ay.weight(iy, jy);
      acc.x = fmaf(wy, row.x, acc.x); acc.y = fmaf(wy, row.y, acc.y);
      acc.z = fmaf(wy, row.z, acc.z); acc.w = fmaf(wy, row.w, acc.w);
    }
    reinterpret_cast<float4*>(dpos)[(long long)blockIdx.x * d4 + c] = acc;
  }
}

// ------------------------------------------------------------------------------------------ head tail (1x1 conv + ReLUs)
// forward (training, unfused): out[b][k][p] = relu?(bias[k] + sum_j w[k][j] a[b][p][j]); a has `cs` channels per pixel
// of which the first 32 are real (the 128 -> 32 conv is carried zero-padded to 64 output channels).
template <typename T>
__global__ void __launch_bounds__(256) head_tail_fwd_kernel(const T* __restrict__ a, int cs, const float* __restrict__ w,
                                                            const float* __restrict__ bias, float* __restrict__ out,
                                                            long long ppi, int batch, int head_c, int relu) {
  const long long total = ppi * batch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float v[32];
#pragma unroll
    for (int j = 0; j < 4; ++j) ld8(a + i * cs + j * 8, v + j * 8);
    const long long b = i / ppi, pix = i - b * ppi;
    for (int k = 0; k < head_c; ++k) {
      float acc = bias[k];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc = fmaf(v[j], w[k * 32 + j], acc);
      out[(b * head_c + k) * ppi + pix] = relu ? fmaxf(acc, 0.f) : acc;
    }
  }
}
// backward: dpre[k] = dout[k] * [out[k] > 0] (or dout if !relu); da[j] = [a[j] > 0] * sum_k dpre[k] w[k][j];
// per-block partials of dw[k][j] = sum dpre[k] a[j] and db[k] = sum dpre[k]  ->  partial[block][head_c][33] (partial NULL:
// da only)
template <typename T>
__global__ void __launch_bounds__(256) head_tail_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ out,
                                                            const T* __restrict__ a, int cs, const float* __restrict__ w,
                                                            T* __restrict__ da, float* __restrict__ partial, long long ppi,
                                                            int batch, int head_c, int relu) {
  const long long total = ppi * batch;
  float pw[3][33];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int j = 0; j < 33; ++j) pw[k][j] = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float v[32], g[32];
#pragma unroll
    for (int j = 0; j < 4; ++j) ld8(a + i * cs + j * 8, v + j * 8);
#pragma unroll
    for (int j = 0; j < 32; ++j) g[j] = 0.f;
    const long long b = i / ppi, pix = i - b * ppi;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (k >= head_c) break;
      const long long idx = (b * head_c + k) * ppi + pix;
      float d = dout[idx];
      if (relu && !(out[idx] > 0.f)) d = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) { g[j] = fmaf(d, w[k * 32 + j], g[j]); pw[k][j] = fmaf(d, v[j], pw[k][j]); }
      pw[k][32] += d;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) g[j] = v[j] > 0.f ? g[j] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) st8(da + i * cs + j * 8, g + j * 8);
    if (cs > 32) {
      const float z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int j = 4; j < cs / 8; ++j) st8(da + i * cs + j * 8, z);
    }
  }
  if (partial == nullptr) return;                              // uniform over the block: no parameter gradient wanted
  // block reduction in a fixed order (warp shuffles, then 8 warps through shared memory)
  __shared__ float sh[8][3 * 33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int j = 0; j < 33; ++j) {
      const float t = warp_sum(pw[k][j]);
      if (lane == 0) sh[warp][k * 33 + j] = t;
    }
  __syncthreads();
  for (int e = threadIdx.x; e < head_c * 33; e += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += sh[q][e];
    partial[(long long)blockIdx.x * head_c * 33 + e] = t;
  }
}

// ------------------------------------------------------------------------------------------ fp32 stream += T gradient
template <typename T>
__global__ void __launch_bounds__(256) add_cast_kernel(const float* __restrict__ ds_in, const T* __restrict__ g,
                                                       float* __restrict__ ds_out, T* __restrict__ copy, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    ld8(g + i * 8, b);
    if (ds_in != nullptr) {
      ld8(ds_in + i * 8, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] += a[j];
    }
    st8(ds_out + i * 8, b);
    if (copy != nullptr) st8(copy + i * 8, b);
  }
}

// ------------------------------------------------------------------------------------------ weight packing (per step)
// w fp32 [N][C][kh][kw] (optionally weight-standardised, timm StdConv2dSame eps 1e-8) ->
//   fwd  T [n_pad][taps * c_pad]   fwd[n][t * c_pad + c]            = w[n][c][t]           (conv_gemm operand)
//   bwd  T [c_pad][taps * n_pad]   bwd[c][(taps-1-t) * n_pad + n]   = w[n][c][t]           (dgrad operand: 180-degree
//                                                                     rotated taps, in/out channels swapped)
// one block per output channel n (zero rows for n >= N).
template <typename T>
__global__ void __launch_bounds__(256) pack_weight_kernel(const float* __restrict__ w, T* __restrict__ fwd, T* __restrict__ bwd,
                                                          int N, int C, int taps, int n_pad, int c_pad, int standardize,
                                                          float eps) {
  const int n = blockIdx.x;
  const int K = C * taps;
  __shared__ double red[2][256];
  __shared__ float s_mean, s_inv;
  float mean = 0.f, inv = 1.f;
  if (n < N && standardize) {
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < K; i += blockDim.x) { const double v = w[(long long)n * K + i]; s += v; q += v * v; }
    red[0][threadIdx.x] = s; red[1][threadIdx.x] = q;
    __syncthreads();
    if (threadIdx.x == 0) {
      double ts = 0.0, tq = 0.0;
      for (int i = 0; i < 256; ++i) { ts += red[0][i]; tq += red[1][i]; }
      const double m = ts / K;
      double var = tq / K - m * m;
      if (var < 0.0) var = 0.0;
      s_mean = (float)m;
      s_inv = (float)(1.0 / (sqrt(var) + (double)eps));
    }
    __syncthreads();
    mean = s_mean; inv = s_inv;
  }
  for (int i = threadIdx.x; i < c_pad * taps; i += blockDim.x) {
    const int t = i / c_pad, c = i - t * c_pad;
    float v = 0.f;
    if (n < N && c < C) v = (w[((long long)n * C + c) * taps + t] - mean) * inv;
    if (fwd != nullptr) stf(fwd + (long long)n * taps * c_pad + i, v);
    if (bwd != nullptr) stf(bwd + ((long long)c * taps + (taps - 1 - t)) * n_pad + n, v);   // only without a fwd buffer
  }
}
// bwd[c][(taps-1-t) * n_pad + n] = fwd[n][t * c_pad + c]: 32 x 32 tiles through shared memory, coalesced both ways
template <typename T>
__global__ void __launch_bounds__(256) pack_transpose_kernel(const T* __restrict__ fwd, T* __restrict__ bwd, int taps,
                                                             int n_pad, int c_pad) {
  __shared__ float tile[32][33];
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32, t = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8)
    tile[r][tx] = (n0 + r < n_pad && c0 + tx < c_pad) ? ldf(fwd + ((long long)(n0 + r) * taps + t) * c_pad + c0 + tx) : 0.f;
  __syncthreads();
  for (int r = ty; r < 32; r += 8)
    if (c0 + r < c_pad && n0 + tx < n_pad)
      stf(bwd + ((long long)(c0 + r) * taps + (taps - 1 - t)) * n_pad + n0 + tx, tile[tx][r]);
}
// gradient of the packed weight gp fp32 [n_pad][taps * c_pad] -> gradient in parameter layout [N][C][taps], through
// the weight standardisation if the layer has one:  dw = (g - mean(g)) / (sigma + eps) - mean(g * what) * what / sigma
__global__ void __launch_bounds__(256) unpack_wgrad_kernel(const float* __restrict__ gp, const float* __restrict__ w,
                                                           float* __restrict__ dw, int N, int C, int taps, int c_pad,
                                                           int standardize, float eps) {
  extern __shared__ float row[];         // the packed gradient row of this output channel: [taps][c_pad], loaded coalesced
  const int n = blockIdx.x;
  const int K = C * taps;
  for (int i = threadIdx.x; i < taps * c_pad; i += blockDim.x) row[i] = gp[(long long)n * taps * c_pad + i];
  __syncthreads();
  if (!standardize) {
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
      const int c = i / taps, t = i - c * taps;
      dw[(long long)n * K + i] = row[t * c_pad + c];
    }
    return;
  }
  __shared__ double red[4][256];
  double s = 0.0, q = 0.0, sg = 0.0, sgw = 0.0;
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int c = i / taps, t = i - c * taps;
    const double v = w[(long long)n * K + i], g = row[t * c_pad + c];
    s += v; q += v * v; sg += g; sgw += g * v;
  }
  red[0][threadIdx.x] = s; red[1][threadIdx.x] = q; red[2][threadIdx.x] = sg; red[3][threadIdx.x] = sgw;
  __syncthreads();
  __shared__ double st[4];
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int i = 0; i < 256; ++i) t += red[threadIdx.x][i];
    st[threadIdx.x] = t;
  }
  __syncthreads();
  const double mean = st[0] / K;
  double var = st[1] / K - mean * mean;
  if (var < 0.0) var = 0.0;
  const double sigma = sqrt(var), sden = sigma + (double)eps;
  const double mg = st[2] / K;
  // mean(g * what) with what = (w - mean) / sden
  const double mgw = (st[3] - mean * st[2]) / (sden * K);
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int c = i / taps, t = i - c * taps;
    const double v = w[(long long)n * K + i], g = row[t * c_pad + c];
    const double what = (v - mean) / sden;
    const double r = (g - mg) / sden - (sigma > 0.0 ? mgw * what / sigma : 0.0);
    dw[(long long)n * K + i] = (float)r;
  }
}

// ---- multi-tensor versions: ONE launch packs / unpacks every layer of a table (the per-layer launches of ~100 small
// kernels cost more in launch gaps than in work).  Tables live in device memory; blockIdx.x -> (item, row) by binary search
// over the items' first block.
struct PackItem {
  const float* w; void* fwd; void* bwd;
  int n, c, taps, n_pad, c_pad, standardize, first_block, first_tile;
};
struct UnpackItem {
  const float* gp; const float* w; float* dw;
  int n, c, taps, c_pad, standardize, first_block, pad0, pad1;
};
template <typename Item>
ODB_DEVINL int find_item(const Item* items, int n_items, int block, int Item::*first) {
  int lo = 0, hi = n_items - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].*first <= block) lo = mid; else hi = mid - 1;
  }
  return lo;
}
template <typename T>
__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const PackItem* __restrict__ items, int n_items, float eps) {
  const PackItem it = items[find_item(items, n_items, (int)blockIdx.x, &PackItem::first_block)];
  const int n = blockIdx.x - it.first_block;
  const int K = it.c * it.taps;
  __shared__ double red[2][256];
  __shared__ float s_mean, s_inv;
  float mean = 0.f, inv = 1.f;
  if (n < it.n && it.standardize) {
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < K; i += blockDim.x) { const double v = it.w[(long long)n * K + i]; s += v; q += v * v; }
    red[0][threadIdx.x] = s; red[1][threadIdx.x] = q;
    __syncthreads();
    if (threadIdx.x == 0) {
      double ts = 0.0, tq = 0.0;
      for (int i = 0; i < 256; ++i) { ts += red[0][i]; tq += red[1][i]; }
      const double m = ts / K;
      double var = tq / K - m * m;
      if (var < 0.0) var = 0.0;
      s_mean = (float)m;
      s_inv = (float)(1.0 / (sqrt(var) + (double)eps));
    }
    __syncthreads();
    mean = s_mean; inv = s_inv;
  }
  T* fwd = static_cast<T*>(it.fwd);
  if (it.taps == 1 && (it.c & 3) == 0 && (it.c_pad & 3) == 0) {
    // linear / 1x1 layers (most of the parameters): four values per thread, 16-byte loads
    T* dst = fwd + (long long)n * it.c_pad;
    const float* src = it.w + (long long)n * it.c;
    for (int c = threadIdx.x * 4; c < it.c_pad; c += blockDim.x * 4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n < it.n && c < it.c) {
        v = *reinterpret_cast<const float4*>(src + c);
        v.x = (v.x - mean) * inv; v.y = (v.y - mean) * inv; v.z = (v.z - mean) * inv; v.w = (v.w - mean) * inv;
      }
      st4(dst + c, v);
    }
    return;
  }
  for (int i = threadIdx.x; i < it.c_pad * it.taps; i += blockDim.x) {
    const int t = i / it.c_pad, c = i - t * it.c_pad;
    float v = 0.f;
    if (n < it.n && c < it.c) v = (it.w[((long long)n * it.c + c) * it.taps + t] - mean) * inv;
    stf(fwd + (long long)n * it.taps * it.c_pad + i, v);
  }
}
// bwd[c][(taps-1-t) * n_pad + n] = fwd[n][t * c_pad + c]: 64 x 64 tiles through shared memory, element pairs both ways
constexpr int kPackTile = 64;
template <typename T>
__global__ void __launch_bounds__(256) pack_transpose_multi_kernel(const PackItem* __restrict__ items, int n_items) {
  const PackItem it = items[find_item(items, n_items, (int)blockIdx.x, &PackItem::first_tile)];
  __shared__ float tile[kPackTile][kPackTile + 1];
  int tl = blockIdx.x - it.first_tile;
  const int tn = (it.n_pad + kPackTile - 1) / kPackTile, tc = (it.c_pad + kPackTile - 1) / kPackTile;
  const int n0 = (tl % tn) * kPackTile; tl /= tn;
  const int c0 = (tl % tc) * kPackTile;
  const int t = tl / tc;
  const T* fwd = static_cast<const T*>(it.fwd);
  T* bwd = static_cast<T*>(it.bwd);
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const bool pairs = ((it.n_pad | it.c_pad) & 1) == 0;
  if (pairs) {
    for (int r = ty; r < kPackTile; r += 8) {
      float2 v = make_float2(0.f, 0.f);
      if (n0 + r < it.n_pad && c0 + 2 * tx < it.c_pad) v = ld2(fwd + ((long long)(n0 + r) * it.taps + t) * it.c_pad + c0 + 2 * tx);
      tile[r][2 * tx] = v.x;
      tile[r][2 * tx + 1] = v.y;
    }
    __syncthreads();
    for (int r = ty; r < kPackTile; r += 8)
      if (c0 + r < it.c_pad && n0 + 2 * tx < it.n_pad)
        st2(bwd + ((long long)(c0 + r) * it.taps + (it.taps - 1 - t)) * it.n_pad + n0 + 2 * tx,
            make_float2(tile[2 * tx][r], tile[2 * tx + 1][r]));
  } else {
    for (int r = ty; r < kPackTile; r += 8)
      for (int q = tx; q < kPackTile; q += 32)
        tile[r][q] = (n0 + r < it.n_pad && c0 + q < it.c_pad) ? ldf(fwd + ((long long)(n0 + r) * it.taps + t) * it.c_pad + c0 + q) : 0.f;
    __syncthreads();
    for (int r = ty; r < kPackTile; r += 8)
      for (int q = tx; q < kPackTile; q += 32)
        if (c0 + r < it.c_pad && n0 + q < it.n_pad)
          stf(bwd + ((long long)(c0 + r) * it.taps + (it.taps - 1 - t)) * it.n_pad + n0 + q, tile[q][r]);
  }
}
__global__ void __launch_bounds__(256) unpack_wgrads_multi_kernel(const UnpackItem* __restrict__ items, int n_items, float eps) {
  extern __shared__ float row[];
  const UnpackItem it = items[find_item(items, n_items, (int)blockIdx.x, &UnpackItem::first_block)];
  const int n = blockIdx.x - it.first_block;
  const int K = it.c * it.taps, taps = it.taps, c_pad = it.c_pad;
  for (int i = threadIdx.x; i < taps * c_pad; i += blockDim.x) row[i] = it.gp[(long long)n * taps * c_pad + i];
  __syncthreads();
  if (!it.standardize) {
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
      const int c = i / taps, t = i - c * taps;
      it.dw[(long long)n * K + i] = row[t * c_pad + c];
    }
    return;
  }
  __shared__ double red[4][256];
  double s = 0.0, q = 0.0, sg = 0.0, sgw = 0.0;
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int c = i / taps, t = i - c * taps;
    const double v = it.w[(long long)n * K + i], g = row[t * c_pad + c];
    s += v; q += v * v; sg += g; sgw += g * v;
  }
  red[0][threadIdx.x] = s; red[1][threadIdx.x] = q; red[2][threadIdx.x] = sg; red[3][threadIdx.x] = sgw;
  __syncthreads();
  __shared__ double st[4];
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int i = 0; i < 256; ++i) t += red[threadIdx.x][i];
    st[threadIdx.x] = t;
  }
  __syncthreads();
  const double mean = st[0] / K;
  double var = st[1] / K - mean * mean;
  if (var < 0.0) var = 0.0;
  const double sigma = sqrt(var), sden = sigma + (double)eps;
  const double mg = st[2] / K;
  const double mgw = (st[3] - mean * st[2]) / (sden * K);
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int c = i / taps, t = i - c * taps;
    const double v = it.w[(long long)n * K + i], g = row[t * c_pad + c];
    const double what = (v - mean) / sden;
    it.dw[(long long)n * K + i] = (float)((g - mg) / sden - (sigma > 0.0 ? mgw * what / sigma : 0.0));
  }
}

// ---- train_depth.py:263 `depth_preds = torch.clamp(depth_preds, 0, 1)` and its backward (sum of the loss gradients,
// passed where 0 <= p <= 1 as torch does)
__global__ void __launch_bounds__(256) clamp01_kernel(const float* __restrict__ p, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = fminf(fmaxf(p[i], 0.f), 1.f);
}
__global__ void __launch_bounds__(256) clamp01_bwd_kernel(const float* __restrict__ p, const float* __restrict__ g1,
                                                          const float* __restrict__ g2, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = p[i];
    const float g = g1[i] + (g2 != nullptr ? g2[i] : 0.f);
    out[i] = (v >= 0.f && v <= 1.f) ? g : 0.f;
  }
}

// ---- small ordered reductions of per-block / per-image partials into parameter gradients
__global__ void gn_param_reduce_kernel(const float* __restrict__ dpar, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       int batch, int c, int accumulate) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double tg = 0.0, tb = 0.0;
  for (int b = 0; b < batch; ++b) {
    tg += (double)dpar[((long long)b * 2 + 0) * c + ch];
    tb += (double)dpar[((long long)b * 2 + 1) * c + ch];
  }
  if (accumulate) { tg += (double)dgamma[ch]; tb += (double)dbeta[ch]; }
  dgamma[ch] = (float)tg;
  dbeta[ch] = (float)tb;
}
// grid ceil(head_c * 33 / 32)
__global__ void __launch_bounds__(256) head_param_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw,
                                                                float* __restrict__ db, int blocks, int head_c, int accumulate) {
  const int e = blockIdx.x * 32 + (threadIdx.x & 31);
  const bool active = e < head_c * 33;
  const float* src = partial + e;
  double t = ordered_sum8(blocks, active, [&](int b) { return __ldg(src + (long long)b * head_c * 33); });
  if (threadIdx.x < 32 && active) {
    const int k = e / 33, j = e % 33;
    float* dst = j < 32 ? dw + k * 32 + j : db + k;
    if (accumulate) t += (double)*dst;
    *dst = (float)t;
  }
}

}  // namespace odb

using namespace odb;

#define ODB_DT(dt, T, what, ...)                                                    \
  do {                                                                              \
    if ((dt) == ODB_DTYPE_BF16) { using T = bf16; __VA_ARGS__; }                    \
    else if ((dt) == ODB_DTYPE_F32) { using T = float; __VA_ARGS__; }               \
    else return fail(ODB_ERR_INVALID, what ": dtype must be ODB_DTYPE_BF16 or ODB_DTYPE_F32"); \
  } while (0)

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

extern "C" int odb_mask_add(const void* a, const void* b, const void* mask, void* out, int64_t n, int32_t dtype,
                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!b || !out || n < 0 || n % 8 || !aligned16(b) || !aligned16(out) || !aligned16(a) || !aligned16(mask))
    return fail(ODB_ERR_INVALID, "mask_add: bad argument (n multiple of 8, 16-byte aligned pointers)");
  if (n == 0) return ODB_OK;
  ODB_DT(dtype, T, "mask_add",
         mask_add_kernel<T><<<grid_for(n / 8), 256, 0, stream>>>(static_cast<const T*>(a), static_cast<const T*>(b),
                                                                 static_cast<const T*>(mask), static_cast<T*>(out), n / 8));
  count_launch();
  return check_launch("mask_add");
}

extern "C" int odb_gelu_fwd(const void* u, void* y, int64_t n, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!u || !y || n < 0 || n % 8 || !aligned16(u) || !aligned16(y)) return fail(ODB_ERR_INVALID, "gelu_fwd: bad argument");
  if (n == 0) return ODB_OK;
  ODB_DT(dtype, T, "gelu_fwd",
         gelu_fwd_kernel<T><<<grid_for(n / 8), 256, 0, stream>>>(static_cast<const T*>(u), static_cast<T*>(y), n / 8));
  count_launch();
  return check_launch("gelu_fwd");
}

extern "C" int odb_gelu_bwd(const void* dy, const void* u, void* du, int64_t n, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dy || !u || !du || n < 0 || n % 8 || !aligned16(u) || !aligned16(dy) || !aligned16(du))
    return fail(ODB_ERR_INVALID, "gelu_bwd: bad argument");
  if (n == 0) return ODB_OK;
  ODB_DT(dtype, T, "gelu_bwd",
         gelu_bwd_kernel<T><<<grid_for(n / 8), 256, 0, stream>>>(static_cast<const T*>(dy), static_cast<const T*>(u),
                                                                 static_cast<T*>(du), n / 8));
  count_launch();
  return check_launch("gelu_bwd");
}

extern "C" int64_t odb_colsum_workspace_bytes(int32_t batches, int64_t rows_per_batch, int32_t n) {
  if (batches < 1 || rows_per_batch < 1 || n < 1) return -1;
  return (int64_t)batches * colsum_slabs(batches, rows_per_batch, n) * n * 4;
}

extern "C" int odb_colsum(const void* x, float* out, void* workspace, int32_t batches, int64_t rows_per_batch, int32_t n,
                          int64_t row_stride, int64_t batch_stride, int32_t accumulate, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !out || !workspace || batches < 1 || batches > 65535 || rows_per_batch < 1 || n < 8 || n % 8 || row_stride % 8 ||
      batch_stride % 8 || !aligned16(x))
    return fail(ODB_ERR_INVALID, "colsum: bad argument");
  const int slabs = colsum_slabs(batches, rows_per_batch, n);
  dim3 grid((n + 63) / 64, (unsigned)slabs, batches);
  float* partial = static_cast<float*>(workspace);
  ODB_DT(dtype, T, "colsum",
         colsum_partial_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), partial, rows_per_batch, n, row_stride,
                                                            batch_stride, slabs));
  count_launch();
  reduce_partials_kernel<<<dim3((n + 31) / 32, batches), 256, 0, stream>>>(partial, out, slabs, n, accumulate);
  count_launch();
  return check_launch("colsum");
}

extern "C" int odb_reduce_partials(const float* partial, float* out, int32_t batches, int32_t parts, int64_t n,
                                   int32_t accumulate, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!partial || !out || batches < 1 || batches > 65535 || parts < 1 || n < 1 || (n + 31) / 32 > 0x7fffffffLL)
    return fail(ODB_ERR_INVALID, "reduce_partials: bad argument");
  reduce_partials_kernel<<<dim3((unsigned)((n + 31) / 32), batches), 256, 0, stream>>>(partial, out, parts, n, accumulate);
  count_launch();
  return check_launch("reduce_partials");
}

constexpr int kLnBwdMaxBlocks = 256;   // one block per SM (register-resident accumulators: 1 block of 8 warps per SM)
extern "C" int64_t odb_layernorm_bwd_workspace_bytes(int32_t cols) { return (int64_t)kLnBwdMaxBlocks * 3 * cols * 4; }

extern "C" int odb_layernorm_bwd(const void* dy, const float* x, const float* gamma, const float* ds_in, float* ds_out,
                                 void* ds_copy, float* dgamma, float* dbeta, float* dcolsum, void* workspace, int64_t rows,
                                 int32_t cols, float eps, int32_t accumulate, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dy || !x || !gamma || !ds_out || !workspace || rows < 1 || (dgamma == nullptr) != (dbeta == nullptr))
    return fail(ODB_ERR_INVALID, "layernorm_bwd: bad argument (dgamma and dbeta both NULL or both set)");
  float* partial = static_cast<float*>(workspace);
  int blocks = num_sms();
  if (blocks > kLnBwdMaxBlocks) blocks = kLnBwdMaxBlocks;
  if ((long long)blocks * 8 > rows) blocks = (int)((rows + 7) / 8);
  const int want_colsum = dcolsum != nullptr, want_params = dgamma != nullptr;
#define ODB_LN_BWD(VPL)                                                                                              \
  ODB_DT(dtype, T, "layernorm_bwd",                                                                                  \
         layernorm_bwd_kernel<VPL, T><<<blocks, 256, 0, stream>>>(static_cast<const T*>(dy), x, gamma, ds_in, ds_out, \
                                                                  static_cast<T*>(ds_copy), partial, (long long)rows, eps, \
                                                                  want_params, want_colsum))
  switch (cols) {
    case 256: ODB_LN_BWD(1); break;
    case 512: ODB_LN_BWD(2); break;
    case 768: ODB_LN_BWD(3); break;
    case 1024: ODB_LN_BWD(4); break;
    default: return fail(ODB_ERR_UNSUPPORTED, "layernorm_bwd: cols must be 256/512/768/1024");
  }
#undef ODB_LN_BWD
  count_launch();
  const int reduced = (want_colsum ? 3 : 2) - (want_params ? 0 : 2);     // partial rows to reduce (0: frozen norm, no colsum)
  if (reduced > 0) {
    ln_param_reduce_kernel<<<(reduced * cols + 31) / 32, 256, 0, stream>>>(partial, dgamma, dbeta, dcolsum, blocks, cols,
                                                                         accumulate);
    count_launch();
  }
  return check_launch("layernorm_bwd");
}

constexpr int kGnBwdMaxC = 1024;
static void gn_bwd_plan(int hw, int c, int* slabs, int* ppb) {
  const int planes = 256 / (c / 8);
  *ppb = planes * 16;
  *slabs = (hw + *ppb - 1) / *ppb;
}
extern "C" int64_t odb_groupnorm_bwd_workspace_bytes(int32_t b, int32_t hw, int32_t c, int32_t groups) {
  if (b < 1 || hw < 1 || c < 8 || c % 8 || c > kGnBwdMaxC || groups < 1 || c % groups || 256 % (c / 8)) return -1;
  int slabs, ppb;
  gn_bwd_plan(hw, c, &slabs, &ppb);
  // slab partials [b][slabs][c][2], coefficients [b][c + 2 groups], dparam shares [b][2][c]
  return ((int64_t)b * slabs * c * 2 + (int64_t)b * (c + 2 * groups) + (int64_t)b * 2 * c) * 4 + 1024;
}

/* dx, dgamma, dbeta of y = relu?(gn(x) ...): g = dy * [mask > 0] (mask NULL: g = dy). */
extern "C" int odb_groupnorm_bwd(const void* dy, const void* mask, const void* x, const float* stats, const float* gamma,
                                 void* dx, float* dgamma, float* dbeta, void* workspace, int32_t b, int32_t hw, int32_t c,
                                 int32_t groups, int32_t accumulate, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dy || !x || !stats || !gamma || !dx || !workspace || (dgamma == nullptr) != (dbeta == nullptr) ||
      odb_groupnorm_bwd_workspace_bytes(b, hw, c, groups) < 0)
    return fail(ODB_ERR_INVALID, "groupnorm_bwd: bad argument (dgamma and dbeta both NULL or both set)");
  const bool want_params = dgamma != nullptr;
  int slabs, ppb;
  gn_bwd_plan(hw, c, &slabs, &ppb);
  float* partial = static_cast<float*>(workspace);
  float* coef = partial + (size_t)b * slabs * c * 2;
  float* dpar = coef + (size_t)b * (c + 2 * groups);
  const int planes = 256 / (c / 8);
  ODB_DT(dtype, T, "groupnorm_bwd",
         groupnorm_bwd_sums_kernel<T><<<dim3(slabs, b), 256, 2 * planes * c * sizeof(float), stream>>>(
             static_cast<const T*>(dy), static_cast<const T*>(mask), static_cast<const T*>(x), partial, hw, c, ppb));
  count_launch();
  const int coef_lanes = 1024 / c > 1 ? 1024 / c : 1;
  groupnorm_bwd_coef_kernel<<<b, 1024, (size_t)(2 * c + 2 * groups + 2 * coef_lanes * c) * sizeof(double), stream>>>(
      partial, stats, gamma, coef, want_params ? dpar : nullptr, slabs, hw, c, groups);
  count_launch();
  long long gx = ((long long)hw * (c / 8) + 255) / 256;
  const long long cap = ((long long)num_sms() * 8 + b - 1) / b;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  ODB_DT(dtype, T, "groupnorm_bwd",
         groupnorm_bwd_apply_kernel<T><<<dim3((unsigned)gx, b), 256, 3 * c * sizeof(float), stream>>>(
             static_cast<const T*>(dy), static_cast<const T*>(mask), static_cast<const T*>(x), coef, static_cast<T*>(dx), hw,
             c, groups));
  count_launch();
  // dgamma / dbeta: ordered sum over the images
  if (want_params) {
    gn_param_reduce_kernel<<<(c + 255) / 256, 256, 0, stream>>>(dpar, dgamma, dbeta, b, c, accumulate);
    count_launch();
  }
  return check_launch("groupnorm_bwd");
}

extern "C" int odb_upsample2x_bwd(const void* dout, void* dz, int32_t b, int32_t h, int32_t w, int32_t c, int32_t dtype,
                                  void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dout || !dz || b < 1 || h < 2 || w < 2 || c < 8 || c % 8 || b > 65535) return fail(ODB_ERR_INVALID, "upsample2x_bwd: bad argument");
  long long gx = ((long long)h * w * (c / 8) + 255) / 256;
  const long long cap = ((long long)num_sms() * 16 + b - 1) / b;
  if (gx > cap) gx = cap;
  ODB_DT(dtype, T, "upsample2x_bwd",
         upsample2x_bwd_kernel<T><<<dim3((unsigned)gx, b), 256, 0, stream>>>(static_cast<const T*>(dout), static_cast<T*>(dz),
                                                                             h, w, c));
  count_launch();
  return check_launch("upsample2x_bwd");
}

extern "C" int odb_stem_pool_bwd(const void* dt, const void* s0, const float* stats, const float* gamma, const float* beta,
                                 void* g_s0, int32_t b, int32_t h, int32_t w, int32_t c, int32_t groups, int32_t dtype,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dt || !s0 || !stats || !gamma || !beta || !g_s0 || b < 1 || h < 2 || w < 2 || (h & 1) || (w & 1) || c < 1 ||
      c % groups || b > 65535)
    return fail(ODB_ERR_INVALID, "stem_pool_bwd: bad argument");
  if (c % 8) return fail(ODB_ERR_INVALID, "stem_pool_bwd: c must be a multiple of 8");
  long long gx = ((long long)h * w * (c / 8) + 255) / 256;
  const long long cap = ((long long)num_sms() * 16 + b - 1) / b;
  if (gx > cap) gx = cap;
  ODB_DT(dtype, T, "stem_pool_bwd",
         stem_pool_bwd_kernel<T><<<dim3((unsigned)gx, b), 256, 2 * c * sizeof(float), stream>>>(
             static_cast<const T*>(dt), static_cast<const T*>(s0), stats, gamma, beta, static_cast<T*>(g_s0), h, w, c, groups));
  count_launch();
  return check_launch("stem_pool_bwd");
}

template <typename T>
static int stem_input_grad_launch(const void* ds0, const void* w, float* dx, int b, int h, int wd, int kpad,
                                  unsigned grid, cudaStream_t stream) {
  static bool configured[kMaxDevices] = {};
  const int dev_ = current_device();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(stem_input_grad_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kSigSmemBytes);
    if (e != cudaSuccess) return fail_cuda(e, "stem_input_grad: cudaFuncSetAttribute");
    configured[dev_] = true;
  }
  launch_pdl(stem_input_grad_kernel<T>, dim3(grid), dim3(256), kSigSmemBytes, stream, static_cast<const T*>(ds0),
             static_cast<const T*>(w), dx, b, h, wd, kpad);
  return ODB_OK;
}

extern "C" int odb_stem_input_grad(const void* ds0, const void* weight, float* dx, int32_t b, int32_t h, int32_t w,
                                   int32_t kpad, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!ds0 || !weight || !dx || b < 1 || h < 2 || w < 2 || (h & 1) || (w & 1) || kpad < 152 || kpad % 8 || kpad > 1024 ||
      !aligned16(ds0) || (reinterpret_cast<uintptr_t>(dx) & 7u))
    return fail(ODB_ERR_INVALID, "stem_input_grad: bad argument (even h, w; kpad a multiple of 8 in [152, 1024]; "
                                 "16-byte aligned ds0, 8-byte aligned dx)");
  // the staged tile is fixed-size (persistent blocks loop over tiles): no limit on h or w
  const long long tiles = (long long)b * ((h / 2 + kSigQH - 1) / kSigQH) * ((w / 2 + kSigQW - 1) / kSigQW);
  const long long cap = (long long)num_sms() * 2;                 // two 90 KiB blocks per SM
  const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
  int rc = ODB_OK;
  ODB_DT(dtype, T, "stem_input_grad", rc = stem_input_grad_launch<T>(ds0, weight, dx, b, h, w, kpad, grid, stream));
  if (rc) return rc;
  count_launch();
  return check_launch("stem_input_grad");
}

extern "C" int odb_pos_embed_resize_bwd(const float* dgrid, float* dpos, int32_t gh, int32_t gw, int32_t d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dgrid || !dpos || gh < 1 || gw < 1 || d < 4 || d % 4 || !aligned16(dgrid) || !aligned16(dpos))
    return fail(ODB_ERR_INVALID, "pos_embed_resize_bwd: bad argument (positive sizes, d a multiple of 4, 16-byte aligned "
                                 "pointers)");
  const int d4 = d / 4;
  const int block = d4 >= 256 ? 256 : (d4 + 31) / 32 * 32;
  const int chunks = (d4 + block - 1) / block;
  const cudaError_t e = launch_pdl(pos_embed_resize_bwd_kernel, dim3(kPosSrc * kPosSrc, chunks < 64 ? chunks : 64),
                                   dim3(block), 0, stream, dgrid, dpos, gh, gw, d4);
  if (e != cudaSuccess) return fail_cuda(e, "pos_embed_resize_bwd");
  count_launch();
  return check_launch("pos_embed_resize_bwd");
}

constexpr int kHeadBwdBlocks = 592;
extern "C" int64_t odb_head_tail_bwd_workspace_bytes(int32_t head_c) { return (int64_t)kHeadBwdBlocks * head_c * 33 * 4; }

extern "C" int odb_head_tail_fwd(const void* a, int32_t channel_stride, const float* w, const float* bias, float* out,
                                 int32_t b, int32_t h, int32_t wd, int32_t head_c, int32_t relu, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!a || !w || !bias || !out || b < 1 || h < 1 || wd < 1 || head_c < 1 || channel_stride < 32 || channel_stride % 8)
    return fail(ODB_ERR_INVALID, "head_tail_fwd: bad argument");
  const long long ppi = (long long)h * wd;
  ODB_DT(dtype, T, "head_tail_fwd",
         head_tail_fwd_kernel<T><<<grid_for(ppi * b), 256, 0, stream>>>(static_cast<const T*>(a), channel_stride, w, bias, out,
                                                                        ppi, b, head_c, relu));
  count_launch();
  return check_launch("head_tail_fwd");
}

extern "C" int odb_head_tail_bwd(const float* dout, const float* out, const void* a, int32_t channel_stride, const float* w,
                                 void* da, float* dw, float* dbias, void* workspace, int32_t b, int32_t h, int32_t wd,
                                 int32_t head_c, int32_t relu, int32_t accumulate, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!dout || !out || !a || !w || !da || !workspace || (dw == nullptr) != (dbias == nullptr) || b < 1 || h < 1 ||
      wd < 1 || head_c < 1 || head_c > 3 || channel_stride < 32 || channel_stride % 8)
    return fail(ODB_ERR_INVALID, "head_tail_bwd: bad argument (head_c <= 3; dw and dbias both NULL or both set)");
  const long long ppi = (long long)h * wd;
  const bool want_params = dw != nullptr;
  float* partial = want_params ? static_cast<float*>(workspace) : nullptr;
  ODB_DT(dtype, T, "head_tail_bwd",
         head_tail_bwd_kernel<T><<<kHeadBwdBlocks, 256, 0, stream>>>(dout, out, static_cast<const T*>(a), channel_stride, w,
                                                                     static_cast<T*>(da), partial, ppi, b, head_c, relu));
  count_launch();
  if (want_params) {
    head_param_reduce_kernel<<<(head_c * 33 + 31) / 32, 256, 0, stream>>>(partial, dw, dbias, kHeadBwdBlocks, head_c,
                                                                         accumulate);
    count_launch();
  }
  return check_launch("head_tail_bwd");
}

extern "C" int odb_add_cast(const float* ds_in, const void* g, float* ds_out, void* copy, int64_t n, int32_t dtype,
                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!g || !ds_out || n < 0 || n % 8 || !aligned16(g) || !aligned16(ds_out) || !aligned16(ds_in) || !aligned16(copy))
    return fail(ODB_ERR_INVALID, "add_cast: bad argument");
  if (n == 0) return ODB_OK;
  ODB_DT(dtype, T, "add_cast",
         add_cast_kernel<T><<<grid_for(n / 8), 256, 0, stream>>>(ds_in, static_cast<const T*>(g), ds_out, static_cast<T*>(copy),
                                                                 n / 8));
  count_launch();
  return check_launch("add_cast");
}

extern "C" int odb_pack_weight(const float* w, void* fwd, void* bwd, int32_t n, int32_t c, int32_t taps, int32_t n_pad,
                               int32_t c_pad, int32_t standardize, float eps, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!w || (!fwd && !bwd) || n < 1 || c < 1 || taps < 1 || n_pad < n || c_pad < c)
    return fail(ODB_ERR_INVALID, "pack_weight: bad argument");
  // with both operands wanted: rows of fwd (coalesced), then bwd as a tiled transpose of fwd; bwd alone: direct
  const bool two_pass = fwd != nullptr && bwd != nullptr;
  ODB_DT(dtype, T, "pack_weight",
         pack_weight_kernel<T><<<n_pad, 256, 0, stream>>>(w, static_cast<T*>(fwd), two_pass ? nullptr : static_cast<T*>(bwd), n,
                                                          c, taps, n_pad, c_pad, standardize, eps));
  count_launch();
  if (two_pass) {
    dim3 grid((n_pad + 31) / 32, (c_pad + 31) / 32, taps);
    ODB_DT(dtype, T, "pack_weight",
           pack_transpose_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(fwd), static_cast<T*>(bwd), taps, n_pad,
                                                              c_pad));
    count_launch();
  }
  return check_launch("pack_weight");
}

extern "C" int odb_unpack_wgrad(const float* gp, const float* w, float* dw, int32_t n, int32_t c, int32_t taps, int32_t c_pad,
                                int32_t standardize, float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!gp || !dw || (standardize && !w) || n < 1 || c < 1 || taps < 1 || c_pad < c)
    return fail(ODB_ERR_INVALID, "unpack_wgrad: bad argument");
  if ((long long)taps * c_pad * 4 > 40 * 1024) return fail(ODB_ERR_UNSUPPORTED, "unpack_wgrad: taps * c_pad too large");
  unpack_wgrad_kernel<<<n, 256, (size_t)taps * c_pad * sizeof(float), stream>>>(gp, w, dw, n, c, taps, c_pad, standardize, eps);
  count_launch();
  return check_launch("unpack_wgrad");
}

extern "C" int odb_clamp01(const float* p, float* out, int64_t n, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !out || n < 0) return fail(ODB_ERR_INVALID, "clamp01: bad argument");
  if (n == 0) return ODB_OK;
  clamp01_kernel<<<grid_for(n), 256, 0, stream>>>(p, out, n);
  count_launch();
  return check_launch("clamp01");
}

extern "C" int odb_clamp01_bwd(const float* p, const float* g1, const float* g2, float* out, int64_t n, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !g1 || !out || n < 0) return fail(ODB_ERR_INVALID, "clamp01_bwd: bad argument");
  if (n == 0) return ODB_OK;
  clamp01_bwd_kernel<<<grid_for(n), 256, 0, stream>>>(p, g1, g2, out, n);
  count_launch();
  return check_launch("clamp01_bwd");
}

extern "C" int odb_pack_weights_multi(const void* items, int32_t n_items, int32_t total_rows, int32_t total_tiles, float eps,
                                      int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!items || n_items < 1 || total_rows < 1 || total_tiles < 0) return fail(ODB_ERR_INVALID, "pack_weights_multi: bad argument");
  const PackItem* it = static_cast<const PackItem*>(items);
  ODB_DT(dtype, T, "pack_weights_multi", pack_weights_multi_kernel<T><<<total_rows, 256, 0, stream>>>(it, n_items, eps));
  count_launch();
  if (total_tiles > 0) {
    ODB_DT(dtype, T, "pack_weights_multi", pack_transpose_multi_kernel<T><<<total_tiles, 256, 0, stream>>>(it, n_items));
    count_launch();
  }
  return check_launch("pack_weights_multi");
}

extern "C" int odb_unpack_wgrads_multi(const void* items, int32_t n_items, int32_t total_rows, int32_t max_row_floats, float eps,
                                       void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!items || n_items < 1 || total_rows < 1 || max_row_floats < 1 || (long long)max_row_floats * 4 > 40 * 1024)
    return fail(ODB_ERR_INVALID, "unpack_wgrads_multi: bad argument (rows of at most 10240 floats)");
  unpack_wgrads_multi_kernel<<<total_rows, 256, (size_t)max_row_floats * sizeof(float), stream>>>(
      static_cast<const UnpackItem*>(items), n_items, eps);
  count_launch();
  return check_launch("unpack_wgrads_multi");
}
