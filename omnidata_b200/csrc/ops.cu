// HBM-bound kernels of the DPT-Hybrid path: LayerNorm, GroupNorm (stats / apply / stem tail),
// stem im2col, bilinear x2 (+ skip add), cls row, ProjectReadout cls term.
// All activations are channels-last bf16; every thread moves 16-byte vectors (8 channels),
// consecutive threads touch consecutive addresses.  What each replaces in the reference is
// documented in include/omnidata_b200.h.
#include "common.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

ODB_DEVINL void load8(const bf16* p, float* v) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
               d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
ODB_DEVINL void store8(bf16* p, const float* v) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// fp32 storage (the ViT residual stream, and every activation in the fp32 correctness mode): the same 8-element
// item is two 16-byte vectors
ODB_DEVINL void load8(const float* p, float* v) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
ODB_DEVINL void store8(float* p, const float* v) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
ODB_DEVINL void store1(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
ODB_DEVINL void store1(float* p, float v) { *p = v; }

// ---- e4m3 storage (the fp8 inference mode's GEMM operands), quantised per row:
//   amax = max |z|, scale = amax / 448, q = cvt.rn.satfinite.e4m3(z * (448 / amax)); an all-zero row: scale 1, q = z * 0.
// Both divisions are IEEE round-to-nearest (__fdiv_rn) although this file is built with fast math.
struct e4m3_t { uint8_t bits; };
ODB_DEVINL float e4m3_inv_scale(float amax) { return amax > 0.f ? __fdiv_rn(448.f, amax) : 0.f; }
ODB_DEVINL float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f; }
// eight values times inv -> eight e4m3 bytes, v[0] in the lowest byte
ODB_DEVINL uint2 quant8_e4m3(const float* v, float inv) {
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint16_t h;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h) : "f"(__fmul_rn(v[2 * k + 1], inv)),
        "f"(__fmul_rn(v[2 * k], inv)));
    w[k] = h;
  }
  return make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
}

// ------------------------------------------------------------------------------------------
// LayerNorm: each warp normalises TWO rows held in registers (cols <= 1024 -> <= 4 vectors per lane
// and row), so six to eight 16-byte loads are in flight per lane before the first reduction.
// TO = e4m3_t: the fp32 results stay in registers until the row's amax is known, then are quantised as above and
// the row scale goes to row_scale[row] (unused otherwise).
template <int VPL, typename TI, typename TO>  // 8-element items per lane and row; cols = VPL * 256
__global__ void __launch_bounds__(256) layernorm_kernel(const TI* __restrict__ x,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta,
                                                        TO* __restrict__ y, long long rows,
                                                        float eps, float* __restrict__ row_scale) {
  constexpr bool E4M3 = std::is_same<TO, e4m3_t>::value;
  grid_dep_wait();
  grid_dep_launch();
  constexpr int COLS = VPL * 256;
  const int lane = threadIdx.x & 31;
  const long long row0 = 2 * ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5));
  if (row0 >= rows) return;
  const bool two = row0 + 1 < rows;
  float v[2][VPL][8];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (r == 1 && !two) break;
    const TI* xr = x + (row0 + r) * COLS;
#pragma unroll
    for (int i = 0; i < VPL; ++i) load8(xr + (i * 32 + lane) * 8, v[r][i]);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (r == 1 && !two) break;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[r][i][j];
    const float mean = warp_sum(s) * (1.0f / COLS);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[r][i][j] - mean;
        q += d * d;
      }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / COLS) + eps);
    TO* yr = y + (row0 + r) * COLS;
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c0 = (i * 32 + lane) * 8;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[r][i][j] - mean) * rstd * g[j] + bb[j];
      if constexpr (E4M3) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[r][i][j] = o[j];
          amax = fmaxf(amax, fabsf(o[j]));
        }
      } else {
        store8(yr + c0, o);
      }
    }
    if constexpr (E4M3) {
      amax = warp_max(amax);
      const float inv = e4m3_inv_scale(amax);
#pragma unroll
      for (int i = 0; i < VPL; ++i)
        *reinterpret_cast<uint2*>(yr + (i * 32 + lane) * 8) = quant8_e4m3(v[r][i], inv);
      if (lane == 0) row_scale[row0 + r] = e4m3_row_scale(amax);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Per-row e4m3 quantisation of a bf16 [rows][cols] tensor (the inputs of attn.proj and mlp.fc2 in the fp8 mode): one
// warp per row, the row held in registers as VPL 16-byte vectors per lane (cols = VPL * 256) between the amax
// reduction and the quantisation; 8-byte e4m3 stores.
template <int VPL>
__global__ void __launch_bounds__(256) rowquant_e4m3_kernel(const bf16* __restrict__ x, e4m3_t* __restrict__ y,
                                                            float* __restrict__ row_scale, long long rows) {
  grid_dep_wait();
  grid_dep_launch();
  constexpr int COLS = VPL * 256;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bf16* xr = x + row * COLS;
  uint4 u[VPL];
#pragma unroll
  for (int i = 0; i < VPL; ++i) u[i] = __ldg(reinterpret_cast<const uint4*>(xr + (i * 32 + lane) * 8));
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&u[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(w[k]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  amax = warp_max(amax);
  const float inv = e4m3_inv_scale(amax);
  e4m3_t* yr = y + row * COLS;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&u[i]);
    float f[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 t = unpack_bf16x2(w[k]);
      f[2 * k] = t.x;
      f[2 * k + 1] = t.y;
    }
    *reinterpret_cast<uint2*>(yr + (i * 32 + lane) * 8) = quant8_e4m3(f, inv);
  }
  if (lane == 0) row_scale[row] = e4m3_row_scale(amax);
}

// ------------------------------------------------------------------------------------------
// GroupNorm statistics, deterministic: block = (image, pixel slab); thread = (channel octet, pixel
// lane) accumulates fp32 partial sums over a short strided run; the block combines them in a FIXED
// order in fp64 and writes one (sum, sum of squares) pair per group to a partials buffer.  The last
// block of an image to finish (ticket counter) reduces the slabs in slab order, in fp64, and
// writes (mean, rstd) — no floating-point atomics anywhere, so results are bit-reproducible
// run to run and independent of the batch size.
constexpr int kGnMaxC = 1024;

template <typename T>
__global__ void __launch_bounds__(256) groupnorm_stats_kernel(
    const T* __restrict__ x, float* __restrict__ stats, double* __restrict__ partial,
    unsigned int* __restrict__ counters, int hw, int c, int groups, int pixels_per_block,
    float eps) {
  __shared__ float s_thr[2][256 * 8];     // per-thread channel partials, [plane][channel]
  __shared__ double s_ch[2][kGnMaxC];     // per-channel block sums
  __shared__ int s_last;
  const int b = blockIdx.y, slab = blockIdx.x, slabs = gridDim.x;
  const int octets = c >> 3;
  const int cpg = c / groups;
  const int p0 = slab * pixels_per_block;
  const int p1 = min(hw, p0 + pixels_per_block);
  const int oct = threadIdx.x % octets;
  const int plane = threadIdx.x / octets;
  const int planes = blockDim.x / octets;
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (plane < planes) {
    const T* base = x + ((long long)b * hw) * c + oct * 8;
    for (int p = p0 + plane; p < p1; p += planes) {
      float v[8];
      load8(base + (long long)p * c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j] += v[j]; q[j] = fmaf(v[j], v[j], q[j]); }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s_thr[0][plane * c + oct * 8 + j] = s[j];
      s_thr[1][plane * c + oct * 8 + j] = q[j];
    }
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    double ts = 0.0, tq = 0.0;
    for (int pl = 0; pl < planes; ++pl) {
      ts += (double)s_thr[0][pl * c + ch];
      tq += (double)s_thr[1][pl * c + ch];
    }
    s_ch[0][ch] = ts;
    s_ch[1][ch] = tq;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    double ts = 0.0, tq = 0.0;
    for (int j = 0; j < cpg; ++j) { ts += s_ch[0][g * cpg + j]; tq += s_ch[1][g * cpg + j]; }
    double* dst = partial + (((long long)b * slabs + slab) * groups + g) * 2;
    dst[0] = ts;
    dst[1] = tq;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(&counters[b], 1u);
    s_last = (ticket == (unsigned int)(slabs - 1));
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    if (threadIdx.x < groups) {
      const int g = threadIdx.x;
      double ts = 0.0, tq = 0.0;
      for (int sl = 0; sl < slabs; ++sl) {
        const double* src = partial + (((long long)b * slabs + sl) * groups + g) * 2;
        ts += src[0];
        tq += src[1];
      }
      const double n = (double)hw * (double)cpg;
      const double mean = ts / n;
      double var = tq / n - mean * mean;
      if (var < 0.0) var = 0.0;
      stats[((long long)b * groups + g) * 2 + 0] = (float)mean;
      stats[((long long)b * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
    if (threadIdx.x == 0) counters[b] = 0u;   // self-reset for the next launch on this stream
  }
}

// Finalize the per-warp partial sums written by the conv epilogue: block = image, one warp per
// group; lane l sums rows l, l+32, ... in fp64 (independent loads, fixed order), then a fixed
// shuffle tree combines the 32 lanes.
__global__ void __launch_bounds__(1024) groupnorm_finalize_kernel(const float* __restrict__ partial,
                                                                  float* __restrict__ stats,
                                                                  int rows, int groups, double count,
                                                                  float eps) {
  grid_dep_wait();
  grid_dep_launch();
  const int b = blockIdx.x;
  const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (g >= groups) return;
  const float* base = partial + ((long long)b * rows) * groups * 2 + g * 2;
  double ts = 0.0, tq = 0.0;
#pragma unroll 4
  for (int r = lane; r < rows; r += 32) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(base + (long long)r * groups * 2));
    ts += (double)v.x;
    tq += (double)v.y;
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    ts += __shfl_down_sync(0xffffffffu, ts, o);
    tq += __shfl_down_sync(0xffffffffu, tq, o);
  }
  if (lane == 0) {
    const double mean = ts / count;
    double var = tq / count - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[((long long)b * groups + g) * 2 + 0] = (float)mean;
    stats[((long long)b * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

struct GnCoef {  // per-channel scale/shift of one image: y = x * a + b
  float a, b;
};
ODB_DEVINL GnCoef gn_coef(const float* stats, const float* gamma, const float* beta, int b,
                          int groups, int cpg, int ch) {
  const int g = ch / cpg;
  const float mean = __ldg(&stats[((long long)b * groups + g) * 2 + 0]);
  const float rstd = __ldg(&stats[((long long)b * groups + g) * 2 + 1]);
  GnCoef k;
  k.a = rstd * __ldg(gamma + ch);
  k.b = __ldg(beta + ch) - mean * k.a;
  return k;
}

// y = relu?( gn(x) + shortcut ).  Each block first folds the statistics and the affine parameters
// of its image into a per-channel (scale, shift) table in shared memory, so the streaming loop is
// one FMA per element; thread = (pixel, channel octet), 16-byte accesses.
template <typename T>
__global__ void __launch_bounds__(256) groupnorm_apply_kernel(
    const T* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
    const float* __restrict__ beta, const T* __restrict__ res,
    const float* __restrict__ res_stats, const float* __restrict__ res_gamma,
    const float* __restrict__ res_beta, T* __restrict__ y, int hw, int c, int groups, int relu) {
  grid_dep_wait();
  grid_dep_launch();
  extern __shared__ float coef[];  // [c] scale, [c] shift, then [c] shortcut scale (shift is folded)
  const int b = blockIdx.y;
  const int octets = c >> 3;
  const int cpg = c / groups;
  const bool res_norm = (res != nullptr) && (res_stats != nullptr);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    GnCoef k = gn_coef(stats, gamma, beta, b, groups, cpg, ch);
    if (res_norm) {
      const GnCoef kr = gn_coef(res_stats, res_gamma, res_beta, b, groups, cpg, ch);
      coef[2 * c + ch] = kr.a;
      k.b += kr.b;
    }
    coef[ch] = k.a;
    coef[c + ch] = k.b;
  }
  __syncthreads();
  // 32-bit indexing inside one image (hw * c < 2^31); c is a power of two on this path
  const unsigned total = (unsigned)hw * (unsigned)octets;
  const unsigned omask = (unsigned)octets - 1u;
  const bool pow2 = (octets & (octets - 1)) == 0;
  const T* xb = x + ((long long)b * hw) * c;
  const T* rb = res ? res + ((long long)b * hw) * c : nullptr;
  T* yb = y + ((long long)b * hw) * c;
  // A thread always lands on the same channel octet (the grid stride is a multiple of the octet
  // count), so its (scale, shift) coefficients are loaded from shared memory ONCE; two independent
  // items per iteration keep all global loads ahead of the math.
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned first = blockIdx.x * blockDim.x + threadIdx.x;
  const bool fixed_oct = pow2 && (stride & omask) == 0;
  float a[8], sh[8], ra[8];
  {
    const unsigned oct = pow2 ? (first & omask) : (first % (unsigned)octets);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      a[j] = coef[oct * 8 + j];
      sh[j] = coef[c + oct * 8 + j];
      ra[j] = res_norm ? coef[2 * c + oct * 8 + j] : 1.0f;
    }
  }
  for (unsigned i0 = first; i0 < total; i0 += 2 * stride) {
    const unsigned i1 = i0 + stride;
    const bool has1 = i1 < total;
    float v[2][8], r[2][8];
    load8(xb + i0 * 8u, v[0]);
    if (has1) load8(xb + i1 * 8u, v[1]);
    if (rb != nullptr) {
      load8(rb + i0 * 8u, r[0]);
      if (has1) load8(rb + i1 * 8u, r[1]);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const unsigned i = u ? i1 : i0;
      if (u && !has1) break;
      if (!fixed_oct) {
        const unsigned oct = pow2 ? (i & omask) : (i % (unsigned)octets);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          a[j] = coef[oct * 8 + j];
          sh[j] = coef[c + oct * 8 + j];
          ra[j] = res_norm ? coef[2 * c + oct * 8 + j] : 1.0f;
        }
      }
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf(v[u][j], a[j], sh[j]);
      if (rb != nullptr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(r[u][j], ra[j], o[j]);
      }
      if (relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j], 0.f);
      }
      store8(yb + i * 8u, o);
    }
  }
}

// Stem: GroupNorm + ReLU + MaxPool 3x3 s2, TF-SAME pad (0,1): window rows/cols 2o..2o+2, clipped.
template <typename T>
__global__ void __launch_bounds__(256) stem_gn_relu_maxpool_kernel(
    const T* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
    const float* __restrict__ beta, T* __restrict__ y, int h, int w, int c, int groups) {
  grid_dep_wait();
  grid_dep_launch();
  extern __shared__ float coef[];  // [c] scale, [c] shift
  const int b = blockIdx.y;
  const int octets = c >> 3;
  const int cpg = c / groups;
  const int oh = h / 2, ow = w / 2;
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    const GnCoef k = gn_coef(stats, gamma, beta, b, groups, cpg, ch);
    coef[ch] = k.a;
    coef[c + ch] = k.b;
  }
  __syncthreads();
  const unsigned total = (unsigned)oh * (unsigned)ow * (unsigned)octets;
  const T* xb = x + (long long)b * h * w * c;
  T* yb = y + (long long)b * oh * ow * c;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned oct = i % (unsigned)octets;
    const unsigned pix = i / (unsigned)octets;
    const int ox = (int)(pix % (unsigned)ow), oy = (int)(pix / (unsigned)ow);
    float a[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] = coef[oct * 8 + j]; sh[j] = coef[c + oct * 8 + j]; }
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = 0.f;  // relu output is >= 0, so 0 is the identity of max
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int iy = 2 * oy + dy;
      if (iy >= h) continue;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int ix = 2 * ox + dx;
        if (ix >= w) continue;
        float v[8];
        load8(xb + ((unsigned)iy * (unsigned)w + (unsigned)ix) * (unsigned)c + oct * 8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], fmaf(v[j], a[j], sh[j]));  // relu folded into max(0,.)
      }
    }
    store8(yb + pix * (unsigned)c + oct * 8, m);
  }
}

// Stem im2col: fp32 NCHW -> bf16 [b*oh*ow][kpad], column (ky*7+kx)*3+ch, TF-SAME pad (2,3), stride 2.
// One block per output row: the 7 input rows x 3 channels it reads are staged ONCE in shared memory
// with coalesced loads (zero-filled borders = the convolution padding), then thread = (output pixel,
// 8-column group) gathers its 8 columns from shared memory through a 160-entry offset table — no
// per-element div/mod, no bounds tests, no redundant global loads (the first version issued 8 scalar
// global loads and ~40 integer ops per 16 output bytes and ran at 1.2 TB/s).
constexpr int kStemMaxW = 1792;                      // staged rows: 21 x (w + 5) floats <= 151 KiB
template <typename T>
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x,
                                                          T* __restrict__ cols, int b, int h,
                                                          int w, int kpad) {
  grid_dep_wait();
  grid_dep_launch();
  extern __shared__ float stage[];                   // [3 ch][7 ky][w + 5], then int off[kpad]
  const int pitch = w + 5;
  int* off = reinterpret_cast<int*>(stage + 21 * pitch);
  const int oh = h / 2, ow = w / 2;
  const int groups8 = kpad >> 3;
  const int oy = blockIdx.x % oh, bi = blockIdx.x / oh;
  const float* xb = x + (long long)bi * 3 * h * w;
  // input rows 2*oy - 2 .. 2*oy + 4, columns -2 .. w + 2
  for (int i = threadIdx.x; i < 21 * pitch; i += blockDim.x) {
    const int r = i / pitch, px = i - r * pitch;     // r = ch * 7 + ky
    const int ch = r / 7, ky = r - ch * 7;
    const int iy = 2 * oy + ky - 2, ix = px - 2;
    stage[i] = (iy >= 0 && iy < h && ix >= 0 && ix < w) ? __ldg(xb + ((long long)ch * h + iy) * w + ix) : 0.f;
  }
  for (int col = threadIdx.x; col < kpad; col += blockDim.x) {
    const int ch = col % 3, kx = (col / 3) % 7, ky = col / 21;
    off[col] = col < 147 ? (ch * 7 + ky) * pitch + kx : -1;
  }
  __syncthreads();
  T* crow = cols + ((long long)bi * oh + oy) * ow * kpad;
  const int total = ow * groups8;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const int ox = i / groups8;
    const int g = i - ox * groups8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int o = off[g * 8 + j];
      v[j] = o >= 0 ? stage[o + 2 * ox] : 0.f;
    }
    store8(crow + i * 8, v);
  }
}

// Patch embedding gather of the plain ViT backbones (timm PatchEmbed: Conv2d(3, D, 16, stride 16),
// modules/midas/vit.py:131 `patch_embed.proj(x)`): fp32 NCHW -> bf16 [b * gh * gw][3 * p * p], column
// (c * p + py) * p + px — the row-major flattening of the conv weight [D][3][p][p], so the conv is one GEMM.
// Thread = (token, 8 consecutive px of one (c, py) row): two float4 loads, one 16-byte store.
template <typename T>
__global__ void __launch_bounds__(256) patchify_kernel(const float* __restrict__ x, T* __restrict__ cols,
                                                       int b, int h, int w, int p) {
  grid_dep_wait();
  grid_dep_launch();
  const int gh = h / p, gw = w / p;
  const int groups = 3 * p * p / 8;                      // 8-column groups per token
  const long long total = (long long)b * gh * gw * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const long long tok = i / groups;
    const int tx = (int)(tok % gw), ty = (int)((tok / gw) % gh), bi = (int)(tok / ((long long)gw * gh));
    const int col = g * 8;
    const int px = col % p, py = (col / p) % p, c = col / (p * p);
    const float* src = x + (((long long)bi * 3 + c) * h + (ty * p + py)) * w + tx * p + px;
    const float4 a = __ldg(reinterpret_cast<const float4*>(src));
    const float4 d = __ldg(reinterpret_cast<const float4*>(src + 4));
    const float v[8] = {a.x, a.y, a.z, a.w, d.x, d.y, d.z, d.w};
    store8(cols + i * 8, v);
  }
}

// Bilinear x2, align_corners=True: src = dst * (n-1)/(2n-1).  out = up(z) (+ res); out_relu = relu(out).
// ncu showed the first two versions of this kernel ISSUE-bound (75-88 % issue slots, ~30 % DRAM):
// four gathers, 32 unpacks and 32 FMAs for every 16 output bytes.  With align_corners=True and an
// exact x2 factor, output columns 2k+1 and 2k+2 both interpolate between source columns k and k+1
// (and likewise for rows), so a thread now owns one SOURCE quad (m..m+1, k..k+1) and produces the
// 2x2 output block {2m+1, 2m+2} x {2k+1, 2k+2} from a single set of four loads; m = -1 / k = -1 and
// m = h-1 / k = w-1 produce the border rows / columns (source index clamped, weight 0 or 1).
// blockDim = (channel octets, quads along x); no integer division, 32-bit index math.
template <typename T>
__global__ void __launch_bounds__(256) upsample2x_add_kernel(const T* __restrict__ z,
                                                             const T* __restrict__ res,
                                                             T* __restrict__ out,
                                                             T* __restrict__ out_relu, int h, int w,
                                                             int c) {
  grid_dep_wait();
  grid_dep_launch();
  const int oh = 2 * h, ow = 2 * w;
  const int k = (int)(blockIdx.x * blockDim.y + threadIdx.y) - 1;   // source quad column, -1 .. w-1
  if (k > w - 1) return;
  const int m = (int)blockIdx.y - 1;                                // source quad row,    -1 .. h-1
  const int bi = blockIdx.z;
  const int ch = threadIdx.x * 8;
  const float sy = (float)(h - 1) / (float)(oh - 1), sx = (float)(w - 1) / (float)(ow - 1);
  const int ys = min(max(m, 0), h - 2), xs = min(max(k, 0), w - 2);
  const T* zb = z + ((size_t)bi * h + ys) * w * c + (size_t)xs * c + ch;
  float q00[8], q01[8], q10[8], q11[8];
  load8(zb, q00);
  load8(zb + c, q01);
  load8(zb + (size_t)w * c, q10);
  load8(zb + (size_t)w * c + c, q11);
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) {
    const int oy = 2 * m + 1 + dy;
    if (oy < 0 || oy >= oh) continue;
    const float wy = fminf(fmaxf(oy * sy - (float)ys, 0.f), 1.f);
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int ox = 2 * k + 1 + dx;
      if (ox < 0 || ox >= ow) continue;
      const float wx = fminf(fmaxf(ox * sx - (float)xs, 0.f), 1.f);
      const float w11 = wy * wx, w10 = wy - w11, w01 = wx - w11, w00 = 1.0f - wy - wx + w11;
      const size_t off = ((size_t)(bi * oh + oy) * ow + ox) * c + ch;
      float o[8];
      if (res != nullptr) {
        float r[8];
        load8(res + off, r);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          o[j] = fmaf(w11, q11[j], fmaf(w10, q10[j], fmaf(w01, q01[j], fmaf(w00, q00[j], r[j]))));
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          o[j] = fmaf(w11, q11[j], fmaf(w10, q10[j], fmaf(w01, q01[j], w00 * q00[j])));
      }
      store8(out + off, o);
      if (out_relu != nullptr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j], 0.f);
        store8(out_relu + off, o);
      }
    }
  }
}

template <typename T>
__global__ void write_cls_row_kernel(T* __restrict__ tokens, const float* __restrict__ cls,
                                     const float* __restrict__ pos0, int tokens_n, int c) {
  grid_dep_wait();
  grid_dep_launch();
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < c; i += blockDim.x)
    store1(tokens + (long long)b * tokens_n * c + i, cls[i] + pos0[i]);
}

// out[b][n] = bias[n] + sum_k w[n][c + k] * tokens[b][0][k];  one warp per (b, n).
template <typename T>
__global__ void __launch_bounds__(256) readout_cls_bias_kernel(const T* __restrict__ w,
                                                               const float* __restrict__ bias,
                                                               const T* __restrict__ tokens,
                                                               float* __restrict__ out, int b_n,
                                                               int tokens_n, int c) {
  grid_dep_wait();
  grid_dep_launch();
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)b_n * c) return;
  const int n = (int)(wid % c), b = (int)(wid / c);
  const T* wr = w + (long long)n * 2 * c + c;
  const T* t = tokens + (long long)b * tokens_n * c;
  float acc = 0.f;
  for (int k = lane * 8; k < c; k += 256) {
    float a[8], x[8];
    load8(wr + k, a);
    load8(t + k, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(a[j], x[j], acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[wid] = acc + __ldg(bias + n);
}

// fp32 -> bf16 copy (the hooked ViT activations: the residual stream is fp32, the readout GEMM reads bf16)
__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst,
                                                            long long n8) {
  grid_dep_wait();
  grid_dep_launch();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float v[8];
    load8(src + i * 8, v);
    store8(dst + i * 8, v);
  }
}

// grid.x of a (blocks per image, image) launch: the per-image block count, capped by the share of
// the chip-wide block budget one image gets
static int per_image_grid(long long items_per_image, int block, int b, int max_blocks_per_sm = 8) {
  long long blocks = (items_per_image + block - 1) / block;
  long long cap = ((long long)num_sms() * max_blocks_per_sm + b - 1) / b;
  if (cap < 1) cap = 1;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace odb

using namespace odb;

// storage type dispatch: T = bf16 (ODB_DTYPE_BF16) or float (ODB_DTYPE_F32)
#define ODB_DTYPE_SWITCH(dt, T, what, ...)                                          \
  do {                                                                              \
    if ((dt) == ODB_DTYPE_BF16) { using T = bf16; __VA_ARGS__; }                    \
    else if ((dt) == ODB_DTYPE_F32) { using T = float; __VA_ARGS__; }               \
    else return fail(ODB_ERR_INVALID, what ": dtype must be ODB_DTYPE_BF16 or ODB_DTYPE_F32"); \
  } while (0)

template <typename TI, typename TO>
static int layernorm_launch(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int32_t cols,
                            float eps, cudaStream_t stream, float* rs = nullptr) {
  const int rpb = 16;   // 8 warps x 2 rows
  const unsigned grid = (unsigned)((rows + rpb - 1) / rpb);
  const TI* xp = static_cast<const TI*>(x);
  TO* yp = static_cast<TO*>(y);
  switch (cols) {
    case 256: launch_pdl(layernorm_kernel<1, TI, TO>, dim3(grid), dim3(256), 0, stream, xp, gamma, beta, yp, (long long)rows, eps, rs); break;
    case 512: launch_pdl(layernorm_kernel<2, TI, TO>, dim3(grid), dim3(256), 0, stream, xp, gamma, beta, yp, (long long)rows, eps, rs); break;
    case 768: launch_pdl(layernorm_kernel<3, TI, TO>, dim3(grid), dim3(256), 0, stream, xp, gamma, beta, yp, (long long)rows, eps, rs); break;
    case 1024: launch_pdl(layernorm_kernel<4, TI, TO>, dim3(grid), dim3(256), 0, stream, xp, gamma, beta, yp, (long long)rows, eps, rs); break;
    default: return fail(ODB_ERR_UNSUPPORTED, "layernorm: cols must be 256/512/768/1024");
  }
  count_launch();
  return check_launch("layernorm");
}

extern "C" int odb_layernorm(const void* x, const float* gamma, const float* beta, void* y,
                             int64_t rows, int32_t cols, float eps, int32_t x_dtype, int32_t y_dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !gamma || !beta || !y || rows < 0) return fail(ODB_ERR_INVALID, "layernorm: bad argument");
  if (rows == 0) return ODB_OK;
  if (x_dtype == ODB_DTYPE_BF16 && y_dtype == ODB_DTYPE_BF16) return layernorm_launch<bf16, bf16>(x, gamma, beta, y, rows, cols, eps, stream);
  if (x_dtype == ODB_DTYPE_F32 && y_dtype == ODB_DTYPE_BF16) return layernorm_launch<float, bf16>(x, gamma, beta, y, rows, cols, eps, stream);
  if (x_dtype == ODB_DTYPE_F32 && y_dtype == ODB_DTYPE_F32) return layernorm_launch<float, float>(x, gamma, beta, y, rows, cols, eps, stream);
  return fail(ODB_ERR_INVALID, "layernorm: (x, y) dtypes must be (bf16, bf16), (f32, bf16) or (f32, f32)");
}

extern "C" int odb_layernorm_e4m3(const void* x, const float* gamma, const float* beta, void* y, float* row_scale,
                                  int64_t rows, int32_t cols, float eps, int32_t x_dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !gamma || !beta || !y || !row_scale || rows < 0) return fail(ODB_ERR_INVALID, "layernorm_e4m3: bad argument");
  if ((reinterpret_cast<uintptr_t>(y) & 7u) != 0) return fail(ODB_ERR_INVALID, "layernorm_e4m3: y must be 8-byte aligned");
  if (rows == 0) return ODB_OK;
  if (x_dtype == ODB_DTYPE_F32) return layernorm_launch<float, e4m3_t>(x, gamma, beta, y, rows, cols, eps, stream, row_scale);
  if (x_dtype == ODB_DTYPE_BF16) return layernorm_launch<bf16, e4m3_t>(x, gamma, beta, y, rows, cols, eps, stream, row_scale);
  return fail(ODB_ERR_INVALID, "layernorm_e4m3: x_dtype must be ODB_DTYPE_F32 or ODB_DTYPE_BF16");
}

extern "C" int odb_rowquant_e4m3(const void* x, void* y, float* row_scale, int64_t rows, int32_t cols, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !y || !row_scale || rows < 0) return fail(ODB_ERR_INVALID, "rowquant_e4m3: bad argument");
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) != 0)
    return fail(ODB_ERR_INVALID, "rowquant_e4m3: x and y must be 16-byte aligned");
  if (rows == 0) return ODB_OK;
  const unsigned grid = (unsigned)((rows + 7) / 8);       // 8 warps, one row each
  const bf16* xp = static_cast<const bf16*>(x);
  e4m3_t* yp = static_cast<e4m3_t*>(y);
  const long long n = rows;
  switch (cols) {
    case 768: launch_pdl(rowquant_e4m3_kernel<3>, dim3(grid), dim3(256), 0, stream, xp, yp, row_scale, n); break;
    case 1024: launch_pdl(rowquant_e4m3_kernel<4>, dim3(grid), dim3(256), 0, stream, xp, yp, row_scale, n); break;
    case 3072: launch_pdl(rowquant_e4m3_kernel<12>, dim3(grid), dim3(256), 0, stream, xp, yp, row_scale, n); break;
    case 4096: launch_pdl(rowquant_e4m3_kernel<16>, dim3(grid), dim3(256), 0, stream, xp, yp, row_scale, n); break;
    default: return fail(ODB_ERR_UNSUPPORTED, "rowquant_e4m3: cols must be 768, 1024, 3072 or 4096");
  }
  count_launch();
  return check_launch("rowquant_e4m3");
}

static int gn_args_ok(int b, int hw, int c, int groups) {
  return b > 0 && hw > 0 && c > 0 && groups > 0 && groups <= 64 && c % 8 == 0 && c % groups == 0 &&
         (c / 8) <= 256 && ((c / groups) >= 8 ? (c / groups) % 8 == 0 : 8 % (c / groups) == 0);
}

static void gn_stats_plan(int b, int hw, int c, int* slabs, int* ppb) {
  // The slab size depends on the layer shape only (never on the batch), so that the order of every
  // floating-point sum — and therefore the result — is identical whatever batch an image sits in.
  (void)b;
  const int planes = 256 / (c / 8);
  *ppb = planes * 8;                      // 8 pixels per thread
  *slabs = (hw + *ppb - 1) / *ppb;
}

extern "C" int64_t odb_groupnorm_scratch_bytes(int32_t b, int32_t hw, int32_t c, int32_t groups) {
  if (!gn_args_ok(b, hw, c, groups)) return -1;
  int slabs, ppb;
  gn_stats_plan(b, hw, c, &slabs, &ppb);
  return 256 + (int64_t)b * 4 + (int64_t)b * slabs * groups * 2 * 8;
}

extern "C" int odb_groupnorm_stats(const void* x, float* stats, void* scratch, int64_t scratch_bytes,
                                   int32_t b, int32_t hw, int32_t c, int32_t groups, float eps,
                                   int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !stats || !scratch || !gn_args_ok(b, hw, c, groups) || c > kGnMaxC)
    return fail(ODB_ERR_INVALID, "groupnorm_stats: bad argument");
  if (scratch_bytes < odb_groupnorm_scratch_bytes(b, hw, c, groups) ||
      (reinterpret_cast<uintptr_t>(scratch) & 255u))
    return fail(ODB_ERR_INVALID, "groupnorm_stats: scratch too small or not 256-byte aligned");
  int slabs, ppb;
  gn_stats_plan(b, hw, c, &slabs, &ppb);
  unsigned int* counters = static_cast<unsigned int*>(scratch);
  const size_t part_off = (((size_t)b * 4) + 255) & ~(size_t)255;
  double* partial = reinterpret_cast<double*>(static_cast<char*>(scratch) + part_off);
  dim3 grid(slabs, b);
  ODB_DTYPE_SWITCH(dtype, T, "groupnorm_stats",
                   groupnorm_stats_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), stats, partial, counters,
                                                                       hw, c, groups, ppb, eps));
  count_launch();
  return check_launch("groupnorm_stats");
}

extern "C" int odb_groupnorm_finalize(const float* partial, float* stats, int32_t b,
                                      int32_t rows_per_image, int32_t groups, double count,
                                      float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!partial || !stats || b < 1 || rows_per_image < 1 || groups < 1 || groups > 32 || count <= 0)
    return fail(ODB_ERR_INVALID, "groupnorm_finalize: bad argument");
  launch_pdl(groupnorm_finalize_kernel, dim3(b), dim3(32 * groups), 0, stream, partial, stats,
             rows_per_image, groups, count, eps);
  count_launch();
  return check_launch("groupnorm_finalize");
}

extern "C" int odb_groupnorm_apply(const void* x, const float* stats, const float* gamma,
                                   const float* beta, const void* res, const float* res_stats,
                                   const float* res_gamma, const float* res_beta, void* y, int32_t b,
                                   int32_t hw, int32_t c, int32_t groups, int32_t relu, int32_t dtype,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !stats || !gamma || !beta || !y || !gn_args_ok(b, hw, c, groups))
    return fail(ODB_ERR_INVALID, "groupnorm_apply: bad argument");
  if (res_stats && (!res || !res_gamma || !res_beta))
    return fail(ODB_ERR_INVALID, "groupnorm_apply: res_stats needs res, res_gamma, res_beta");
  // blocks per image: enough for one 8-element item per thread, capped so that the whole grid
  // (gx * b blocks) stays within ~8 resident blocks per SM
  const int gx = per_image_grid((long long)hw * (c / 8), 256, b);
  dim3 grid(gx, b);
  ODB_DTYPE_SWITCH(dtype, T, "groupnorm_apply",
                   launch_pdl(groupnorm_apply_kernel<T>, grid, dim3(256), 3 * c * sizeof(float), stream,
                              static_cast<const T*>(x), stats, gamma, beta, static_cast<const T*>(res), res_stats,
                              res_gamma, res_beta, static_cast<T*>(y), hw, c, groups, relu));
  count_launch();
  return check_launch("groupnorm_apply");
}

extern "C" int odb_stem_gn_relu_maxpool(const void* x, const float* stats, const float* gamma,
                                        const float* beta, void* y, int32_t b, int32_t h, int32_t w,
                                        int32_t c, int32_t groups, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !stats || !gamma || !beta || !y || h < 2 || w < 2 || (h & 1) || (w & 1) ||
      !gn_args_ok(b, h * w, c, groups))
    return fail(ODB_ERR_INVALID, "stem_gn_relu_maxpool: bad argument");
  const int gx = per_image_grid((long long)(h / 2) * (w / 2) * (c / 8), 256, b);
  dim3 grid(gx, b);
  ODB_DTYPE_SWITCH(dtype, T, "stem_gn_relu_maxpool",
                   launch_pdl(stem_gn_relu_maxpool_kernel<T>, grid, dim3(256), 2 * c * sizeof(float), stream,
                              static_cast<const T*>(x), stats, gamma, beta, static_cast<T*>(y), h, w, c, groups));
  count_launch();
  return check_launch("stem_gn_relu_maxpool");
}

template <typename T>
static int stem_im2col_launch(const float* x, void* cols, int32_t b, int32_t h, int32_t w, int32_t kpad, size_t smem,
                              cudaStream_t stream) {
  static bool configured[kMaxDevices] = {};
  const int dev_ = current_device();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(stem_im2col_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         21 * (kStemMaxW + 5) * (int)sizeof(float) + 4096);
    if (e != cudaSuccess) return fail_cuda(e, "stem_im2col: cudaFuncSetAttribute");
    configured[dev_] = true;
  }
  launch_pdl(stem_im2col_kernel<T>, dim3(b * (h / 2)), dim3(256), smem, stream, x, static_cast<T*>(cols), b, h, w, kpad);
  return ODB_OK;
}

extern "C" int odb_stem_im2col(const float* x, void* cols, int32_t b, int32_t h, int32_t w,
                               int32_t kpad, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !cols || b < 1 || h < 2 || w < 2 || (h & 1) || (w & 1) || kpad < 152 || kpad % 8)
    return fail(ODB_ERR_INVALID, "stem_im2col: bad argument");
  if (w > kStemMaxW) return fail(ODB_ERR_UNSUPPORTED, "stem_im2col: width above 1792 not supported");
  const size_t smem = (size_t)21 * (w + 5) * sizeof(float) + (size_t)kpad * sizeof(int);
  if (kpad > 1024) return fail(ODB_ERR_INVALID, "stem_im2col: kpad too large");
  int rc = ODB_OK;
  ODB_DTYPE_SWITCH(dtype, T, "stem_im2col", rc = stem_im2col_launch<T>(x, cols, b, h, w, kpad, smem, stream));
  if (rc) return rc;
  count_launch();
  return check_launch("stem_im2col");
}

extern "C" int odb_patchify(const float* x, void* cols, int32_t b, int32_t h, int32_t w, int32_t patch,
                            int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !cols || b < 1 || patch < 8 || patch % 8 || h < patch || w < patch || h % patch || w % patch ||
      (reinterpret_cast<uintptr_t>(x) & 15u) || (w % 4))
    return fail(ODB_ERR_INVALID, "patchify: bad argument (patch a multiple of 8 dividing h and w)");
  const long long total = (long long)b * (h / patch) * (w / patch) * (3 * patch * patch / 8);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  ODB_DTYPE_SWITCH(dtype, T, "patchify",
                   launch_pdl(patchify_kernel<T>, dim3((unsigned)blocks), dim3(256), 0, stream, x, static_cast<T*>(cols), b,
                              h, w, patch));
  count_launch();
  return check_launch("patchify");
}

extern "C" int odb_upsample2x_add(const void* z, const void* res, void* out, void* out_relu,
                                  int32_t b, int32_t h, int32_t w, int32_t c, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!z || !out || b < 1 || h < 1 || w < 1 || c < 8 || c % 8)
    return fail(ODB_ERR_INVALID, "upsample2x_add: bad argument");
  const int octets = c / 8;
  if (h + 1 > 65535 || b > 65535 || octets > 256 || (256 % octets) != 0 || h < 2 || w < 2)
    return fail(ODB_ERR_INVALID, "upsample2x_add: extent / channel count unsupported (h, w >= 2)");
  const int quads = 256 / octets;                       // source quads along x per block
  dim3 block(octets, quads);
  dim3 grid((w + 1 + quads - 1) / quads, h + 1, b);     // quad columns -1..w-1, quad rows -1..h-1
  ODB_DTYPE_SWITCH(dtype, T, "upsample2x_add",
                   launch_pdl(upsample2x_add_kernel<T>, grid, block, 0, stream, static_cast<const T*>(z),
                              static_cast<const T*>(res), static_cast<T*>(out), static_cast<T*>(out_relu), h, w, c));
  count_launch();
  return check_launch("upsample2x_add");
}

extern "C" int odb_write_cls_row(void* tokens, const float* cls, const float* pos0, int32_t b,
                                 int32_t tokens_n, int32_t c, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!tokens || !cls || !pos0 || b < 1 || tokens_n < 1 || c < 1)
    return fail(ODB_ERR_INVALID, "write_cls_row: bad argument");
  ODB_DTYPE_SWITCH(dtype, T, "write_cls_row",
                   launch_pdl(write_cls_row_kernel<T>, dim3(b), dim3(256), 0, stream, static_cast<T*>(tokens), cls, pos0,
                              tokens_n, c));
  count_launch();
  return check_launch("write_cls_row");
}

extern "C" int odb_readout_cls_bias(const void* w, const float* bias, const void* tokens, float* out,
                                    int32_t b, int32_t tokens_n, int32_t c, int32_t dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!w || !bias || !tokens || !out || b < 1 || tokens_n < 1 || c < 8 || c % 8)
    return fail(ODB_ERR_INVALID, "readout_cls_bias: bad argument");
  const long long warps = (long long)b * c;
  const unsigned grid = (unsigned)((warps + 7) / 8);
  ODB_DTYPE_SWITCH(dtype, T, "readout_cls_bias",
                   launch_pdl(readout_cls_bias_kernel<T>, dim3(grid), dim3(256), 0, stream, static_cast<const T*>(w), bias,
                              static_cast<const T*>(tokens), out, b, tokens_n, c));
  count_launch();
  return check_launch("readout_cls_bias");
}

extern "C" int odb_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!src || !dst || n < 0 || n % 8 || (reinterpret_cast<uintptr_t>(src) & 15u) || (reinterpret_cast<uintptr_t>(dst) & 15u))
    return fail(ODB_ERR_INVALID, "cast_f32_bf16: n must be a multiple of 8, pointers 16-byte aligned");
  if (n == 0) return ODB_OK;
  long long blocks = (n / 8 + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  launch_pdl(cast_f32_bf16_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, src, static_cast<bf16*>(dst),
             (long long)(n / 8));
  count_launch();
  return check_launch("cast_f32_bf16");
}
