// Image pre- and post-processing either side of the DPT forward, on the device
// (omnidata_tools/torch/demo.py:74-76,92-95: Resize(384, BILINEAR) + CenterCrop(384) + ToTensor
// [+ Normalize(0.5, 0.5)];  :142-150: bicubic resize to 512, clamp, 1 - x / ToPILImage).
//
// The reference resizes with Pillow: an antialiased two-pass (horizontal, then vertical) triangle
// filter in 8-bit fixed point (ImagingResample, PRECISION_BITS = 22) with an 8-bit intermediate
// image.  These kernels reproduce that arithmetic exactly — the coefficient tables come from the host
// (omnidata_b200/imageproc.py restates Pillow's precompute_coeffs / normalize_coeffs_8bpc), the
// accumulation is the same int32 sum with the same rounding constant and clip — so the tensor that
// enters the network is bit-identical to the reference's.  Only the rows / columns that survive the
// centre crop are computed.
//
// HBM-bound byte kernels: one thread per output pixel, all channels; coalesced along x.
#include "common.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kPilPrecisionBits = 22;   // Pillow: 32 - 8 - 2

ODB_DEVINL uint8_t pil_clip8(int v) {
  v >>= kPilPrecisionBits;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Horizontal pass: tmp[r][x][c] = clip8((2^21 + sum_t kk[x][t] * src[row0 + r][xmin[x] + t][c]) >> 22)
template <int C>
__global__ void __launch_bounds__(256) resize_h_u8_kernel(
    const uint8_t* __restrict__ src, long long src_pitch, const int32_t* __restrict__ bounds,
    const int32_t* __restrict__ kk, int ksize, int row0, int nrows, int ncols, uint8_t* __restrict__ tmp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (x >= ncols || r >= nrows) return;
  const int xmin = bounds[2 * x], cnt = bounds[2 * x + 1];
  const int32_t* k = kk + static_cast<long long>(x) * ksize;
  const uint8_t* s = src + static_cast<long long>(row0 + r) * src_pitch + static_cast<long long>(xmin) * C;
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 1 << (kPilPrecisionBits - 1);
  for (int t = 0; t < cnt; ++t) {
    const int w = __ldg(k + t);
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] += static_cast<int>(s[t * C + c]) * w;
  }
  uint8_t* o = tmp + (static_cast<long long>(r) * ncols + x) * C;
#pragma unroll
  for (int c = 0; c < C; ++c) o[c] = pil_clip8(acc[c]);
}

// Vertical pass + ToTensor (+ Normalize): out[c][y][x] = (clip8(...) / 255 - mean) / std, fp32 NCHW.
// A single-channel image is replicated to three planes (demo.py:137-138).
template <int C>
__global__ void __launch_bounds__(256) resize_v_u8_to_f32_kernel(
    const uint8_t* __restrict__ tmp, int row0, int ncols, const int32_t* __restrict__ bounds,
    const int32_t* __restrict__ kk, int ksize, int out_h, float mean, float stdv, int normalize,
    float* __restrict__ out, uint8_t* __restrict__ out_u8) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= ncols || y >= out_h) return;
  const int ymin = bounds[2 * y], cnt = bounds[2 * y + 1];
  const int32_t* k = kk + static_cast<long long>(y) * ksize;
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 1 << (kPilPrecisionBits - 1);
  for (int t = 0; t < cnt; ++t) {
    const int w = __ldg(k + t);
    const uint8_t* s = tmp + (static_cast<long long>(ymin - row0 + t) * ncols + x) * C;
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] += static_cast<int>(s[c]) * w;
  }
  const long long plane = static_cast<long long>(out_h) * ncols;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const uint8_t u = pil_clip8(acc[c]);
    if (out_u8 != nullptr) out_u8[(static_cast<long long>(y) * ncols + x) * C + c] = u;
    // ToTensor: uint8 -> float32, true division by 255; Normalize: (t - mean) / std (IEEE ops, no fast-math)
    float v = __fdiv_rn(static_cast<float>(u), 255.0f);
    if (normalize) v = __fdiv_rn(__fsub_rn(v, mean), stdv);
    if (C == 1) {
      out[0 * plane + static_cast<long long>(y) * ncols + x] = v;
      out[1 * plane + static_cast<long long>(y) * ncols + x] = v;
      out[2 * plane + static_cast<long long>(y) * ncols + x] = v;
    } else {
      out[c * plane + static_cast<long long>(y) * ncols + x] = v;
    }
  }
}

// torch upsample_bicubic2d, align_corners = False, A = -0.75 (F.interpolate(mode='bicubic'), demo.py:143)
ODB_DEVINL float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
ODB_DEVINL float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
ODB_DEVINL void cubic_coeffs(float t, float* w) {
  const float A = -0.75f;
  w[0] = cubic2(t + 1.f, A);
  w[1] = cubic1(t, A);
  w[2] = cubic1(1.f - t, A);
  w[3] = cubic2(2.f - t, A);
}

// out = post(bicubic(pre(in))): pre = clamp to [0,1] (flags bit 0), post = clamp to [0,1] (bit 1), 1 - x (bit 2)
__global__ void __launch_bounds__(256) bicubic_resize_f32_kernel(const float* __restrict__ in, int planes,
                                                                 int ih, int iw, int oh, int ow, int flags,
                                                                 float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int pl = blockIdx.z;
  if (x >= ow || y >= oh || pl >= planes) return;
  const float sh = static_cast<float>(ih) / static_cast<float>(oh);
  const float sw = static_cast<float>(iw) / static_cast<float>(ow);
  const float ry = __fmaf_rn(sh, static_cast<float>(y) + 0.5f, -0.5f);
  const float rx = __fmaf_rn(sw, static_cast<float>(x) + 0.5f, -0.5f);
  const float fy = floorf(ry), fx = floorf(rx);
  const int iy = static_cast<int>(fy), ix = static_cast<int>(fx);
  float wy[4], wx[4];
  cubic_coeffs(ry - fy, wy);
  cubic_coeffs(rx - fx, wx);
  const float* src = in + static_cast<long long>(pl) * ih * iw;
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int yy = iy - 1 + j;
    yy = yy < 0 ? 0 : (yy > ih - 1 ? ih - 1 : yy);
    float row = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int xx = ix - 1 + i;
      xx = xx < 0 ? 0 : (xx > iw - 1 ? iw - 1 : xx);
      float v = __ldg(src + static_cast<long long>(yy) * iw + xx);
      if (flags & 1) v = fminf(fmaxf(v, 0.f), 1.f);
      row = __fmaf_rn(v, wx[i], row);
    }
    acc = __fmaf_rn(row, wy[j], acc);
  }
  if (flags & 2) acc = fminf(fmaxf(acc, 0.f), 1.f);
  if (flags & 4) acc = 1.0f - acc;
  out[(static_cast<long long>(pl) * oh + y) * ow + x] = acc;
}

// Antialiased bilinear resampling of fp32 planes (F.interpolate(mode="bilinear", align_corners=False, antialias=True)):
// the same triangle filter as Pillow's, its per-axis (xmin, count) bounds and normalised fp32 weights from the host
// (omnidata_b200/imageproc.py bilinear_aa_weights).  Horizontal pass in -> tmp [planes][ih][ow], then vertical pass
// tmp -> out [planes][oh][ow]; fp32 fused multiply-adds in tap order.
__global__ void __launch_bounds__(256) resample_h_f32_kernel(const float* __restrict__ in, int ih, int iw, int ow,
                                                             const int32_t* __restrict__ bounds,
                                                             const float* __restrict__ wts, int ksize,
                                                             float* __restrict__ tmp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= ow) return;
  const long long row = (long long)blockIdx.z * ih + blockIdx.y;
  const int xmin = __ldg(bounds + 2 * x), cnt = __ldg(bounds + 2 * x + 1);
  const float* src = in + row * iw + xmin;
  const float* k = wts + (long long)x * ksize;
  float acc = 0.f;
  for (int t = 0; t < cnt; ++t) acc = __fmaf_rn(__ldg(k + t), __ldg(src + t), acc);
  tmp[row * ow + x] = acc;
}

__global__ void __launch_bounds__(256) resample_v_f32_kernel(const float* __restrict__ tmp, int ih, int oh, int ow,
                                                             const int32_t* __restrict__ bounds,
                                                             const float* __restrict__ wts, int ksize,
                                                             float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= ow) return;
  const int y = blockIdx.y, pl = blockIdx.z;
  const int ymin = __ldg(bounds + 2 * y), cnt = __ldg(bounds + 2 * y + 1);
  const float* src = tmp + ((long long)pl * ih + ymin) * ow + x;
  const float* k = wts + (long long)y * ksize;
  float acc = 0.f;
  for (int t = 0; t < cnt; ++t) acc = __fmaf_rn(__ldg(k + t), __ldg(src + (long long)t * ow), acc);
  out[((long long)pl * oh + y) * ow + x] = acc;
}

// ToPILImage for a float CHW tensor: (x * 255) truncated to uint8, HWC (torchvision to_pil_image)
__global__ void __launch_bounds__(256) f32_chw_to_u8_hwc_kernel(const float* __restrict__ in, int c, int h, int w,
                                                                int clamp01, uint8_t* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(h) * w;
  if (i >= n) return;
  for (int ch = 0; ch < c; ++ch) {
    float v = in[ch * n + i];
    if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
    const float s = __fmul_rn(v, 255.0f);
    out[i * c + ch] = static_cast<uint8_t>(static_cast<int>(s));   // truncation, as numpy astype(uint8) on [0,255]
  }
}

}  // namespace odb

using namespace odb;

extern "C" int odb_pil_resize_crop_to_tensor(const void* src, int32_t src_h, int32_t src_w, int32_t channels,
                                             int64_t src_pitch, const int32_t* bounds_h, const int32_t* kk_h,
                                             int32_t ksize_h, const int32_t* bounds_v, const int32_t* kk_v,
                                             int32_t ksize_v, int32_t row0, int32_t nrows, int32_t out_h,
                                             int32_t out_w, int32_t normalize, float mean, float stdv, void* tmp,
                                             float* out, void* out_u8, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!src || !bounds_h || !kk_h || !bounds_v || !kk_v || !tmp || !out || src_h < 1 || src_w < 1 ||
      (channels != 1 && channels != 3) || ksize_h < 1 || ksize_v < 1 || row0 < 0 || nrows < 1 ||
      row0 + nrows > src_h || out_h < 1 || out_w < 1 || src_pitch < (int64_t)src_w * channels)
    return fail(ODB_ERR_INVALID, "pil_resize_crop_to_tensor: bad argument");
  const dim3 block(256);
  const dim3 grid_h((out_w + 255) / 256, nrows);
  const dim3 grid_v((out_w + 255) / 256, out_h);
  const uint8_t* s = static_cast<const uint8_t*>(src);
  uint8_t* t = static_cast<uint8_t*>(tmp);
  if (channels == 3) {
    resize_h_u8_kernel<3><<<grid_h, block, 0, stream>>>(s, src_pitch, bounds_h, kk_h, ksize_h, row0, nrows, out_w, t);
    count_launch();
    resize_v_u8_to_f32_kernel<3><<<grid_v, block, 0, stream>>>(t, row0, out_w, bounds_v, kk_v, ksize_v, out_h, mean,
                                                              stdv, normalize, out, static_cast<uint8_t*>(out_u8));
  } else {
    resize_h_u8_kernel<1><<<grid_h, block, 0, stream>>>(s, src_pitch, bounds_h, kk_h, ksize_h, row0, nrows, out_w, t);
    count_launch();
    resize_v_u8_to_f32_kernel<1><<<grid_v, block, 0, stream>>>(t, row0, out_w, bounds_v, kk_v, ksize_v, out_h, mean,
                                                              stdv, normalize, out, static_cast<uint8_t*>(out_u8));
  }
  count_launch();
  return check_launch("pil_resize_crop_to_tensor");
}

extern "C" int odb_bicubic_resize_f32(const float* in, int32_t planes, int32_t in_h, int32_t in_w, int32_t out_h,
                                      int32_t out_w, int32_t flags, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!in || !out || planes < 1 || in_h < 1 || in_w < 1 || out_h < 1 || out_w < 1 || out_h > 65535 || planes > 65535)
    return fail(ODB_ERR_INVALID, "bicubic_resize_f32: bad argument");
  const dim3 grid((out_w + 255) / 256, out_h, planes);
  bicubic_resize_f32_kernel<<<grid, 256, 0, stream>>>(in, planes, in_h, in_w, out_h, out_w, flags, out);
  count_launch();
  return check_launch("bicubic_resize_f32");
}

extern "C" int odb_resize_bilinear_f32(const float* in, int32_t planes, int32_t in_h, int32_t in_w, int32_t out_h,
                                       int32_t out_w, const int32_t* bounds_h, const float* weights_h, int32_t ksize_h,
                                       const int32_t* bounds_v, const float* weights_v, int32_t ksize_v, float* tmp,
                                       float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!in || !out || !tmp || !bounds_h || !weights_h || !bounds_v || !weights_v || planes < 1 || planes > 65535 ||
      in_h < 1 || in_w < 1 || out_h < 1 || out_w < 1 || in_h > 65535 || out_h > 65535 || ksize_h < 1 || ksize_v < 1)
    return fail(ODB_ERR_INVALID, "resize_bilinear_f32: bad argument");
  resample_h_f32_kernel<<<dim3((out_w + 255) / 256, in_h, planes), 256, 0, stream>>>(in, in_h, in_w, out_w, bounds_h,
                                                                                    weights_h, ksize_h, tmp);
  count_launch();
  resample_v_f32_kernel<<<dim3((out_w + 255) / 256, out_h, planes), 256, 0, stream>>>(tmp, in_h, out_h, out_w,
                                                                                     bounds_v, weights_v, ksize_v, out);
  count_launch();
  return check_launch("resize_bilinear_f32");
}

extern "C" int odb_f32_chw_to_u8_hwc(const float* in, int32_t c, int32_t h, int32_t w, int32_t clamp01, void* out,
                                     void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!in || !out || c < 1 || c > 4 || h < 1 || w < 1) return fail(ODB_ERR_INVALID, "f32_chw_to_u8_hwc: bad argument");
  const long long n = (long long)h * w;
  f32_chw_to_u8_hwc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(in, c, h, w, clamp01,
                                                                            static_cast<uint8_t*>(out));
  count_launch();
  return check_launch("f32_chw_to_u8_hwc");
}
