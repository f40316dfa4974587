// Deterministic block-level reductions and exact order statistics shared by the loss and refocus kernels:
// fixed-order fp64 block sum, and a 4-pass radix select (integer histograms) for the k-th smallest value.
#pragma once
#include "common.cuh"

namespace odb {

constexpr int kLossThreads = 1024;

ODB_DEVINL double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
// fixed-order block sum (result valid in thread 0)
ODB_DEVINL double block_sum_d(double v, double* scratch /* [32] shared */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_d(v);
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (warp == 0) {
    r = lane < (int)(blockDim.x >> 5) ? scratch[lane] : 0.0;
    r = warp_sum_d(r);
  }
  return r;
}
// block minimum / maximum (result valid in thread 0); exact, so the order does not matter
template <bool kMin>
ODB_DEVINL double block_extreme_d(double v, double* scratch /* [32] shared */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_down_sync(0xffffffffu, v, o);
    v = kMin ? fmin(v, u) : fmax(v, u);
  }
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  double r = v;
  if (warp == 0) {
    r = lane < (int)(blockDim.x >> 5) ? scratch[lane] : (kMin ? INFINITY : -INFINITY);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double u = __shfl_down_sync(0xffffffffu, r, o);
      r = kMin ? fmin(r, u) : fmax(r, u);
    }
  }
  return r;
}
ODB_DEVINL double block_min_d(double v, double* scratch) { return block_extreme_d<true>(v, scratch); }
ODB_DEVINL double block_max_d(double v, double* scratch) { return block_extreme_d<false>(v, scratch); }
ODB_DEVINL uint32_t sortable_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
ODB_DEVINL float key_to_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Exact k-th smallest (0-based rank) of the selected elements of `vals`; `pred(i)` says whether
// element i takes part.  Whole block cooperates; returns the key in every thread.
template <typename Pred>
ODB_DEVINL uint32_t block_radix_select(const float* vals, long long n, unsigned long long rank, Pred pred,
                                       uint32_t* hist /* [256] shared */, uint32_t* bcast /* [2] shared */) {
  uint32_t prefix = 0, himask = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      if (!pred(i)) continue;
      const uint32_t k = sortable_key(vals[i]);
      if (((k ^ prefix) & himask) == 0) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cum = 0;
      uint32_t d = 0;
      for (; d < 256; ++d) {
        if (cum + hist[d] > rank) break;
        cum += hist[d];
      }
      if (d > 255) d = 255;
      bcast[0] = d;
      bcast[1] = (uint32_t)cum;
    }
    __syncthreads();
    prefix |= bcast[0] << shift;
    himask |= 0xFFu << shift;
    rank -= bcast[1];
    __syncthreads();
  }
  return prefix;
}

}  // namespace odb
