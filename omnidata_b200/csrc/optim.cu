// Optimizer step of the depth train step (SURVEY.md 8 row a21): Depth.configure_optimizers =
// torch.optim.Adam(self.parameters(), lr) (train_depth.py:381-383; default betas (0.9, 0.999), eps 1e-8,
// no weight decay, no amsgrad) behind the Trainer's gradient_clip_val = 10 (train_depth.py:425: PL clips
// the global L2 norm with torch.nn.utils.clip_grad_norm_).
//
// All parameters / gradients / moments live in ONE flat fp32 buffer each (the model is 123 M parameters:
// 493 MB per buffer), so the whole step is two launches: a deterministic sum of squares (fixed-order
// fp64 partials, last-block finalize -> the clip coefficient on the device, no host sync) and one fused
// update pass.  HBM-bound: 16 B read + 12 B written per parameter.
#include "common.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kOptThreads = 256;
constexpr int kMaxNormBlocks = 2048;      // fixes the workspace size (no device query needed)
constexpr int kMaxSegments = 1024;        // entries of a segment table (the DPT-Hybrid has 368 parameter tensors)

ODB_DEVINL double opt_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// Both kernels walk a virtual index space: the concatenation of the segments [start, end) of the flat buffers, in table
// order (table NULL: the one segment [0, n)).  Every start is a multiple of 4 and every segment but the last has a
// length that is a multiple of 4, so an aligned group of 4 virtual indices never straddles two segments and maps to one
// 16-byte aligned float4.  With one segment the virtual index is the buffer index: the whole-buffer entry points are
// this case, with the arithmetic and summation order they always had.
struct SegMap {
  long long vbeg[kMaxSegments];           // virtual index of each segment's first element
  long long start[kMaxSegments];          // its buffer index
};

// block-wide: s <- the table (exclusive scan of the lengths by warp 0); the caller synchronises
ODB_DEVINL void load_segments(const long long* __restrict__ table, int nseg, SegMap& s) {
  if (table == nullptr) {
    if (threadIdx.x == 0) { s.vbeg[0] = 0; s.start[0] = 0; }
    return;
  }
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x, per = (nseg + 31) / 32;
  const int k0 = min(nseg, lane * per), k1 = min(nseg, k0 + per);
  long long own = 0;
  for (int k = k0; k < k1; ++k) own += table[2 * k + 1] - table[2 * k];
  long long incl = own;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  long long run = incl - own;
  for (int k = k0; k < k1; ++k) {
    s.vbeg[k] = run;
    s.start[k] = table[2 * k];
    run += table[2 * k + 1] - table[2 * k];
  }
}

// buffer index of virtual index i: the last segment whose vbeg <= i
ODB_DEVINL long long seg_index(const SegMap& s, int nseg, long long i) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (s.vbeg[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return s.start[lo] + (i - s.vbeg[lo]);
}

// partial[blockIdx.x] = sum of g^2 over the block's contiguous slab of the n virtual indices; the last block to finish
// adds the partials in index order and writes out2 = (total_norm, clip_coef = min(1, max_norm / (total_norm + 1e-6)))
__global__ void __launch_bounds__(kOptThreads) grad_norm_kernel(const float* __restrict__ g,
                                                                const long long* __restrict__ table, int nseg, long long n,
                                                                long long per_block, double* __restrict__ partial,
                                                                unsigned int* __restrict__ ticket, float max_norm,
                                                                float* __restrict__ out2) {
  __shared__ double scratch[kOptThreads / 32];
  __shared__ bool last;
  __shared__ SegMap seg;
  load_segments(table, nseg, seg);
  __syncthreads();
  const long long lo = (long long)blockIdx.x * per_block;
  long long hi = lo + per_block;
  if (hi > n) hi = n;
  double acc = 0.0;
  // per_block is a multiple of 4 * blockDim: 16-byte loads, each thread a fixed set of elements
  for (long long i = lo + 4LL * threadIdx.x; i < hi; i += 4LL * kOptThreads) {
    if (i + 3 < hi) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(g + seg_index(seg, nseg, i)));
      acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    } else {
      for (long long j = i; j < hi; ++j) {
        const float e = g[seg_index(seg, nseg, j)];
        acc += (double)e * e;
      }
    }
  }
  acc = opt_warp_sum(acc);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kOptThreads / 32; ++w) s += scratch[w];
    partial[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double s = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) s += reinterpret_cast<volatile double*>(partial)[b];
    const float norm = (float)sqrt(s);
    const float coef = max_norm / (norm + 1e-6f);      // clip_grad_norm_: max_norm / (total_norm + 1e-6), clamped to 1
    out2[0] = norm;
    out2[1] = coef < 1.0f ? coef : 1.0f;
    *ticket = 0;                                       // re-armed for the next step
  }
}

// torch.optim.Adam single-tensor update (adam.py _single_tensor_adam, maximize / amsgrad / weight_decay off):
//   g' = g * clip;  m = lerp(m, g', 1 - beta1);  v = v * beta2 + (1 - beta2) g'^2
//   p -= (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// over the n virtual indices of the segment table; elements outside the segments are not touched
__global__ void __launch_bounds__(kOptThreads) adam_step_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                                float* __restrict__ m, float* __restrict__ v,
                                                                const long long* __restrict__ table, int nseg,
                                                                long long n, const float* __restrict__ clip2,
                                                                float w1, float beta2, float w2, float step_size,
                                                                float bc2_sqrt, float eps,
                                                                const float* __restrict__ step_scalars) {
  __shared__ SegMap seg;
  load_segments(table, nseg, seg);
  __syncthreads();
  const float clip = clip2 != nullptr ? clip2[1] : 1.0f;
  if (step_scalars != nullptr) {       // captured in a CUDA graph: the step-dependent scalars come from device memory
    step_size = step_scalars[0];
    bc2_sqrt = step_scalars[1];
  }
  const long long stride = 4LL * gridDim.x * blockDim.x;
  for (long long i = 4LL * (blockIdx.x * (long long)blockDim.x + threadIdx.x); i < n; i += stride) {
    if (i + 3 < n) {
      const long long b = seg_index(seg, nseg, i);
      float4 pv = *reinterpret_cast<float4*>(p + b);
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + b));
      float4 mv = *reinterpret_cast<float4*>(m + b);
      float4 vv = *reinterpret_cast<float4*>(v + b);
      float* pp = &pv.x; const float* gp = &gv.x; float* mp = &mv.x; float* vp = &vv.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float gg = __fmul_rn(gp[k], clip);
        mp[k] = __fadd_rn(mp[k], __fmul_rn(w1, __fsub_rn(gg, mp[k])));
        vp[k] = __fadd_rn(__fmul_rn(vp[k], beta2), __fmul_rn(__fmul_rn(w2, gg), gg));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vp[k]), bc2_sqrt), eps);
        pp[k] = __fsub_rn(pp[k], __fmul_rn(step_size, __fdiv_rn(mp[k], denom)));
      }
      *reinterpret_cast<float4*>(p + b) = pv;
      *reinterpret_cast<float4*>(m + b) = mv;
      *reinterpret_cast<float4*>(v + b) = vv;
    } else {
      for (long long jv = i; jv < n; ++jv) {
        const long long j = seg_index(seg, nseg, jv);
        const float gg = __fmul_rn(g[j], clip);
        const float mm = __fadd_rn(m[j], __fmul_rn(w1, __fsub_rn(gg, m[j])));
        const float vv = __fadd_rn(__fmul_rn(v[j], beta2), __fmul_rn(__fmul_rn(w2, gg), gg));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), bc2_sqrt), eps);
        m[j] = mm; v[j] = vv;
        p[j] = __fsub_rn(p[j], __fmul_rn(step_size, __fdiv_rn(mm, denom)));
      }
    }
  }
}

static int clip_grad_norm_launch(const float* grads, const int64_t* table, int nseg, int64_t n, float max_norm,
                                 void* workspace, float* out2, cudaStream_t stream) {
  int max_blocks = num_sms() * 8;
  if (max_blocks > kMaxNormBlocks) max_blocks = kMaxNormBlocks;
  const long long quantum = 4LL * kOptThreads;
  long long per_block = (n + max_blocks - 1) / max_blocks;
  per_block = (per_block + quantum - 1) / quantum * quantum;
  const int blocks = (int)((n + per_block - 1) / per_block);
  // layout of the workspace: [ticket (zero-initialised by the caller once; the kernel re-arms it)] [partials]
  unsigned int* ticket = static_cast<unsigned int*>(workspace);
  double* partial = reinterpret_cast<double*>(static_cast<char*>(workspace) + 256);
  grad_norm_kernel<<<blocks, kOptThreads, 0, stream>>>(grads, reinterpret_cast<const long long*>(table), nseg, n, per_block,
                                                       partial, ticket, max_norm, out2);
  count_launch();
  return check_launch("clip_grad_norm");
}

static int adam_step_launch(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const int64_t* table,
                            int nseg, int64_t n, const float* clip2, float lr, float beta1, float beta2, float eps,
                            int64_t step, const float* step_scalars, cudaStream_t stream) {
  // scalar preparation as torch does it on the host (python floats = doubles), then one rounding to fp32
  float host2[2];
  odb_adam_step_scalars(lr, beta1, beta2, step, host2);
  const float step_size = host2[0], bc2_sqrt = host2[1];
  const float w1 = (float)(1.0 - (double)beta1), w2 = (float)(1.0 - (double)beta2);
  long long blocks = (n / 4 + kOptThreads - 1) / kOptThreads;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  adam_step_kernel<<<(unsigned)blocks, kOptThreads, 0, stream>>>(params, grads, exp_avg, exp_avg_sq,
                                                                 reinterpret_cast<const long long*>(table), nseg, n, clip2,
                                                                 w1, beta2, w2, step_size, bc2_sqrt, eps, step_scalars);
  count_launch();
  return check_launch("adam_step");
}

static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_grad_norm_workspace_bytes(void) { return (int64_t)kMaxNormBlocks * 8 + 256; }

extern "C" int odb_clip_grad_norm(const float* grads, int64_t n, float max_norm, void* workspace, float* out2,
                                  void* stream_) {
  if (!grads || !workspace || !out2 || n < 1 || misaligned16(grads) || (reinterpret_cast<uintptr_t>(workspace) & 7u))
    return fail(ODB_ERR_INVALID, "clip_grad_norm: bad argument (16-byte aligned gradients, workspace required)");
  return clip_grad_norm_launch(grads, nullptr, 1, n, max_norm, workspace, out2, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_clip_grad_norm_segments(const float* grads, const int64_t* segments, int32_t num_segments, int64_t total,
                                           float max_norm, void* workspace, float* out2, void* stream_) {
  if (!grads || !segments || !workspace || !out2 || num_segments < 1 || num_segments > kMaxSegments || total < 1 ||
      misaligned16(grads) || misaligned16(segments) || (reinterpret_cast<uintptr_t>(workspace) & 7u))
    return fail(ODB_ERR_INVALID, "clip_grad_norm_segments: bad argument (16-byte aligned gradients and segment table, "
                                 "1..1024 segments, total >= 1, workspace required)");
  return clip_grad_norm_launch(grads, segments, num_segments, total, max_norm, workspace, out2,
                               static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_adam_step_scalars(float lr, float beta1, float beta2, int64_t step, float* out2) {
  if (out2 == nullptr || step < 1) return fail(ODB_ERR_INVALID, "adam_step_scalars: bad argument");
  // scalar preparation as torch does it on the host (python floats = doubles), then one rounding to fp32
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  out2[0] = (float)((double)lr / bc1);
  out2[1] = (float)sqrt(bc2);
  return ODB_OK;
}

extern "C" int odb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                             const float* clip2, float lr, float beta1, float beta2, float eps, int64_t step,
                             const float* step_scalars, void* stream_) {
  if (step_scalars != nullptr && step < 1) step = 1;     // unused: the scalars are read from device memory
  if (!params || !grads || !exp_avg || !exp_avg_sq || n < 1 || step < 1 || misaligned16(params) || misaligned16(grads) ||
      misaligned16(exp_avg) || misaligned16(exp_avg_sq))
    return fail(ODB_ERR_INVALID, "adam_step: bad argument (16-byte aligned flat fp32 buffers, step >= 1)");
  return adam_step_launch(params, grads, exp_avg, exp_avg_sq, nullptr, 1, n, clip2, lr, beta1, beta2, eps, step,
                          step_scalars, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_adam_step_segments(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                                      const int64_t* segments, int32_t num_segments, int64_t total, const float* clip2,
                                      float lr, float beta1, float beta2, float eps, int64_t step, const float* step_scalars,
                                      void* stream_) {
  if (step_scalars != nullptr && step < 1) step = 1;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !segments || num_segments < 1 || num_segments > kMaxSegments ||
      total < 1 || step < 1 || misaligned16(params) || misaligned16(grads) || misaligned16(exp_avg) ||
      misaligned16(exp_avg_sq) || misaligned16(segments))
    return fail(ODB_ERR_INVALID, "adam_step_segments: bad argument (16-byte aligned flat fp32 buffers and segment table, "
                                 "1..1024 segments, total >= 1, step >= 1)");
  return adam_step_launch(params, grads, exp_avg, exp_avg_sq, segments, num_segments, total, clip2, lr, beta1, beta2, eps,
                          step, step_scalars, static_cast<cudaStream_t>(stream_));
}
