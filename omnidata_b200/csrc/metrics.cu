// Evaluation metrics of depth and surface-normal predictions against ground truth (omnidata_b200/metrics.py
// DepthMetrics / NormalMetrics; definitions in DESIGN.md §3 "Evaluation metrics", restated in float64 by
// oracle/metrics_oracle.py).
//
// Every image is cut into fixed slabs of kSlab pixels, so the partition depends on H x W only and never on the batch.
// Per-pixel arithmetic is fp64; each slab's sums are combined by block_sum_d (fixed order), the slabs of an image by
// slab_reduce_kernel (fixed order), and the per-image results are folded into the running state one image after the
// other, in image order.  No floating-point atomics: the state after a dataset does not depend on how it was split into
// batches, and repeat runs give the same bits.  The normal-angle histogram is filled with integer atomics, which are
// order-independent.
//
//   depth:  depth_moments_kernel (slabs) -> slab_reduce_kernel (images) -> depth_error_kernel (slabs, each CTA solves
//           its image's scale / shift) -> slab_reduce_kernel -> depth_fold_kernel (one thread, image order)
//   normal: normal_angle_kernel (slabs, histogram) -> slab_reduce_kernel -> normal_fold_kernel (one thread)
//           normal_median_kernel: block prefix scan over the histogram
//
// Built without fast-math: the metrics promise IEEE fp64 arithmetic, and d-hat and the angle (angle_deg, fp64.cuh) are
// written with explicit round-to-nearest operations (no fma contraction) so that the float64 oracle reproduces them
// operation by operation.
#include <cmath>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "select.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kMetricThreads = 256;
constexpr int kSlabIters = kSlab / kMetricThreads;
constexpr int kMedianThreads = 1024;

// Slab partials [b][slab][8] over V of the image: (n, Sp, Spp, Sy, Spy, non-finite predictions), y = g (depth space) or
// 1 / g (disparity space).  grid (slabs, b)
__global__ void __launch_bounds__(kMetricThreads) depth_moments_kernel(const float* __restrict__ pred,
                                                                       const float* __restrict__ gt, const void* mask,
                                                                       int mask_kind, long long hw, int disparity,
                                                                       double min_depth, double max_depth,
                                                                       double* __restrict__ part) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const long long base = (long long)b * hw;
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (int k = 0; k < kSlabIters; ++k) {
    const long long i = blockIdx.x * kSlab + k * kMetricThreads + threadIdx.x;
    if (i >= hw || !mask_valid(mask, mask_kind, base + i)) continue;
    const double g = gt[base + i];
    if (!depth_valid(g, min_depth, max_depth)) continue;
    const double p = pred[base + i];
    const double y = disparity ? 1.0 / g : g;
    acc[0] += 1.0;
    acc[1] += p;
    acc[2] = fma(p, p, acc[2]);
    acc[3] += y;
    acc[4] = fma(p, y, acc[4]);
    acc[5] += isfinite(p) ? 0.0 : 1.0;
  }
  double* out = part + ((long long)b * gridDim.x + blockIdx.x) * kPartStride;
  for (int q = 0; q < 6; ++q) {
    const double r = block_sum_d(acc[q], scratch);
    if (threadIdx.x == 0) out[q] = r;
  }
}

// out[b][q] = sum over the image's slabs of part[b][slab][q], q < nq, in a fixed order; the minimum or the maximum
// instead where bit q of min_mask or max_mask is set.  grid (b)
__global__ void __launch_bounds__(kMetricThreads) slab_reduce_kernel(const double* __restrict__ part, int slabs, int nq,
                                                                     unsigned min_mask, unsigned max_mask,
                                                                     double* __restrict__ out) {
  __shared__ double scratch[32];
  const int b = blockIdx.x;
  const double* p = part + (long long)b * slabs * kPartStride;
  for (int q = 0; q < nq; ++q) {
    double r;
    if ((min_mask | max_mask) >> q & 1u) {
      const bool lo = min_mask >> q & 1u;
      double acc = lo ? INFINITY : -INFINITY;
      for (int s = threadIdx.x; s < slabs; s += kMetricThreads) {
        const double v = p[(long long)s * kPartStride + q];
        acc = lo ? fmin(acc, v) : fmax(acc, v);
      }
      r = lo ? block_min_d(acc, scratch) : block_max_d(acc, scratch);
    } else {
      double acc = 0.0;
      for (int s = threadIdx.x; s < slabs; s += kMetricThreads) acc += p[(long long)s * kPartStride + q];
      r = block_sum_d(acc, scratch);
    }
    if (threadIdx.x == 0) out[(long long)b * kPartStride + q] = r;
  }
}

// compute_scale_and_shift (L/midas_loss.py:10-30) in fp64 on the image's moments: s = t = 0 where det <= 0
ODB_DEVINL void depth_scale_shift(const double* m, double& s, double& t) {
  const double a00 = m[2], a01 = m[1], a11 = m[0], b0 = m[4], b1 = m[3];
  const double det = a00 * a11 - a01 * a01;
  s = t = 0.0;
  if (det > 0.0) {
    s = (a11 * b0 - a01 * b1) / det;
    t = (-a01 * b0 + a00 * b1) / det;
  }
}

// Slab partials [b][slab][8] over V: (S|e|/g, Se^2/g, Se^2, S(ln dh - ln g)^2, #(r < 1.25), #(r < 1.25^2),
// #(r < 1.25^3)), e = dh - g, r = max(dh / g, g / dh); each CTA solves its image's (s, t) from mom, or takes (1, 0)
// without `align` (a metric prediction, depth space).  grid (slabs, b)
__global__ void __launch_bounds__(kMetricThreads) depth_error_kernel(const float* __restrict__ pred,
                                                                     const float* __restrict__ gt, const void* mask,
                                                                     int mask_kind, long long hw, int disparity,
                                                                     double min_depth, double max_depth,
                                                                     const double* __restrict__ mom, int align,
                                                                     double* __restrict__ part) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const long long base = (long long)b * hw;
  double s = 1.0, t = 0.0;
  if (align) depth_scale_shift(mom + (long long)b * kPartStride, s, t);
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < kSlabIters; ++k) {
    const long long i = blockIdx.x * kSlab + k * kMetricThreads + threadIdx.x;
    if (i >= hw || !mask_valid(mask, mask_kind, base + i)) continue;
    const double g = gt[base + i];
    if (!depth_valid(g, min_depth, max_depth)) continue;
    const double d = depth_hat((double)pred[base + i], s, t, disparity, min_depth, max_depth);
    const double e = d - g;
    const double e2 = e * e;
    const double lg = log(d) - log(g);
    const double r = fmax(d / g, g / d);
    acc[0] += fabs(e) / g;
    acc[1] += e2 / g;
    acc[2] += e2;
    acc[3] += lg * lg;
    acc[4] += r < 1.25 ? 1.0 : 0.0;
    acc[5] += r < 1.5625 ? 1.0 : 0.0;
    acc[6] += r < 1.953125 ? 1.0 : 0.0;
  }
  double* out = part + ((long long)b * gridDim.x + blockIdx.x) * kPartStride;
  for (int q = 0; q < 7; ++q) {
    const double r = block_sum_d(acc[q], scratch);
    if (threadIdx.x == 0) out[q] = r;
  }
}

// One thread, images in order: records[b][12] = (n, AbsRel, SqRel, RMSE, RMSE_log, #delta1, #delta2, #delta3, s, t,
// det <= 0, non-finite predictions) (s = 1, t = 0 and never det <= 0 without `align`); the state adds each image with
// n > 0:
// sums[7] += (AbsRel, SqRel, RMSE, RMSE_log, delta1, delta2, delta3), counts[4] += (images, excluded, det <= 0, pixels).
// A non-finite prediction on a valid pixel makes the image's metrics NaN.
__global__ void depth_fold_kernel(const double* __restrict__ mom, const double* __restrict__ err, int b_n, int align,
                                  double* __restrict__ records, double* __restrict__ sums,
                                  long long* __restrict__ counts) {
  if (threadIdx.x != 0) return;
  for (int b = 0; b < b_n; ++b) {
    const double* m = mom + (long long)b * kPartStride;
    const double* e = err + (long long)b * kPartStride;
    double* r = records + (long long)b * ODB_DEPTH_RECORD;
    const double n = m[0];
    double s = 1.0, t = 0.0;
    if (align) depth_scale_shift(m, s, t);
    const bool degenerate = align && n > 0.0 && m[2] * m[0] - m[1] * m[1] <= 0.0;
    const double bad = m[5] > 0.0 ? NAN : 0.0;                      // NaN + x = NaN, 0 + x = x
    const double v[7] = {e[0] / n + bad, e[1] / n + bad, sqrt(e[2] / n) + bad, sqrt(e[3] / n) + bad,
                         e[4] / n + bad, e[5] / n + bad, e[6] / n + bad};
    r[0] = n;
    for (int q = 0; q < 4; ++q) r[1 + q] = n > 0.0 ? v[q] : NAN;
    for (int q = 0; q < 3; ++q) r[5 + q] = e[4 + q] + bad;
    r[8] = s;
    r[9] = t;
    r[10] = degenerate ? 1.0 : 0.0;
    r[11] = m[5];
    if (n > 0.0) {
      for (int q = 0; q < 7; ++q) sums[q] += v[q];
      counts[0] += 1;
      counts[2] += degenerate ? 1 : 0;
      counts[3] += (long long)n;
    } else {
      counts[1] += 1;
    }
  }
}

// Per-pixel angle theta = atan2(|a x b|, a . b) in degrees, a = 2 p - 1, b = 2 g - 1; the pixel takes part where the
// mask is nonzero and both |a|, |b| > 1e-6.  Slab partials [b][slab][8] = (n, S theta, S theta^2, #non-finite,
// #(theta < 11.25), #(theta < 22.5), #(theta < 30)); hist[floor(4096 theta)] += 1 for the finite ones (integer
// atomics, aggregated over the lanes of a warp that hit the same bin).  grid (slabs, b)
__global__ void __launch_bounds__(kMetricThreads) normal_angle_kernel(const float* __restrict__ pred,
                                                                      const float* __restrict__ gt, const void* mask,
                                                                      int mask_kind, long long hw,
                                                                      double* __restrict__ part,
                                                                      unsigned long long* __restrict__ hist) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const float* P = pred + (long long)b * 3 * hw;
  const float* G = gt + (long long)b * 3 * hw;
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < kSlabIters; ++k) {                             // every lane runs every iteration (__match_any_sync)
    const long long i = blockIdx.x * kSlab + k * kMetricThreads + threadIdx.x;
    int bin = -1;
    if (i < hw && mask_valid(mask, mask_kind, (long long)b * hw + i)) {
      double a[3], c[3];
      for (int ch = 0; ch < 3; ++ch) {
        a[ch] = __dsub_rn(__dmul_rn(2.0, (double)P[ch * hw + i]), 1.0);
        c[ch] = __dsub_rn(__dmul_rn(2.0, (double)G[ch * hw + i]), 1.0);
      }
      const double na = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(a[0], a[0]), __dmul_rn(a[1], a[1])), __dmul_rn(a[2], a[2])));
      const double nc = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(c[0], c[0]), __dmul_rn(c[1], c[1])), __dmul_rn(c[2], c[2])));
      if (!(na <= 1e-6) && !(nc <= 1e-6)) {                           // NaN norms take part (and count as non-finite)
        const double th = angle_deg(a, c);
        if (isfinite(th)) {
          acc[0] += 1.0;
          acc[1] += th;
          acc[2] = fma(th, th, acc[2]);
          acc[4] += th < 11.25 ? 1.0 : 0.0;
          acc[5] += th < 22.5 ? 1.0 : 0.0;
          acc[6] += th < 30.0 ? 1.0 : 0.0;
          bin = min((int)(th * ODB_NORMAL_HIST_PER_DEGREE), ODB_NORMAL_HIST_BINS - 1);
        } else {
          acc[3] += 1.0;
        }
      }
    }
    const unsigned same = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(hist + bin, (unsigned long long)__popc(same));
  }
  double* out = part + ((long long)b * gridDim.x + blockIdx.x) * kPartStride;
  for (int q = 0; q < 7; ++q) {
    const double r = block_sum_d(acc[q], scratch);
    if (threadIdx.x == 0) out[q] = r;
  }
}

// One thread, images in order: sums[2] += (S theta, S theta^2), counts[5] += (n, #non-finite, #<11.25, #<22.5, #<30)
__global__ void normal_fold_kernel(const double* __restrict__ img, int b_n, double* __restrict__ sums,
                                   long long* __restrict__ counts) {
  if (threadIdx.x != 0) return;
  for (int b = 0; b < b_n; ++b) {
    const double* m = img + (long long)b * kPartStride;
    sums[0] += m[1];
    sums[1] += m[2];
    counts[0] += (long long)m[0];
    counts[1] += (long long)m[3];
    for (int q = 0; q < 3; ++q) counts[2 + q] += (long long)m[4 + q];
  }
}

// out[2] = (bin, (bin + 0.5) / 4096) of the bin holding the 0-based rank floor((N - 1) / 2) of the N counted angles;
// (-1, NaN) when N = 0.  One CTA: every thread owns a contiguous run of bins, an exclusive scan over the runs' totals
// finds the run holding the rank, and its owner walks it.
__global__ void __launch_bounds__(kMedianThreads) normal_median_kernel(const unsigned long long* __restrict__ hist,
                                                                       double* __restrict__ out) {
  __shared__ unsigned long long warp_tot[32];
  __shared__ unsigned long long s_total;
  constexpr int kRun = (ODB_NORMAL_HIST_BINS + kMedianThreads - 1) / kMedianThreads;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lo = threadIdx.x * kRun, hi = min(lo + kRun, ODB_NORMAL_HIST_BINS);
  unsigned long long own = 0;
  for (int i = lo; i < hi; ++i) own += hist[i];
  unsigned long long incl = own;                                      // inclusive scan within the warp
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int w = 0; w < kMedianThreads / 32; ++w) {
      const unsigned long long v = warp_tot[w];
      warp_tot[w] = run;
      run += v;
    }
    s_total = run;
    out[0] = -1.0;
    out[1] = NAN;
  }
  __syncthreads();
  const unsigned long long total = s_total;
  if (total == 0) return;
  const unsigned long long rank = (total - 1) / 2;
  unsigned long long before = warp_tot[warp] + incl - own;           // angles in the runs before this thread's
  if (rank < before || rank >= before + own) return;
  for (int i = lo; i < hi; ++i) {
    before += hist[i];
    if (rank < before) {
      out[0] = (double)i;
      out[1] = ((double)i + 0.5) / ODB_NORMAL_HIST_PER_DEGREE;
      return;
    }
  }
}

void launch_slab_reduce(const double* part, int images, int slabs, int nq, unsigned min_mask, unsigned max_mask,
                        double* out, cudaStream_t stream) {
  slab_reduce_kernel<<<images, kMetricThreads, 0, stream>>>(part, slabs, nq, min_mask, max_mask, out);
  count_launch();
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_metrics_workspace_bytes(int32_t b, int32_t h, int32_t w) {
  if (!planes_ok(b, h, w)) return -1;
  return ((int64_t)b * slab_count(h, w) + 2 * (int64_t)b) * kPartStride * (int64_t)sizeof(double);
}

static int depth_update(const char* name, const char* bad_argument, const float* pred, const float* gt,
                        const void* mask, int32_t mask_dtype, int32_t b, int32_t h, int32_t w, int32_t space,
                        int align, double min_depth, double max_depth, void* workspace, double* records,
                        double* state_sums, int64_t* state_counts, cudaStream_t stream) {
  const bool disparity = space == ODB_SPACE_DISPARITY;
  if (!pred || !gt || !workspace || !records || !state_sums || !state_counts || !planes_ok(b, h, w) ||
      !metric_mask_ok(mask, mask_dtype) || !aligned(pred, 4) || !aligned(gt, 4) || !aligned(workspace, 8) ||
      !aligned(records, 8) || !aligned(state_sums, 8) || !aligned(state_counts, 8) ||
      (space != ODB_SPACE_DEPTH && !disparity) || !std::isfinite(min_depth) || min_depth < 0.0 ||
      std::isnan(max_depth) || !(max_depth > min_depth) || (disparity && !std::isfinite(max_depth)))
    return fail(ODB_ERR_INVALID, bad_argument);
  const int slabs = slab_count(h, w);
  const long long hw = (long long)h * w;
  double* part = static_cast<double*>(workspace);
  double* mom = part + (long long)b * slabs * kPartStride;
  double* err = mom + (long long)b * kPartStride;
  const int disp = disparity ? 1 : 0;
  depth_moments_kernel<<<dim3(slabs, b), kMetricThreads, 0, stream>>>(pred, gt, mask, mask_dtype, hw, disp, min_depth,
                                                                      max_depth, part);
  count_launch();
  slab_reduce_kernel<<<b, kMetricThreads, 0, stream>>>(part, slabs, 6, 0u, 0u, mom);
  count_launch();
  depth_error_kernel<<<dim3(slabs, b), kMetricThreads, 0, stream>>>(pred, gt, mask, mask_dtype, hw, disp, min_depth,
                                                                    max_depth, mom, align, part);
  count_launch();
  slab_reduce_kernel<<<b, kMetricThreads, 0, stream>>>(part, slabs, 7, 0u, 0u, err);
  count_launch();
  depth_fold_kernel<<<1, 32, 0, stream>>>(mom, err, b, align, records, state_sums,
                                          reinterpret_cast<long long*>(state_counts));
  count_launch();
  return check_launch(name);
}

extern "C" int odb_depth_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype,
                                        int32_t b, int32_t h, int32_t w, int32_t space, double min_depth,
                                        double max_depth, void* workspace, double* records, double* state_sums,
                                        int64_t* state_counts, void* stream_) {
  return depth_update("depth_metrics_update", "depth_metrics_update: bad argument", pred, gt, mask, mask_dtype, b, h,
                      w, space, 1, min_depth, max_depth, workspace, records, state_sums, state_counts,
                      static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_depth_metrics_update_metric(const float* pred, const float* gt, const void* mask,
                                               int32_t mask_dtype, int32_t b, int32_t h, int32_t w, double min_depth,
                                               double max_depth, void* workspace, double* records, double* state_sums,
                                               int64_t* state_counts, void* stream_) {
  return depth_update("depth_metrics_update_metric", "depth_metrics_update_metric: bad argument", pred, gt, mask,
                      mask_dtype, b, h, w, ODB_SPACE_DEPTH, 0, min_depth, max_depth, workspace, records,
                      state_sums, state_counts, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_normal_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype,
                                         int32_t b, int32_t h, int32_t w, void* workspace, double* state_sums,
                                         int64_t* state_counts, int64_t* hist, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!pred || !gt || !workspace || !state_sums || !state_counts || !hist || !planes_ok(b, h, w) ||
      !metric_mask_ok(mask, mask_dtype) || !aligned(pred, 4) || !aligned(gt, 4) || !aligned(workspace, 8) ||
      !aligned(state_sums, 8) || !aligned(state_counts, 8) || !aligned(hist, 8))
    return fail(ODB_ERR_INVALID, "normal_metrics_update: bad argument");
  const int slabs = slab_count(h, w);
  double* part = static_cast<double*>(workspace);
  double* img = part + (long long)b * slabs * kPartStride;
  normal_angle_kernel<<<dim3(slabs, b), kMetricThreads, 0, stream>>>(pred, gt, mask, mask_dtype, (long long)h * w,
                                                                     part, reinterpret_cast<unsigned long long*>(hist));
  count_launch();
  slab_reduce_kernel<<<b, kMetricThreads, 0, stream>>>(part, slabs, 7, 0u, 0u, img);
  count_launch();
  normal_fold_kernel<<<1, 32, 0, stream>>>(img, b, state_sums, reinterpret_cast<long long*>(state_counts));
  count_launch();
  return check_launch("normal_metrics_update");
}

extern "C" int odb_normal_metrics_median(const int64_t* hist, double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!hist || !out || !aligned(hist, 8) || !aligned(out, 8))
    return fail(ODB_ERR_INVALID, "normal_metrics_median: bad argument");
  normal_median_kernel<<<1, kMedianThreads, 0, stream>>>(reinterpret_cast<const unsigned long long*>(hist), out);
  count_launch();
  return check_launch("normal_metrics_median");
}
