// fp64 routines shared by the post-processing kernels: the SPD band solve of the tiled, ensemble and sparse alignments
// (tiled.cu, ensemble.cu, sparse.cu), the angle between two vectors of the normal metrics and the normal ensemble merge
// (metrics.cu, ensemble.cu), and the valid set and clamped depth of the depth metrics and the sparse alignment
// (metrics.cu, sparse.cu), and the round-to-nearest linear interpolation of the TSDF raycast and the tracker's bilinear
// lookups (volume.cu, track.cu).  Callers are built without fast-math.
#pragma once
#include "common.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr double kRadToDeg = 180.0 / 3.141592653589793;
constexpr size_t kBandSmemMax = 200 * 1024;      // band + right-hand side of a band solve in shared memory up to this

ODB_DEVINL bool mask_valid(const void* mask, int kind, long long i) {
  if (kind == ODB_MASK_U8) return static_cast<const uint8_t*>(mask)[i] != 0;
  if (kind == ODB_MASK_F32) return static_cast<const float*>(mask)[i] != 0.0f;
  return true;
}

// a + t (b - a), each operation rounded to nearest
ODB_DEVINL double lerp_rn(double a, double b, double t) { return __dadd_rn(a, __dmul_rn(t, __dsub_rn(b, a))); }

ODB_DEVINL bool depth_valid(double g, double min_depth, double max_depth) {
  return isfinite(g) && g > min_depth && g <= max_depth;           // max_depth = +inf when not given
}

// d-hat = clamp(s p + t, min, max) (depth space) or clamp(1 / max(s p + t, 1 / max), min, max) (disparity space)
ODB_DEVINL double depth_hat(double p, double s, double t, int disparity, double min_depth, double max_depth) {
  const double a = __dadd_rn(__dmul_rn(s, p), t);
  const double d = disparity ? __drcp_rn(fmax(a, __drcp_rn(max_depth))) : a;
  return fmin(fmax(d, min_depth), max_depth);
}

// Solves A x = rhs in place for A symmetric positive definite of order n with half-bandwidth w - 1 (w = n: dense).
// The lower band is stored row-wise, band[r * w + q] = A[r][r - q] (entries with q > r are not read); it is
// overwritten by the Cholesky factor, rhs by x.  Every thread of the CTA calls it (block-strided loops,
// __syncthreads); band and rhs lie in shared or global memory, and x is visible to all threads on return.
ODB_DEVINL void band_cholesky_solve(double* band, double* rhs, int n, int w) {
  // A = L L^T, in place, column by column; each trailing element is updated by one thread
  for (int k = 0; k < n; ++k) {
    const int m = min(w - 1, n - 1 - k);
    const double d = sqrt(band[(long long)k * w]);
    for (int r = 1 + threadIdx.x; r <= m; r += blockDim.x) band[(long long)(k + r) * w + r] /= d;
    __syncthreads();
    if (threadIdx.x == 0) band[(long long)k * w] = d;
    for (int e = threadIdx.x; e < m * m; e += blockDim.x) {
      const int r = e / m + 1, c = e - (r - 1) * m + 1;
      if (c <= r)
        band[(long long)(k + r) * w + (r - c)] -= band[(long long)(k + r) * w + r] * band[(long long)(k + c) * w + c];
    }
    __syncthreads();
  }
  // L y = rhs, then L^T x = y (column-oriented; rhs is overwritten by y, then by x).  Step k reads rhs[k] and updates
  // the entries after (before) it, so thread 0's store of rhs[k] needs no barrier of its own
  for (int k = 0; k < n; ++k) {
    const int m = min(w - 1, n - 1 - k);
    const double yk = rhs[k] / band[(long long)k * w];
    for (int r = 1 + threadIdx.x; r <= m; r += blockDim.x) rhs[k + r] -= band[(long long)(k + r) * w + r] * yk;
    __syncthreads();
    if (threadIdx.x == 0) rhs[k] = yk;
  }
  __syncthreads();
  for (int k = n - 1; k >= 0; --k) {
    const int m = min(w - 1, k);
    const double xk = rhs[k] / band[(long long)k * w];
    for (int q = 1 + threadIdx.x; q <= m; q += blockDim.x) rhs[k - q] -= band[(long long)k * w + q] * xk;
    __syncthreads();
    if (threadIdx.x == 0) rhs[k] = xk;
  }
  __syncthreads();
}

// atan2(|p x q|, p . q) in degrees, every product and sum rounded to nearest (no fma contraction), so that the float64
// oracles reproduce it operation by operation
ODB_DEVINL double angle_deg(const double p[3], const double q[3]) {
  const double cx = __dsub_rn(__dmul_rn(p[1], q[2]), __dmul_rn(p[2], q[1]));
  const double cy = __dsub_rn(__dmul_rn(p[2], q[0]), __dmul_rn(p[0], q[2]));
  const double cz = __dsub_rn(__dmul_rn(p[0], q[1]), __dmul_rn(p[1], q[0]));
  const double cr = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz)));
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn(p[0], q[0]), __dmul_rn(p[1], q[1])), __dmul_rn(p[2], q[2]));
  return __dmul_rn(atan2(cr, dot), kRadToDeg);
}

}  // namespace odb
