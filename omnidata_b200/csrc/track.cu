// Camera tracking (omnidata_b200/track.py FrameTracker): one frame's pose, and with `affine` the scale and shift of its
// depth, solved against a model depth map rendered at a reference pose (normally TSDFVolume.raycast) by point-to-plane
// ICP with projective association (KinectFusion, Newcombe et al. 2011).  Definition in DESIGN.md §3 "Camera tracking"
// and include/omnidata_b200.h; oracle/track_oracle.py restates it in float64, oracle/photometric_oracle.py the
// photometric term.
//
//   track_intensity_kernel  (photometric only) one thread per reference pixel: luminance and Sobel gradient of
//                        ref_rgb into the fp32 planes the tracker keeps
//   track_setup_kernel   one thread: the state from init_pose (by value) and init_nodes (device)
//   track_step_kernel    one Gauss-Newton iteration per launch.  Per fixed chunk of kChunk pixels: association, residual,
//                        Huber weight and Jacobian row of each pixel, and the chunk's fp64 partial sums (warp butterfly,
//                        then the warps in order).  The CTA takes an integer ticket; the last one folds the partials in
//                        chunk order (ordered_sum8), solves the scaled 8 x 8 (6 x 6) normal equations by Cholesky, writes
//                        the next state and re-arms the ticket.  Templated on kPhoto: the photometric instantiation
//                        adds each correspondence's colour term to the same sums, so the geometric arithmetic exists
//                        once
//   track_output_kernel  one thread: pose, nodes and record (init_pose / init_nodes for a failed frame)
//
// The state (pose, M = ref^-1 T, s, t, done flag, status, counters) lives in the workspace.  Every CTA copies it to
// shared memory before it does anything else, so strictly before it takes the ticket; the last CTA, which rewrites it,
// takes the ticket after every other CTA of the launch has read it.  One buffer is therefore enough.  A stopped frame's
// later launches return after reading the done flag, so the launch sequence is fixed and a call can be captured in a
// CUDA graph.  The association, the Jacobian and the exponential are explicit round-to-nearest fp64 operations (no
// contraction into FMAs), so that the oracle reproduces every association decision.  No floating-point atomics; built
// without fast-math.
#include <cmath>
#include <string>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "se3.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kTrkThreads = 256;
constexpr int kChunk = 8 * kTrkThreads;           // pixels per CTA: depends on nothing but this constant
constexpr int kUnknowns = 8;
constexpr int kTri = kUnknowns * (kUnknowns + 1) / 2;
// partial sums: 0..35 the upper triangle of sum w J J^T (row-major, i <= j), 36..43 sum w J e, then these
constexpr int kG = kTri, kCount = kG + kUnknowns, kWE2 = kCount + 1, kWSum = kCount + 2, kDown = kCount + 3,
              kValid = kCount + 4, kSums = kCount + 5;
// the photometric instantiation's four more: count, sum w_c e_c^2, sum w_c and the count with w_c < 1
constexpr int kPCount = kSums, kPWE2 = kSums + 1, kPWSum = kSums + 2, kPDown = kSums + 3, kSumsRgbd = kSums + 4;
constexpr int kPart = 64;                         // doubles per chunk partial (two ordered_sum8 column blocks)
constexpr double kPivotMin = 1e-6;                // smallest Cholesky pivot of the unit-diagonal matrix (not tuned)
// state [kState] doubles
constexpr int kT = 0, kM = 12, kS = 24, kSh = 25, kDone = 26, kStatus = 27, kIters = 28, kCorr = 29, kRms = 30,
              kFrac = 31, kNValid = 32, kState = 34;
constexpr int kStatusOk = 0, kNoOverlap = 1, kDegenerate = 2, kNonfinite = 3;
// luminance weights (ITU-R BT.601) and the largest depth step inside a gradient window, relative to its centre
constexpr double kLumR = 0.299, kLumG = 0.587, kLumB = 0.114, kStepRel = 0.05;

struct TrkParams {
  int h, w, affine, unknowns;
  double fx, fy, cx, cy, tol, robust, max_dist, min_overlap;
  double photometric, photometric_robust;         // lambda and delta_c (the photometric instantiation only)
  double ref[12], init[12];                       // R row-major (9), then t (3), of camera-to-world
};

static int trk_chunks(int h, int w) { return (int)(((long long)h * w + kChunk - 1) / kChunk); }

// Y = (0.299 R + 0.587 G) + 0.114 B
ODB_DEVINL double luminance(float r, float g, float b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(kLumR, (double)r), __dmul_rn(kLumG, (double)g)), __dmul_rn(kLumB, (double)b));
}

// A reference pixel is usable with a surface, a finite colour and a usable normal; its luminance Y in fp64
ODB_DEVINL bool usable_pixel(const float* __restrict__ ref, const float* __restrict__ rgb,
                             const float* __restrict__ nrm, long long hw, long long q, double& d, double& Y) {
  const float dq = ref[q], r = rgb[q], g = rgb[hw + q], b = rgb[2 * hw + q];
  if (!(isfinite(dq) && dq > 0.f && isfinite(r) && isfinite(g) && isfinite(b) && isfinite(nrm[q]) &&
        isfinite(nrm[hw + q]) && isfinite(nrm[2 * hw + q])))
    return false;
  d = dq;
  Y = luminance(r, g, b);
  return true;
}

// ig [3][h][w] = (Y, g_u, g_v) rounded to fp32: Y NaN unless the pixel is usable; the 3 x 3 Sobel gradient / 8 NaN
// unless the window lies in the image, all 9 pixels are usable and none lies further in depth from the centre than
// kStepRel of the centre's depth (depth_normals keeps one-sided normals at a depth step, so the normals alone do not
// keep occlusion edges out)
__global__ void __launch_bounds__(kTrkThreads) track_intensity_kernel(const float* __restrict__ ref,
                                                                      const float* __restrict__ rgb,
                                                                      const float* __restrict__ nrm, int h, int w,
                                                                      float* __restrict__ ig) {
  const long long hw = (long long)h * w;
  const long long i = (long long)blockIdx.x * kTrkThreads + threadIdx.x;
  if (i >= hw) return;
  const int y = (int)(i / w), x = (int)(i - (long long)y * w);
  double dc = 0.0, Yc = 0.0;
  const bool uc = usable_pixel(ref, rgb, nrm, hw, i, dc, Yc);
  float gu = NAN, gv = NAN;
  if (uc && x >= 1 && x <= w - 2 && y >= 1 && y <= h - 2) {
    const double lim = __dmul_rn(kStepRel, dc);
    double Yw[9];
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      double dk = 0.0;
      Yw[k] = 0.0;
      if (!usable_pixel(ref, rgb, nrm, hw, i + (long long)(k / 3 - 1) * w + (k % 3 - 1), dk, Yw[k]) ||
          !(fabs(__dsub_rn(dk, dc)) <= lim))
        ok = false;
    }
    if (ok) {                                     // Yw[3 j + k]: row y + j - 1, column x + k - 1
      const double dx0 = __dsub_rn(Yw[2], Yw[0]), dx1 = __dsub_rn(Yw[5], Yw[3]), dx2 = __dsub_rn(Yw[8], Yw[6]);
      const double dy0 = __dsub_rn(Yw[6], Yw[0]), dy1 = __dsub_rn(Yw[7], Yw[1]), dy2 = __dsub_rn(Yw[8], Yw[2]);
      gu = (float)__ddiv_rn(__dadd_rn(__dadd_rn(dx0, __dmul_rn(2.0, dx1)), dx2), 8.0);
      gv = (float)__ddiv_rn(__dadd_rn(__dadd_rn(dy0, __dmul_rn(2.0, dy1)), dy2), 8.0);
    }
  }
  ig[i] = uc ? (float)Yc : NAN;
  ig[hw + i] = gu;
  ig[2 * hw + i] = gv;
}

// prec: the photometric record columns 8..10 (NULL without the photometric term), zero until a step writes them
__global__ void track_setup_kernel(TrkParams P, const double* __restrict__ init_nodes, double* __restrict__ st,
                                   double* __restrict__ prec) {
  if (threadIdx.x != 0) return;
  if (prec) prec[0] = prec[1] = prec[2] = 0.0;
  const double s = P.affine ? init_nodes[0] : 1.0, t = P.affine ? init_nodes[1] : 0.0;
  for (int k = 0; k < 12; ++k) st[kT + k] = P.init[k];
  relative_pose(P.ref, P.init, st + kM);
  st[kS] = s;
  st[kSh] = t;
  const bool bad = !(isfinite(s) && isfinite(t));
  st[kDone] = bad ? 1.0 : 0.0;
  st[kStatus] = bad ? kNonfinite : kStatusOk;
  for (int k = kIters; k < kState; ++k) st[k] = 0.0;
}

// w J J^T and w J e added to the sums (upper triangle row-major, then the gradient)
template <int N>
ODB_DEVINL void add_row(double (&acc)[N], const double (&J)[kUnknowns], double wt, double e) {
  int k = 0;
#pragma unroll
  for (int p = 0; p < kUnknowns; ++p) {
    const double wj = wt * J[p];
#pragma unroll
    for (int c = p; c < kUnknowns; ++c) acc[k++] += wj * J[c];
    acc[kG + p] += wj * e;
  }
}

// the Jacobian row (m, P x m, m.(a r), m.r) with m = Rm^T g for a residual whose gradient with respect to Q is g
ODB_DEVINL void jacobian_row(const double* M, const double g[3], const double Pp[3], const double r[3], double a,
                             double (&J)[kUnknowns]) {
  double m[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    m[j] = __dadd_rn(__dadd_rn(__dmul_rn(M[j], g[0]), __dmul_rn(M[3 + j], g[1])), __dmul_rn(M[6 + j], g[2]));
  const double ar[3] = {__dmul_rn(a, r[0]), __dmul_rn(a, r[1]), a};
  J[0] = m[0];
  J[1] = m[1];
  J[2] = m[2];
  J[3] = __dsub_rn(__dmul_rn(Pp[1], m[2]), __dmul_rn(Pp[2], m[1]));
  J[4] = __dsub_rn(__dmul_rn(Pp[2], m[0]), __dmul_rn(Pp[0], m[2]));
  J[5] = __dsub_rn(__dmul_rn(Pp[0], m[1]), __dmul_rn(Pp[1], m[0]));
  J[6] = dot3_rn(m, ar);
  J[7] = dot3_rn(m, r);
}

// The photometric inputs of one pixel's term (kPhoto): the frame's rgb [3][h][w] and the reference's (Y, g_u, g_v)
struct PhotoIn {
  const float* rgb;
  const float* ig;
};

// One pixel's terms added to acc (nothing when it has no correspondence); with kPhoto also its photometric term
template <bool kPhoto, int N>
ODB_DEVINL void pixel_terms(const float* __restrict__ pred, const float* __restrict__ ref,
                            const float* __restrict__ nrm, const PhotoIn& C, const TrkParams& P, const double* M,
                            double s, double t, long long i, double (&acc)[N]) {
  const long long hw = (long long)P.h * P.w;
  const float af = pred[i];
  if (!isfinite(af)) return;
  const double a = af, z = __dadd_rn(__dmul_rn(s, a), t);
  if (!(z > 0.0)) return;
  acc[kValid] += 1.0;
  const int y = (int)(i / P.w), x = (int)(i - (long long)y * P.w);
  const double r[3] = {__ddiv_rn(__dsub_rn((double)x, P.cx), P.fx), __ddiv_rn(__dsub_rn((double)y, P.cy), P.fy), 1.0};
  const double Pp[3] = {__dmul_rn(z, r[0]), __dmul_rn(z, r[1]), z};
  double Q[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) Q[k] = __dadd_rn(dot3_rn(M + 3 * k, Pp), M[9 + k]);
  if (!(Q[2] > 0.0)) return;
  const double uf = __dadd_rn(__ddiv_rn(__dmul_rn(P.fx, Q[0]), Q[2]), P.cx);
  const double vf = __dadd_rn(__ddiv_rn(__dmul_rn(P.fy, Q[1]), Q[2]), P.cy);
  const double u = floor(__dadd_rn(uf, 0.5)), v = floor(__dadd_rn(vf, 0.5));
  if (!(u >= 0.0 && u <= (double)(P.w - 1) && v >= 0.0 && v <= (double)(P.h - 1))) return;
  const long long q = (long long)v * P.w + (long long)u;
  const float dq = ref[q], c0 = nrm[q], c1 = nrm[hw + q], c2 = nrm[2 * hw + q];
  if (!(isfinite(dq) && dq > 0.f && isfinite(c0) && isfinite(c1) && isfinite(c2))) return;
  const double n[3] = {__dsub_rn(__dmul_rn(2.0, (double)c0), 1.0), __dsub_rn(__dmul_rn(2.0, (double)c1), 1.0),
                       __dsub_rn(__dmul_rn(2.0, (double)c2), 1.0)};
  const double d = dq;
  const double Vq[3] = {__dmul_rn(d, __ddiv_rn(__dsub_rn(u, P.cx), P.fx)),
                        __dmul_rn(d, __ddiv_rn(__dsub_rn(v, P.cy), P.fy)), d};
  const double df[3] = {__dsub_rn(Q[0], Vq[0]), __dsub_rn(Q[1], Vq[1]), __dsub_rn(Q[2], Vq[2])};
  if (!(__dsqrt_rn(dot3_rn(df, df)) <= P.max_dist)) return;
  const double e = dot3_rn(n, df), ae = fabs(e);
  const double wt = ae <= P.robust ? 1.0 : __ddiv_rn(P.robust, ae);
  {
    double J[kUnknowns];
    jacobian_row(M, n, Pp, r, a, J);
    add_row(acc, J, wt, e);
  }
  acc[kCount] += 1.0;
  acc[kWE2] += wt * e * e;
  acc[kWSum] += wt;
  acc[kDown] += ae > P.robust ? 1.0 : 0.0;
  if constexpr (kPhoto) {
    // bilinear lookup of (Y, g_u, g_v) at the unrounded projection (u, v), x first
    const double bu = floor(uf), bv = floor(vf);
    if (!(bu >= 0.0 && bu <= (double)(P.w - 2) && bv >= 0.0 && bv <= (double)(P.h - 2))) return;
    const long long b0 = (long long)bv * P.w + (long long)bu;
    const double fu = __dsub_rn(uf, bu), fv = __dsub_rn(vf, bv);
    double I[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* pl = C.ig + c * hw + b0;
      const float x00 = pl[0], x10 = pl[1], x01 = pl[P.w], x11 = pl[P.w + 1];
      if (!(isfinite(x00) && isfinite(x10) && isfinite(x01) && isfinite(x11))) return;
      I[c] = lerp_rn(lerp_rn(x00, x10, fu), lerp_rn(x01, x11, fu), fv);
    }
    const double Yf = luminance(C.rgb[i], C.rgb[hw + i], C.rgb[2 * hw + i]);
    if (!isfinite(Yf)) return;
    const double ec = __dsub_rn(I[0], Yf), aec = fabs(ec);
    const double wc = aec <= P.photometric_robust ? 1.0 : __ddiv_rn(P.photometric_robust, aec);
    // d e_c / d Q = (g_u, g_v) d(u, v) / d Q
    const double gfu = __dmul_rn(I[1], P.fx), gfv = __dmul_rn(I[2], P.fy);
    const double g3[3] = {__ddiv_rn(gfu, Q[2]), __ddiv_rn(gfv, Q[2]),
                          -__ddiv_rn(__dadd_rn(__dmul_rn(gfu, Q[0]), __dmul_rn(gfv, Q[1])), __dmul_rn(Q[2], Q[2]))};
    double J[kUnknowns];
    jacobian_row(M, g3, Pp, r, a, J);
    add_row(acc, J, __dmul_rn(P.photometric, wc), ec);
    acc[kPCount] += 1.0;
    acc[kPWE2] += wc * ec * ec;
    acc[kPWSum] += wc;
    acc[kPDown] += aec > P.photometric_robust ? 1.0 : 0.0;
  }
}

ODB_DEVINL int tri_index(int i, int j) {          // i <= j
  return i * kUnknowns - i * (i - 1) / 2 + (j - i);
}

// The last CTA, thread 0: status, solve result and the next state from the folded sums tot and the factor in band / rhs
ODB_DEVINL void track_update(const TrkParams& P, const double* tot, const double* band, const double* rhs,
                             const double* scale, int code, double* st) {
  const int n = P.unknowns;
  st[kIters] += 1.0;
  st[kCorr] = tot[kCount];
  st[kNValid] = tot[kValid];
  st[kRms] = tot[kWSum] > 0.0 ? sqrt(tot[kWE2] / tot[kWSum]) : 0.0;
  st[kFrac] = tot[kCount] > 0.0 ? tot[kDown] / tot[kCount] : 0.0;
  double x[kUnknowns] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (code == kStatusOk) {
    for (int k = 0; k < n; ++k) {
      const double l = band[k * n];                 // the factor's diagonal: sqrt of the k-th pivot
      if (!(__dmul_rn(l, l) >= kPivotMin)) code = kDegenerate;
    }
  }
  if (code == kStatusOk) {
#pragma unroll
    for (int k = 0; k < kUnknowns; ++k) {
      if (k < n) x[k] = __ddiv_rn(rhs[k], scale[k]);
      if (!isfinite(x[k])) code = kNonfinite;
    }
  }
  double Tn[12];
  if (code == kStatusOk) {
    double Re[9], u[3];
    se3_exp(x, Re, u);
    const double* T = st + kT;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j)
        Tn[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(T[3 * i], Re[j]), __dmul_rn(T[3 * i + 1], Re[3 + j])),
                                  __dmul_rn(T[3 * i + 2], Re[6 + j]));
      Tn[9 + i] = __dadd_rn(dot3_rn(T + 3 * i, u), T[9 + i]);
    }
#pragma unroll
    for (int k = 0; k < 12; ++k)
      if (!isfinite(Tn[k])) code = kNonfinite;
  }
  if (code != kStatusOk) {
    st[kStatus] = code;
    st[kDone] = 1.0;
    return;
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) st[kT + k] = Tn[k];
  relative_pose(P.ref, Tn, st + kM);
  st[kS] = __dadd_rn(st[kS], x[6]);
  st[kSh] = __dadd_rn(st[kSh], x[7]);
  const double vv[3] = {x[0], x[1], x[2]}, om[3] = {x[3], x[4], x[5]};
  if (__dsqrt_rn(dot3_rn(om, om)) <= P.tol && __dsqrt_rn(dot3_rn(vv, vv)) <= P.tol && fabs(x[6]) <= P.tol &&
      fabs(x[7]) <= P.tol)
    st[kDone] = 1.0;
}

// kPhoto: prec = the record's photometric columns 8..10, written by the last CTA of every launch that runs
template <bool kPhoto>
__global__ void __launch_bounds__(kTrkThreads) track_step_kernel(const float* __restrict__ pred,
                                                                 const float* __restrict__ ref,
                                                                 const float* __restrict__ nrm, PhotoIn C, TrkParams P,
                                                                 double* __restrict__ st, double* __restrict__ part,
                                                                 unsigned int* __restrict__ ticket,
                                                                 double* __restrict__ prec) {
  constexpr int nsums = kPhoto ? kSumsRgbd : kSums;   // partial sums per chunk
  __shared__ double S[kDone + 1];
  __shared__ double red[kTrkThreads / 32][nsums];
  __shared__ bool last;
  if (threadIdx.x <= kDone) S[threadIdx.x] = st[threadIdx.x];
  __syncthreads();
  if (S[kDone] != 0.0) return;
  double acc[nsums];
#pragma unroll
  for (int k = 0; k < nsums; ++k) acc[k] = 0.0;
  const long long hw = (long long)P.h * P.w;
#pragma unroll 1
  for (int k = 0; k < kChunk / kTrkThreads; ++k) {
    const long long i = (long long)blockIdx.x * kChunk + k * kTrkThreads + threadIdx.x;
    if (i < hw) pixel_terms<kPhoto>(pred, ref, nrm, C, P, S + kM, S[kS], S[kSh], i, acc);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < nsums; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < nsums) {
    double v = 0.0;
#pragma unroll
    for (int q = 0; q < kTrkThreads / 32; ++q) v += red[q][threadIdx.x];
    part[(long long)blockIdx.x * kPart + threadIdx.x] = v;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // fold the partials in chunk order: columns 0..31, then 32..nsums-1
  __shared__ double tot[kPart];
  const int col = threadIdx.x & 31;
  const double lo = ordered_sum8(gridDim.x, true, [&](int c) { return __ldcg(part + (long long)c * kPart + col); });
  if (threadIdx.x < 32) tot[col] = lo;
  __syncthreads();
  const double hi = ordered_sum8(gridDim.x, 32 + col < nsums,
                                 [&](int c) { return __ldcg(part + (long long)c * kPart + 32 + col); });
  if (threadIdx.x < 32) tot[32 + col] = hi;
  __syncthreads();
  // unit-diagonal scaling D^-1 H D^-1 y = -D^-1 g, x = D^-1 y; the lower band of band_cholesky_solve with w = n
  __shared__ double band[kUnknowns * kUnknowns], rhs[kUnknowns], scale[kUnknowns];
  __shared__ int code;
  const int n = P.unknowns;
  if (threadIdx.x == 0) {
    int c = kStatusOk;
    for (int k = 0; k < nsums; ++k)
      if (!isfinite(tot[k])) c = kNonfinite;
    if (c == kStatusOk && !(tot[kValid] > 0.0 && tot[kCount] >= __dmul_rn(P.min_overlap, tot[kValid]) &&
                            tot[kCount] > 0.0))
      c = kNoOverlap;
    if (c == kStatusOk)
      for (int k = 0; k < n; ++k) {
        const double hkk = tot[tri_index(k, k)];
        if (!(hkk > 0.0)) c = kDegenerate;
        scale[k] = __dsqrt_rn(hkk);
      }
    if (c == kStatusOk)
      for (int r = 0; r < n; ++r) {
        for (int q = 0; q <= r; ++q) {
          const int cc = r - q;
          band[r * n + q] = __ddiv_rn(tot[tri_index(cc, r)], __dmul_rn(scale[r], scale[cc]));
        }
        rhs[r] = -__ddiv_rn(tot[kG + r], scale[r]);
      }
    code = c;
  }
  __syncthreads();
  if (code == kStatusOk) band_cholesky_solve(band, rhs, n, n);
  if (threadIdx.x == 0) {
    track_update(P, tot, band, rhs, scale, code, st);
    if constexpr (kPhoto) {
      prec[0] = tot[kPCount];
      prec[1] = tot[kPWSum] > 0.0 ? sqrt(tot[kPWE2] / tot[kPWSum]) : 0.0;
      prec[2] = tot[kPCount] > 0.0 ? tot[kPDown] / tot[kPCount] : 0.0;
    }
    *ticket = 0u;                                   // re-armed for the next launch
  }
}

__global__ void track_output_kernel(TrkParams P, const double* __restrict__ init_nodes, const double* __restrict__ st,
                                    double* __restrict__ pose, double* __restrict__ nodes,
                                    double* __restrict__ record) {
  if (threadIdx.x != 0) return;
  const bool ok = st[kStatus] == (double)kStatusOk;
  const double* T = ok ? st + kT : P.init;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) pose[4 * r + c] = T[3 * r + c];
    pose[4 * r + 3] = T[9 + r];
  }
  pose[12] = pose[13] = pose[14] = 0.0;
  pose[15] = 1.0;
  double s = 1.0, t = 0.0;
  if (ok) {
    s = st[kS];
    t = st[kSh];
  } else if (P.affine) {
    s = init_nodes[0];
    t = init_nodes[1];
  }
  nodes[0] = s;
  nodes[1] = t;
  record[0] = st[kCorr];
  record[1] = st[kStatus];
  record[2] = st[kRms];
  record[3] = st[kFrac];
  record[4] = st[kIters];
  record[5] = s;
  record[6] = t;
  record[7] = st[kNValid];
}

// info [n][n] = sum w J J^T of the last step that ran: columns 0..kTri-1 of the chunk partials folded in chunk order by
// ordered_sum8 exactly as that step's last CTA folded them, so the matrix is the one its Cholesky factored (unscaled)
__global__ void __launch_bounds__(kTrkThreads) track_information_kernel(const double* __restrict__ part, int chunks,
                                                                        int n, double* __restrict__ info) {
  __shared__ double tot[kPart];
  const int col = threadIdx.x & 31;
  const double lo = ordered_sum8(chunks, true, [&](int c) { return __ldcg(part + (long long)c * kPart + col); });
  if (threadIdx.x < 32) tot[col] = lo;
  __syncthreads();
  const double hi = ordered_sum8(chunks, 32 + col < kTri,
                                 [&](int c) { return __ldcg(part + (long long)c * kPart + 32 + col); });
  if (threadIdx.x < 32) tot[32 + col] = hi;
  __syncthreads();
  if (threadIdx.x < n * n) {
    const int p = threadIdx.x / n, q = threadIdx.x - p * n;
    info[threadIdx.x] = tot[p <= q ? tri_index(p, q) : tri_index(q, p)];
  }
}

}  // namespace odb

using namespace odb;

extern "C" int odb_track_information(const void* workspace, int32_t h, int32_t w, int32_t unknowns, double* info,
                                     void* stream_) {
  if (!workspace || !info || !planes_ok(1, h, w) || (unknowns != 6 && unknowns != 8) || !aligned(workspace, 8) ||
      !aligned(info, 8))
    return fail(ODB_ERR_INVALID, "track_information: bad argument");
  const double* part = static_cast<const double*>(workspace) + 1 + kState;
  track_information_kernel<<<1, kTrkThreads, 0, static_cast<cudaStream_t>(stream_)>>>(part, trk_chunks(h, w),
                                                                                      unknowns, info);
  count_launch();
  return check_launch("track_information");
}

extern "C" int64_t odb_track_workspace_bytes(int32_t h, int32_t w) {
  if (!planes_ok(1, h, w)) return -1;
  return (1 + kState + (int64_t)trk_chunks(h, w) * kPart) * (int64_t)sizeof(double);
}

// odb_track_frame (rgb NULL) and odb_track_frame_rgbd
static int track_frame(const char* name, const float* pred, const float* rgb, const float* ref_depth,
                       const float* ref_rgb, const float* ref_normals, float* ref_intensity, int32_t h, int32_t w,
                       double fx, double fy, double cx, double cy, const double* ref_pose, const double* init_pose,
                       const double* init_nodes, int32_t affine, int32_t iterations, double tol, double robust,
                       double max_dist, double min_overlap, double photometric, double photometric_robust,
                       void* workspace, double* pose, double* nodes, double* record, cudaStream_t stream) {
  const bool photo = rgb != nullptr;
  if (!pred || !ref_depth || !ref_normals || !ref_pose || !init_pose || !workspace || !pose || !nodes || !record ||
      (affine != 0 && affine != 1) || (init_nodes == nullptr) != (affine == 0) || !planes_ok(1, h, w) ||
      !(std::isfinite(fx) && fx > 0.0 && std::isfinite(fy) && fy > 0.0 && std::isfinite(cx) && std::isfinite(cy)) ||
      iterations < 1 || iterations > 100 || !(std::isfinite(tol) && tol > 0.0) ||
      !(std::isfinite(robust) && robust > 0.0) || !(std::isfinite(max_dist) && max_dist > 0.0) ||
      !(min_overlap > 0.0 && min_overlap <= 1.0) || !aligned(pred, 4) || !aligned(ref_depth, 4) ||
      !aligned(ref_normals, 4) || !aligned(init_nodes, 8) || !aligned(workspace, 8) || !aligned(pose, 8) ||
      !aligned(nodes, 8) || !aligned(record, 8) ||
      (photo && (!ref_rgb || !ref_intensity || !(std::isfinite(photometric) && photometric > 0.0) ||
                 !(std::isfinite(photometric_robust) && photometric_robust > 0.0) || !aligned(rgb, 4) ||
                 !aligned(ref_rgb, 4) || !aligned(ref_intensity, 4))))
    return fail(ODB_ERR_INVALID, (std::string(name) + ": bad argument").c_str());
  TrkParams P;
  if (!pose_ok(ref_pose, P.ref) || !pose_ok(init_pose, P.init))
    return fail(ODB_ERR_INVALID,
                (std::string(name) + ": a pose is not a finite rigid camera-to-world matrix").c_str());
  P.h = h;
  P.w = w;
  P.affine = affine;
  P.unknowns = affine ? 8 : 6;
  P.fx = fx; P.fy = fy; P.cx = cx; P.cy = cy;
  P.tol = tol;
  P.robust = robust;
  P.max_dist = max_dist;
  P.min_overlap = min_overlap;
  P.photometric = photometric;
  P.photometric_robust = photometric_robust;
  double* ws = static_cast<double*>(workspace);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(ws);
  double* st = ws + 1;
  double* part = st + kState;
  double* prec = photo ? record + ODB_TRACK_RECORD : nullptr;
  cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(double), stream);
  if (e != cudaSuccess) return fail_cuda(e, (std::string(name) + ": cudaMemsetAsync").c_str());
  const int chunks = trk_chunks(h, w);
  if (photo) {
    track_intensity_kernel<<<(unsigned)(((long long)h * w + kTrkThreads - 1) / kTrkThreads), kTrkThreads, 0,
                             stream>>>(ref_depth, ref_rgb, ref_normals, h, w, ref_intensity);
    count_launch();
  }
  track_setup_kernel<<<1, 32, 0, stream>>>(P, init_nodes, st, prec);
  count_launch();
  const PhotoIn C{rgb, ref_intensity};
  for (int it = 0; it < iterations; ++it) {
    if (photo)
      track_step_kernel<true><<<chunks, kTrkThreads, 0, stream>>>(pred, ref_depth, ref_normals, C, P, st, part,
                                                                  ticket, prec);
    else
      track_step_kernel<false><<<chunks, kTrkThreads, 0, stream>>>(pred, ref_depth, ref_normals, C, P, st, part,
                                                                   ticket, nullptr);
    count_launch();
  }
  track_output_kernel<<<1, 32, 0, stream>>>(P, init_nodes, st, pose, nodes, record);
  count_launch();
  return check_launch(name);
}

extern "C" int odb_track_frame(const float* pred, const float* ref_depth, const float* ref_normals, int32_t h,
                               int32_t w, double fx, double fy, double cx, double cy, const double* ref_pose,
                               const double* init_pose, const double* init_nodes, int32_t affine, int32_t iterations,
                               double tol, double robust, double max_dist, double min_overlap, void* workspace,
                               double* pose, double* nodes, double* record, void* stream_) {
  return track_frame("track_frame", pred, nullptr, ref_depth, nullptr, ref_normals, nullptr, h, w, fx, fy, cx, cy,
                     ref_pose, init_pose, init_nodes, affine, iterations, tol, robust, max_dist, min_overlap, 0.0, 0.0,
                     workspace, pose, nodes, record, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_track_frame_rgbd(const float* pred, const float* rgb, const float* ref_depth, const float* ref_rgb,
                                    const float* ref_normals, float* ref_intensity, int32_t h, int32_t w, double fx,
                                    double fy, double cx, double cy, const double* ref_pose, const double* init_pose,
                                    const double* init_nodes, int32_t affine, int32_t iterations, double tol,
                                    double robust, double max_dist, double min_overlap, double photometric,
                                    double photometric_robust, void* workspace, double* pose, double* nodes,
                                    double* record, void* stream_) {
  if (!rgb) return fail(ODB_ERR_INVALID, "track_frame_rgbd: bad argument");
  return track_frame("track_frame_rgbd", pred, rgb, ref_depth, ref_rgb, ref_normals, ref_intensity, h, w, fx, fy, cx,
                     cy, ref_pose, init_pose, init_nodes, affine, iterations, tol, robust, max_dist, min_overlap,
                     photometric, photometric_robust, workspace, pose, nodes, record,
                     static_cast<cudaStream_t>(stream_));
}
