// Depth-normal fusion (omnidata_b200/fusion.py DepthNormalFusion, depth_normals): a depth prediction a and a surface
// normal prediction of the same frame are combined into one depth map z whose back-projection agrees with the normals,
// with the depth's unknown shift t recovered from them.  Definition in DESIGN.md §3 "Depth-normal fusion" and
// include/omnidata_b200.h; oracle/fusion_oracle.py restates it in float64.
//
// Pixel (x, y) has the ray r = ((x - cx) / fx, (y - cy) / fy, 1).  A kept 4-neighbour edge (p, q) has the coefficients
// alpha = m.r_p, beta = m.r_q of the mean normal m of its two ends, and the residual e = beta z_q - alpha z_p.  With
// N = the Gram operator of the residuals and s(v) = S_V v / (|V| (1 + kappa)), the energy
//   E(z, t) = lambda S_V (z - a - t)^2 + lambda kappa |V| t^2 + S_kept e^2
// reduces, after eliminating t, to the SPD system M z = lambda (z - s(z)) + N z = lambda (a - s(a)) = b, solved by
// Jacobi-preconditioned conjugate gradients in fp64 from z0 = a:
//
//   fusion_range_kernel   per 4096-pixel slab: (min, max, |V|, S a) of a over V, folded by launch_slab_reduce
//   fusion_edges_kernel   per 64 x 16 tile: the coefficients of each pixel's right and down edge
//   fusion_setup_kernel   per tile: inverse Jacobi diagonal, r0 = -N a, z0 = D^-1 r0; the last CTA of the image sets
//                         up its scalars
//   fusion_matvec_kernel  per tile: p = z + beta p (shared tile with a one-pixel halo), q = lambda p + N p, partials
//                         (p.p, S p, p.N p); last CTA: alpha
//   fusion_update_kernel  per tile: x += alpha p, r -= alpha (q - lambda s(p)), z = D^-1 r, partials (r.z, r.r); last
//                         CTA: beta, convergence
//   fusion_shift_kernel   per tile: S_V (x - a); last CTA: t
//   fusion_apply_kernel   per tile: out = x rounded once (NaN off V), S_V (x - a - t)^2; last CTA: the record
//
// Per-image scalars live in the workspace.  Every tile CTA writes its partials, takes an integer ticket, and the last
// CTA of the image folds the partials in tile order (ordered_sum8) and re-arms the ticket: two launches per CG
// iteration.  Once an image has converged its CTAs return after reading its flag, so its state is never written again
// and the remaining launches of a call cost launch overhead only.  Tile partition and fold order depend on h and w only:
// results are bit-reproducible and independent of the batch.  No floating-point atomics.  Built without fast-math; the
// coefficients and depth_normals are written with explicit round-to-nearest operations so that the oracle reproduces
// them operation by operation.
#include <cmath>
#include <initializer_list>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "select.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kFusThreads = 256;
constexpr int kTW = 64, kTH = 16;                 // CG tile; each thread owns one column, rows ty, ty + 4, ...
constexpr int kRowsPerThread = kTH / (kFusThreads / kTW);
constexpr double kKappa = 1e-6;                   // ridge on t (the ensemble's): t stays defined on a fronto-parallel scene
constexpr int kTilePart = 4;                      // doubles per tile partial
// per-image scalars [b][8]
constexpr int kRho = 0, kAlpha = 1, kBeta = 2, kLamSp = 3, kDone = 4, kIters = 5, kRR = 6, kBB = 7;
// per-image info [b][kPartStride]: launch_slab_reduce writes 0..3, the folds the rest
constexpr int kMin = 0, kMax = 1, kN = 2, kSumA = 3, kStatus = 4, kKept = 5, kShift = 6;

struct FusGeom {
  int h, w, tiles_x, tiles;
  double fx, fy, cx, cy, ax, ay, az, jump, lam;
  int shift;
};

struct FusWs {                // workspace carve-up (odb_fusion_workspace_bytes)
  unsigned int* ticket;       // [b]
  double *info, *scal, *slab, *part;
  double2 *cr, *cd;           // (alpha, beta) of the right / down edge of each pixel, 0 when dropped
  double *dinv, *x, *r, *z, *p[2], *q;
};

static int fus_tiles(int h, int w) { return ((w + kTW - 1) / kTW) * ((h + kTH - 1) / kTH); }

// bytes before the per-pixel planes: tickets, info, scalars, slab partials, tile partials
static int64_t fus_head_doubles(int64_t b, int h, int w) {
  return b + b * kPartStride + b * 8 + b * slab_count(h, w) * kPartStride + b * fus_tiles(h, w) * kTilePart;
}

static FusWs fus_ws(void* workspace, int b, int h, int w, bool planes) {
  FusWs W;
  double* d = static_cast<double*>(workspace);
  W.ticket = reinterpret_cast<unsigned int*>(d);
  d += b;                                          // one double per ticket keeps the rest 8-byte aligned
  W.info = d;
  d += (int64_t)b * kPartStride;
  W.scal = d;
  d += (int64_t)b * 8;
  W.slab = d;
  d += (int64_t)b * slab_count(h, w) * kPartStride;
  W.part = d;
  d += (int64_t)b * fus_tiles(h, w) * kTilePart;
  if (planes) {
    const int64_t n = (int64_t)b * h * w;
    d = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(d) + 15) & ~uintptr_t(15));
    W.cr = reinterpret_cast<double2*>(d);
    W.cd = W.cr + n;
    d += 4 * n;
    W.dinv = d;
    W.x = d + n;
    W.r = d + 2 * n;
    W.z = d + 3 * n;
    W.p[0] = d + 4 * n;
    W.p[1] = d + 5 * n;
    W.q = d + 6 * n;
  }
  return W;
}

ODB_DEVINL double ray_x(int x, const FusGeom& G) { return __ddiv_rn(__dsub_rn((double)x, G.cx), G.fx); }
ODB_DEVINL double ray_y(int y, const FusGeom& G) { return __ddiv_rn(__dsub_rn((double)y, G.cy), G.fy); }
ODB_DEVINL double dot3(const double u[3], const double v[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(u[0], v[0]), __dmul_rn(u[1], v[1])), __dmul_rn(u[2], v[2]));
}

// V: mask != 0 and a finite
ODB_DEVINL bool in_v(const float* a, const void* mask, int kind, long long i) {
  return mask_valid(mask, kind, i) && isfinite(a[i]);
}

// n = axes (2 clamp(c, 0, 1) - 1), usable when finite and |n| >= 0.5; then normalised
ODB_DEVINL bool unit_normal(const float* c, long long plane, long long i, const FusGeom& G, double n[3]) {
  const double ax[3] = {G.ax, G.ay, G.az};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float v = c[k * plane + i];
    if (!isfinite(v)) return false;
    n[k] = ax[k] * __dsub_rn(__dmul_rn(2.0, fmin(fmax((double)v, 0.0), 1.0)), 1.0);
  }
  const double len = __dsqrt_rn(dot3(n, n));
  if (!(len >= 0.5)) return false;
#pragma unroll
  for (int k = 0; k < 3; ++k) n[k] = __ddiv_rn(n[k], len);
  return true;
}

// Edge from pixel p (index i, position (x, y)) to q = p + (dx, dy) (index j).  Kept when both ends are in V with
// usable normals, n_p . n_q > 0 and |a_q - a_p| <= thr; then (alpha, beta) = (m.r_p, m.r_q), m = normalise(n_p + n_q).
ODB_DEVINL double2 edge_coef(const float* a, const float* c, const void* mask, int kind, long long plane, long long i,
                             long long j, int x, int y, int dx, int dy, double thr, const FusGeom& G) {
  const double2 none = make_double2(0.0, 0.0);
  if (!in_v(a, mask, kind, i) || !in_v(a, mask, kind, j)) return none;
  if (!(fabs(__dsub_rn((double)a[j], (double)a[i])) <= thr)) return none;
  double np[3], nq[3];
  if (!unit_normal(c, plane, i, G, np) || !unit_normal(c, plane, j, G, nq)) return none;
  if (!(dot3(np, nq) > 0.0)) return none;
  double m[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = __dadd_rn(np[k], nq[k]);
  const double len = __dsqrt_rn(dot3(m, m));
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = __ddiv_rn(m[k], len);
  const double rp[3] = {ray_x(x, G), ray_y(y, G), 1.0};
  const double rq[3] = {ray_x(x + dx, G), ray_y(y + dy, G), 1.0};
  return make_double2(dot3(m, rp), dot3(m, rq));
}

// Slab partials [b][slab][8] = (min a, max a, |V|, S a) over V.  grid (slabs, b)
__global__ void __launch_bounds__(kFusThreads) fusion_range_kernel(const float* __restrict__ a, const void* mask,
                                                                   int kind, long long hw, double* __restrict__ part) {
  __shared__ double scratch[32];
  const long long base = (long long)blockIdx.y * hw;
  double lo = INFINITY, hi = -INFINITY, n = 0.0, s = 0.0;
  for (int k = 0; k < kSlab / kFusThreads; ++k) {
    const long long i = blockIdx.x * kSlab + k * kFusThreads + threadIdx.x;
    if (i >= hw || !in_v(a, mask, kind, base + i)) continue;
    const double v = a[base + i];
    lo = fmin(lo, v);
    hi = fmax(hi, v);
    n += 1.0;
    s += v;
  }
  double* out = part + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * kPartStride;
  const double r0 = block_min_d(lo, scratch);
  if (threadIdx.x == 0) out[0] = r0;
  const double r1 = block_max_d(hi, scratch);
  if (threadIdx.x == 0) out[1] = r1;
  const double r2 = block_sum_d(n, scratch);
  if (threadIdx.x == 0) out[2] = r2;
  const double r3 = block_sum_d(s, scratch);
  if (threadIdx.x == 0) out[3] = r3;
}

// Writes the CTA's kq partial sums (fixed-order block sums) and takes the image's ticket; true in every thread of the
// image's last CTA, which then sees every partial of the image (read with ld.cg).
template <int kq>
ODB_DEVINL bool tile_partials_last(const double (&acc)[kq], double* part, unsigned int* ticket, double* scratch) {
  __shared__ bool last;
  const int b = blockIdx.y;
  double* out = part + ((long long)b * gridDim.x + blockIdx.x) * kTilePart;
#pragma unroll
  for (int k = 0; k < kq; ++k) {
    const double v = block_sum_d(acc[k], scratch);
    if (threadIdx.x == 0) out[k] = v;
  }
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(ticket + b, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last) __threadfence();
  return last;
}

// In the last CTA: the image's sum of partial k over its tiles, in tile order, returned to threads < 32 (column k)
ODB_DEVINL double fold_tiles(const double* part, int kq) {
  const int b = blockIdx.y, col = threadIdx.x & 31;
  const double* p = part + (long long)b * gridDim.x * kTilePart;
  return ordered_sum8(gridDim.x, col < kq, [&](int t) { return __ldcg(p + (long long)t * kTilePart + col); });
}

ODB_DEVINL void tile_origin(const FusGeom& G, int& x0, int& y0) {
  const int t = blockIdx.x, ty = t / G.tiles_x;
  x0 = (t - ty * G.tiles_x) * kTW;
  y0 = ty * kTH;
}

// Per pixel: the coefficients of its right and down edges (0 when dropped).  grid (tiles, b)
__global__ void __launch_bounds__(kFusThreads) fusion_edges_kernel(const float* __restrict__ a,
                                                                   const float* __restrict__ c, const void* mask,
                                                                   int kind, FusGeom G, FusWs W) {
  const int b = blockIdx.y;
  const double* info = W.info + (long long)b * kPartStride;
  const double thr = __dmul_rn(G.jump, __dsub_rn(info[kMax], info[kMin]));
  const long long plane = (long long)G.h * G.w, pb = (long long)b * plane;
  const float* ab = a + pb;
  const float* cb = c + 3 * pb;
  const void* mb = mask == nullptr ? nullptr
                   : kind == ODB_MASK_U8 ? (const void*)(static_cast<const uint8_t*>(mask) + pb)
                                         : (const void*)(static_cast<const float*>(mask) + pb);
  int x0, y0;
  tile_origin(G, x0, y0);
  const int x = x0 + threadIdx.x % kTW;
#pragma unroll 1
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = y0 + threadIdx.x / kTW + k * (kFusThreads / kTW);
    if (x >= G.w || y >= G.h) continue;
    const long long i = (long long)y * G.w + x;
    W.cr[pb + i] = x + 1 < G.w ? edge_coef(ab, cb, mb, kind, plane, i, i + 1, x, y, 1, 0, thr, G)
                               : make_double2(0.0, 0.0);
    W.cd[pb + i] = y + 1 < G.h ? edge_coef(ab, cb, mb, kind, plane, i, i + G.w, x, y, 0, 1, thr, G)
                               : make_double2(0.0, 0.0);
  }
}

ODB_DEVINL bool kept(double2 e) { return e.x != 0.0 || e.y != 0.0; }

// Per pixel: D^-1, x0 = a, r0 = -N a, z0 = D^-1 r0 (all 0 off V).  Partials (kept edges, r.z, r.r, b.b); the last CTA
// sets the status (1: V empty, 2: a constant on V, else 3 until converged), the scalars and the done flag.
__global__ void __launch_bounds__(kFusThreads) fusion_setup_kernel(const float* __restrict__ a, const void* mask,
                                                                   int kind, FusGeom G, double tol, FusWs W) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const double* info = W.info + (long long)b * kPartStride;
  const double nv = info[kN], denom = __dmul_rn(nv, 1.0 + kKappa);
  const double sa = G.shift ? __ddiv_rn(info[kSumA], denom) : 0.0;
  const double diag0 = G.shift ? __dmul_rn(G.lam, __dsub_rn(1.0, __drcp_rn(denom))) : G.lam;
  const long long pb = (long long)b * G.h * G.w;
  int x0, y0;
  tile_origin(G, x0, y0);
  const int x = x0 + threadIdx.x % kTW;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = y0 + threadIdx.x / kTW + k * (kFusThreads / kTW);
    if (x >= G.w || y >= G.h) continue;
    const long long i = pb + (long long)y * G.w + x;
    const double2 R = W.cr[i], D = W.cd[i];
    acc[0] += (kept(R) ? 1.0 : 0.0) + (kept(D) ? 1.0 : 0.0);
    double dinv = 0.0, xv = 0.0, rv = 0.0, zv = 0.0;
    if (in_v(a, mask, kind, i)) {
      const double2 L = x > 0 ? W.cr[i - 1] : make_double2(0.0, 0.0);
      const double2 U = y > 0 ? W.cd[i - G.w] : make_double2(0.0, 0.0);
      const double av = a[i];
      double na = 0.0;                            // (N a)_p over the kept edges (their far ends are in V)
      if (kept(R)) na += R.x * (R.x * av - R.y * (double)a[i + 1]);
      if (kept(D)) na += D.x * (D.x * av - D.y * (double)a[i + G.w]);
      if (kept(L)) na += L.y * (L.y * av - L.x * (double)a[i - 1]);
      if (kept(U)) na += U.y * (U.y * av - U.x * (double)a[i - G.w]);
      dinv = 1.0 / (diag0 + R.x * R.x + D.x * D.x + L.y * L.y + U.y * U.y);
      xv = av;
      rv = -na;
      zv = dinv * rv;
      const double bv = G.lam * (av - sa);
      acc[1] += rv * zv;
      acc[2] += rv * rv;
      acc[3] += bv * bv;
    }
    W.dinv[i] = dinv;
    W.x[i] = xv;
    W.r[i] = rv;
    W.z[i] = zv;
  }
  if (!tile_partials_last<4>(acc, W.part, W.ticket, scratch)) return;
  const double s = fold_tiles(W.part, 4);
  __shared__ double tot[4];
  if (threadIdx.x < 4) tot[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double* in = W.info + (long long)b * kPartStride;
    double* S = W.scal + (long long)b * 8;
    const int status = nv == 0.0 ? 1 : !(in[kMax] > in[kMin]) ? 2 : 3;
    in[kStatus] = status;
    in[kKept] = tot[0];
    S[kRho] = tot[1];
    S[kRR] = tot[2];
    S[kBB] = tot[3];
    S[kAlpha] = S[kBeta] = S[kLamSp] = S[kIters] = 0.0;
    bool done = status != 3;
    if (!done && sqrt(tot[2]) <= tol * sqrt(tot[3])) {
      in[kStatus] = 0;
      done = true;
    }
    S[kDone] = done ? 1.0 : 0.0;
    W.ticket[b] = 0;
  }
}

// p = z + beta p_old (p = z on the first iteration) over the tile and its one-pixel halo in shared memory; writes p and
// q = lambda p + N p over the tile.  Partials (p.p, S p, p.N p); the last CTA: alpha = rho / p.M p.
__global__ void __launch_bounds__(kFusThreads) fusion_matvec_kernel(FusGeom G, int first, const double* __restrict__ p_old,
                                                                    double* __restrict__ p_new, FusWs W) {
  __shared__ double P[kTH + 2][kTW + 2];
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  double* S = W.scal + (long long)b * 8;
  if (S[kDone] != 0.0) return;
  const double beta = S[kBeta];
  const long long pb = (long long)b * G.h * G.w;
  int x0, y0;
  tile_origin(G, x0, y0);
  for (int e = threadIdx.x; e < (kTH + 2) * (kTW + 2); e += kFusThreads) {
    const int ly = e / (kTW + 2), lx = e - ly * (kTW + 2);
    const int y = y0 + ly - 1, x = x0 + lx - 1;
    double v = 0.0;
    if (x >= 0 && x < G.w && y >= 0 && y < G.h) {
      const long long i = pb + (long long)y * G.w + x;
      v = first ? W.z[i] : W.z[i] + beta * p_old[i];
    }
    P[ly][lx] = v;
  }
  __syncthreads();
  const int lx = threadIdx.x % kTW, x = x0 + lx;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int ly = threadIdx.x / kTW + k * (kFusThreads / kTW), y = y0 + ly;
    if (x >= G.w || y >= G.h) continue;
    const long long i = pb + (long long)y * G.w + x;
    const double pc = P[ly + 1][lx + 1];
    const double2 R = W.cr[i], D = W.cd[i];
    const double2 L = x > 0 ? W.cr[i - 1] : make_double2(0, 0);
    const double2 U = y > 0 ? W.cd[i - G.w] : make_double2(0, 0);
    const double np = R.x * (R.x * pc - R.y * P[ly + 1][lx + 2]) + D.x * (D.x * pc - D.y * P[ly + 2][lx + 1]) +
                      L.y * (L.y * pc - L.x * P[ly + 1][lx]) + U.y * (U.y * pc - U.x * P[ly][lx + 1]);
    p_new[i] = pc;
    W.q[i] = G.lam * pc + np;
    acc[0] += pc * pc;
    acc[1] += pc;
    acc[2] += pc * np;
  }
  if (!tile_partials_last<3>(acc, W.part, W.ticket, scratch)) return;
  const double s = fold_tiles(W.part, 3);
  __shared__ double tot[3];
  if (threadIdx.x < 3) tot[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    const double denom = W.info[(long long)b * kPartStride + kN] * (1.0 + kKappa);
    const double pmp = G.shift ? G.lam * (tot[0] - tot[1] * tot[1] / denom) + tot[2] : G.lam * tot[0] + tot[2];
    S[kAlpha] = S[kRho] / pmp;
    S[kLamSp] = G.shift ? G.lam * tot[1] / denom : 0.0;
    if (!(pmp > 0.0)) S[kDone] = 1.0;              // p = 0 or lost definiteness: stop (status stays 3)
    W.ticket[b] = 0;
  }
}

// x += alpha p, r -= alpha (q - lambda s(p)), z = D^-1 r on V.  Partials (r.z, r.r); the last CTA: beta, the iteration
// count and the stopping rule |r| <= tol |b|.
__global__ void __launch_bounds__(kFusThreads) fusion_update_kernel(FusGeom G, const double* __restrict__ p,
                                                                    double tol, FusWs W) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  double* S = W.scal + (long long)b * 8;
  if (S[kDone] != 0.0) return;
  const double alpha = S[kAlpha], lsp = S[kLamSp];
  const long long pb = (long long)b * G.h * G.w;
  int x0, y0;
  tile_origin(G, x0, y0);
  const int x = x0 + threadIdx.x % kTW;
  double acc[2] = {0.0, 0.0};
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = y0 + threadIdx.x / kTW + k * (kFusThreads / kTW);
    if (x >= G.w || y >= G.h) continue;
    const long long i = pb + (long long)y * G.w + x;
    const double dinv = W.dinv[i];
    if (dinv == 0.0) continue;
    W.x[i] += alpha * p[i];
    const double r = W.r[i] - alpha * (W.q[i] - lsp);
    const double z = dinv * r;
    W.r[i] = r;
    W.z[i] = z;
    acc[0] += r * z;
    acc[1] += r * r;
  }
  if (!tile_partials_last<2>(acc, W.part, W.ticket, scratch)) return;
  const double s = fold_tiles(W.part, 2);
  __shared__ double tot[2];
  if (threadIdx.x < 2) tot[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    S[kBeta] = tot[0] / S[kRho];
    S[kRho] = tot[0];
    S[kRR] = tot[1];
    S[kIters] += 1.0;
    if (sqrt(tot[1]) <= tol * sqrt(S[kBB])) {
      S[kDone] = 1.0;
      W.info[(long long)b * kPartStride + kStatus] = 0.0;
    }
    W.ticket[b] = 0;
  }
}

// S_V (x - a); the last CTA: t = that / (|V| (1 + kappa)) with shift, else 0 (NaN for status 1 and 2)
__global__ void __launch_bounds__(kFusThreads) fusion_shift_kernel(const float* __restrict__ a, FusGeom G, FusWs W) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const long long pb = (long long)b * G.h * G.w;
  int x0, y0;
  tile_origin(G, x0, y0);
  const int x = x0 + threadIdx.x % kTW;
  double acc[1] = {0.0};
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = y0 + threadIdx.x / kTW + k * (kFusThreads / kTW);
    if (x >= G.w || y >= G.h) continue;
    const long long i = pb + (long long)y * G.w + x;
    if (W.dinv[i] != 0.0) acc[0] += W.x[i] - (double)a[i];
  }
  if (!tile_partials_last<1>(acc, W.part, W.ticket, scratch)) return;
  const double s = fold_tiles(W.part, 1);
  if (threadIdx.x == 0) {
    double* in = W.info + (long long)b * kPartStride;
    const int status = (int)in[kStatus];
    in[kShift] = status == 1 || status == 2 ? NAN : G.shift ? s / (in[kN] * (1.0 + kKappa)) : 0.0;
    W.ticket[b] = 0;
  }
}

// out = x rounded to fp32 on V, NaN off V and for status 1 / 2.  S_V (x - a - t)^2; the last CTA writes the record
// (|V|, status, kept edges, iterations, |r| / |b|, t, RMS over V of z - a - t, 0).
__global__ void __launch_bounds__(kFusThreads) fusion_apply_kernel(const float* __restrict__ a, FusGeom G, FusWs W,
                                                                   float* __restrict__ out,
                                                                   double* __restrict__ records) {
  __shared__ double scratch[32];
  const int b = blockIdx.y;
  const double* in = W.info + (long long)b * kPartStride;
  const int status = (int)in[kStatus];
  const bool solved = status == 0 || status == 3;
  const double t = in[kShift];
  const long long pb = (long long)b * G.h * G.w;
  int x0, y0;
  tile_origin(G, x0, y0);
  const int x = x0 + threadIdx.x % kTW;
  double acc[1] = {0.0};
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = y0 + threadIdx.x / kTW + k * (kFusThreads / kTW);
    if (x >= G.w || y >= G.h) continue;
    const long long i = pb + (long long)y * G.w + x;
    float o = NAN;
    if (solved && W.dinv[i] != 0.0) {
      const double xv = W.x[i], e = xv - (double)a[i] - t;
      o = (float)xv;
      acc[0] += e * e;
    }
    out[i] = o;
  }
  if (!tile_partials_last<1>(acc, W.part, W.ticket, scratch)) return;
  const double s = fold_tiles(W.part, 1);
  if (threadIdx.x == 0) {
    const double* S = W.scal + (long long)b * 8;
    double* rec = records + (long long)b * ODB_FUSION_RECORD;
    rec[0] = in[kN];
    rec[1] = status;
    rec[2] = in[kKept];
    rec[3] = S[kIters];
    rec[4] = solved ? sqrt(S[kRR]) / sqrt(S[kBB]) : NAN;
    rec[5] = t;
    rec[6] = solved ? sqrt(s / in[kN]) : NAN;
    rec[7] = 0.0;
    W.ticket[b] = 0;
  }
}

// X = z r, component k, at pixel (x, y)
ODB_DEVINL void back_project(double z, int x, int y, const FusGeom& G, double X[3]) {
  X[0] = __dmul_rn(z, ray_x(x, G));
  X[1] = __dmul_rn(z, ray_y(y, G));
  X[2] = z;
}

// The tangent along one axis at p from its neighbours m (before) and n (after): central difference X_n - X_m with
// both edges kept, else the one-sided difference over the kept edge; false with neither.
ODB_DEVINL bool tangent(bool km, bool kn, const double Xm[3], const double Xp[3], const double Xn[3], double t[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = __dsub_rn(kn ? Xn[k] : Xp[k], km ? Xm[k] : Xp[k]);
  return km || kn;
}

// V and a at (x, y) (absolute index within the batch)
ODB_DEVINL bool valid_at(const float* a, const void* mask, int kind, long long pb, int x, int y, const FusGeom& G,
                         double& v) {
  if (x < 0 || x >= G.w || y < 0 || y >= G.h) return false;
  const long long i = pb + (long long)y * G.w + x;
  if (!in_v(a, mask, kind, i)) return false;
  v = a[i];
  return true;
}

// The encoded normal of the depth map at (x, y): NaN off V or where a tangent is missing
ODB_DEVINL float3 normal_at(const float* a, const void* mask, int kind, long long pb, int x, int y, double thr,
                            const FusGeom& G) {
  const float3 none = make_float3(NAN, NAN, NAN);
  double ap, al = 0, ar = 0, au = 0, ad = 0;
  if (!valid_at(a, mask, kind, pb, x, y, G, ap)) return none;
  const bool kl = valid_at(a, mask, kind, pb, x - 1, y, G, al) && fabs(__dsub_rn(ap, al)) <= thr;
  const bool kr = valid_at(a, mask, kind, pb, x + 1, y, G, ar) && fabs(__dsub_rn(ar, ap)) <= thr;
  const bool ku = valid_at(a, mask, kind, pb, x, y - 1, G, au) && fabs(__dsub_rn(ap, au)) <= thr;
  const bool kd = valid_at(a, mask, kind, pb, x, y + 1, G, ad) && fabs(__dsub_rn(ad, ap)) <= thr;
  double Xp[3], Xl[3], Xr[3], Xu[3], Xd[3], tx[3], ty[3];
  back_project(ap, x, y, G, Xp);
  back_project(al, x - 1, y, G, Xl);
  back_project(ar, x + 1, y, G, Xr);
  back_project(au, x, y - 1, G, Xu);
  back_project(ad, x, y + 1, G, Xd);
  if (!tangent(kl, kr, Xl, Xp, Xr, tx) || !tangent(ku, kd, Xu, Xp, Xd, ty)) return none;
  double n[3] = {__dsub_rn(__dmul_rn(ty[1], tx[2]), __dmul_rn(ty[2], tx[1])),
                 __dsub_rn(__dmul_rn(ty[2], tx[0]), __dmul_rn(ty[0], tx[2])),
                 __dsub_rn(__dmul_rn(ty[0], tx[1]), __dmul_rn(ty[1], tx[0]))};
  const double len = __dsqrt_rn(dot3(n, n));
#pragma unroll
  for (int k = 0; k < 3; ++k) n[k] = __ddiv_rn(n[k], len);
  const double sg = dot3(n, Xp) > 0.0 ? -1.0 : 1.0;
  return make_float3((float)__dmul_rn(__dadd_rn(G.ax * (sg * n[0]), 1.0), 0.5),
                     (float)__dmul_rn(__dadd_rn(G.ay * (sg * n[1]), 1.0), 0.5),
                     (float)__dmul_rn(__dadd_rn(G.az * (sg * n[2]), 1.0), 0.5));
}

// out fp32 [b][3][h][w]: the normals of the depth map, in the model's encoding (axes n + 1) / 2; NaN where p is not in
// V or a tangent is missing.  Each thread writes 4 consecutive pixels of a row (16-byte stores when `vec`).
// grid (ceil(ceil(w / 4) / 64), h, b)
__global__ void __launch_bounds__(kFusThreads / 4) depth_normals_kernel(const float* __restrict__ a, const void* mask,
                                                                        int kind, FusGeom G,
                                                                        const double* __restrict__ info, int vec,
                                                                        float* __restrict__ out) {
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y, b = blockIdx.z;
  if (x0 >= G.w) return;
  const long long plane = (long long)G.h * G.w, pb = (long long)b * plane;
  const double* in = info + (long long)b * kPartStride;
  const double thr = __dmul_rn(G.jump, __dsub_rn(in[kMax], in[kMin]));
  float3 o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = normal_at(a, mask, kind, pb, min(x0 + j, G.w - 1), y, thr, G);
  float* row = out + (long long)b * 3 * plane + (long long)y * G.w + x0;
  if (vec) {
    *reinterpret_cast<float4*>(row) = make_float4(o[0].x, o[1].x, o[2].x, o[3].x);
    *reinterpret_cast<float4*>(row + plane) = make_float4(o[0].y, o[1].y, o[2].y, o[3].y);
    *reinterpret_cast<float4*>(row + 2 * plane) = make_float4(o[0].z, o[1].z, o[2].z, o[3].z);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (x0 + j >= G.w) break;
      row[j] = o[j].x;
      row[j + plane] = o[j].y;
      row[j + 2 * plane] = o[j].z;
    }
  }
}

static bool fusion_geom(int32_t h, int32_t w, double fx, double fy, double cx, double cy, int32_t ax, int32_t ay,
                        int32_t az, double jump, FusGeom& G) {
  if (!(std::isfinite(fx) && fx > 0.0 && std::isfinite(fy) && fy > 0.0 && std::isfinite(cx) && std::isfinite(cy)))
    return false;
  for (int32_t s : {ax, ay, az})
    if (s != 1 && s != -1) return false;
  if (!(std::isfinite(jump) && jump > 0.0)) return false;
  G.h = h;
  G.w = w;
  G.tiles_x = (w + kTW - 1) / kTW;
  G.tiles = fus_tiles(h, w);
  G.fx = fx; G.fy = fy; G.cx = cx; G.cy = cy;
  G.ax = ax; G.ay = ay; G.az = az;
  G.jump = jump;
  G.lam = 0.0;
  G.shift = 0;
  return true;
}

static void launch_range(const float* a, const void* mask, int32_t kind, int b, int h, int w, const FusWs& W,
                         cudaStream_t stream) {
  const int slabs = slab_count(h, w);
  fusion_range_kernel<<<dim3(slabs, b), kFusThreads, 0, stream>>>(a, mask, kind, (long long)h * w, W.slab);
  count_launch();
  launch_slab_reduce(W.slab, b, slabs, 4, 1u << kMin, 1u << kMax, W.info, stream);
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_fusion_workspace_bytes(int32_t b, int32_t h, int32_t w) {
  if (!planes_ok(b, h, w)) return -1;
  return (fus_head_doubles(b, h, w) + 2 + 11 * (int64_t)b * h * w) * (int64_t)sizeof(double);
}

extern "C" int64_t odb_depth_normals_workspace_bytes(int32_t b, int32_t h, int32_t w) {
  if (!planes_ok(b, h, w)) return -1;
  return fus_head_doubles(b, h, w) * (int64_t)sizeof(double);
}

extern "C" int odb_depth_normal_fusion(const float* depth, const float* normals, const void* mask, int32_t mask_dtype,
                                       int32_t b, int32_t h, int32_t w, double fx, double fy, double cx, double cy,
                                       int32_t axis_x, int32_t axis_y, int32_t axis_z, double jump, double weight,
                                       int32_t shift, int32_t iterations, double tol, void* workspace, float* out,
                                       double* records, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FusGeom G;
  if (!depth || !normals || !workspace || !out || !records || !planes_ok(b, h, w) ||
      !metric_mask_ok(mask, mask_dtype) || !aligned(depth, 4) || !aligned(normals, 4) || !aligned(workspace, 16) ||
      !aligned(out, 4) || !aligned(records, 8) ||
      !fusion_geom(h, w, fx, fy, cx, cy, axis_x, axis_y, axis_z, jump, G) || !(std::isfinite(weight) && weight > 0.0) ||
      (shift != 0 && shift != 1) || iterations < 1 || iterations > 10000 || !(std::isfinite(tol) && tol > 0.0))
    return fail(ODB_ERR_INVALID, "depth_normal_fusion: bad argument");
  G.lam = weight;
  G.shift = shift;
  const FusWs W = fus_ws(workspace, b, h, w, true);
  cudaError_t e = cudaMemsetAsync(W.ticket, 0, (size_t)b * sizeof(double), stream);
  if (e != cudaSuccess) return fail_cuda(e, "depth_normal_fusion: cudaMemsetAsync");
  launch_range(depth, mask, mask_dtype, b, h, w, W, stream);
  const dim3 grid(G.tiles, b);
  fusion_edges_kernel<<<grid, kFusThreads, 0, stream>>>(depth, normals, mask, mask_dtype, G, W);
  count_launch();
  fusion_setup_kernel<<<grid, kFusThreads, 0, stream>>>(depth, mask, mask_dtype, G, tol, W);
  count_launch();
  for (int it = 0; it < iterations; ++it) {
    fusion_matvec_kernel<<<grid, kFusThreads, 0, stream>>>(G, it == 0 ? 1 : 0, W.p[it & 1], W.p[(it + 1) & 1], W);
    count_launch();
    fusion_update_kernel<<<grid, kFusThreads, 0, stream>>>(G, W.p[(it + 1) & 1], tol, W);
    count_launch();
  }
  fusion_shift_kernel<<<grid, kFusThreads, 0, stream>>>(depth, G, W);
  count_launch();
  fusion_apply_kernel<<<grid, kFusThreads, 0, stream>>>(depth, G, W, out, records);
  count_launch();
  return check_launch("depth_normal_fusion");
}

extern "C" int odb_depth_normals(const float* depth, const void* mask, int32_t mask_dtype, int32_t b, int32_t h,
                                 int32_t w, double fx, double fy, double cx, double cy, int32_t axis_x, int32_t axis_y,
                                 int32_t axis_z, double jump, void* workspace, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FusGeom G;
  if (!depth || !workspace || !out || !planes_ok(b, h, w) || !metric_mask_ok(mask, mask_dtype) || !aligned(depth, 4) ||
      !aligned(workspace, 8) || !aligned(out, 4) || !fusion_geom(h, w, fx, fy, cx, cy, axis_x, axis_y, axis_z, jump, G))
    return fail(ODB_ERR_INVALID, "depth_normals: bad argument");
  const FusWs W = fus_ws(workspace, b, h, w, false);
  launch_range(depth, mask, mask_dtype, b, h, w, W, stream);
  const int vec = w % 4 == 0 && aligned(out, 16) ? 1 : 0;
  const int quads = (w + 3) / 4, per = kFusThreads / 4;
  depth_normals_kernel<<<dim3((quads + per - 1) / per, h, b), per, 0, stream>>>(depth, mask, mask_dtype, G, W.info,
                                                                                vec, out);
  count_launch();
  return check_launch("depth_normals");
}
