// SE(3) pose-graph optimisation (omnidata_b200/posegraph.py PoseGraph): Gauss-Newton over N camera-to-world poses with
// relative-pose edges, node 0 fixed.  Definition in DESIGN.md §3 "Loop closure and pose graphs" and
// include/omnidata_b200.h; oracle/posegraph_oracle.py restates it in float64.
//
//   pg_setup_kernel      one CTA: the incidence lists (each node's edges in ascending edge id, built in a fixed order
//                        from the device edge list), the working poses and the state
//   per Gauss-Newton iteration:
//   pg_edge_kernel       one thread per edge: the residual r = Log(Z^-1 Ti^-1 Tj), J_i = -Ad(Tj^-1 Ti), J_j = I and the
//                        edge's blocks Ji^T W Ji, Ji^T W Jj (Jj^T W Jj = W is the input), gradient pieces and flags
//   pg_node_kernel       one thread per free unknown: its diagonal and gradient entries gathered over the node's
//                        incidence list, the unit-diagonal scale and the right-hand side -g / scale
//   pg_fill_kernel       one CTA per 64 x 64 tile of the lower triangle of the dense scaled H: every entry gathered over
//                        the incidence list of its row's node (zero where no edge joins the two nodes).  No scatter, no
//                        atomics
//   per 64-wide panel of the blocked right-looking Cholesky (the forward substitution rides along):
//   pg_factor_kernel     one CTA: factors the diagonal block, checks the pivots, solves L11 y = b for the panel (panel
//                        0 first reduces the edge and node flags to the status)
//   pg_trsm_kernel       one CTA per 32 rows below the panel: L21 = A21 L11^-T, and b -= L21 y for those rows
//   pg_trailing_kernel   one CTA per 64 x 64 tile of the trailing lower triangle: C -= L21_i L21_j^T as fp64 FMAs in a
//                        fixed k order
//   per panel, last to first:
//   pg_backsub_kernel    one CTA per 64-row tile below the panel: L^T x partials; the last CTA (integer ticket) folds
//                        them in tile order and solves L11^T x = y - s for the panel
//   pg_update_kernel     one CTA: delta = x / scale, T_k <- T_k exp(delta_k), the stop rule
//   pg_output_kernel     one CTA: poses (the input poses, bit for bit, unless the status is ok), costs and the record
//
// The panel solve below the diagonal block runs on many CTAs rather than the factoring CTA: one CTA would walk up to
// 6138 rows x 64 columns serially per panel.  A stopped solve's later launches return after reading the done flag, so
// the launch sequence is fixed for (N, E, iterations) and a call can be captured in a CUDA graph.  No floating-point
// atomics; built without fast-math; bit-reproducible.
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "se3.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kPgThreads = 256;
constexpr int kPanel = 64;                        // Cholesky panel and tile width
constexpr int kTrsmRows = 32;                     // rows per CTA of the panel solve
constexpr int kPad = kPanel + 1;
constexpr double kPgPivotMin = 1e-12;             // smallest pivot of the unit-diagonal matrix (not tuned)
constexpr double kHalfPi = 1.5707963267948966;
constexpr int kPgOk = 0, kPgDegenerate = 1, kPgNonfinite = 2;
// state doubles
constexpr int kPgDone = 0, kPgStatus = 1, kPgIters = 2, kPgMaxDelta = 3, kPgState = 8;
// per-edge doubles: Ji^T W Ji (36), Ji^T W Jj (36), Ji^T W r (6), W r (6), r^T W r, flag
constexpr int kEHii = 0, kEHij = 36, kEGi = 72, kEGj = 78, kECost = 84, kEFlag = 85, kEdge = 86;

struct PgArgs {
  int N, E, n, panels;
  double tol;
  const int* edges;                               // [E][2]
  const double* poses;                            // [N][16] the input
  const double* meas;                             // [E][16]
  const double* info;                             // [E][36]
  double* st;                                     // state
  double* T;                                      // [N][12] working poses (R row-major, t)
  double* eb;                                     // [E][kEdge]
  double* scale;                                  // [n]
  double* rhs;                                    // [n]: -g / scale, then y, then x
  double* nflag;                                  // [n]
  double* part;                                   // [panels][kPanel]
  double* H;                                      // [n][n] row-major, lower triangle
  unsigned int* ticket;
  int* inc_off;                                   // [N + 1]
  int* inc;                                       // [2E]: 2 e + side (0: the node is i, 1: it is j)
};

static int pg_panels(int n) { return (n + kPanel - 1) / kPanel; }

ODB_DEVINL void load_pose16(const double* P, double* T) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) T[3 * r + c] = P[4 * r + c];
    T[9 + r] = P[4 * r + 3];
  }
}

ODB_DEVINL bool edge_ok(const int* edges, int e, int N, int& i, int& j) {
  i = edges[2 * e];
  j = edges[2 * e + 1];
  return i >= 0 && i < N && j >= 0 && j < N && i != j;
}

// r = Log(Z^-1 Ti^-1 Tj) in (v, omega) order, and D = Ti^-1 Tj.  SO(3): w = vee(R - R^T) / 2, theta = atan2(|w|,
// (tr R - 1) / 2), omega = (theta / |w|) w (|w| = sin theta); SE(3): v = V^-1 u, V^-1 = I - W / 2 + c W^2, c = (1 -
// A / (2 B)) / theta^2 with se3_exp's A, B; below kSeriesTheta theta / |w| = 1 + theta^2 / 6 + 7 theta^4 / 360 and
// c = 1 / 12 + theta^2 / 720 + theta^4 / 30240.  Returns theta.
ODB_DEVINL double edge_residual(const double* Ti, const double* Tj, const double* Zp, double r[6], double D[12]) {
  double Z[12], M[12];
  load_pose16(Zp, Z);
  relative_pose(Ti, Tj, D);
  relative_pose(Z, D, M);
  const double w[3] = {__dmul_rn(0.5, __dsub_rn(M[7], M[5])), __dmul_rn(0.5, __dsub_rn(M[2], M[6])),
                       __dmul_rn(0.5, __dsub_rn(M[3], M[1]))};
  const double s = __dsqrt_rn(dot3_rn(w, w));
  const double cth = __dmul_rn(0.5, __dsub_rn(__dadd_rn(__dadd_rn(M[0], M[4]), M[8]), 1.0));
  const double th = atan2(s, cth), th2 = __dmul_rn(th, th);
  double f, c;
  if (th < kSeriesTheta) {
    const double th4 = __dmul_rn(th2, th2);
    f = __dadd_rn(__dadd_rn(1.0, __ddiv_rn(th2, 6.0)), __ddiv_rn(__dmul_rn(7.0, th4), 360.0));
    c = __dadd_rn(__dadd_rn(1.0 / 12.0, __ddiv_rn(th2, 720.0)), __ddiv_rn(th4, 30240.0));
  } else {
    double A, B;
    se3_coefficients(th2, th, A, B, nullptr);
    f = __ddiv_rn(th, s);
    c = __ddiv_rn(__dsub_rn(1.0, __ddiv_rn(A, __dmul_rn(2.0, B))), th2);
  }
  const double om[3] = {__dmul_rn(f, w[0]), __dmul_rn(f, w[1]), __dmul_rn(f, w[2])};
  const double o2 = dot3_rn(om, om);
  const double W[9] = {0.0, -om[2], om[1], om[2], 0.0, -om[0], -om[1], om[0], 0.0};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double Vi[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double w2 = i == j ? __dsub_rn(__dmul_rn(om[i], om[j]), o2) : __dmul_rn(om[i], om[j]);
      const double id = i == j ? 1.0 : 0.0;
      Vi[j] = __dadd_rn(__dsub_rn(id, __dmul_rn(0.5, W[3 * i + j])), __dmul_rn(c, w2));
    }
    r[i] = dot3_rn(Vi, M + 9);
    r[3 + i] = om[i];
  }
  return th;
}

// r^T W r, W row-major 6 x 6: sum over rows p of r_p (sum over q of W_pq r_q), in order
ODB_DEVINL double quad6(const double* W, const double r[6], double Wr[6]) {
  double cost = 0.0;
#pragma unroll
  for (int p = 0; p < 6; ++p) {
    double a = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) a = __dadd_rn(a, __dmul_rn(__ldg(W + 6 * p + q), r[q]));
    Wr[p] = a;
    cost = __dadd_rn(cost, __dmul_rn(r[p], a));
  }
  return cost;
}

__global__ void __launch_bounds__(1024) pg_setup_kernel(PgArgs A) {
  __shared__ int cnt[1024];
  const int k = threadIdx.x;
  int c = 0;
  if (k < A.N)
    for (int e = 0; e < A.E; ++e) {
      int i, j;
      if (edge_ok(A.edges, e, A.N, i, j)) c += (i == k) + (j == k);
    }
  cnt[k] = c;
  __syncthreads();
  if (k == 0) {
    int s = 0;
    for (int q = 0; q < A.N; ++q) {
      A.inc_off[q] = s;
      s += cnt[q];
    }
    A.inc_off[A.N] = s;
    for (int q = 0; q < kPgState; ++q) A.st[q] = 0.0;
    *A.ticket = 0u;
  }
  __syncthreads();
  if (k < A.N) {
    int pos = A.inc_off[k];
    for (int e = 0; e < A.E; ++e) {
      int i, j;
      if (!edge_ok(A.edges, e, A.N, i, j)) continue;
      if (i == k) A.inc[pos++] = 2 * e;
      if (j == k) A.inc[pos++] = 2 * e + 1;
    }
    double T[12];
    load_pose16(A.poses + 16 * k, T);
#pragma unroll
    for (int q = 0; q < 12; ++q) A.T[12 * k + q] = T[q];
  }
}

__global__ void __launch_bounds__(128) pg_edge_kernel(PgArgs A) {
  if (A.st[kPgDone] != 0.0) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) A.st[kPgIters] += 1.0;
  const int e = blockIdx.x * 128 + threadIdx.x;
  if (e >= A.E) return;
  double* out = A.eb + (long long)e * kEdge;
  int i, j;
  if (!edge_ok(A.edges, e, A.N, i, j)) {
    for (int q = 0; q < kEdge; ++q) out[q] = 0.0;
    return;
  }
  double Ti[12], Tj[12], r[6], D[12];
#pragma unroll
  for (int q = 0; q < 12; ++q) {
    Ti[q] = A.T[12 * i + q];
    Tj[q] = A.T[12 * j + q];
  }
  const double th = edge_residual(Ti, Tj, A.meas + 16LL * e, r, D);
  const double* W = A.info + 36LL * e;
  double Wr[6];
  const double cost = quad6(W, r, Wr);
  // Ad(D^-1) = [[Ra, [ta]x Ra], [0, Ra]] with Ra = RD^T, ta = -RD^T tD
  double Ra[9], ta[3], S[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) Ra[3 * a + b] = D[3 * b + a];
#pragma unroll
  for (int a = 0; a < 3; ++a) ta[a] = -dot3_rn(Ra + 3 * a, D + 9);
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    S[b] = __dsub_rn(__dmul_rn(ta[1], Ra[6 + b]), __dmul_rn(ta[2], Ra[3 + b]));
    S[3 + b] = __dsub_rn(__dmul_rn(ta[2], Ra[b]), __dmul_rn(ta[0], Ra[6 + b]));
    S[6 + b] = __dsub_rn(__dmul_rn(ta[0], Ra[3 + b]), __dmul_rn(ta[1], Ra[b]));
  }
  // Ad[m][q]: rows 0..2 = [Ra S], rows 3..5 = [0 Ra]
  auto ad = [&](int m, int q) -> double {
    if (m < 3) return q < 3 ? Ra[3 * m + q] : S[3 * m + q - 3];
    return q < 3 ? 0.0 : Ra[3 * (m - 3) + q - 3];
  };
  // B = W Ad; Ji^T W Jj = -Ad^T W = -B^T; Ji^T W Ji = Ad^T B; Ji^T W r = -Ad^T W r
  double B[36];
#pragma unroll
  for (int p = 0; p < 6; ++p)
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      double a = 0.0;
#pragma unroll
      for (int m = 0; m < 6; ++m) a = __dadd_rn(a, __dmul_rn(__ldg(W + 6 * p + m), ad(m, q)));
      B[6 * p + q] = a;
    }
  bool finite = isfinite(cost);
#pragma unroll
  for (int p = 0; p < 6; ++p) {
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      double a = 0.0;
#pragma unroll
      for (int m = 0; m < 6; ++m) a = __dadd_rn(a, __dmul_rn(ad(m, p), B[6 * m + q]));
      out[kEHii + 6 * p + q] = a;
      out[kEHij + 6 * p + q] = -B[6 * q + p];
      finite = finite && isfinite(a) && isfinite(B[6 * q + p]);
    }
    double g = 0.0;
#pragma unroll
    for (int m = 0; m < 6; ++m) g = __dadd_rn(g, __dmul_rn(ad(m, p), Wr[m]));
    out[kEGi + p] = -g;
    out[kEGj + p] = Wr[p];
    finite = finite && isfinite(g);
  }
  out[kECost] = cost;
  out[kEFlag] = finite && th <= kHalfPi ? (double)kPgOk : (double)kPgNonfinite;
}

// entry (p, q) of the diagonal block of node a: sum over its incident edges in ascending id of Ji^T W Ji (a = i) or
// W (a = j)
ODB_DEVINL double diag_entry(const PgArgs& A, int a, int p, int q) {
  double s = 0.0;
  for (int k = A.inc_off[a]; k < A.inc_off[a + 1]; ++k) {
    const int e = A.inc[k] >> 1;
    s += (A.inc[k] & 1) ? __ldg(A.info + 36LL * e + 6 * p + q) : A.eb[(long long)e * kEdge + kEHii + 6 * p + q];
  }
  return s;
}

__global__ void __launch_bounds__(kPgThreads) pg_node_kernel(PgArgs A) {
  if (A.st[kPgDone] != 0.0) return;
  const int u = blockIdx.x * kPgThreads + threadIdx.x;
  if (u >= A.n) return;
  const int a = u / 6 + 1, p = u - (u / 6) * 6;
  const double d = diag_entry(A, a, p, p);
  double g = 0.0;
  for (int k = A.inc_off[a]; k < A.inc_off[a + 1]; ++k) {
    const int e = A.inc[k] >> 1;
    g += A.eb[(long long)e * kEdge + ((A.inc[k] & 1) ? kEGj : kEGi) + p];
  }
  const double sc = __dsqrt_rn(d);
  A.scale[u] = sc;
  A.rhs[u] = -__ddiv_rn(g, sc);
  A.nflag[u] = !(isfinite(d) && isfinite(g)) ? kPgNonfinite : (d > 0.0 ? kPgOk : kPgDegenerate);
}

// tile index t of a lower triangle of tiles -> (ti, tj), tj <= ti
ODB_DEVINL void tri_tile(int t, int& ti, int& tj) {
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while (i * (i + 1) / 2 > t) --i;
  while ((i + 1) * (i + 2) / 2 <= t) ++i;
  ti = i;
  tj = t - i * (i + 1) / 2;
}

__global__ void __launch_bounds__(kPgThreads) pg_fill_kernel(PgArgs A) {
  if (A.st[kPgDone] != 0.0) return;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int n = A.n;
  for (int idx = threadIdx.x; idx < kPanel * kPanel; idx += kPgThreads) {
    const int r = ti * kPanel + idx / kPanel, c = tj * kPanel + (idx & (kPanel - 1));
    if (r >= n || c > r) continue;
    const int a = r / 6 + 1, p = r - (r / 6) * 6, b = c / 6 + 1, q = c - (c / 6) * 6;
    double s = 0.0;
    if (a == b) {
      s = diag_entry(A, a, p, q);
    } else {                                      // a > b: the edges joining them, ascending
      for (int k = A.inc_off[a]; k < A.inc_off[a + 1]; ++k) {
        const int e = A.inc[k] >> 1, side = A.inc[k] & 1;
        if (A.edges[2 * e + (side ^ 1)] != b) continue;
        const double* hij = A.eb + (long long)e * kEdge + kEHij;
        s += side ? hij[6 * q + p] : hij[6 * p + q];        // a = j: (Ji^T W Jj)^T; a = i: Ji^T W Jj
      }
    }
    A.H[(long long)r * n + c] = __ddiv_rn(s, __dmul_rn(A.scale[r], A.scale[c]));
  }
}

__global__ void __launch_bounds__(kPgThreads) pg_factor_kernel(PgArgs A, int panel) {
  __shared__ double L[kPanel][kPad];
  __shared__ int code;
  if (A.st[kPgDone] != 0.0) return;
  if (panel == 0) {
    // the status of this linearisation: the largest flag over the nodes' unknowns and the edges
    __shared__ int red[kPgThreads];
    int f = 0;
    for (int u = threadIdx.x; u < A.n; u += kPgThreads) f = max(f, (int)A.nflag[u]);
    for (int e = threadIdx.x; e < A.E; e += kPgThreads) f = max(f, (int)A.eb[(long long)e * kEdge + kEFlag]);
    red[threadIdx.x] = f;
    __syncthreads();
    if (threadIdx.x == 0) {
      int m = 0;
      for (int t = 0; t < kPgThreads; ++t) m = max(m, red[t]);
      code = m;
      if (m != kPgOk) {
        A.st[kPgStatus] = m;
        A.st[kPgDone] = 1.0;
      }
    }
    __syncthreads();
    if (code != kPgOk) return;
  }
  const int n = A.n, k0 = panel * kPanel, m = min(kPanel, n - k0);
  for (int idx = threadIdx.x; idx < kPanel * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, c = idx & (kPanel - 1);
    if (r < m && c <= r) L[r][c] = A.H[(long long)(k0 + r) * n + k0 + c];
  }
  __syncthreads();
  for (int k = 0; k < m; ++k) {
    const double l = __dsqrt_rn(L[k][k]);
    if (!(__dmul_rn(l, l) >= kPgPivotMin)) {      // every thread reads the same pivot
      if (threadIdx.x == 0) {
        A.st[kPgStatus] = kPgDegenerate;
        A.st[kPgDone] = 1.0;
      }
      return;
    }
    for (int r = k + 1 + threadIdx.x; r < m; r += kPgThreads) L[r][k] = __ddiv_rn(L[r][k], l);
    __syncthreads();
    if (threadIdx.x == 0) L[k][k] = l;
    const int t = m - 1 - k;
    for (int e = threadIdx.x; e < t * t; e += kPgThreads) {
      const int r = k + 1 + e / t, c = k + 1 + e % t;
      if (c <= r) L[r][c] = __fma_rn(-L[r][k], L[c][k], L[r][c]);
    }
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < kPanel * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, c = idx & (kPanel - 1);
    if (r < m && c <= r) A.H[(long long)(k0 + r) * n + k0 + c] = L[r][c];
  }
  // L11 y = b for the panel's entries of b (already reduced by the earlier panels' rows)
  __shared__ double b[kPanel];
  if (threadIdx.x < m) b[threadIdx.x] = A.rhs[k0 + threadIdx.x];
  __syncthreads();
  for (int k = 0; k < m; ++k) {
    const double yk = __ddiv_rn(b[k], L[k][k]);
    for (int r = k + 1 + threadIdx.x; r < m; r += kPgThreads) b[r] = __fma_rn(-L[r][k], yk, b[r]);
    __syncthreads();
    if (threadIdx.x == 0) b[k] = yk;
    __syncthreads();
  }
  if (threadIdx.x < m) A.rhs[k0 + threadIdx.x] = b[threadIdx.x];
}

// L21 = A21 L11^-T for kTrsmRows rows below a full panel, then b -= L21 y for them
__global__ void __launch_bounds__(kPgThreads) pg_trsm_kernel(PgArgs A, int panel) {
  __shared__ double L[kPanel * (kPanel + 1) / 2];  // packed lower triangle, row r at r (r + 1) / 2
  __shared__ double X[kTrsmRows][kPad];
  if (A.st[kPgDone] != 0.0) return;
  const int n = A.n, k0 = panel * kPanel, r0 = k0 + kPanel + blockIdx.x * kTrsmRows;
  const int mr = min(kTrsmRows, n - r0);
  for (int idx = threadIdx.x; idx < kPanel * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, c = idx & (kPanel - 1);
    if (c <= r) L[r * (r + 1) / 2 + c] = A.H[(long long)(k0 + r) * n + k0 + c];
  }
  for (int idx = threadIdx.x; idx < kTrsmRows * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, c = idx & (kPanel - 1);
    X[r][c] = r < mr ? A.H[(long long)(r0 + r) * n + k0 + c] : 0.0;
  }
  __syncthreads();
  for (int c = 0; c < kPanel; ++c) {
    const double lcc = L[c * (c + 1) / 2 + c];
    if (threadIdx.x < kTrsmRows) X[threadIdx.x][c] = __ddiv_rn(X[threadIdx.x][c], lcc);
    __syncthreads();
    const int t = kPanel - 1 - c;
    for (int e = threadIdx.x; e < kTrsmRows * t; e += kPgThreads) {
      const int r = e / t, q = c + 1 + e % t;
      X[r][q] = __fma_rn(-X[r][c], L[q * (q + 1) / 2 + c], X[r][q]);
    }
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < kTrsmRows * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, c = idx & (kPanel - 1);
    if (r < mr) A.H[(long long)(r0 + r) * n + k0 + c] = X[r][c];
  }
  if (threadIdx.x < mr) {
    double s = A.rhs[r0 + threadIdx.x];
    for (int c = 0; c < kPanel; ++c) s = __fma_rn(-X[threadIdx.x][c], A.rhs[k0 + c], s);
    A.rhs[r0 + threadIdx.x] = s;
  }
}

// C(ti, tj) -= L21(ti) L21(tj)^T over the panel's 64 columns, k in order, 4 x 4 outputs per thread
__global__ void __launch_bounds__(kPgThreads) pg_trailing_kernel(PgArgs A, int panel) {
  __shared__ double As[kPanel / 2][kPanel + 2], Bs[kPanel / 2][kPanel + 2];
  if (A.st[kPgDone] != 0.0) return;
  int li, lj;
  tri_tile(blockIdx.x, li, lj);
  const int n = A.n, k0 = panel * kPanel;
  const int r0 = (panel + 1 + li) * kPanel, c0 = (panel + 1 + lj) * kPanel;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    const int kb = k0 + half * (kPanel / 2);
    __syncthreads();
    for (int idx = threadIdx.x; idx < kPanel * (kPanel / 2); idx += kPgThreads) {
      const int r = idx / (kPanel / 2), k = idx & (kPanel / 2 - 1);
      As[k][r] = r0 + r < n ? A.H[(long long)(r0 + r) * n + kb + k] : 0.0;
      Bs[k][r] = c0 + r < n ? A.H[(long long)(c0 + r) * n + kb + k] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kPanel / 2; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        a[i] = As[k][ty + 16 * i];
        b[i] = Bs[k][tx + 16 * i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fma_rn(a[i], b[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = r0 + ty + 16 * i, c = c0 + tx + 16 * j;
      if (r < n && c <= r) {
        double* h = A.H + (long long)r * n + c;
        *h = __dsub_rn(*h, acc[i][j]);
      }
    }
}

// x of the panel: s = L21^T x over the rows below (per 64-row tile, then the tiles in order), L11^T x = y - s
__global__ void __launch_bounds__(kPgThreads) pg_backsub_kernel(PgArgs A, int panel) {
  __shared__ double red[4][kPanel];
  __shared__ double L[kPanel][kPad];
  __shared__ double b[kPanel];
  __shared__ bool last;
  if (A.st[kPgDone] != 0.0) return;
  const int n = A.n, k0 = panel * kPanel, m = min(kPanel, n - k0);
  const int c = threadIdx.x & (kPanel - 1), g = threadIdx.x >> 6;
  const int r0 = k0 + kPanel + blockIdx.x * kPanel;
  double s = 0.0;
  if (c < m)
    for (int r = r0 + g; r < min(n, r0 + kPanel); r += 4) s = __fma_rn(A.H[(long long)r * n + k0 + c], A.rhs[r], s);
  red[g][c] = s;
  __syncthreads();
  if (threadIdx.x < kPanel) {
    A.part[(long long)blockIdx.x * kPanel + c] =
        __dadd_rn(__dadd_rn(__dadd_rn(red[0][c], red[1][c]), red[2][c]), red[3][c]);
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(A.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int idx = threadIdx.x; idx < kPanel * kPanel; idx += kPgThreads) {
    const int r = idx / kPanel, q = idx & (kPanel - 1);
    if (r < m && q <= r) L[r][q] = A.H[(long long)(k0 + r) * n + k0 + q];
  }
  if (threadIdx.x < m) {
    double t = 0.0;
    for (int q = 0; q < (int)gridDim.x; ++q) t = __dadd_rn(t, __ldcg(A.part + (long long)q * kPanel + threadIdx.x));
    b[threadIdx.x] = __dsub_rn(A.rhs[k0 + threadIdx.x], t);
  }
  __syncthreads();
  for (int k = m - 1; k >= 0; --k) {
    const double xk = __ddiv_rn(b[k], L[k][k]);
    for (int q = threadIdx.x; q < k; q += kPgThreads) b[q] = __fma_rn(-L[k][q], xk, b[q]);
    __syncthreads();
    if (threadIdx.x == 0) b[k] = xk;
    __syncthreads();
  }
  if (threadIdx.x < m) A.rhs[k0 + threadIdx.x] = b[threadIdx.x];
  if (threadIdx.x == 0) *A.ticket = 0u;              // re-armed for the next launch
}

constexpr int kUpdThreads = 512;                  // two nodes per thread (N <= 1024)

__global__ void __launch_bounds__(kUpdThreads) pg_update_kernel(PgArgs A) {
  __shared__ double mx[kUpdThreads];
  __shared__ int bad[kUpdThreads];
  if (A.st[kPgDone] != 0.0) return;
  double Tn[2][12], dmax = 0.0;
  int nb = 0;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int k = 1 + threadIdx.x + s * kUpdThreads;
    if (k >= A.N) continue;
    double x[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) x[q] = __ddiv_rn(A.rhs[6 * (k - 1) + q], A.scale[6 * (k - 1) + q]);
    const double v[3] = {x[0], x[1], x[2]}, om[3] = {x[3], x[4], x[5]};
    const double d = fmax(__dsqrt_rn(dot3_rn(v, v)), __dsqrt_rn(dot3_rn(om, om)));
    if (!isfinite(d)) nb = 1;
    else dmax = fmax(dmax, d);
    double T[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) T[q] = A.T[12 * k + q];
    se3_right_update(T, x, Tn[s]);
#pragma unroll
    for (int q = 0; q < 12; ++q)
      if (!isfinite(Tn[s][q])) nb = 1;
  }
  mx[threadIdx.x] = dmax;
  bad[threadIdx.x] = nb;
  __syncthreads();
  for (int o = kUpdThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      mx[threadIdx.x] = fmax(mx[threadIdx.x], mx[threadIdx.x + o]);
      bad[threadIdx.x] |= bad[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (bad[0]) {
    if (threadIdx.x == 0) {
      A.st[kPgStatus] = kPgNonfinite;
      A.st[kPgDone] = 1.0;
    }
    return;
  }
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int k = 1 + threadIdx.x + s * kUpdThreads;
    if (k < A.N)
#pragma unroll
      for (int q = 0; q < 12; ++q) A.T[12 * k + q] = Tn[s][q];
  }
  if (threadIdx.x == 0) {
    A.st[kPgMaxDelta] = mx[0];
    if (mx[0] <= A.tol) A.st[kPgDone] = 1.0;
  }
}

// sum of r^T W r over the edges at poses src (R, t layout; src16: [N][16] instead), fixed order
ODB_DEVINL double graph_cost(const PgArgs& A, const double* src, bool src16, double* red) {
  double s = 0.0;
  for (int e = threadIdx.x; e < A.E; e += kPgThreads) {
    int i, j;
    if (!edge_ok(A.edges, e, A.N, i, j)) continue;
    double Ti[12], Tj[12], r[6], D[12], Wr[6];
    if (src16) {
      load_pose16(src + 16 * i, Ti);
      load_pose16(src + 16 * j, Tj);
    } else {
#pragma unroll
      for (int q = 0; q < 12; ++q) {
        Ti[q] = src[12 * i + q];
        Tj[q] = src[12 * j + q];
      }
    }
    edge_residual(Ti, Tj, A.meas + 16LL * e, r, D);
    s = __dadd_rn(s, quad6(A.info + 36LL * e, r, Wr));
  }
  red[threadIdx.x] = s;
  __syncthreads();
  double t = 0.0;
  for (int q = 0; q < kPgThreads; ++q) t = __dadd_rn(t, red[q]);
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(kPgThreads) pg_output_kernel(PgArgs A, double* __restrict__ out,
                                                               double* __restrict__ record) {
  __shared__ double red[kPgThreads];
  const bool ok = A.st[kPgStatus] == (double)kPgOk;
  for (int k = threadIdx.x; k < A.N; k += kPgThreads) {
    if (ok) {
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) out[16 * k + 4 * r + c] = A.T[12 * k + 3 * r + c];
        out[16 * k + 4 * r + 3] = A.T[12 * k + 9 + r];
      }
      out[16 * k + 12] = out[16 * k + 13] = out[16 * k + 14] = 0.0;
      out[16 * k + 15] = 1.0;
    } else {
      for (int q = 0; q < 16; ++q) out[16 * k + q] = A.poses[16 * k + q];
    }
  }
  const double c_in = graph_cost(A, A.poses, true, red);
  const double c_out = ok ? graph_cost(A, A.T, false, red) : c_in;
  if (threadIdx.x == 0) {
    record[0] = A.st[kPgStatus];
    record[1] = A.st[kPgIters];
    record[2] = c_in;
    record[3] = c_out;
    record[4] = A.st[kPgMaxDelta];
    record[5] = A.N;
    record[6] = A.E;
  }
}

// workspace layout: ticket, state, T, edge blocks, scale, rhs, nflag, part, H (doubles), then inc_off, inc (int32)
static int64_t pg_layout(int N, int E, PgArgs* a, void* ws) {
  const int64_t n = 6LL * (N - 1), panels = pg_panels((int)n);
  const int64_t doubles = 1 + kPgState + 12LL * N + (int64_t)kEdge * E + 3 * n + panels * kPanel + n * n;
  const int64_t ints = (N + 1) + 2LL * E;
  if (a) {
    double* d = static_cast<double*>(ws);
    a->ticket = reinterpret_cast<unsigned int*>(d);
    a->st = d + 1;
    a->T = a->st + kPgState;
    a->eb = a->T + 12LL * N;
    a->scale = a->eb + (int64_t)kEdge * E;
    a->rhs = a->scale + n;
    a->nflag = a->rhs + n;
    a->part = a->nflag + n;
    a->H = a->part + panels * kPanel;
    a->inc_off = reinterpret_cast<int*>(a->H + n * n);
    a->inc = a->inc_off + N + 1;
  }
  return doubles * 8 + ints * 4;
}

static bool pg_sizes_ok(int32_t N, int32_t E) {
  return N >= 2 && N <= ODB_POSEGRAPH_MAX_NODES && E >= 1 && (int64_t)E <= 8LL * N;
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_posegraph_workspace_bytes(int32_t n_nodes, int32_t n_edges) {
  if (!pg_sizes_ok(n_nodes, n_edges)) return -1;
  return pg_layout(n_nodes, n_edges, nullptr, nullptr);
}

extern "C" int odb_posegraph_optimize(int32_t n_nodes, int32_t n_edges, const int32_t* edges, const double* poses,
                                      const double* measurements, const double* information, int32_t iterations,
                                      double tol, void* workspace, double* poses_out, double* record, void* stream_) {
  if (!pg_sizes_ok(n_nodes, n_edges) || !edges || !poses || !measurements || !information || !workspace ||
      !poses_out || !record || iterations < 1 || iterations > 100 || !(std::isfinite(tol) && tol > 0.0) ||
      !aligned(edges, 4) || !aligned(poses, 8) || !aligned(measurements, 8) || !aligned(information, 8) ||
      !aligned(workspace, 8) || !aligned(poses_out, 8) || !aligned(record, 8))
    return fail(ODB_ERR_INVALID, "posegraph_optimize: bad argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PgArgs A;
  pg_layout(n_nodes, n_edges, &A, workspace);
  A.N = n_nodes;
  A.E = n_edges;
  A.n = 6 * (n_nodes - 1);
  A.panels = pg_panels(A.n);
  A.tol = tol;
  A.edges = edges;
  A.poses = poses;
  A.meas = measurements;
  A.info = information;
  const int P = A.panels;
  pg_setup_kernel<<<1, 1024, 0, stream>>>(A);
  count_launch();
  for (int it = 0; it < iterations; ++it) {
    pg_edge_kernel<<<(n_edges + 127) / 128, 128, 0, stream>>>(A);
    pg_node_kernel<<<(A.n + kPgThreads - 1) / kPgThreads, kPgThreads, 0, stream>>>(A);
    pg_fill_kernel<<<P * (P + 1) / 2, kPgThreads, 0, stream>>>(A);
    count_launch();
    count_launch();
    count_launch();
    for (int p = 0; p < P; ++p) {
      pg_factor_kernel<<<1, kPgThreads, 0, stream>>>(A, p);
      count_launch();
      const int below = A.n - (p + 1) * kPanel;
      if (below <= 0) continue;
      pg_trsm_kernel<<<(below + kTrsmRows - 1) / kTrsmRows, kPgThreads, 0, stream>>>(A, p);
      const int q = P - 1 - p;
      pg_trailing_kernel<<<q * (q + 1) / 2, kPgThreads, 0, stream>>>(A, p);
      count_launch();
      count_launch();
    }
    for (int p = P - 1; p >= 0; --p) {
      pg_backsub_kernel<<<P - 1 - p > 0 ? P - 1 - p : 1, kPgThreads, 0, stream>>>(A, p);
      count_launch();
    }
    pg_update_kernel<<<1, kUpdThreads, 0, stream>>>(A);
    count_launch();
  }
  pg_output_kernel<<<1, kPgThreads, 0, stream>>>(A, poses_out, record);
  count_launch();
  return check_launch("posegraph_optimize");
}
