// SE(3) arithmetic shared by the camera tracker (track.cu) and the pose-graph solve (posegraph.cu): the exponential of
// a twist in the camera-frame convention T <- T exp(xi), xi = (v, omega), and its inverse, the logarithm.  Every
// operation is an explicit round-to-nearest fp64 operation (no contraction into FMAs), so that the float64 oracles
// (oracle/track_oracle.py, oracle/posegraph_oracle.py) restate them operation by operation.  Callers are built without
// fast-math.
#pragma once
#include "common.cuh"

namespace odb {

constexpr double kSeriesTheta = 1e-2;             // |omega| below this: series for the coefficients
constexpr double kPi = 3.141592653589793;

ODB_DEVINL double dot3_rn(const double u[3], const double v[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(u[0], v[0]), __dmul_rn(u[1], v[1])), __dmul_rn(u[2], v[2]));
}

// A = sin(theta) / theta and B = (1 - cos(theta)) / theta^2 of th2 = theta^2, th = theta (C unused when null:
// C = (theta - sin(theta)) / theta^3); below kSeriesTheta the Taylor series to theta^4
ODB_DEVINL void se3_coefficients(double th2, double th, double& A, double& B, double* C) {
  if (th < kSeriesTheta) {
    const double th4 = __dmul_rn(th2, th2);
    A = __dadd_rn(__dsub_rn(1.0, __ddiv_rn(th2, 6.0)), __ddiv_rn(th4, 120.0));
    B = __dadd_rn(__dsub_rn(0.5, __ddiv_rn(th2, 24.0)), __ddiv_rn(th4, 720.0));
    if (C) *C = __dadd_rn(__dsub_rn(1.0 / 6.0, __ddiv_rn(th2, 120.0)), __ddiv_rn(th4, 5040.0));
  } else {
    double sn, cs;                                  // sin(theta), cos(theta); no Payne-Hanek path (no stack frame)
    sincospi(__ddiv_rn(th, kPi), &sn, &cs);
    A = __ddiv_rn(sn, th);
    B = __ddiv_rn(__dsub_rn(1.0, cs), th2);
    if (C) *C = __ddiv_rn(__dsub_rn(th, sn), __dmul_rn(th2, th));
  }
}

// exp of the twist (v, omega): R = I + A W + B W^2, u = (I + B W + C W^2) v with W = [omega]x, W^2 = omega omega^T -
// theta^2 I, A = sin(theta) / theta, B = (1 - cos(theta)) / theta^2, C = (theta - sin(theta)) / theta^3; below
// kSeriesTheta the Taylor series to theta^4
ODB_DEVINL void se3_exp(const double xi[6], double R[9], double u[3]) {
  const double om[3] = {xi[3], xi[4], xi[5]};
  const double th2 = dot3_rn(om, om), th = __dsqrt_rn(th2);
  double A, B, C;
  se3_coefficients(th2, th, A, B, &C);
  const double W[9] = {0.0, -om[2], om[1], om[2], 0.0, -om[0], -om[1], om[0], 0.0};
  double V[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double w2 = i == j ? __dsub_rn(__dmul_rn(om[i], om[j]), th2) : __dmul_rn(om[i], om[j]);
      const double id = i == j ? 1.0 : 0.0;
      R[3 * i + j] = __dadd_rn(__dadd_rn(id, __dmul_rn(A, W[3 * i + j])), __dmul_rn(B, w2));
      V[3 * i + j] = __dadd_rn(__dadd_rn(id, __dmul_rn(B, W[3 * i + j])), __dmul_rn(C, w2));
    }
#pragma unroll
  for (int i = 0; i < 3; ++i) u[i] = dot3_rn(V + 3 * i, xi);
}

// M = ref^-1 T of two poses stored as R row-major (9), then t (3): Rm = Rref^T R, tm = Rref^T (t - tref)
ODB_DEVINL void relative_pose(const double* ref, const double* T, double* M) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
      M[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(ref[i], T[j]), __dmul_rn(ref[3 + i], T[3 + j])),
                               __dmul_rn(ref[6 + i], T[6 + j]));
    M[9 + i] = __dadd_rn(__dadd_rn(__dmul_rn(ref[i], __dsub_rn(T[9], ref[9])),
                                   __dmul_rn(ref[3 + i], __dsub_rn(T[10], ref[10]))),
                         __dmul_rn(ref[6 + i], __dsub_rn(T[11], ref[11])));
  }
}

// Tn = T exp(xi): Rn = R Re, tn = R u + t
ODB_DEVINL void se3_right_update(const double* T, const double xi[6], double* Tn) {
  double Re[9], u[3];
  se3_exp(xi, Re, u);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
      Tn[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(T[3 * i], Re[j]), __dmul_rn(T[3 * i + 1], Re[3 + j])),
                                __dmul_rn(T[3 * i + 2], Re[6 + j]));
    Tn[9 + i] = __dadd_rn(dot3_rn(T + 3 * i, u), T[9 + i]);
  }
}

}  // namespace odb
