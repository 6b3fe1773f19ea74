// se(3) helpers shared by the pose solver (gn.cu), the bundle adjustments (lba.cu), the keyframe matching (kfmatch.cu),
// the batched front-end's epilogue (pipeline.cu) and the loop-closure decision (loopclosure.cu).
// Conventions of stvo-pl's auxiliar.h as used by pl-slam (SURVEY Appendix A.4; ordering x = [t; w] confirmed at
// src/mapHandler.cpp:3513-3514); same operation order as oracle/gn.c.
#pragma once
#include <math.h>

__device__ inline void d_skew(const double* w, double* S) {
  S[0] = 0; S[1] = -w[2]; S[2] = w[1];
  S[3] = w[2]; S[4] = 0; S[5] = -w[0];
  S[6] = -w[1]; S[7] = w[0]; S[8] = 0;
}
__device__ inline void d_mul3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// Q = R P + t of the row-major 4x4 T, each row summed ((r0 x + r1 y) + r2 z) + t (no contraction: --fmad=false)
__device__ __forceinline__ void d_transform(const double* T, const double* P, double* Q) {
#pragma unroll
  for (int i = 0; i < 3; ++i) Q[i] = T[4 * i] * P[0] + T[4 * i + 1] * P[1] + T[4 * i + 2] * P[2] + T[4 * i + 3];
}

__device__ inline void d_logmap(const double* T, double* x) {
  double V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, w[3] = {0, 0, 0};
  const double Vt[3] = {T[3], T[7], T[11]};
  double cosine = (T[0] + T[5] + T[10] - 1.0) / 2.0;
  cosine = cosine > 1.0 ? 1.0 : (cosine < -1.0 ? -1.0 : cosine);
  double sine = sqrt(1.0 - cosine * cosine);
  sine = sine > 1.0 ? 1.0 : sine;
  const double theta = acos(cosine);
  if (theta > 0.000001) {
    const double k = theta / (2.0 * sine);
    w[0] = k * (T[9] - T[6]);
    w[1] = k * (T[2] - T[8]);
    w[2] = k * (T[4] - T[1]);
    double s[9], s2[9];
    d_skew(w, s);
    for (int i = 0; i < 9; ++i) s[i] /= theta;
    d_mul3(s, s, s2);
    for (int i = 0; i < 9; ++i) {
      const double I = (i % 4 == 0) ? 1.0 : 0.0;
      V[i] = I + s[i] * (1.0 - cosine) / theta + s2[i] * (theta - sine) / theta;
    }
  }
  const double det = V[0] * (V[4] * V[8] - V[5] * V[7]) - V[1] * (V[3] * V[8] - V[5] * V[6]) +
                     V[2] * (V[3] * V[7] - V[4] * V[6]);
  const double id = 1.0 / det;
  const double Vi[9] = {(V[4] * V[8] - V[5] * V[7]) * id, (V[2] * V[7] - V[1] * V[8]) * id,
                        (V[1] * V[5] - V[2] * V[4]) * id, (V[5] * V[6] - V[3] * V[8]) * id,
                        (V[0] * V[8] - V[2] * V[6]) * id, (V[2] * V[3] - V[0] * V[5]) * id,
                        (V[3] * V[7] - V[4] * V[6]) * id, (V[1] * V[6] - V[0] * V[7]) * id,
                        (V[0] * V[4] - V[1] * V[3]) * id};
  for (int i = 0; i < 3; ++i) x[i] = Vi[3 * i] * Vt[0] + Vi[3 * i + 1] * Vt[1] + Vi[3 * i + 2] * Vt[2];
  x[3] = w[0];
  x[4] = w[1];
  x[5] = w[2];
}

// T = expmap_se3(x) (row-major 4x4), computed directly (same operation order as oracle/gn.c orc_expmap_se3)
__device__ inline void d_expmap(const double* x, double* T) {
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {x[0], x[1], x[2]};
  const double* w = x + 3;
  const double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(theta < 0.000001)) {
    double s[9], s2[9], V[9];
    d_skew(w, s);
    for (int i = 0; i < 9; ++i) s[i] /= theta;
    d_mul3(s, s, s2);
    const double sn = sin(theta), cs = cos(theta);
    for (int i = 0; i < 9; ++i) {
      const double I = (i % 4 == 0) ? 1.0 : 0.0;
      R[i] = I + s[i] * sn + s2[i] * (1.0 - cs);
      V[i] = I + s[i] * (1.0 - cs) / theta + s2[i] * (theta - sn) / theta;
    }
    const double t0 = t[0], t1 = t[1], t2 = t[2];
    for (int i = 0; i < 3; ++i) t[i] = V[3 * i] * t0 + V[3 * i + 1] * t1 + V[3 * i + 2] * t2;
  }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[4 * i + j] = R[3 * i + j];
    T[4 * i + 3] = t[i];
  }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
}
// Ti = inverse_se3(T) = [R^T, -R^T t]  (Ti may be T)
__host__ __device__ inline void d_inverse_se3(const double* T, double* Ti) {
  double out[16];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out[4 * i + j] = T[4 * j + i];
    out[4 * i + 3] = -(T[i] * T[3] + T[4 + i] * T[7] + T[8 + i] * T[11]);
  }
  out[12] = out[13] = out[14] = 0;
  out[15] = 1;
  for (int i = 0; i < 16; ++i) Ti[i] = out[i];
}

// Cyclic Jacobi on the symmetric part of a 6x6 matrix: A (36 entries) ends diagonal, its diagonal the eigenvalues
// (unsorted).  Host and device give the same bits: the device is built --fmad=false, the host has no FMA contraction, and
// sqrt and the division are correctly rounded on both.
__host__ __device__ inline void plf_sym6_jacobi(const double* A_in, double* A) {
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) A[6 * i + j] = 0.5 * (A_in[6 * i + j] + A_in[6 * j + i]);
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0;
    for (int i = 0; i < 6; ++i)
      for (int j = i + 1; j < 6; ++j) off += A[6 * i + j] * A[6 * i + j];
    if (off < 1e-300) break;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) {
        const double apq = A[6 * p + q];
        if (apq == 0.0) continue;
        const double theta = (A[6 * q + q] - A[6 * p + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; ++k) {  // A <- J^T A J
          const double akp = A[6 * k + p], akq = A[6 * k + q];
          A[6 * k + p] = c * akp - s * akq;
          A[6 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 6; ++k) {
          const double apk = A[6 * p + k], aqk = A[6 * q + k];
          A[6 * p + k] = c * apk - s * aqk;
          A[6 * q + k] = s * apk + c * aqk;
        }
      }
  }
}

// Largest eigenvalue of a symmetric 6x6 matrix (Eigen's SelfAdjointEigenSolver sorts ascending and
// MapHandler::isLoopClosure reads element 5, src/mapHandler.cpp:3883-3885).
__host__ __device__ inline double plf_sym6_max_eig(const double* A_in) {
  double A[36];
  plf_sym6_jacobi(A_in, A);
  double m = A[0];
  for (int i = 1; i < 6; ++i) m = A[7 * i] > m ? A[7 * i] : m;
  return m;
}

// T <- T * inverse_se3(expmap_se3(x)),  x = [t; w]
__device__ inline void d_update_pose(double* T, const double* x) {
  double Ei[16];
  d_expmap(x, Ei);
  d_inverse_se3(Ei, Ei);
  double out[16];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double a = 0;
      for (int k = 0; k < 4; ++k) a += T[4 * i + k] * Ei[4 * k + j];
      out[4 * i + j] = a;
    }
  for (int i = 0; i < 16; ++i) T[i] = out[i];
}
