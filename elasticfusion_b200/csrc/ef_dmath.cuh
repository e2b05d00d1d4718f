// Small dense linear algebra in double (and a float 3x3 solve) usable from host and device code.
// This is what lets the Gauss-Newton loop of RGBDOdometry::getIncrementalTransformation
// (reference Core/Utils/RGBDOdometry.cpp:259-571) run entirely on the GPU: the 6x6 normal equations are solved by
// one thread of the reduction kernel's last block instead of Eigen on the host after a blocking D2H copy.
// Algorithms: LDL^T with diagonal pivoting (what Eigen::LDLT does, RGBDOdometry.cpp:356,526-534), cofactor 3x3
// inverse, Gauss-Jordan NxN inverse (also the host's covariance, RGBDOdometry.cpp:573-575), Rodrigues (OdometryProvider.h:34-71), orthogonal polar factor by Newton
// iteration (== U*V^T of the JacobiSVD at RGBDOdometry.cpp:566-570), SE3 log (Sophus, ElasticFusion.cpp:371-374).
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

namespace efm {

#define EFM_HD __host__ __device__ __forceinline__

EFM_HD void mul3(const double* a, const double* b, double* c) {
  double r[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r[i * 3 + j] = a[i * 3 + 0] * b[0 * 3 + j] + a[i * 3 + 1] * b[1 * 3 + j] + a[i * 3 + 2] * b[2 * 3 + j];
  for (int i = 0; i < 9; ++i) c[i] = r[i];
}
EFM_HD void mulv3(const double* a, const double* v, double* o) {
  double r[3];
  for (int i = 0; i < 3; ++i) r[i] = a[i * 3 + 0] * v[0] + a[i * 3 + 1] * v[1] + a[i * 3 + 2] * v[2];
  for (int i = 0; i < 3; ++i) o[i] = r[i];
}
EFM_HD void mul4(const double* a, const double* b, double* c) {
  double r[16];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double s = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
      r[i * 4 + j] = s;
    }
  for (int i = 0; i < 16; ++i) c[i] = r[i];
}

template <typename T>
EFM_HD void inv3(const T* m, T* o) {
  T c00 = m[4] * m[8] - m[5] * m[7];
  T c01 = m[5] * m[6] - m[3] * m[8];
  T c02 = m[3] * m[7] - m[4] * m[6];
  T det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  T id = T(1) / det;
  T r[9];
  r[0] = c00 * id;
  r[1] = (m[2] * m[7] - m[1] * m[8]) * id;
  r[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  r[3] = c01 * id;
  r[4] = (m[0] * m[8] - m[2] * m[6]) * id;
  r[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  r[6] = c02 * id;
  r[7] = (m[1] * m[6] - m[0] * m[7]) * id;
  r[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  for (int i = 0; i < 9; ++i) o[i] = r[i];
}

// The reference's packed normal equations (JtJJtrSE3 for N = 6, JtJJtrSO3 for N = 3, types.cuh:98-104): the upper triangle of
// [A | b] row by row. Unpacked into the symmetric N x N A and b; the residual terms that follow the packed system are left alone.
template <int N>
EFM_HD void unpack_normal_eq(const float* h, float* A, float* b) {
  int shift = 0;
  for (int i = 0; i < N; ++i)
    for (int j = i; j < N + 1; ++j) {
      const float value = h[shift++];
      if (j == N)
        b[i] = value;
      else
        A[j * N + i] = A[i * N + j] = value;
    }
}

// Gauss-Jordan inverse with partial pivoting, N <= 6
template <int N>
EFM_HD void inv_n(const double* m, double* o) {
  double a[N][2 * N];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      a[i][j] = m[i * N + j];
      a[i][N + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < N; ++c) {
    int p = c;
    for (int r = c + 1; r < N; ++r)
      if (fabs(a[r][c]) > fabs(a[p][c])) p = r;
    if (p != c)
      for (int j = 0; j < 2 * N; ++j) {
        double t = a[c][j];
        a[c][j] = a[p][j];
        a[p][j] = t;
      }
    double d = a[c][c];
    for (int j = 0; j < 2 * N; ++j) a[c][j] /= d;
    for (int r = 0; r < N; ++r)
      if (r != c) {
        double f = a[r][c];
        if (f != 0)
          for (int j = 0; j < 2 * N; ++j) a[r][j] -= f * a[c][j];
      }
  }
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) o[i * N + j] = a[i][N + j];
}

// x = A^-1 b for symmetric A via L D L^T with diagonal pivoting; near-zero pivots contribute 0 (Eigen LDLT).
template <typename T, int N>
EFM_HD void ldlt_solve(const T* A_, const T* b_, T* x, T tiny) {
  T A[N][N];
  T bb[N];
  T invd[N];
  int perm[N];
  for (int i = 0; i < N; ++i) {
    perm[i] = i;
    invd[i] = T(0);
    bb[i] = b_[i];
    for (int j = 0; j < N; ++j) A[i][j] = A_[i * N + j];
  }
  for (int k = 0; k < N; ++k) {
    int p = k;
    T big = fabs(A[k][k]);
    for (int i = k + 1; i < N; ++i)
      if (fabs(A[i][i]) > big) {
        big = fabs(A[i][i]);
        p = i;
      }
    if (p != k) {
      for (int j = 0; j < N; ++j) {
        T t = A[k][j];
        A[k][j] = A[p][j];
        A[p][j] = t;
      }
      for (int i = 0; i < N; ++i) {
        T t = A[i][k];
        A[i][k] = A[i][p];
        A[i][p] = t;
      }
      T t = bb[k];
      bb[k] = bb[p];
      bb[p] = t;
      int ti = perm[k];
      perm[k] = perm[p];
      perm[p] = ti;
    }
    T d = A[k][k];
    if (d == T(0)) continue;
    const T rd = T(1) / d;  // one division per pivot (double division is a ~40-instruction dependent sequence on the GPU)
    invd[k] = (fabs(d) > tiny) ? rd : T(0);
    for (int i = k + 1; i < N; ++i) A[i][k] *= rd;
    for (int i = k + 1; i < N; ++i)
      for (int j = k + 1; j <= i; ++j) {
        A[i][j] -= A[i][k] * d * A[j][k];
        A[j][i] = A[i][j];
      }
  }
  T y[N];
  for (int i = 0; i < N; ++i) {
    T s = bb[i];
    for (int j = 0; j < i; ++j) s -= A[i][j] * y[j];
    y[i] = s;
  }
  for (int i = 0; i < N; ++i) y[i] = y[i] * invd[i];
  T z[N];
  for (int i = N - 1; i >= 0; --i) {
    T s = y[i];
    for (int j = i + 1; j < N; ++j) s -= A[j][i] * z[j];
    z[i] = s;
  }
  for (int i = 0; i < N; ++i) x[perm[i]] = z[i];
}
EFM_HD void solve_sym6(const double* A, const double* b, double* x) { ldlt_solve<double, 6>(A, b, x, 1.0 / DBL_MAX); }

// 1/d to full double precision without the ~40-instruction IEEE division sequence: hardware reciprocal seed (rcp.approx.ftz.f64,
// ~20 good bits) + three Newton steps. Used only where a 1-ulp difference is irrelevant (pivot reciprocals of the solve).
__device__ __forceinline__ double fast_rcp(double d) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  r = r * (2.0 - d * r);
  r = r * (2.0 - d * r);
  r = r * (2.0 - d * r);
  return r;
}

// Register-resident L D L^T solve (no pivoting, fully unrolled: every index is a compile-time constant, so nothing goes
// to local memory). For the symmetric positive-definite normal equations of the tracker this equals the pivoted solve to
// rounding (~1e-13 relative); a vanishing pivot contributes 0 like Eigen::LDLT does. Used on the device, where a
// single thread runs the solve and dependent local-memory traffic would dominate.
template <int N>
__device__ __forceinline__ void ldlt_solve_unrolled(const double* A_, const double* b_, double* x) {
  double L[N][N], D[N], invD[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double d = A_[j * N + j];
#pragma unroll
    for (int k = 0; k < N; ++k)
      if (k < j) d -= L[j][k] * L[j][k] * D[k];
    D[j] = d;
    invD[j] = (fabs(d) > 1e-300) ? fast_rcp(d) : 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i)
      if (i > j) {
        double v = A_[i * N + j];
#pragma unroll
        for (int k = 0; k < N; ++k)
          if (k < j) v -= L[i][k] * L[j][k] * D[k];
        L[i][j] = v * invD[j];
      }
  }
  double y[N];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double v = b_[i];
#pragma unroll
    for (int k = 0; k < N; ++k)
      if (k < i) v -= L[i][k] * y[k];
    y[i] = v;
  }
#pragma unroll
  for (int i = 0; i < N; ++i) y[i] *= invD[i];
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double v = y[i];
#pragma unroll
    for (int k = 0; k < N; ++k)
      if (k > i) v -= L[k][i] * x[k];
    x[i] = v;
  }
}
EFM_HD void solve_sym3f(const float* A, const float* b, float* x) { ldlt_solve<float, 3>(A, b, x, 1.0f / FLT_MAX); }

EFM_HD void rodrigues(const double* src, double* dst) {
  const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int k = 0; k < 9; ++k) dst[k] = I[k];
  double rx = src[0], ry = src[1], rz = src[2];
  double theta = sqrt(rx * rx + ry * ry + rz * rz);
  if (theta >= DBL_EPSILON) {
    double c, s;
#ifdef __CUDA_ARCH__
    sincos(theta, &s, &c);  // one range reduction for both
#else
    c = cos(theta);
    s = sin(theta);
#endif
    const double c1 = 1. - c;
    double itheta = theta ? 1. / theta : 0.;
    rx *= itheta;
    ry *= itheta;
    rz *= itheta;
    double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int k = 0; k < 9; ++k) dst[k] = c * I[k] + c1 * rrt[k] + s * r_x[k];
  }
}

EFM_HD void polar_orthogonal(const double* m, double* o) {
  double X[9];
  for (int k = 0; k < 9; ++k) X[k] = m[k];
  for (int it = 0; it < 30; ++it) {
    double Xi[9], Nn[9], delta = 0;
    inv3<double>(X, Xi);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        Nn[r * 3 + c] = 0.5 * (X[r * 3 + c] + Xi[c * 3 + r]);
        delta += fabs(Nn[r * 3 + c] - X[r * 3 + c]);
      }
    for (int k = 0; k < 9; ++k) X[k] = Nn[k];
    // converged to rounding (9 entries x a few ulp of values <= 1). The input is a float rotation (off by ~1e-7) and the iteration
    // is quadratic, so this is the third pass; a tighter bound is never met and ran all 30 passes on one thread (8 us per frame).
    if (delta < 4e-15) break;
  }
  for (int k = 0; k < 9; ++k) o[k] = X[k];
}

EFM_HD void se3_inverse(const double* T, double* o) {
  double r[16];
  for (int i = 0; i < 16; ++i) r[i] = 0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[i * 4 + j] = T[j * 4 + i];
  for (int i = 0; i < 3; ++i) r[i * 4 + 3] = -(r[i * 4 + 0] * T[3] + r[i * 4 + 1] * T[7] + r[i * 4 + 2] * T[11]);
  r[15] = 1;
  for (int i = 0; i < 16; ++i) o[i] = r[i];
}

EFM_HD double se3_log_norm(const double* T) {
  double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  double t[3] = {T[3], T[7], T[11]};
  double cs = (R[0] + R[4] + R[8] - 1.0) * 0.5;
  cs = cs > 1 ? 1 : (cs < -1 ? -1 : cs);
  double ax[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
  double sn = 0.5 * sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
  double theta = atan2(sn, cs);
  double w[3];
  double k = (theta < 1e-10) ? 0.5 : theta / (2.0 * sn);
  for (int i = 0; i < 3; ++i) w[i] = k * ax[i];
  double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double W2[9];
  mul3(W, W, W2);
  double coef = (theta < 1e-5) ? 1.0 / 12.0 : (1.0 - (theta * sin(theta)) / (2.0 * (1.0 - cos(theta)))) / (theta * theta);
  double u[3];
  for (int i = 0; i < 3; ++i) {
    u[i] = 0;
    for (int j = 0; j < 3; ++j) u[i] += (((i == j) ? 1.0 : 0.0) - 0.5 * W[i * 3 + j] + coef * W2[i * 3 + j]) * t[j];
  }
  return sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2] + w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
}

}  // namespace efm
