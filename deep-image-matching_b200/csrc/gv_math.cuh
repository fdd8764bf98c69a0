// gv_math.cuh - the arithmetic of fundamental-matrix RANSAC, written once for host and device: the CUDA kernels of gv.cu call it per
// thread, the self-test library drives the very same functions on the CPU (tests without a GPU).
// Replaces the estimator inside the reference's geometric_verification (utils/geometric_verification.py:45-179: pydegensac /
// OpenCV findFundamentalMat); RANSAC is stochastic, so parity is statistical (inlier sets on data with known geometry).
#pragma once
#include <math.h>
#include <stdint.h>
#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace gv {

struct Norm {  // Hartley normalisation x' = s (x - c)
  float cx, cy, s;
};

__host__ __device__ inline uint32_t hash3(uint32_t a, uint32_t b, uint32_t c) {  // counter-based RNG (no state to carry)
  uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du;
  h ^= h >> 15;
  h *= 0x2C1B3C6Du;
  h ^= h >> 12;
  h *= 0x297A2D39u;
  h ^= h >> 15;
  return h;
}

// K distinct indices in [0, n) for hypothesis `hyp` (n >= K): rejection of repeats on one counter stream
template <int K>
__host__ __device__ inline void sample_distinct(uint32_t seed, uint32_t hyp, int n, int idx[K]) {
  uint32_t ctr = 0;
  for (int k = 0; k < K; ++k) {
    while (true) {
      const int c = static_cast<int>(hash3(seed, hyp, ctr++) % static_cast<uint32_t>(n));
      bool dup = false;
      for (int j = 0; j < k; ++j) dup |= idx[j] == c;
      if (!dup) {
        idx[k] = c;
        break;
      }
    }
  }
}

// 8 distinct indices in [0, n) for hypothesis `hyp` (n >= 8)
__host__ __device__ inline void sample8(uint32_t seed, uint32_t hyp, int n, int idx[8]) { sample_distinct<8>(seed, hyp, n, idx); }

// 7 distinct indices: the draws of sample8 stopped after the seventh
__host__ __device__ inline void sample7(uint32_t seed, uint32_t hyp, int n, int idx[7]) { sample_distinct<7>(seed, hyp, n, idx); }

// Null vector of an 8 x 9 system by Gauss-Jordan elimination with partial (row) pivoting and a free column chosen as the worst
// pivot column: returns false for (near-)degenerate samples.  a: row-major [8][9], destroyed.
__host__ __device__ inline bool null9(float a[8][9], float f[9]) {
  int piv_col[8];
  bool used[9] = {false, false, false, false, false, false, false, false, false};
  for (int r = 0; r < 8; ++r) {
    // pivot = largest |a[i][c]| over rows i >= r and unused columns c
    int pr = r, pc = -1;
    float best = 0.f;
    for (int i = r; i < 8; ++i)
      for (int c = 0; c < 9; ++c)
        if (!used[c] && fabsf(a[i][c]) > best) best = fabsf(a[i][c]), pr = i, pc = c;
    if (pc < 0 || best < 1e-7f) return false;
    if (pr != r)
      for (int c = 0; c < 9; ++c) {
        const float t = a[r][c];
        a[r][c] = a[pr][c];
        a[pr][c] = t;
      }
    used[pc] = true;
    piv_col[r] = pc;
    const float inv = 1.f / a[r][pc];
    for (int c = 0; c < 9; ++c) a[r][c] *= inv;
    for (int i = 0; i < 8; ++i)
      if (i != r) {
        const float m = a[i][pc];
        if (m != 0.f)
          for (int c = 0; c < 9; ++c) a[i][c] -= m * a[r][c];
      }
  }
  int fc = 0;
  while (used[fc]) ++fc;  // the free column
  f[fc] = 1.f;
  for (int r = 0; r < 8; ++r) f[piv_col[r]] = -a[r][fc];
  float nrm = 0.f;
  for (int c = 0; c < 9; ++c) nrm += f[c] * f[c];
  nrm = 1.f / sqrtf(nrm);
  for (int c = 0; c < 9; ++c) f[c] *= nrm;
  return true;
}

// symmetric 3x3 eigen-decomposition by cyclic Jacobi: A = V diag(w) V^T (A destroyed; V columns = eigenvectors)
__host__ __device__ inline void jacobi3(float A[3][3], float V[3][3], float w[3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) V[i][j] = i == j ? 1.f : 0.f;
  for (int sweep = 0; sweep < 12; ++sweep) {
    const float off = fabsf(A[0][1]) + fabsf(A[0][2]) + fabsf(A[1][2]);
    if (off < 1e-12f) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (fabsf(A[p][q]) < 1e-20f) continue;
        const float theta = (A[q][q] - A[p][p]) / (2.f * A[p][q]);
        const float t = (theta >= 0.f ? 1.f : -1.f) / (fabsf(theta) + sqrtf(theta * theta + 1.f));
        const float c = 1.f / sqrtf(t * t + 1.f), s = t * c;
        for (int k = 0; k < 3; ++k) {  // A <- A J
          const float akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {  // A <- J^T A
          const float apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const float vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; ++i) w[i] = A[i][i];
}

// rank-2 projection: F <- F - (F v)(v^T) with v the right singular vector of the smallest singular value (= the closest rank-2
// matrix in Frobenius norm, what the SVD clamp of the 8-point algorithm computes)
__host__ __device__ inline void rank2(float F[9]) {
  float M[3][3], V[3][3], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i][j] = F[0 + i] * F[0 + j] + F[3 + i] * F[3 + j] + F[6 + i] * F[6 + j];  // F^T F
  jacobi3(M, V, w);
  int k = 0;
  if (w[1] < w[k]) k = 1;
  if (w[2] < w[k]) k = 2;
  const float v[3] = {V[0][k], V[1][k], V[2][k]};
  for (int r = 0; r < 3; ++r) {
    const float fv = F[3 * r] * v[0] + F[3 * r + 1] * v[1] + F[3 * r + 2] * v[2];
    for (int c = 0; c < 3; ++c) F[3 * r + c] -= fv * v[c];
  }
}

// F = T1^T Fn T0 with T = [[s,0,-s cx],[0,s,-s cy],[0,0,1]], scaled to unit Frobenius norm; false for a zero matrix
__host__ __device__ inline bool denormalise(const float f[9], Norm n0, Norm n1, float F[9]) {
  float G[9];  // Fn T0
  for (int r = 0; r < 3; ++r) {
    G[3 * r] = f[3 * r] * n0.s;
    G[3 * r + 1] = f[3 * r + 1] * n0.s;
    G[3 * r + 2] = f[3 * r + 2] - n0.s * (f[3 * r] * n0.cx + f[3 * r + 1] * n0.cy);
  }
  for (int c = 0; c < 3; ++c) {
    F[c] = n1.s * G[c];
    F[3 + c] = n1.s * G[3 + c];
    F[6 + c] = G[6 + c] - n1.s * (n1.cx * G[c] + n1.cy * G[3 + c]);
  }
  float nrm = 0.f;
  for (int c = 0; c < 9; ++c) nrm += F[c] * F[c];
  if (!(nrm > 0.f)) return false;
  nrm = 1.f / sqrtf(nrm);
  for (int c = 0; c < 9; ++c) F[c] *= nrm;
  return true;
}

// normalised 8-point algorithm on 8 correspondences given in ORIGINAL pixels; F maps image 0 -> epipolar lines of image 1
// (x1^T F x0 = 0).  n0 / n1: Hartley normalisations of the whole match set.
__host__ __device__ inline bool eight_point(const float* k0, const float* k1, const int idx[8], Norm n0, Norm n1, float F[9]) {
  float a[8][9];
  for (int r = 0; r < 8; ++r) {
    const float x0 = (k0[2 * idx[r]] - n0.cx) * n0.s, y0 = (k0[2 * idx[r] + 1] - n0.cy) * n0.s;
    const float x1 = (k1[2 * idx[r]] - n1.cx) * n1.s, y1 = (k1[2 * idx[r] + 1] - n1.cy) * n1.s;
    a[r][0] = x1 * x0, a[r][1] = x1 * y0, a[r][2] = x1;
    a[r][3] = y1 * x0, a[r][4] = y1 * y0, a[r][5] = y1;
    a[r][6] = x0, a[r][7] = y0, a[r][8] = 1.f;
  }
  float f[9];
  if (!null9(a, f)) return false;
  rank2(f);
  return denormalise(f, n0, n1, F);
}

// Gauss-Jordan elimination of a 7 x 9 system, as null9 with two free columns: the two null vectors f1 / f2 (unit norm), false for a
// (near-)degenerate sample.  a: row-major [7][9], destroyed.
__host__ __device__ inline bool null9x2(float a[7][9], float f1[9], float f2[9]) {
  int piv_col[7];
  bool used[9] = {false, false, false, false, false, false, false, false, false};
  for (int r = 0; r < 7; ++r) {
    int pr = r, pc = -1;
    float best = 0.f;
    for (int i = r; i < 7; ++i)
      for (int c = 0; c < 9; ++c)
        if (!used[c] && fabsf(a[i][c]) > best) best = fabsf(a[i][c]), pr = i, pc = c;
    if (pc < 0 || best < 1e-7f) return false;
    if (pr != r)
      for (int c = 0; c < 9; ++c) {
        const float t = a[r][c];
        a[r][c] = a[pr][c];
        a[pr][c] = t;
      }
    used[pc] = true;
    piv_col[r] = pc;
    const float inv = 1.f / a[r][pc];
    for (int c = 0; c < 9; ++c) a[r][c] *= inv;
    for (int i = 0; i < 7; ++i)
      if (i != r) {
        const float m = a[i][pc];
        if (m != 0.f)
          for (int c = 0; c < 9; ++c) a[i][c] -= m * a[r][c];
      }
  }
  int fc[2], k = 0;
  for (int c = 0; c < 9; ++c)
    if (!used[c]) fc[k++] = c;
  float* out[2] = {f1, f2};
  for (int v = 0; v < 2; ++v) {
    float* f = out[v];
    f[fc[v]] = 1.f;
    f[fc[1 - v]] = 0.f;
    for (int r = 0; r < 7; ++r) f[piv_col[r]] = -a[r][fc[v]];
    float nrm = 0.f;
    for (int c = 0; c < 9; ++c) nrm += f[c] * f[c];
    nrm = 1.f / sqrtf(nrm);
    for (int c = 0; c < 9; ++c) f[c] *= nrm;
  }
  return true;
}

__host__ __device__ inline double det3(const double m[9]) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// real roots of c3 a^3 + c2 a^2 + c1 a + c0 in ascending order (a quadratic or linear equation when the leading terms vanish); returns
// their number (0 .. 3)
__host__ __device__ inline int real_roots3(double c3, double c2, double c1, double c0, double r[3]) {
  const double scale = fmax(fmax(fabs(c3), fabs(c2)), fmax(fabs(c1), fabs(c0)));
  if (!(scale > 0.0)) return 0;
  int m = 0;
  if (fabs(c3) > 1e-10 * scale) {
    const double a = c2 / c3, b = c1 / c3, c = c0 / c3;
    const double Q = (a * a - 3.0 * b) / 9.0, R = (2.0 * a * a * a - 9.0 * a * b + 27.0 * c) / 54.0;
    if (R * R < Q * Q * Q) {  // three real roots (trigonometric form)
      const double th = acos(fmin(1.0, fmax(-1.0, R / sqrt(Q * Q * Q)))), sq = -2.0 * sqrt(Q);
      r[0] = sq * cos(th / 3.0) - a / 3.0;
      r[1] = sq * cos((th + 6.283185307179586) / 3.0) - a / 3.0;
      r[2] = sq * cos((th - 6.283185307179586) / 3.0) - a / 3.0;
      m = 3;
    } else {  // one real root (Cardano)
      const double A = (R > 0.0 ? -1.0 : 1.0) * cbrt(fabs(R) + sqrt(R * R - Q * Q * Q));
      r[0] = A + (A != 0.0 ? Q / A : 0.0) - a / 3.0;
      m = 1;
    }
    for (int i = 0; i < m; ++i)  // two Newton steps against the cancellation of the closed forms
      for (int it = 0; it < 2; ++it) {
        const double x = r[i], f = ((c3 * x + c2) * x + c1) * x + c0, d = (3.0 * c3 * x + 2.0 * c2) * x + c1;
        if (d != 0.0) r[i] = x - f / d;
      }
  } else if (fabs(c2) > 1e-10 * scale) {
    const double disc = c1 * c1 - 4.0 * c2 * c0;
    if (disc < 0.0) return 0;
    const double q = -0.5 * (c1 + (c1 >= 0.0 ? 1.0 : -1.0) * sqrt(disc));
    r[m++] = q / c2;
    if (q != 0.0) r[m++] = c0 / q;
  } else if (fabs(c1) > 1e-10 * scale) {
    r[m++] = -c0 / c1;
  }
  for (int i = 1; i < m; ++i)
    for (int j = i; j > 0 && r[j] < r[j - 1]; --j) {
      const double t = r[j];
      r[j] = r[j - 1];
      r[j - 1] = t;
    }
  return m;
}

// normalised 7-point algorithm on 7 correspondences given in ORIGINAL pixels (layout and convention of eight_point): the null space
// (F1, F2) of the 7 x 9 system, the real roots alpha of det(alpha F1 + (1 - alpha) F2) = 0 (cubic in double), each root's matrix
// denormalised.  Returns the number of models written to F[0 .. 2] (0: degenerate sample or no real root); model r is root r in
// ascending order of alpha.
__host__ __device__ inline int seven_point(const float* k0, const float* k1, const int idx[7], Norm n0, Norm n1, float F[3][9]) {
  float a[7][9];
  for (int r = 0; r < 7; ++r) {
    const float x0 = (k0[2 * idx[r]] - n0.cx) * n0.s, y0 = (k0[2 * idx[r] + 1] - n0.cy) * n0.s;
    const float x1 = (k1[2 * idx[r]] - n1.cx) * n1.s, y1 = (k1[2 * idx[r] + 1] - n1.cy) * n1.s;
    a[r][0] = x1 * x0, a[r][1] = x1 * y0, a[r][2] = x1;
    a[r][3] = y1 * x0, a[r][4] = y1 * y0, a[r][5] = y1;
    a[r][6] = x0, a[r][7] = y0, a[r][8] = 1.f;
  }
  float f1[9], f2[9];
  if (!null9x2(a, f1, f2)) return 0;
  // d(alpha) = det(F2 + alpha (F1 - F2)) = c0 + c1 alpha + c2 alpha^2 + c3 alpha^3, from its values at 0, 1, -1 and 2
  double d[4];
  const double at[4] = {0.0, 1.0, -1.0, 2.0};
  for (int k = 0; k < 4; ++k) {
    double m[9];
    for (int c = 0; c < 9; ++c) m[c] = static_cast<double>(f2[c]) + at[k] * (static_cast<double>(f1[c]) - static_cast<double>(f2[c]));
    d[k] = det3(m);
  }
  const double c0 = d[0], c2 = 0.5 * (d[1] + d[2]) - c0, s = 0.5 * (d[1] - d[2]);  // s = c1 + c3
  const double c3 = ((d[3] - c0 - 4.0 * c2) - 2.0 * s) / 6.0, c1 = s - c3;
  double r[3];
  const int m = real_roots3(c3, c2, c1, c0, r);
  int out = 0;
  for (int k = 0; k < m; ++k) {
    float f[9];
    for (int c = 0; c < 9; ++c) f[c] = static_cast<float>(r[k] * f1[c] + (1.0 - r[k]) * f2[c]);
    if (denormalise(f, n0, n1, F[out])) ++out;
  }
  return out;
}

// hypotheses LO-RANSAC must run for `confidence` when the best model explains `best` of n matches: ceil(log(1 - confidence) /
// log(1 - w^7)), w = best / n; 1 when w = 1, `cap` when w^7 is too small to bound it (and never more than cap)
__host__ __device__ inline int lo_needed(int best, int n, float confidence, int cap) {
  if (best >= n) return 1;
  const double w = static_cast<double>(best) / n, p = pow(w, 7.0);
  if (!(p > 0.0)) return cap;
  const double den = log(1.0 - p);
  if (!(den < 0.0)) return cap;
  const double need = ceil(log(1.0 - static_cast<double>(confidence)) / den);
  return need < static_cast<double>(cap) ? static_cast<int>(need) : cap;
}

// positions in [0, m) of the 16 distinct inliers that inner LO iteration `it` after wave `wave` fits: the counter RNG of the pair's
// seed on stream numbers 2^31 + 32 wave + it, above every hypothesis index (m >= 16)
__host__ __device__ inline void lo_sample16(uint32_t seed, int wave, int it, int m, int pos[16]) {
  sample_distinct<16>(seed, 0x80000000u + 32u * static_cast<uint32_t>(wave) + static_cast<uint32_t>(it), m, pos);
}

// the normal-matrix row a of one correspondence in normalised coordinates: sum a^T a over inliers is what refit_from_normal solves
__host__ __device__ inline void normal_row(float x0, float y0, float x1, float y1, Norm n0, Norm n1, float a[9]) {
  const float u0 = (x0 - n0.cx) * n0.s, v0 = (y0 - n0.cy) * n0.s, u1 = (x1 - n1.cx) * n1.s, v1 = (y1 - n1.cy) * n1.s;
  a[0] = u1 * u0, a[1] = u1 * v0, a[2] = u1, a[3] = v1 * u0, a[4] = v1 * v0, a[5] = v1, a[6] = u0, a[7] = v0, a[8] = 1.f;
}

// squared Sampson distance of a correspondence (first-order geometric error, pixels^2)
__host__ __device__ inline float sampson2(const float F[9], float x0, float y0, float x1, float y1) {
  const float l0 = F[0] * x0 + F[1] * y0 + F[2], l1 = F[3] * x0 + F[4] * y0 + F[5], l2 = F[6] * x0 + F[7] * y0 + F[8];  // F x0
  const float m0 = F[0] * x1 + F[3] * y1 + F[6], m1 = F[1] * x1 + F[4] * y1 + F[7];                                      // F^T x1
  const float e = x1 * l0 + y1 * l1 + l2;
  const float d = l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1;
  return d > 0.f ? e * e / d : 3.4e38f;
}

// least-squares refit on a set of correspondences: smallest eigenvector of the 9x9 normal matrix (cyclic Jacobi), rank 2, denormalise.
// N: upper-triangular-complete symmetric 9x9 sum of a^T a over the NORMALISED inlier correspondences.
__host__ __device__ inline bool refit_from_normal(float N[9][9], Norm n0, Norm n1, float F[9]) {
  float V[9][9];
  for (int i = 0; i < 9; ++i)
    for (int j = 0; j < 9; ++j) V[i][j] = i == j ? 1.f : 0.f;
  for (int sweep = 0; sweep < 30; ++sweep) {
    float off = 0.f;
    for (int p = 0; p < 8; ++p)
      for (int q = p + 1; q < 9; ++q) off += fabsf(N[p][q]);
    if (off < 1e-9f) break;
    for (int p = 0; p < 8; ++p)
      for (int q = p + 1; q < 9; ++q) {
        if (fabsf(N[p][q]) < 1e-30f) continue;
        const float theta = (N[q][q] - N[p][p]) / (2.f * N[p][q]);
        const float t = (theta >= 0.f ? 1.f : -1.f) / (fabsf(theta) + sqrtf(theta * theta + 1.f));
        const float c = 1.f / sqrtf(t * t + 1.f), s = t * c;
        for (int k = 0; k < 9; ++k) {
          const float akp = N[k][p], akq = N[k][q];
          N[k][p] = c * akp - s * akq;
          N[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 9; ++k) {
          const float apk = N[p][k], aqk = N[q][k];
          N[p][k] = c * apk - s * aqk;
          N[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 9; ++k) {
          const float vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int k = 0;
  for (int i = 1; i < 9; ++i)
    if (N[i][i] < N[k][k]) k = i;
  float f[9];
  for (int i = 0; i < 9; ++i) f[i] = V[i][k];
  rank2(f);
  return denormalise(f, n0, n1, F);
}

}  // namespace gv
