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

// F (pixels) in the normalised coordinates, Fn = T1^-T F T0^-1 (the inverse of denormalise, up to scale)
__host__ __device__ inline void normalise_f(const float F[9], Norm n0, Norm n1, float Fn[9]) {
  const float i0 = 1.f / n0.s, i1 = 1.f / n1.s;
  float G[9];  // T1^-T F
  for (int c = 0; c < 3; ++c) {
    G[c] = i1 * F[c];
    G[3 + c] = i1 * F[3 + c];
    G[6 + c] = n1.cx * F[c] + n1.cy * F[3 + c] + F[6 + c];
  }
  for (int r = 0; r < 3; ++r) {  // G T0^-1
    Fn[3 * r] = i0 * G[3 * r];
    Fn[3 * r + 1] = i0 * G[3 * r + 1];
    Fn[3 * r + 2] = n0.cx * G[3 * r] + n0.cy * G[3 * r + 1] + G[3 * r + 2];
  }
}

// samples of K points a RANSAC must draw for `confidence` when the best model explains `best` of n candidates: ceil(log(1 -
// confidence) / log(1 - w^K)), w = best / n; 1 when w = 1, `cap` when w^K is too small to bound it (and never more than cap)
template <int K>
__host__ __device__ inline int ransac_needed(int best, int n, float confidence, int cap) {
  if (best >= n) return 1;
  const double w = static_cast<double>(best) / n, p = pow(w, static_cast<double>(K));
  if (!(p > 0.0)) return cap;
  const double den = log(1.0 - p);
  if (!(den < 0.0)) return cap;
  const double need = ceil(log(1.0 - static_cast<double>(confidence)) / den);
  return need < static_cast<double>(cap) ? static_cast<int>(need) : cap;
}

// hypotheses LO-RANSAC must run: 7-point samples
__host__ __device__ inline int lo_needed(int best, int n, float confidence, int cap) { return ransac_needed<7>(best, n, confidence, cap); }

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

// ------------------------------------------------------------------ DEGENSAC (Chum, Werner, Matas, CVPR 2005)
// In the Hartley-normalised coordinates of the 7-point solver; a correspondence c is (x, y, x', y').

// H-inlier threshold of degensac: transfer error |x' - H x| below kDegHFactor * threshold, in image-1 pixels, both in the degeneracy
// test of a sample and when an H is scored over all matches.  The transfer error carries the noise of both images and the error of an
// H solved from three noisy points, where the Sampson distance of F carries one first-order residual: twice the F threshold keeps the
// plane's points together without taking in off-plane points of small parallax.
constexpr float kDegHFactor = 2.f;

// the squared H-inlier threshold in normalised units of image 1, for the squared F threshold thr2 in pixels
__host__ __device__ inline float deg_t2n(float thr2, Norm n1) { return kDegHFactor * kDegHFactor * thr2 * n1.s * n1.s; }

// squared transfer error |x' - H x|^2 of a correspondence, in the units of x'; 3.4e38 when H x is at infinity
__host__ __device__ inline float transfer2(const float H[9], float x0, float y0, float x1, float y1) {
  const float u = H[0] * x0 + H[1] * y0 + H[2], v = H[3] * x0 + H[4] * y0 + H[5], w = H[6] * x0 + H[7] * y0 + H[8];
  if (w == 0.f) return 3.4e38f;
  const float iw = 1.f / w, dx = x1 - u * iw, dy = y1 - v * iw;
  return dx * dx + dy * dy;
}

__host__ __device__ inline void cross3(const float a[3], const float b[3], float c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1], c[1] = a[2] * b[0] - a[0] * b[2], c[2] = a[0] * b[1] - a[1] * b[0];
}

// G = [e]_x M (3 x 3, row-major)
__host__ __device__ inline void skew_times(const float e[3], const float M[9], float G[9]) {
  for (int c = 0; c < 3; ++c) {
    G[c] = -e[2] * M[3 + c] + e[1] * M[6 + c];
    G[3 + c] = e[2] * M[c] - e[0] * M[6 + c];
    G[6 + c] = -e[1] * M[c] + e[0] * M[3 + c];
  }
}

// The homography compatible with F (x'^T F x = 0) that maps three correspondences c[0..2] (Hartley & Zisserman, Result 13.6):
// H = A - e' (M^-1 b)^T with A = [e']_x F, e' the left null vector of F, M the rows x_i^T and
// b_i = (x'_i x A x_i)^T (x'_i x e') / |x'_i x e'|^2.  False when it is ill-conditioned: F of rank < 2 (no e'), a point x'_i at the
// epipole, or three (nearly) collinear x_i.
__host__ __device__ inline bool h_from_f3(const float F[9], const float c[3][4], float H[9]) {
  float e[3] = {0.f, 0.f, 0.f}, ee = 0.f, ff = 0.f;
  for (int k = 0; k < 9; ++k) ff += F[k] * F[k];
  for (int a = 0; a < 2; ++a)  // e' = the longest cross product of two columns of F (F^T e' = 0)
    for (int b = a + 1; b < 3; ++b) {
      const float p[3] = {F[a], F[3 + a], F[6 + a]}, q[3] = {F[b], F[3 + b], F[6 + b]};
      float x[3];
      cross3(p, q, x);
      const float s = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
      if (s > ee) ee = s, e[0] = x[0], e[1] = x[1], e[2] = x[2];
    }
  if (!(ee > 1e-10f * ff * ff)) return false;
  const float ie = 1.f / sqrtf(ee);
  for (int k = 0; k < 3; ++k) e[k] *= ie;
  float A[9];
  skew_times(e, F, A);
  float b[3], x[3][3];
  for (int i = 0; i < 3; ++i) {
    x[i][0] = c[i][0], x[i][1] = c[i][1], x[i][2] = 1.f;
    const float xp[3] = {c[i][2], c[i][3], 1.f};
    const float ax[3] = {A[0] * x[i][0] + A[1] * x[i][1] + A[2], A[3] * x[i][0] + A[4] * x[i][1] + A[5], A[6] * x[i][0] + A[7] * x[i][1] + A[8]};
    float p[3], q[3];
    cross3(xp, ax, p);
    cross3(xp, e, q);
    const float qq = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
    if (!(qq > 1e-10f * (xp[0] * xp[0] + xp[1] * xp[1] + 1.f))) return false;
    b[i] = (p[0] * q[0] + p[1] * q[1] + p[2] * q[2]) / qq;
  }
  // M^-1 = [x1 x x2 | x2 x x0 | x0 x x1] / det M (columns)
  float adj[3][3];
  cross3(x[1], x[2], adj[0]);
  cross3(x[2], x[0], adj[1]);
  cross3(x[0], x[1], adj[2]);
  const float det = x[0][0] * adj[0][0] + x[0][1] * adj[0][1] + x[0][2] * adj[0][2];
  float nx = 1.f;
  for (int i = 0; i < 3; ++i) nx *= x[i][0] * x[i][0] + x[i][1] * x[i][1] + 1.f;
  if (!(det * det > 1e-10f * nx)) return false;
  const float id = 1.f / det;
  float v[3];
  for (int k = 0; k < 3; ++k) v[k] = (b[0] * adj[0][k] + b[1] * adj[1][k] + b[2] * adj[2][k]) * id;
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) H[3 * r + k] = A[3 * r + k] - e[r] * v[k];
  return true;
}

// DEGENSAC's degeneracy test of a 7-point model F of the sample u[0..6]: for each of the five triplets {0,1,2}, {3,4,5}, {0,1,6},
// {3,4,6}, {2,5,6} (every 5 of the 7 points contain one), H from F and the triplet, and the sample points whose squared transfer error
// is below t2.  Returns the first triplet whose H maps 5 or more of them (the sample is dominated by a plane; its H in H), -1 if none.
__host__ __device__ inline int degenerate7(const float F[9], const float u[7][4], float t2, float H[9]) {
  const int tri[5][3] = {{0, 1, 2}, {3, 4, 5}, {0, 1, 6}, {3, 4, 6}, {2, 5, 6}};
  for (int t = 0; t < 5; ++t) {
    float c[3][4], G[9];
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 4; ++k) c[i][k] = u[tri[t][i]][k];
    if (!h_from_f3(F, c, G)) continue;
    int on = 0;
    for (int j = 0; j < 7; ++j) on += transfer2(G, u[j][0], u[j][1], u[j][2], u[j][3]) < t2;
    if (on >= 5) {
      for (int k = 0; k < 9; ++k) H[k] = G[k];
      return t;
    }
  }
  return -1;
}

// H in pixels from H in normalised coordinates: T1^-1 Hn T0, scaled to unit Frobenius norm; false for a zero matrix
__host__ __device__ inline bool h_denormalise(const float h[9], Norm n0, Norm n1, float H[9]) {
  float G[9];  // Hn T0
  for (int r = 0; r < 3; ++r) {
    G[3 * r] = h[3 * r] * n0.s;
    G[3 * r + 1] = h[3 * r + 1] * n0.s;
    G[3 * r + 2] = h[3 * r + 2] - n0.s * (h[3 * r] * n0.cx + h[3 * r + 1] * n0.cy);
  }
  const float is = 1.f / n1.s;
  for (int c = 0; c < 3; ++c) {
    H[c] = G[c] * is + n1.cx * G[6 + c];
    H[3 + c] = G[3 + c] * is + n1.cy * G[6 + c];
    H[6 + c] = G[6 + c];
  }
  float nrm = 0.f;
  for (int c = 0; c < 9; ++c) nrm += H[c] * H[c];
  if (!(nrm > 0.f)) return false;
  nrm = 1.f / sqrtf(nrm);
  for (int c = 0; c < 9; ++c) H[c] *= nrm;
  return true;
}

// Plane and parallax: F = [e']_x H with e' = (H x_a x x'_a) x (H x_b x x'_b), where the parallax lines of two off-plane
// correspondences a, b meet; rank 2 by construction.  False when the lines (nearly) coincide or vanish (a point on the plane).
__host__ __device__ inline bool plane_parallax(const float H[9], const float a[4], const float b[4], float F[9]) {
  float l[2][3];
  for (int s = 0; s < 2; ++s) {
    const float* c = s ? b : a;
    const float hx[3] = {H[0] * c[0] + H[1] * c[1] + H[2], H[3] * c[0] + H[4] * c[1] + H[5], H[6] * c[0] + H[7] * c[1] + H[8]};
    const float xp[3] = {c[2], c[3], 1.f};
    cross3(hx, xp, l[s]);
  }
  float e[3];
  cross3(l[0], l[1], e);
  const float ee = e[0] * e[0] + e[1] * e[1] + e[2] * e[2];
  const float l0 = l[0][0] * l[0][0] + l[0][1] * l[0][1] + l[0][2] * l[0][2], l1 = l[1][0] * l[1][0] + l[1][1] * l[1][1] + l[1][2] * l[1][2];
  if (!(ee > 1e-12f * l0 * l1)) return false;
  const float ie = 1.f / sqrtf(ee);
  for (int k = 0; k < 3; ++k) e[k] *= ie;
  skew_times(e, H, F);
  return true;
}

// plane-and-parallax draws per step: at most kPpMax, in chunks of kPpChunk with confidence stopping between chunks
constexpr int kPpMax = 1024, kPpChunk = 256;

// the positions in [0, m) of plane-and-parallax draw d after wave `wave`: the counter RNG of the pair's seed on stream numbers
// 3 * 2^30 + 2^16 wave + d, above the 7-point (< 2^16) and local-optimisation (2^31 + 32 wave + it) streams (m >= 2, d < 2^16)
__host__ __device__ inline void pp_sample2(uint32_t seed, int wave, int d, int m, int pos[2]) {
  sample_distinct<2>(seed, 0xC0000000u + 65536u * static_cast<uint32_t>(wave) + static_cast<uint32_t>(d), m, pos);
}

}  // namespace gv
