// gv.cu - geometric verification on the GPU (dimb_gv_*): fundamental-matrix RANSAC over the matches of a batch of pairs, the step
// that follows _match_pairs in the reference (utils/geometric_verification.py:45-179 -> pydegensac.findFundamentalMatrix /
// cv2.findFundamentalMat, called per pair from matchers/matcher_base.py:298-340).  At hundreds of pairs per second per GPU the
// CPU estimator becomes the bottleneck of the pipeline (SURVEY 8f rank 4).
//
// Per pair: Hartley normalisation of the matched keypoints; H hypotheses (8 random correspondences each, counter-based RNG ->
// reproducible), each solved by the normalised 8-point algorithm and scored by its Sampson inlier count over all matches by ONE
// thread (gv_math.cuh); the best hypothesis is refitted twice by least squares on its inliers and the final inlier mask is written.
// Two estimators share that frame:
//   ransac8 (estimator 0): no adaptive stopping, every hypothesis runs in parallel, H = max(64, min(max_iters, 8192)).
//   lo-ransac (estimator 1): 7-point hypotheses (up to 3 models each) in waves of kLoWave; after each wave one CTA per pair adopts
//     the wave's best model if it beats the pair's best and runs local optimisation on it (inner RANSAC on 16-inlier least-squares
//     fits, each iterated 4 times), then applies confidence stopping.  Up to min(max_iters, 65536) hypotheses; every wave is
//     enqueued and a pair that has stopped returns at once, so nothing waits for the host.  The finalize step is shared.
//   degensac (estimator 3; 2 stays refused, as it was before degensac existed): lo-ransac's waves plus DEGENSAC's treatment of
//     dominant planes (Chum, Werner, Matas, CVPR 2005).  A 7-point model whose sample is dominated by a plane (gv::degenerate7) also
//     has that plane's H scored; when a wave's best H beats the pair's best H, plane and parallax (gv_pp_kernel) recovers
//     F = [e']_x H from pairs of the matches off that plane, and the best such F competes with the wave's best model for adoption and
//     local optimisation.
// RANSAC is stochastic in the reference too (pydegensac's own RNG), so parity is statistical: tests compare inlier sets on data
// with known geometry and against OpenCV on the same matches.  Every reduction runs in a fixed order (integer atomics only), so a
// pair's result is a function of its matches, its seed and the configuration alone: bitwise reproducible across calls and batches.
//
// dimb_gv_verify_dev adds what an image set needs after matching: keypoints straight from the float16 feature store, a seed per pair
// (independent of the pair's position in the call), and in the last pass of the finalize kernel the ordered compaction of the inlier
// rows of the match table plus the per-pair inlier gate.
#include <memory>
#include <vector>

#include "common.cuh"
#include "gv_math.cuh"

namespace {

struct GvPair {
  const void *k0, *k1;         // keypoints of image 0 / 1: (N,2) x,y, float32 or float16 (f16)
  const long long* matches;    // [n][2] indices into k0 / k1, or null: k0[i] <-> k1[i]
  const int* n_dev;            // device count (or null: n_host)
  int n_host, cap;
  unsigned seed;               // RNG stream of this pair
  int f16[2], round_fp16[2];   // per side: float16 keypoints / round float32 keypoints to fp16 first (the features.h5 round trip)
};

// Optional outputs of dimb_gv_verify_dev: the inlier rows of each match table in order, and the gated count.
struct GvCompact {
  long long* verified;  // [P][cap][2], or null: no compaction (the older entries)
  int* n_verified;      // [P]
  int min_inliers;
  float min_ratio;
};

__device__ __forceinline__ int gv_count(const GvPair& p) { return min(p.n_dev ? *p.n_dev : p.n_host, p.cap); }
__device__ __forceinline__ float gv_kpt(const void* k, long long i, int f16, int r16) {
  if (f16) return __half2float(static_cast<const __half*>(k)[i]);
  const float v = static_cast<const float*>(k)[i];
  return r16 ? __half2float(__float2half_rn(v)) : v;
}
__device__ __forceinline__ void gv_point(const GvPair& p, int i, float& x0, float& y0, float& x1, float& y1) {
  const long long a = p.matches ? p.matches[2 * i] : i, b = p.matches ? p.matches[2 * i + 1] : i;
  x0 = gv_kpt(p.k0, 2 * a, p.f16[0], p.round_fp16[0]), y0 = gv_kpt(p.k0, 2 * a + 1, p.f16[0], p.round_fp16[0]);
  x1 = gv_kpt(p.k1, 2 * b, p.f16[1], p.round_fp16[1]), y1 = gv_kpt(p.k1, 2 * b + 1, p.f16[1], p.round_fp16[1]);
}
// the gate of dimb_gv_verify_dev (float32 comparison of the ratio, as documented in dimb200.h)
__device__ __forceinline__ bool gv_gate(int n_inl, int n_raw, const GvCompact& c) {
  return n_inl >= c.min_inliers && static_cast<float>(n_inl) >= c.min_ratio * static_cast<float>(n_raw);
}

// one CTA per pair: centroid + mean distance of both point sets -> Hartley normalisations; packed coordinates [cap][4]
__global__ void gv_prepare_kernel(const GvPair* pairs, float* xy, gv::Norm* norms, unsigned long long* best, int cap) {
  const GvPair p = pairs[blockIdx.x];
  const int n = gv_count(p), t = threadIdx.x;
  float* out = xy + static_cast<size_t>(blockIdx.x) * cap * 4;
  __shared__ float red[4][32];
  __shared__ float mean[4];
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = t; i < n; i += blockDim.x) {
    float c[4];
    gv_point(p, i, c[0], c[1], c[2], c[3]);
    for (int k = 0; k < 4; ++k) out[4 * i + k] = c[k], s[k] += c[k];
  }
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if ((t & 31) == 0) red[k][t >> 5] = s[k];
  }
  __syncthreads();
  if (t < 4) {
    float a = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) a += red[t][w];
    mean[t] = n ? a / n : 0.f;
  }
  __syncthreads();
  float d[2] = {0.f, 0.f};
  for (int i = t; i < n; i += blockDim.x) {
    d[0] += sqrtf((out[4 * i] - mean[0]) * (out[4 * i] - mean[0]) + (out[4 * i + 1] - mean[1]) * (out[4 * i + 1] - mean[1]));
    d[1] += sqrtf((out[4 * i + 2] - mean[2]) * (out[4 * i + 2] - mean[2]) + (out[4 * i + 3] - mean[3]) * (out[4 * i + 3] - mean[3]));
  }
  __syncthreads();
  for (int k = 0; k < 2; ++k) {
    for (int o = 16; o; o >>= 1) d[k] += __shfl_xor_sync(0xffffffffu, d[k], o);
    if ((t & 31) == 0) red[k][t >> 5] = d[k];
  }
  __syncthreads();
  if (t < 2) {
    float a = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) a += red[t][w];
    const float md = n ? a / n : 1.f;
    norms[2 * blockIdx.x + t] = gv::Norm{mean[2 * t], mean[2 * t + 1], md > 0.f ? 1.41421356f / md : 1.f};
  }
  if (t == 0) best[blockIdx.x] = 0ull;
}

// grid (ceil(H / 128), P): one hypothesis per thread; best = max over (inliers << 32 | ~hyp) (ties -> lowest hypothesis index)
__global__ void gv_hypotheses_kernel(const GvPair* pairs, const float* xy, const gv::Norm* norms, unsigned long long* best, int cap, int H,
                                     float thr2) {
  const int pi = blockIdx.y, h = blockIdx.x * blockDim.x + threadIdx.x;
  const GvPair p = pairs[pi];
  const int n = gv_count(p);
  if (n < 8 || h >= H) return;
  const float* pts = xy + static_cast<size_t>(pi) * cap * 4;
  int idx[8];
  gv::sample8(p.seed, h, n, idx);
  float k0[16], k1[16];
  int id8[8];
  for (int k = 0; k < 8; ++k) {
    k0[2 * k] = pts[4 * idx[k]], k0[2 * k + 1] = pts[4 * idx[k] + 1], k1[2 * k] = pts[4 * idx[k] + 2], k1[2 * k + 1] = pts[4 * idx[k] + 3];
    id8[k] = k;
  }
  float F[9];
  if (!gv::eight_point(k0, k1, id8, norms[2 * pi], norms[2 * pi + 1], F)) return;
  int cnt = 0;
  const float4* p4 = reinterpret_cast<const float4*>(pts);
  for (int i = 0; i < n; ++i) {
    const float4 c = __ldg(p4 + i);
    cnt += gv::sampson2(F, c.x, c.y, c.z, c.w) < thr2;
  }
  atomicMax(&best[pi], (static_cast<unsigned long long>(cnt) << 32) | (0xffffffffu - static_cast<unsigned>(h)));
}

// one CTA per pair: best hypothesis -> two least-squares refits on its inliers -> mask, count, F; with cmp.verified also the inlier
// rows of the match table in order (ballot + warp prefix + block prefix per 256-row chunk) and the gated count
constexpr int kFinThreads = 256, kFinWarps = kFinThreads / 32;

// lo-ransac state of one pair (zeroed before the first wave)
struct GvLo {
  unsigned long long wave_key;  // best (count << 32 | ~(3 h + root)) of the current wave; 0: no model yet
  float F[9];                   // the adopted model; its count is best[pair] >> 32
  int lim;                      // hypotheses the pair runs: min(H, the confidence bound of its best model); 0 before the first wave
  int run;                      // hypotheses run so far
  int done;
};
constexpr int kLoWave = 1024, kLoMaxIters = 65536, kLoInner = 20, kLoSample = 16, kLoLsq = 4;
__device__ __forceinline__ int gv_lo_lim(const GvLo& s, int H) { return s.lim ? s.lim : H; }

// degensac state of one pair next to its GvLo (zeroed before the first wave)
struct GvDeg {
  unsigned long long wave_hkey;  // best (H count << 32 | ~(3 h + root)) of the current wave's plane-dominated models; 0: none
  int hbest;                     // the best H count the pair has seen
  int pp_cnt;                    // Sampson count of the plane-and-parallax model of the current wave, -1: none
  float F[9];                    // that model
};
static_assert(gv::kPpChunk == kFinThreads, "gv_pp_kernel runs one plane-and-parallax draw per thread and chunk");


// kLo: the model is the one lo-ransac adopted (lo[pair].F) rather than hypothesis best[pair] re-solved
template <bool kLo>
__global__ void __launch_bounds__(kFinThreads)
gv_finalize_kernel(const GvPair* pairs, const float* xy, const gv::Norm* norms, const unsigned long long* best, int cap, float thr2,
                   float* Fout, unsigned char* mask, int* n_inl, GvCompact cmp, const GvLo* lo) {
  const int pi = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const GvPair p = pairs[pi];
  const int n = gv_count(p);
  unsigned char* mk = mask + static_cast<size_t>(pi) * cap;
  float* Fo = Fout + 9 * pi;
  long long* vo = cmp.verified ? cmp.verified + static_cast<size_t>(pi) * cap * 2 : nullptr;
  __shared__ float F[9];
  __shared__ float Nm[45];
  __shared__ float part[kFinWarps][45];  // per-warp partials of the normal matrix, summed in warp order (no float atomics)
  __shared__ int wcnt[kFinWarps];
  __shared__ int ok, cnt;
  if (n < 8 || (best[pi] >> 32) < 8) {  // fewer than 8 matches / no usable model: every match stays (reference :107-111 returns all ones)
    for (int i = t; i < n; i += blockDim.x) {
      mk[i] = 1;
      if (vo) vo[2 * i] = p.matches[2 * i], vo[2 * i + 1] = p.matches[2 * i + 1];
    }
    if (t < 9) Fo[t] = 0.f;
    if (t == 0) {
      n_inl[pi] = n;
      if (vo) cmp.n_verified[pi] = gv_gate(n, n, cmp) ? n : 0;
    }
    return;
  }
  const gv::Norm n0 = norms[2 * pi], n1 = norms[2 * pi + 1];
  const float* pts = xy + static_cast<size_t>(pi) * cap * 4;
  if (kLo) {
    if (t < 9) F[t] = lo[pi].F[t];
  } else if (t == 0) {
    const unsigned h = 0xffffffffu - static_cast<unsigned>(best[pi] & 0xffffffffu);
    int idx[8], id8[8];
    float k0[16], k1[16], f[9];
    gv::sample8(p.seed, h, n, idx);
    for (int k = 0; k < 8; ++k) {
      k0[2 * k] = pts[4 * idx[k]], k0[2 * k + 1] = pts[4 * idx[k] + 1], k1[2 * k] = pts[4 * idx[k] + 2], k1[2 * k + 1] = pts[4 * idx[k] + 3];
      id8[k] = k;
    }
    gv::eight_point(k0, k1, id8, n0, n1, f);
    for (int k = 0; k < 9; ++k) F[k] = f[k];
  }
  __syncthreads();
  for (int round = 0; round < 2; ++round) {
    if (t == 0) cnt = 0;
    __syncthreads();
    float acc[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) acc[k] = 0.f;
    int c = 0;
    for (int i = t; i < n; i += blockDim.x) {
      const float x0 = pts[4 * i], y0 = pts[4 * i + 1], x1 = pts[4 * i + 2], y1 = pts[4 * i + 3];
      if (gv::sampson2(F, x0, y0, x1, y1) < thr2) {
        const float u0 = (x0 - n0.cx) * n0.s, v0 = (y0 - n0.cy) * n0.s, u1 = (x1 - n1.cx) * n1.s, v1 = (y1 - n1.cy) * n1.s;
        const float a[9] = {u1 * u0, u1 * v0, u1, v1 * u0, v1 * v0, v1, u0, v0, 1.f};
        int k = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r)
#pragma unroll
          for (int q = r; q < 9; ++q) acc[k++] += a[r] * a[q];
        ++c;
      }
    }
#pragma unroll
    for (int k = 0; k < 45; ++k) {
      float v = acc[k];
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) part[wid][k] = v;
    }
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) atomicAdd(&cnt, c);
    __syncthreads();
    if (t < 45) {
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < kFinWarps; ++w) a += part[w][t];
      Nm[t] = a;
    }
    __syncthreads();
    if (t == 0) {
      ok = 0;
      if (cnt >= 8) {
        float N9[9][9], f[9];
        int k = 0;
        for (int r = 0; r < 9; ++r)
          for (int q = r; q < 9; ++q) N9[r][q] = N9[q][r] = Nm[k++];
        if (gv::refit_from_normal(N9, n0, n1, f)) {
          // keep the refit only if it does not lose inliers (checked below by the caller loop: count with the new model)
          for (int j = 0; j < 9; ++j) Nm[j] = f[j];
          ok = 1;
        }
      }
    }
    __syncthreads();
    if (ok) {  // candidate model in Nm[0..8]: accept if it explains at least as many matches
      __shared__ int c_new;
      if (t == 0) c_new = 0;
      __syncthreads();
      float f[9];
      for (int j = 0; j < 9; ++j) f[j] = Nm[j];
      int cn = 0;
      for (int i = t; i < n; i += blockDim.x) cn += gv::sampson2(f, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]) < thr2;
      for (int o = 16; o; o >>= 1) cn += __shfl_xor_sync(0xffffffffu, cn, o);
      if ((t & 31) == 0) atomicAdd(&c_new, cn);
      __syncthreads();
      if (t < 9 && c_new >= cnt) F[t] = f[t];
      __syncthreads();
    }
  }
  // last pass, in chunks of kFinThreads rows: mask; prefix of the inlier flags -> output row of each inlier (order kept)
  int total = 0;
  for (int base = 0; base < n; base += kFinThreads) {
    const int i = base + t;
    const bool in = i < n && gv::sampson2(F, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]) < thr2;
    if (i < n) mk[i] = in;
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) wcnt[wid] = __popc(bal);
    __syncthreads();
    int off = total + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) off += wcnt[w];
    if (in && vo) vo[2 * off] = p.matches[2 * i], vo[2 * off + 1] = p.matches[2 * i + 1];
    for (int w = 0; w < kFinWarps; ++w) total += wcnt[w];
    __syncthreads();  // wcnt is rewritten by the next chunk
  }
  if (t < 9) Fo[t] = F[t];
  if (t == 0) {
    n_inl[pi] = total;
    if (vo) cmp.n_verified[pi] = gv_gate(total, n, cmp) ? total : 0;
  }
}

// ------------------------------------------------------------------ lo-ransac
// grid (kLoWave / 128, P): hypothesis h = wave * kLoWave + thread of the pair's wave, for h < its limit; 7 points, up to 3 models,
// each scored over all matches; wave_key = max over (count << 32 | ~(3 h + root)) (ties -> lowest hypothesis, then lowest root).
// kDeg (degensac): the first model of the hypothesis that gv::degenerate7 finds dominated by a plane also has that plane's H scored
// (matches within gv::kDegHFactor * threshold transfer error) into deg[pair].wave_hkey, keyed as wave_key.
template <bool kDeg>
__global__ void __launch_bounds__(128)
gv_lo_hypotheses_kernel(const GvPair* pairs, const float* xy, const gv::Norm* norms, GvLo* lo, int cap, int wave, int H, float thr2,
                        GvDeg* deg) {
  const int pi = blockIdx.y, h = wave * kLoWave + blockIdx.x * blockDim.x + threadIdx.x;
  GvLo& s = lo[pi];
  if (s.done) return;
  const GvPair p = pairs[pi];
  const int n = gv_count(p);
  if (n < 8 || h >= gv_lo_lim(s, H)) return;
  const float* pts = xy + static_cast<size_t>(pi) * cap * 4;
  int idx[7], id7[7];
  gv::sample7(p.seed, h, n, idx);
  float k0[14], k1[14];
  for (int k = 0; k < 7; ++k) {
    k0[2 * k] = pts[4 * idx[k]], k0[2 * k + 1] = pts[4 * idx[k] + 1], k1[2 * k] = pts[4 * idx[k] + 2], k1[2 * k + 1] = pts[4 * idx[k] + 3];
    id7[k] = k;
  }
  float F[3][9];
  float Hp[9];
  int hr = -1;  // kDeg: the model whose plane H (pixels) is scored
  int m;
  if constexpr (kDeg) {
    const gv::Norm n0 = norms[2 * pi], n1 = norms[2 * pi + 1];
    float u[7][4];
    m = gv::seven_point(k0, k1, id7, n0, n1, F);
    for (int k = 0; k < 7; ++k)
      u[k][0] = (k0[2 * k] - n0.cx) * n0.s, u[k][1] = (k0[2 * k + 1] - n0.cy) * n0.s, u[k][2] = (k1[2 * k] - n1.cx) * n1.s,
      u[k][3] = (k1[2 * k + 1] - n1.cy) * n1.s;
    for (int r = 0; r < m; ++r) {
      float Fn[9], Hn[9];
      gv::normalise_f(F[r], n0, n1, Fn);
      if (gv::degenerate7(Fn, u, gv::deg_t2n(thr2, n1), Hn) < 0) continue;
      if (gv::h_denormalise(Hn, n0, n1, Hp)) hr = r;
      break;
    }
  } else {
    m = gv::seven_point(k0, k1, id7, norms[2 * pi], norms[2 * pi + 1], F);
  }
  if (m == 0) return;
  int cnt[3] = {0, 0, 0}, hc = 0;
  const float4* p4 = reinterpret_cast<const float4*>(pts);
  for (int i = 0; i < n; ++i) {
    const float4 c = __ldg(p4 + i);
#pragma unroll
    for (int r = 0; r < 3; ++r)
      if (r < m) cnt[r] += gv::sampson2(F[r], c.x, c.y, c.z, c.w) < thr2;
    if constexpr (kDeg)
      if (hr >= 0) hc += gv::transfer2(Hp, c.x, c.y, c.z, c.w) < gv::kDegHFactor * gv::kDegHFactor * thr2;
  }
  unsigned long long key = 0ull;
  for (int r = 0; r < m; ++r)
    key = max(key, (static_cast<unsigned long long>(cnt[r]) << 32) | (0xffffffffu - static_cast<unsigned>(3 * h + r)));
  atomicMax(&s.wave_key, key);
  if constexpr (kDeg)
    if (hr >= 0)
      atomicMax(&deg[pi].wave_hkey, (static_cast<unsigned long long>(hc) << 32) | (0xffffffffu - static_cast<unsigned>(3 * h + hr)));
}

// CTA-wide count of the matches whose Sampson distance to F is below thr2 and, with `normal`, the sum of their normal-matrix rows
// into Nm (45 upper-triangular entries).  Per-thread partials, warp shuffles, warps summed in order: a fixed order, no float atomics.
// Every thread gets the count.
__device__ int gv_lo_sums(const float* Fs, const float* pts, int n, float thr2, gv::Norm n0, gv::Norm n1, bool normal,
                          float (*part)[45], int* wcnt, float* Nm) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  float f[9];
  for (int j = 0; j < 9; ++j) f[j] = Fs[j];
  float acc[45];
#pragma unroll
  for (int k = 0; k < 45; ++k) acc[k] = 0.f;
  int c = 0;
  for (int i = t; i < n; i += blockDim.x) {
    const float x0 = pts[4 * i], y0 = pts[4 * i + 1], x1 = pts[4 * i + 2], y1 = pts[4 * i + 3];
    if (gv::sampson2(f, x0, y0, x1, y1) < thr2) {
      ++c;
      if (normal) {
        float a[9];
        gv::normal_row(x0, y0, x1, y1, n0, n1, a);
        int k = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r)
#pragma unroll
          for (int q = r; q < 9; ++q) acc[k++] += a[r] * a[q];
      }
    }
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) wcnt[wid] = c;
  if (normal) {
#pragma unroll
    for (int k = 0; k < 45; ++k) {
      float v = acc[k];
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) part[wid][k] = v;
    }
  }
  __syncthreads();
  if (normal && t < 45) {
    float a = 0.f;
    for (int w = 0; w < kFinWarps; ++w) a += part[w][t];
    Nm[t] = a;
  }
  int total = 0;
  for (int w = 0; w < kFinWarps; ++w) total += wcnt[w];
  __syncthreads();  // wcnt / part are rewritten by the next call; Nm is complete
  return total;
}

// the indices of the matches within thr2 of F, in order (ballot + warp prefix + block prefix per chunk), into out; returns their number
__device__ int gv_lo_inliers(const float* Fs, const float* pts, int n, float thr2, int* out, int* wcnt) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  float f[9];
  for (int j = 0; j < 9; ++j) f[j] = Fs[j];
  int total = 0;
  for (int base = 0; base < n; base += kFinThreads) {
    const int i = base + t;
    const bool in = i < n && gv::sampson2(f, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]) < thr2;
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) wcnt[wid] = __popc(bal);
    __syncthreads();
    int off = total + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) off += wcnt[w];
    if (in) out[off] = i;
    for (int w = 0; w < kFinWarps; ++w) total += wcnt[w];
    __syncthreads();
  }
  return total;
}

// refit_from_normal on the 45 sums Nm (one thread)
__device__ bool gv_lo_refit(const float* Nm, gv::Norm n0, gv::Norm n1, float f[9]) {
  float N9[9][9];
  int k = 0;
  for (int r = 0; r < 9; ++r)
    for (int q = r; q < 9; ++q) N9[r][q] = N9[q][r] = Nm[k++];
  return gv::refit_from_normal(N9, n0, n1, f);
}

// one CTA per running pair, after the hypotheses of wave `wave`: adopt the wave's best model if it beats the pair's best, then local
// optimisation - kLoInner times: the inliers at 2x the threshold (fewer than kLoSample: stop), a least-squares fit of kLoSample of them
// drawn on the LO stream, kLoLsq least-squares refits on that fit's inliers, the result adopted if it explains more matches.  Then
// confidence stopping: the pair is done once it has run min(its limit, the hypotheses its best model calls for).  inl: [P][cap] scratch.
// kDeg (degensac): the wave's plane-and-parallax model (deg[pair]) is adopted instead when it explains at least 8 matches and at least
// as many as the pair's best and the wave's best model.
template <bool kDeg>
__global__ void __launch_bounds__(kFinThreads)
gv_lo_kernel(const GvPair* pairs, const float* xy, const gv::Norm* norms, unsigned long long* best, GvLo* lo, int* inl, int cap, int wave,
             int H, float thr2, float confidence, const GvDeg* deg) {
  const int pi = blockIdx.x, t = threadIdx.x;
  GvLo* s = lo + pi;
  if (s->done) return;
  const GvPair p = pairs[pi];
  const int n = gv_count(p), lim = gv_lo_lim(*s, H);
  if (n < 8) {  // finalize keeps every match; no hypothesis ran
    if (t == 0) s->done = 1;
    return;
  }
  const gv::Norm n0 = norms[2 * pi], n1 = norms[2 * pi + 1];
  const float* pts = xy + static_cast<size_t>(pi) * cap * 4;
  __shared__ float F[9], G[9], Nm[45];
  __shared__ float part[kFinWarps][45];
  __shared__ int wcnt[kFinWarps];
  __shared__ int adopt, ok, cur;
  if (t == 0) {
    const unsigned long long key = s->wave_key;
    s->wave_key = 0ull;
    cur = static_cast<int>(best[pi] >> 32);
    bool pp = false;
    if constexpr (kDeg) {
      const int pc = deg[pi].pp_cnt;
      pp = pc >= 8 && pc >= cur && pc >= static_cast<int>(key >> 32);
      if (pp) {
        for (int j = 0; j < 9; ++j) F[j] = deg[pi].F[j];
        cur = pc;
      }
    }
    adopt = pp || (key != 0ull && static_cast<int>(key >> 32) > cur);
    if (adopt && !pp) {  // re-solve the winning hypothesis
      const unsigned id = 0xffffffffu - static_cast<unsigned>(key & 0xffffffffu);
      int idx[7], id7[7];
      float k0[14], k1[14], M[3][9];
      gv::sample7(p.seed, id / 3, n, idx);
      for (int k = 0; k < 7; ++k) {
        k0[2 * k] = pts[4 * idx[k]], k0[2 * k + 1] = pts[4 * idx[k] + 1], k1[2 * k] = pts[4 * idx[k] + 2], k1[2 * k + 1] = pts[4 * idx[k] + 3];
        id7[k] = k;
      }
      gv::seven_point(k0, k1, id7, n0, n1, M);
      for (int j = 0; j < 9; ++j) F[j] = M[id % 3][j];
      cur = static_cast<int>(key >> 32);
    }
  }
  __syncthreads();
  if (adopt) {
    int* list = inl + static_cast<size_t>(pi) * cap;
    for (int it = 0; it < kLoInner; ++it) {
      const int m = gv_lo_inliers(F, pts, n, 4.f * thr2, list, wcnt);
      if (m < kLoSample) break;
      if (t == 0) {
        int pos[kLoSample];
        gv::lo_sample16(p.seed, wave, it, m, pos);
        float N9[9][9] = {}, f[9];
        for (int k = 0; k < kLoSample; ++k) {
          const int i = list[pos[k]];
          float a[9];
          gv::normal_row(pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3], n0, n1, a);
          for (int r = 0; r < 9; ++r)
            for (int q = 0; q < 9; ++q) N9[r][q] += a[r] * a[q];
        }
        ok = gv::refit_from_normal(N9, n0, n1, f);
        if (ok)
          for (int j = 0; j < 9; ++j) G[j] = f[j];
      }
      __syncthreads();
      if (!ok) continue;
      for (int r = 0; r < kLoLsq; ++r) {
        const int c = gv_lo_sums(G, pts, n, thr2, n0, n1, true, part, wcnt, Nm);
        if (t == 0) {
          float f[9];
          ok = c >= 8 && gv_lo_refit(Nm, n0, n1, f);
          if (ok)
            for (int j = 0; j < 9; ++j) G[j] = f[j];
        }
        __syncthreads();
        if (!ok) break;
      }
      const int c = gv_lo_sums(G, pts, n, thr2, n0, n1, false, part, wcnt, Nm);
      if (t == 0 && c > cur) {
        cur = c;
        for (int j = 0; j < 9; ++j) F[j] = G[j];
      }
      __syncthreads();
    }
  }
  if (t == 0) {
    if (adopt) {
      best[pi] = static_cast<unsigned long long>(cur) << 32;
      for (int j = 0; j < 9; ++j) s->F[j] = F[j];
    }
    const int run = min(lim, (wave + 1) * kLoWave), need = min(lim, gv::lo_needed(cur, n, confidence, H));
    s->run = run;
    s->lim = need;
    s->done = run >= need;
  }
}

// ------------------------------------------------------------------ degensac
// The indices of the matches whose squared transfer error to H (pixels) is not below t2, in order (as gv_lo_inliers); their number.
__device__ int gv_pp_outside(const float* Hs, const float* pts, int n, float t2, int* out, int* wcnt) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  float h[9];
  for (int j = 0; j < 9; ++j) h[j] = Hs[j];
  int total = 0;
  for (int base = 0; base < n; base += kFinThreads) {
    const int i = base + t;
    const bool off = i < n && !(gv::transfer2(h, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]) < t2);
    const unsigned bal = __ballot_sync(0xffffffffu, off);
    if (lane == 0) wcnt[wid] = __popc(bal);
    __syncthreads();
    int o = total + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) o += wcnt[w];
    if (off) out[o] = i;
    for (int w = 0; w < kFinWarps; ++w) total += wcnt[w];
    __syncthreads();
  }
  return total;
}

// one CTA per running pair, between the hypotheses and gv_lo_kernel of wave `wave`: if the wave's best H beats the pair's best H, plane
// and parallax on it - the m matches off the plane in order, up to gv::kPpMax draws of two of them (one per thread in chunks of
// gv::kPpChunk, stream gv::pp_sample2), F = [e']_x H of each scored by its Sampson count over all matches; the best (lowest draw on
// ties) into deg[pair].  Between chunks, confidence stopping on the off-plane inlier fraction (count - (n - m)) / m of 2-point samples.
// inl: [P][cap] scratch (gv_lo_kernel reuses it after).
__global__ void __launch_bounds__(kFinThreads)
gv_pp_kernel(const GvPair* pairs, const float* xy, const gv::Norm* norms, const GvLo* lo, GvDeg* deg, int* inl, int cap, int wave,
             float thr2, float confidence) {
  const int pi = blockIdx.x, t = threadIdx.x;
  if (lo[pi].done) return;
  GvDeg* d = deg + pi;
  const GvPair p = pairs[pi];
  const int n = gv_count(p);
  const gv::Norm n0 = norms[2 * pi], n1 = norms[2 * pi + 1];
  const float* pts = xy + static_cast<size_t>(pi) * cap * 4;
  __shared__ float Hn[9], Hp[9], Fb[9];
  __shared__ int wcnt[kFinWarps];
  __shared__ int go;
  __shared__ unsigned long long ckey;
  if (t == 0) {
    const unsigned long long key = d->wave_hkey;
    d->wave_hkey = 0ull;
    d->pp_cnt = -1;
    go = 0;
    if (key != 0ull && static_cast<int>(key >> 32) > d->hbest) {  // re-solve the winning model's plane
      d->hbest = static_cast<int>(key >> 32);
      const unsigned id = 0xffffffffu - static_cast<unsigned>(key & 0xffffffffu);
      int idx[7], id7[7];
      float k0[14], k1[14], M[3][9], Mn[9], u[7][4], h[9];
      gv::sample7(p.seed, id / 3, n, idx);
      for (int k = 0; k < 7; ++k) {
        k0[2 * k] = pts[4 * idx[k]], k0[2 * k + 1] = pts[4 * idx[k] + 1], k1[2 * k] = pts[4 * idx[k] + 2], k1[2 * k + 1] = pts[4 * idx[k] + 3];
        id7[k] = k;
        u[k][0] = (k0[2 * k] - n0.cx) * n0.s, u[k][1] = (k0[2 * k + 1] - n0.cy) * n0.s, u[k][2] = (k1[2 * k] - n1.cx) * n1.s,
        u[k][3] = (k1[2 * k + 1] - n1.cy) * n1.s;
      }
      const int m = gv::seven_point(k0, k1, id7, n0, n1, M);
      const int r = static_cast<int>(id % 3);
      if (r < m) gv::normalise_f(M[r], n0, n1, Mn);
      if (r < m && gv::degenerate7(Mn, u, gv::deg_t2n(thr2, n1), h) >= 0) {
        float g[9];
        go = gv::h_denormalise(h, n0, n1, g);
        for (int j = 0; j < 9; ++j) Hn[j] = h[j], Hp[j] = g[j];
      }
    }
  }
  __syncthreads();
  if (!go) return;
  int* list = inl + static_cast<size_t>(pi) * cap;
  const int m = gv_pp_outside(Hp, pts, n, gv::kDegHFactor * gv::kDegHFactor * thr2, list, wcnt);
  if (m < 2) return;
  float h[9];
  for (int j = 0; j < 9; ++j) h[j] = Hn[j];
  const float4* p4 = reinterpret_cast<const float4*>(pts);
  unsigned long long bkey = 0ull;  // best (count << 32 | ~draw) so far; 0: no model
  int need = gv::kPpMax;
  for (int base = 0; base < need; base += gv::kPpChunk) {
    const int dr = base + t;
    int pos[2];
    gv::pp_sample2(p.seed, wave, dr, m, pos);
    float a[4], b[4], fn[9], f[9];
    for (int s = 0; s < 2; ++s) {
      const int i = list[pos[s]];
      float* c = s ? b : a;
      c[0] = (pts[4 * i] - n0.cx) * n0.s, c[1] = (pts[4 * i + 1] - n0.cy) * n0.s, c[2] = (pts[4 * i + 2] - n1.cx) * n1.s,
      c[3] = (pts[4 * i + 3] - n1.cy) * n1.s;
    }
    unsigned long long key = 0ull;
    if (gv::plane_parallax(h, a, b, fn) && gv::denormalise(fn, n0, n1, f)) {
      int c = 0;
      for (int i = 0; i < n; ++i) {
        const float4 q = __ldg(p4 + i);
        c += gv::sampson2(f, q.x, q.y, q.z, q.w) < thr2;
      }
      key = (static_cast<unsigned long long>(c) << 32) | (0xffffffffu - static_cast<unsigned>(dr));
    }
    if (t == 0) ckey = 0ull;
    __syncthreads();
    atomicMax(&ckey, key);
    __syncthreads();
    const unsigned long long top = ckey;
    if (key != 0ull && key == top && top > bkey)
      for (int j = 0; j < 9; ++j) Fb[j] = f[j];
    bkey = max(bkey, top);
    const int bc = bkey ? static_cast<int>(bkey >> 32) : -1;
    need = gv::ransac_needed<2>(max(0, bc - (n - m)), m, confidence, gv::kPpMax);
    __syncthreads();  // Fb complete; ckey is reset by the next chunk
  }
  if (t == 0 && bkey) {
    d->pp_cnt = static_cast<int>(bkey >> 32);
    for (int j = 0; j < 9; ++j) d->F[j] = Fb[j];
  }
}

// The estimator of a gv_run call: 0 ransac8, 1 lo-ransac, 3 degensac (confidence read by lo-ransac and degensac only).  lo_slot,
// lo_slot + 1: the context scratch slots of lo-ransac's state, also used by degensac (52 for dimb_gv_estimate, 54 for
// dimb_gv_verify_dev); deg_slot: degensac's state (56 / 57).  gv_run's d_lo (optional) receives the address of the per-pair lo-ransac
// state, whose `run` is the hypotheses count.
struct GvEstimator {
  int kind, max_iters;
  float confidence;
  int lo_slot, deg_slot;
};

int gv_check_estimator(const dimb_gv_conf& c) {
  if (c.estimator == 0) return DIMB_OK;
  if ((c.estimator != 1 && c.estimator != 3) || !(c.confidence > 0.f && c.confidence < 1.f) || c.max_iters < 1) return DIMB_ERR_ARG;
  return DIMB_OK;
}

// slot0 .. slot0 + 3: the context scratch slots of the calling entry (40 for the float32 entries, 48 for dimb_gv_verify_dev)
int gv_run(dimb_ctx* ctx, cudaStream_t st, const std::vector<GvPair>& hp, int cap, float threshold, const GvEstimator& est, float* d_F,
           unsigned char* d_mask, int* d_ninl, const GvCompact& cmp, int slot0, GvLo** d_lo = nullptr) {
  const int P = static_cast<int>(hp.size());
  GvPair* d_pairs;
  float* d_xy;
  gv::Norm* d_norm;
  unsigned long long* d_best;
  DIMB_TRY(dimb_scratch(ctx, slot0, P * sizeof(GvPair), reinterpret_cast<void**>(&d_pairs)));
  DIMB_TRY(dimb_scratch(ctx, slot0 + 1, static_cast<size_t>(P) * cap * 4 * sizeof(float), reinterpret_cast<void**>(&d_xy)));
  DIMB_TRY(dimb_scratch(ctx, slot0 + 2, 2 * P * sizeof(gv::Norm), reinterpret_cast<void**>(&d_norm)));
  DIMB_TRY(dimb_scratch(ctx, slot0 + 3, P * sizeof(unsigned long long), reinterpret_cast<void**>(&d_best)));
  GvLo* lo = nullptr;
  GvDeg* deg = nullptr;
  int* d_inl = nullptr;
  if (est.kind != 0) {
    DIMB_TRY(dimb_scratch(ctx, est.lo_slot, P * sizeof(GvLo), reinterpret_cast<void**>(&lo)));
    DIMB_TRY(dimb_scratch(ctx, est.lo_slot + 1, static_cast<size_t>(P) * cap * sizeof(int), reinterpret_cast<void**>(&d_inl)));
    if (d_lo) *d_lo = lo;
  }
  if (est.kind == 3) DIMB_TRY(dimb_scratch(ctx, est.deg_slot, P * sizeof(GvDeg), reinterpret_cast<void**>(&deg)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_pairs, hp.data(), P * sizeof(GvPair), cudaMemcpyHostToDevice, st));
  const float thr2 = threshold * threshold;
  if (est.kind == 1) {
    const int H = std::min(est.max_iters, kLoMaxIters);
    ProfScope prof(ctx, st, "gv.lo_ransac");
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(lo, 0, P * sizeof(GvLo), st));
    gv_prepare_kernel<<<P, 256, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap);
    DIMB_LAUNCH_CHECK(ctx);
    for (int w = 0; w * kLoWave < H; ++w) {
      gv_lo_hypotheses_kernel<false><<<dim3(kLoWave / 128, P), 128, 0, st>>>(d_pairs, d_xy, d_norm, lo, cap, w, H, thr2, nullptr);
      DIMB_LAUNCH_CHECK(ctx);
      gv_lo_kernel<false><<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, d_best, lo, d_inl, cap, w, H, thr2, est.confidence, nullptr);
      DIMB_LAUNCH_CHECK(ctx);
    }
    gv_finalize_kernel<true><<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap, thr2, d_F, d_mask, d_ninl, cmp, lo);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  }
  if (est.kind == 3) {
    const int H = std::min(est.max_iters, kLoMaxIters);
    ProfScope prof(ctx, st, "gv.degensac");
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(lo, 0, P * sizeof(GvLo), st));
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(deg, 0, P * sizeof(GvDeg), st));
    gv_prepare_kernel<<<P, 256, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap);
    DIMB_LAUNCH_CHECK(ctx);
    for (int w = 0; w * kLoWave < H; ++w) {
      gv_lo_hypotheses_kernel<true><<<dim3(kLoWave / 128, P), 128, 0, st>>>(d_pairs, d_xy, d_norm, lo, cap, w, H, thr2, deg);
      DIMB_LAUNCH_CHECK(ctx);
      gv_pp_kernel<<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, lo, deg, d_inl, cap, w, thr2, est.confidence);
      DIMB_LAUNCH_CHECK(ctx);
      gv_lo_kernel<true><<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, d_best, lo, d_inl, cap, w, H, thr2, est.confidence, deg);
      DIMB_LAUNCH_CHECK(ctx);
    }
    gv_finalize_kernel<true><<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap, thr2, d_F, d_mask, d_ninl, cmp, lo);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  }
  const int H = std::max(64, std::min(est.max_iters, 8192));
  ProfScope prof(ctx, st, "gv.ransac");
  gv_prepare_kernel<<<P, 256, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap);
  DIMB_LAUNCH_CHECK(ctx);
  gv_hypotheses_kernel<<<dim3(ceil_div(H, 128), P), 128, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap, H, thr2);
  DIMB_LAUNCH_CHECK(ctx);
  gv_finalize_kernel<false><<<P, kFinThreads, 0, st>>>(d_pairs, d_xy, d_norm, d_best, cap, thr2, d_F, d_mask, d_ninl, cmp, nullptr);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace

extern "C" {

// Host entry: matched keypoints kpts0[i] <-> kpts1[i] (n,2) float32 pixels, verified with the estimator of conf (its gate fields are
// not read).  F [9] row-major with x1^T F x0 = 0 (zeros when n < 8 or no model was found - the reference returns F = None and an
// all-True mask then), mask [n] 0/1, n_inliers, n_hypotheses (optional): the hypotheses that ran.
int dimb_gv_estimate(dimb_ctx* ctx, const float* kpts0, const float* kpts1, int n, const dimb_gv_conf* conf, unsigned seed, float* F,
                     unsigned char* mask, int* n_inliers, int* n_hypotheses) {
  if (!ctx || n < 0 || (n > 0 && (!kpts0 || !kpts1)) || !conf || !F || !mask || !n_inliers || !(conf->threshold > 0.f))
    return DIMB_ERR_ARG;
  DIMB_TRY(gv_check_estimator(*conf));
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (n_hypotheses) *n_hypotheses = 0;
  if (n == 0) {
    for (int i = 0; i < 9; ++i) F[i] = 0.f;
    *n_inliers = 0;
    return DIMB_OK;
  }
  cudaStream_t st = 0;
  float *d_k0, *d_k1, *d_F;
  unsigned char* d_mask;
  int* d_n;
  DIMB_TRY(dimb_scratch(ctx, 44, static_cast<size_t>(n) * 2 * sizeof(float), reinterpret_cast<void**>(&d_k0)));
  DIMB_TRY(dimb_scratch(ctx, 45, static_cast<size_t>(n) * 2 * sizeof(float), reinterpret_cast<void**>(&d_k1)));
  DIMB_TRY(dimb_scratch(ctx, 46, 9 * sizeof(float) + sizeof(int), reinterpret_cast<void**>(&d_F)));
  DIMB_TRY(dimb_scratch(ctx, 47, n, reinterpret_cast<void**>(&d_mask)));
  d_n = reinterpret_cast<int*>(d_F + 9);
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_k0, kpts0, static_cast<size_t>(n) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_k1, kpts1, static_cast<size_t>(n) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
  std::vector<GvPair> hp(1);
  hp[0] = GvPair{d_k0, d_k1, nullptr, nullptr, n, n, seed, {0, 0}, {0, 0}};
  GvLo* d_lo = nullptr;
  DIMB_TRY(gv_run(ctx, st, hp, n, conf->threshold, GvEstimator{conf->estimator, conf->max_iters, conf->confidence, 52, 56}, d_F, d_mask, d_n,
                  GvCompact{}, 40, &d_lo));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(F, d_F, 9 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(n_inliers, d_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(mask, d_mask, n, cudaMemcpyDeviceToHost, st));
  if (n_hypotheses && d_lo) DIMB_CUDA_OK(ctx, cudaMemcpyAsync(n_hypotheses, &d_lo->run, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  if (n_hypotheses && !d_lo && n >= 8) *n_hypotheses = std::max(64, std::min(conf->max_iters, 8192));
  return DIMB_OK;
}

// ransac8 through dimb_gv_estimate
int dimb_gv_fundamental(dimb_ctx* ctx, const float* kpts0, const float* kpts1, int n, float threshold, int max_iters, unsigned seed, float* F,
                        unsigned char* mask, int* n_inliers) {
  const dimb_gv_conf conf{threshold, max_iters, 0, 0.f, 0, 0.f};
  return dimb_gv_estimate(ctx, kpts0, kpts1, n, &conf, seed, F, mask, n_inliers, nullptr);
}

// Batch on device buffers, asynchronous on `stream`: pair p verifies d_matches[p][0..d_n_matches[p]) (the output layout of
// dimb_lg_match_dev / dimb_pipe_*: [P][cap][2] int64, [P] counts) against the keypoint arrays d_kpts0[p] / d_kpts1[p] ((N,2) float32).
// Outputs (device): d_F [P][9], d_mask [P][cap] (0/1 per match), d_n_inliers [P].
int dimb_gv_fundamental_batch_dev(dimb_ctx* ctx, int P, const float* const* d_kpts0, const float* const* d_kpts1, const int64_t* d_matches,
                                  const int* d_n_matches, int cap, float threshold, int max_iters, unsigned seed, float* d_F,
                                  unsigned char* d_mask, int* d_n_inliers, void* stream) {
  if (!ctx || P < 1 || !d_kpts0 || !d_kpts1 || !d_matches || !d_n_matches || cap < 1 || !d_F || !d_mask || !d_n_inliers || threshold <= 0.f)
    return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  std::vector<GvPair> hp(P);
  for (int p = 0; p < P; ++p)
    hp[p] = GvPair{d_kpts0[p], d_kpts1[p], reinterpret_cast<const long long*>(d_matches) + static_cast<size_t>(p) * cap * 2, d_n_matches + p, 0, cap,
                   seed + 0x9E37u * static_cast<unsigned>(p), {0, 0}, {0, 0}};
  return gv_run(ctx, static_cast<cudaStream_t>(stream), hp, cap, threshold, GvEstimator{0, max_iters, 0.f, 0, 0}, d_F, d_mask, d_n_inliers,
                GvCompact{}, 40);
}

// P pairs of an image set, asynchronous on `stream`: keypoints from dimb_feats_dev (feature-store slots or float32 extractor
// outputs), one seed per pair, the inlier rows of each match table compacted in order and gated (contract in dimb200.h).
int dimb_gv_verify_dev(dimb_ctx* ctx, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                       const int* d_n_matches, int cap, const unsigned* seeds, const dimb_gv_conf* conf, int64_t* d_verified,
                       int* d_n_verified, float* d_F, unsigned char* d_mask, int* d_n_inliers, void* stream) {
  if (!ctx || P < 1 || !f0 || !f1 || !d_matches || !d_n_matches || cap < 1 || !seeds || !conf || !d_verified || !d_n_verified || !d_F ||
      !d_mask || !d_n_inliers)
    return DIMB_ERR_ARG;
  if (!(conf->threshold > 0.f) || conf->min_inliers < 0 || !(conf->min_inlier_ratio >= 0.f && conf->min_inlier_ratio <= 1.f))
    return DIMB_ERR_ARG;
  DIMB_TRY(gv_check_estimator(*conf));
  for (int p = 0; p < P; ++p)
    if (!f0[p].keypoints || !f1[p].keypoints) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  std::vector<GvPair> hp(P);
  for (int p = 0; p < P; ++p)
    hp[p] = GvPair{f0[p].keypoints, f1[p].keypoints, reinterpret_cast<const long long*>(d_matches) + static_cast<size_t>(p) * cap * 2,
                   d_n_matches + p, 0, cap, seeds[p], {f0[p].f16 ? 1 : 0, f1[p].f16 ? 1 : 0},
                   {f0[p].round_fp16 ? 1 : 0, f1[p].round_fp16 ? 1 : 0}};
  const GvCompact cmp{reinterpret_cast<long long*>(d_verified), d_n_verified, conf->min_inliers, conf->min_inlier_ratio};
  return gv_run(ctx, static_cast<cudaStream_t>(stream), hp, cap, conf->threshold,
                GvEstimator{conf->estimator, conf->max_iters, conf->confidence, 54, 57}, d_F, d_mask, d_n_inliers, cmp, 48);
}

}  // extern "C"
