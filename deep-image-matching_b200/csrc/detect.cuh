// detect.cuh - the dense-score-map -> keypoint-list machinery shared by the SuperPoint and ALIKED extractors:
// simple_nms (identical in both reference models: superpoint.py:47-63, aliked.py:66-89), threshold + border
// compaction in row-major order, and top-k selection (radix select + bitonic sort).
#pragma once
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kNmsTile = 64;
constexpr int kChunk = 4096;       // pixels per compaction chunk
constexpr int kSelThreads = 1024;
constexpr int kMaxTopK = 16384;

// ------------------------------------------------------------------ simple_nms (superpoint.py:47-63)
// Tile of 64x64 outputs + halo 5r; every stage is a separable (2r+1)^2 window max in shared memory.
// 1024 threads as 32 x 32 (one CTA per SM - shared memory bound - so the warps have to come from the CTA itself): loops run over (row, column) directly - no integer divisions in the hot loops.
template <int RT>  // RT > 0: compile-time radius (window in registers); RT = -1: runtime radius
__device__ __forceinline__ void win_max(const float* src, float* tmp, float* dst, int S, int PS, int k, int r_rt) {
  const int r = RT >= 0 ? RT : r_rt;
  // src valid on margin k-r; writes dst on margin k.  Each thread produces a run of 8 outputs from a register
  // sliding window (8 + 2r loads instead of 8 * (2r+1)).
  const int nthr = blockDim.x;
  {  // row pass: runs of 8 columns; lanes walk down the rows so that a warp's smem accesses hit 32 different rows
    const int rows = S - 2 * (k - r), cols = S - 2 * k, segs = (cols + 7) >> 3;
    for (int t = threadIdx.x; t < rows * segs; t += nthr) {
      const int seg = t / rows, i = k - r + (t - seg * rows);
      const int j0 = k + seg * 8, n = min(8, S - k - j0);
      const float* p = src + i * PS + j0;
      if (RT >= 0 && n == 8) {
        float w[8 + 2 * (RT >= 0 ? RT : 0)];
#pragma unroll
        for (int d = 0; d < 8 + 2 * RT; ++d) w[d] = p[d - RT];
#pragma unroll
        for (int o = 0; o < 8; ++o) {
          float m = w[o];
#pragma unroll
          for (int d = 1; d <= 2 * RT; ++d) m = fmaxf(m, w[o + d]);
          tmp[i * PS + j0 + o] = m;
        }
      } else {
        for (int o = 0; o < n; ++o) {
          float m = p[o];
          for (int d = 1; d <= r; ++d) m = fmaxf(m, fmaxf(p[o - d], p[o + d]));
          tmp[i * PS + j0 + o] = m;
        }
      }
    }
  }
  __syncthreads();
  {  // column pass: runs of 8 rows; lanes along columns (conflict-free)
    const int cols = S - 2 * k, segs = (cols + 7) >> 3;
    for (int t = threadIdx.x; t < cols * segs; t += nthr) {
      const int seg = t / cols, j = k + (t - seg * cols);
      const int i0 = k + seg * 8, n = min(8, S - k - i0);
      const float* p = tmp + i0 * PS + j;
      if (RT >= 0 && n == 8) {
        float w[8 + 2 * (RT >= 0 ? RT : 0)];
#pragma unroll
        for (int d = 0; d < 8 + 2 * RT; ++d) w[d] = p[(d - RT) * PS];
#pragma unroll
        for (int o = 0; o < 8; ++o) {
          float m = w[o];
#pragma unroll
          for (int d = 1; d <= 2 * RT; ++d) m = fmaxf(m, w[o + d]);
          dst[(i0 + o) * PS + j] = m;
        }
      } else {
        for (int o = 0; o < n; ++o) {
          float m = p[o * PS];
          for (int d = 1; d <= r; ++d) m = fmaxf(m, fmaxf(p[(o - d) * PS], p[(o + d) * PS]));
          dst[(i0 + o) * PS + j] = m;
        }
      }
    }
  }
  __syncthreads();
}

template <int RT>
__global__ void __launch_bounds__(1024) sp_nms_kernel(const float* __restrict__ scores, float* __restrict__ out, int H, int W, int r,
                                                     int T) {
  extern __shared__ float nsm[];
  const int S = T + 10 * r, PS = S | 1;  // odd row pitch: the row pass walks lanes down the rows, an even pitch costs 2-way bank conflicts
  float* s0 = nsm;             // scores, -inf outside the image
  float* xa = s0 + S * PS;     // mask-as-float / suppressed scores
  float* tmp = xa + S * PS;
  float* wm = tmp + S * PS;    // window max
  unsigned char* msk = reinterpret_cast<unsigned char*>(wm + S * PS);  // max_mask
  unsigned char* sup = msk + S * PS;                                   // supp_mask of the current round
  const int b = blockIdx.z, ty0 = blockIdx.y * T - 5 * r, tx0 = blockIdx.x * T - 5 * r;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, nty = blockDim.x >> 5;
  const float* sc = scores + static_cast<size_t>(b) * H * W;
  for (int i = ty; i < S; i += nty) {
    const int gy = ty0 + i;
    for (int j = tx; j < S; j += 32) {
      const int gx = tx0 + j;
      const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
      s0[i * PS + j] = in ? sc[static_cast<size_t>(gy) * W + gx] : -INFINITY;
    }
  }
  __syncthreads();
  // max_mask = scores == max_pool(scores)                              margin r
  win_max<RT>(s0, tmp, wm, S, PS, r, r);
  for (int i = ty; i < S; i += nty)
    for (int j = tx; j < S; j += 32) {
      const int e = i * PS + j;
      const bool v = i >= r && i < S - r && j >= r && j < S - r;
      const bool in = s0[e] != -INFINITY;  // inside the image (scores are softmax outputs > 0)
      const unsigned char m = (v && in && s0[e] == wm[e]) ? 1 : 0;
      msk[e] = m;
      xa[e] = m ? 1.f : 0.f;
    }
  __syncthreads();
  for (int round = 0; round < 2; ++round) {
    const int kb = r + 2 * r * round;  // margin on which max_mask is valid: r, then 3r
    // supp_mask = max_pool(max_mask.float()) > 0                        margin kb + r
    win_max<RT>(xa, tmp, wm, S, PS, kb + r, r);
    for (int i = ty; i < S; i += nty)
      for (int j = tx; j < S; j += 32) {
        const int e = i * PS + j, k = kb + r;
        const bool v = i >= k && i < S - k && j >= k && j < S - k;
        const bool in = s0[e] != -INFINITY;
        const unsigned char sp = (v && in && wm[e] > 0.f) ? 1 : 0;
        sup[e] = sp;
        // supp_scores = where(supp_mask, 0, scores); -inf outside the image (max_pool2d padding)
        xa[e] = in ? (sp ? 0.f : s0[e]) : -INFINITY;
      }
    __syncthreads();
    // new_max_mask = supp_scores == max_pool(supp_scores)               margin kb + 2r
    win_max<RT>(xa, tmp, wm, S, PS, kb + 2 * r, r);
    for (int i = ty; i < S; i += nty)
      for (int j = tx; j < S; j += 32) {
        const int e = i * PS + j, k = kb + 2 * r;
        const bool v = i >= k && i < S - k && j >= k && j < S - k;
        unsigned char m = 0;
        if (v && s0[e] != -INFINITY) m = (msk[e] | ((xa[e] == wm[e]) && !sup[e])) ? 1 : 0;  // max_mask | (new_max_mask & ~supp_mask)
        msk[e] = m;
      }
    __syncthreads();
    if (round == 0) {
      for (int i = ty; i < S; i += nty)
        for (int j = tx; j < S; j += 32) xa[i * PS + j] = msk[i * PS + j] ? 1.f : 0.f;
      __syncthreads();
    }
  }
  float* o = out + static_cast<size_t>(b) * H * W;
  for (int i = 5 * r + ty; i < 5 * r + T; i += nty) {
    const int gy = ty0 + i;
    if (gy >= H) break;
    for (int j = 5 * r + tx; j < 5 * r + T; j += 32) {
      const int gx = tx0 + j;
      if (gx < W) o[static_cast<size_t>(gy) * W + gx] = msk[i * PS + j] ? s0[i * PS + j] : 0.f;
    }
  }
}

// ------------------------------------------------------------------ simple_nms, second cut (default for radii 1..5)
// Same arithmetic (exact float equality, -inf outside the image, the reference's five max-pools), a third of the instructions:
//   * max_mask / supp_mask live as BIT rows (one 32-bit word per 32 columns, built with __ballot_sync): the two binary max-pools of
//     the reference (max_pool(max_mask.float()) > 0) become funnel shifts and ORs over a few hundred words per tile;
//   * only the three float max-pools remain; each is a row pass (register sliding window, lanes walking down the rows) into `tmp`
//     and a column pass whose result is consumed in registers - compared, balloted into the mask words, or written out - so no
//     window-max, mask-as-float or suppressed-score array exists;
//   * window maxima by doubling (max of 2, of 4, of 8 neighbours) instead of 2r compares per output.
// Region = 64 x 64 outputs + 5r halo; columns are rounded up to whole mask words and framed by 8 columns of -inf.
template <int R>
struct Nms2 {
  static constexpr int S = kNmsTile + 10 * R;     // region rows / meaningful columns
  static constexpr int NW = (S + 31) / 32;         // mask words per row
  static constexpr int SW = NW * 32;               // computed columns
  static constexpr int PAD = 8;                    // -inf frame (>= R)
  static constexpr int PS = (SW + 2 * PAD) | 1;    // odd pitch: the row passes walk lanes down the rows
  static constexpr int NWP = NW + 2;               // mask row pitch: one zero word on either side
  static constexpr int kThreads = 512;
  static constexpr size_t kSmem = static_cast<size_t>(2) * S * PS * 4 + static_cast<size_t>(4) * S * NWP * 4;
};

// m[o] = max(w[o .. o + 2R]), o = 0..7
template <int R>
__device__ __forceinline__ void window_max8(const float (&w)[8 + 2 * R], float (&m)[8]) {
  constexpr int K = 2 * R + 1, N = 8 + 2 * R;
  if constexpr (R == 0) {
#pragma unroll
    for (int o = 0; o < 8; ++o) m[o] = w[o];
  } else {
    float p2[N - 1];
#pragma unroll
    for (int d = 0; d < N - 1; ++d) p2[d] = fmaxf(w[d], w[d + 1]);
    if constexpr (K == 3) {
#pragma unroll
      for (int o = 0; o < 8; ++o) m[o] = fmaxf(p2[o], w[o + 2]);
    } else {
      float p4[N - 3];
#pragma unroll
      for (int d = 0; d < N - 3; ++d) p4[d] = fmaxf(p2[d], p2[d + 2]);
      if constexpr (K < 8) {
#pragma unroll
        for (int o = 0; o < 8; ++o) m[o] = fmaxf(p4[o], p4[o + K - 4]);
      } else {
        float p8[N - 7];
#pragma unroll
        for (int d = 0; d < N - 7; ++d) p8[d] = fmaxf(p4[d], p4[d + 4]);
#pragma unroll
        for (int o = 0; o < 8; ++o) m[o] = fmaxf(p8[o], p8[o + K - 8]);
      }
    }
  }
}

// row pass of one max-pool over rows [K0 - R, S - K0 + R) (K0 = margin of the pool's output): tmp = window max along x of
// (USE_SUP ? where(supp, 0, s0) : s0).  Only the 8-column segments that overlap the output columns [K0, S - K0) are computed.
template <int R, int K0, bool USE_SUP>
__device__ __forceinline__ void nms2_row_pass(const float* __restrict__ s0, float* __restrict__ tmp, const uint32_t* __restrict__ SUP) {
  using G = Nms2<R>;
  constexpr int S = G::S, PS = G::PS, PAD = G::PAD, NWP = G::NWP;
  constexpr int row_lo = K0 - R, rows = S - 2 * (K0 - R), seg_lo = K0 >> 3, nseg = ((S - K0 - 1) >> 3) + 1 - seg_lo;
  for (int t = threadIdx.x; t < rows * nseg; t += G::kThreads) {
    const int sg = t / rows, i = row_lo + (t - sg * rows), j0 = (seg_lo + sg) * 8;
    const float* p = s0 + i * PS + PAD + j0 - R;
    float w[8 + 2 * R];
#pragma unroll
    for (int d = 0; d < 8 + 2 * R; ++d) w[d] = p[d];
    if (USE_SUP) {
      const int a = j0 - R + 32;  // first window column, shifted by the zero pad word
      const uint32_t bits = __funnelshift_r(SUP[i * NWP + (a >> 5)], SUP[i * NWP + (a >> 5) + 1], a & 31);
#pragma unroll
      for (int d = 0; d < 8 + 2 * R; ++d)
        if ((bits >> d) & 1u) w[d] = 0.f;  // supp_scores = where(supp_mask, 0, scores); supp is never set outside the image
    }
    float m[8];
    window_max8<R>(w, m);
    float* o = tmp + i * PS + PAD + j0;
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = m[q];
  }
}

// supp_mask = max_pool(max_mask) > 0 as bit rows: horizontal dilation by funnel shifts, vertical by OR-ing 2R+1 rows; & inside-image
template <int R>
__device__ __forceinline__ void nms2_dilate(const uint32_t* __restrict__ M, uint32_t* __restrict__ HB, uint32_t* __restrict__ SUP,
                                            const uint32_t* __restrict__ IN) {
  using G = Nms2<R>;
  constexpr int S = G::S, NW = G::NW, NWP = G::NWP;
  for (int it = threadIdx.x; it < S * NW; it += G::kThreads) {
    const int i = it / NW, w = it - i * NW;
    const uint32_t l = M[i * NWP + w], c = M[i * NWP + 1 + w], r = M[i * NWP + 2 + w];
    uint32_t h = c;
#pragma unroll
    for (int d = 1; d <= R; ++d) h |= __funnelshift_l(l, c, d) | __funnelshift_r(c, r, d);
    HB[i * NWP + 1 + w] = h;
  }
  __syncthreads();
  for (int it = threadIdx.x; it < S * NW; it += G::kThreads) {
    const int i = it / NW, w = it - i * NW;
    uint32_t v = 0;
#pragma unroll
    for (int d = -R; d <= R; ++d) {
      const int ii = i + d;
      if (ii >= 0 && ii < S) v |= HB[ii * NWP + 1 + w];
    }
    SUP[i * NWP + 1 + w] = v & IN[i * NWP + 1 + w];
  }
  __syncthreads();
}

// column pass of one max-pool with its consumer.  STAGE 0: max_mask = scores == max_pool(scores).  STAGE 1: max_mask |=
// (supp_scores == max_pool(supp_scores)) & ~supp_mask.  STAGE 2: the same, then where(max_mask, scores, 0) -> global (tile centre).
template <int R, int K0, int STAGE>
__device__ __forceinline__ void nms2_col_pass(const float* __restrict__ s0, const float* __restrict__ tmp, uint32_t* __restrict__ M,
                                              const uint32_t* __restrict__ SUP, const uint32_t* __restrict__ IN, float* __restrict__ o,
                                              int H, int W, int ty0, int tx0) {
  using G = Nms2<R>;
  constexpr int S = G::S, PS = G::PS, PAD = G::PAD, NWP = G::NWP;
  constexpr int nchunk = (S - 2 * K0 + 7) / 8, w_lo = K0 >> 5, nw = ((S - K0 - 1) >> 5) + 1 - w_lo;
  const int lane = threadIdx.x & 31;
  for (int it = threadIdx.x >> 5; it < nchunk * nw; it += G::kThreads / 32) {
    const int ch = it / nw, w = w_lo + (it - ch * nw), i0 = K0 + ch * 8, c = w * 32 + lane;
    float win[8 + 2 * R];
#pragma unroll
    for (int d = 0; d < 8 + 2 * R; ++d) win[d] = tmp[min(i0 - R + d, S - 1) * PS + PAD + c];
    float m[8];
    window_max8<R>(win, m);
    const bool colv = c >= K0 && c < S - K0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int i = i0 + q;
      if (i >= S - K0) break;  // warp-uniform
      const float sv = s0[i * PS + PAD + c];
      const bool in = (IN[i * NWP + 1 + w] >> lane) & 1u;
      if (STAGE == 0) {
        const uint32_t bal = __ballot_sync(0xffffffffu, colv && in && sv == m[q]);
        if (lane == 0) M[i * NWP + 1 + w] = bal;
      } else {
        const bool sup = (SUP[i * NWP + 1 + w] >> lane) & 1u;
        const uint32_t fresh = __ballot_sync(0xffffffffu, colv && in && !sup && sv == m[q]);
        if (STAGE == 1) {
          if (lane == 0) M[i * NWP + 1 + w] |= fresh;  // one thread reads and writes the word: no intra-warp hazard
        } else {
          const uint32_t mw = M[i * NWP + 1 + w] | fresh;  // M is read-only in the last stage
          const int gy = ty0 + i, gx = tx0 + c;  // K0 = 5R: rows are the tile centre by construction
          if (colv && gy < H && gx < W) o[static_cast<size_t>(gy) * W + gx] = ((mw >> lane) & 1u) ? sv : 0.f;
        }
      }
    }
  }
}

template <int R>
__global__ void __launch_bounds__(512) sp_nms2_kernel(const float* __restrict__ scores, float* __restrict__ out, int H, int W) {
  using G = Nms2<R>;
  constexpr int S = G::S, NW = G::NW, SW = G::SW, PS = G::PS, PAD = G::PAD, NWP = G::NWP;
  extern __shared__ float nsm2[];
  float* s0 = nsm2;                // scores, -inf outside the image and in the frame
  float* tmp = s0 + S * PS;        // row-pass result of the current pool
  uint32_t* M = reinterpret_cast<uint32_t*>(tmp + S * PS);  // max_mask bit rows
  uint32_t* SUP = M + S * NWP;     // supp_mask of the current round
  uint32_t* IN = SUP + S * NWP;    // inside-the-image bits
  uint32_t* HB = IN + S * NWP;     // horizontally dilated max_mask
  const int b = blockIdx.z, ty0 = blockIdx.y * kNmsTile - 5 * R, tx0 = blockIdx.x * kNmsTile - 5 * R;
  const int tid = threadIdx.x, lane = tid & 31;
  const float* sc = scores + static_cast<size_t>(b) * H * W;
  for (int i = tid; i < 4 * S * NWP; i += G::kThreads) M[i] = 0u;
  for (int i = tid; i < S * 2 * PAD; i += G::kThreads) {
    const int row = i / (2 * PAD), c = i - row * 2 * PAD;
    s0[row * PS + (c < PAD ? c : SW + c)] = -INFINITY;
  }
  __syncthreads();
  for (int it = tid >> 5; it < S * NW; it += G::kThreads / 32) {
    const int i = it / NW, w = it - i * NW, c = w * 32 + lane, gy = ty0 + i, gx = tx0 + c;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    s0[i * PS + PAD + c] = in ? sc[static_cast<size_t>(gy) * W + gx] : -INFINITY;
    const uint32_t bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) IN[i * NWP + 1 + w] = bal;
  }
  __syncthreads();
  float* o = out + static_cast<size_t>(b) * H * W;
  // max_mask = scores == max_pool(scores)                                           valid on margin R
  nms2_row_pass<R, R, false>(s0, tmp, SUP);
  __syncthreads();
  nms2_col_pass<R, R, 0>(s0, tmp, M, SUP, IN, o, H, W, ty0, tx0);
  __syncthreads();
  // round 0: supp on margin 2R, new maxima on margin 3R
  nms2_dilate<R>(M, HB, SUP, IN);
  nms2_row_pass<R, 3 * R, true>(s0, tmp, SUP);
  __syncthreads();
  nms2_col_pass<R, 3 * R, 1>(s0, tmp, M, SUP, IN, o, H, W, ty0, tx0);
  __syncthreads();
  // round 1: supp on margin 4R, final mask on margin 5R = the 64 x 64 centre
  nms2_dilate<R>(M, HB, SUP, IN);
  nms2_row_pass<R, 5 * R, true>(s0, tmp, SUP);
  __syncthreads();
  nms2_col_pass<R, 5 * R, 2>(s0, tmp, M, SUP, IN, o, H, W, ty0, tx0);
}

// ------------------------------------------------------------------ candidate compaction in row-major order
__device__ __forceinline__ bool sp_is_cand(float v, int p, int W, int H, float thr, int border) {
  const int y = p / W, x = p - y * W;
  return v > thr && y >= border && y < H - border && x >= border && x < W - border;  // superpoint.py:183,66-71
}

__global__ void __launch_bounds__(256) sp_count_kernel(const float* __restrict__ nms, int* __restrict__ chunk_count, int H, int W,
                                                       float thr, int border, int nchunks, const float* __restrict__ thr_dev) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const float* s = nms + static_cast<size_t>(b) * H * W;
  if (thr_dev) thr = thr_dev[b];  // threshold decided on the device (ALIKED's mean fallback)
  int cnt = 0;
  const int base = chunk * kChunk + threadIdx.x * 16;
  for (int i = 0; i < 16; ++i) {
    const int p = base + i;
    if (p < H * W && sp_is_cand(s[p], p, W, H, thr, border)) ++cnt;
  }
  __shared__ int red[8];
#pragma unroll
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    chunk_count[b * nchunks + chunk] = t;
  }
}

__global__ void sp_scan_kernel(const int* __restrict__ chunk_count, int* __restrict__ chunk_off, int* __restrict__ cand_count,
                               int nchunks) {
  // one thread block per image; nchunks is small (H*W/4096): serial scan by thread 0 is fine
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < nchunks; ++i) {
      chunk_off[b * nchunks + i] = acc;
      acc += chunk_count[b * nchunks + i];
    }
    cand_count[b] = acc;
  }
}

__global__ void __launch_bounds__(256) sp_compact_kernel(const float* __restrict__ nms, const int* __restrict__ chunk_off,
                                                         int* __restrict__ cand_idx, float* __restrict__ cand_score, int H,
                                                         int W, float thr, int border, int nchunks,
                                                         const float* __restrict__ thr_dev) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const float* s = nms + static_cast<size_t>(b) * H * W;
  if (thr_dev) thr = thr_dev[b];
  const int base = chunk * kChunk + threadIdx.x * 16;
  float v[16];
  int cnt = 0;
  unsigned flags = 0;
  for (int i = 0; i < 16; ++i) {
    const int p = base + i;
    v[i] = p < H * W ? s[p] : 0.f;
    if (p < H * W && sp_is_cand(v[i], p, W, H, thr, border)) {
      flags |= 1u << i;
      ++cnt;
    }
  }
  // block exclusive scan of cnt (256 threads)
  __shared__ int wsum[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) wsum[wid] = inc;
  __syncthreads();
  int woff = 0;
  for (int i = 0; i < wid; ++i) woff += wsum[i];
  int pos = chunk_off[b * nchunks + chunk] + woff + inc - cnt;
  int* ci = cand_idx + static_cast<size_t>(b) * H * W;
  float* cs = cand_score + static_cast<size_t>(b) * H * W;
  for (int i = 0; i < 16; ++i)
    if (flags & (1u << i)) {
      ci[pos] = base + i;
      cs[pos] = v[i];
      ++pos;
    }
}

// ------------------------------------------------------------------ top-k (superpoint.py:74-78): radix select + bitonic sort
// One CTA per image, K <= kMaxTopK.  If count <= K (or K < 0): keep everything in row-major order.  Otherwise pick the K
// largest scores (ties at the cut resolved by smaller pixel index) and order them score-desc, index-asc.
// kSortAll (ALIKED's top-k mode, torch.topk returns sorted values): count <= K keeps every candidate too, but sorted; sel_count is K
// and topk_fill_kernel writes slots count .. K-1.
template <bool kSortAll>
__global__ void __launch_bounds__(kSelThreads) sp_select_kernel(const int* __restrict__ cand_idx, const float* __restrict__ cand_score,
                                                                const int* __restrict__ cand_count, int* __restrict__ sel_idx,
                                                                float* __restrict__ sel_score, int* __restrict__ sel_count,
                                                                int HW, int K, int cap, int sort_cap) {
  extern __shared__ unsigned long long keys[];  // sort_cap entries
  __shared__ unsigned hist[256];
  __shared__ unsigned s_prefix, s_remaining, s_ngreater, s_tiepos;
  const int b = blockIdx.x, t = threadIdx.x;
  const int C = cand_count[b];
  const int* ci = cand_idx + static_cast<size_t>(b) * HW;
  const float* cs = cand_score + static_cast<size_t>(b) * HW;
  int* oi = sel_idx + static_cast<size_t>(b) * cap;
  float* os = sel_score + static_cast<size_t>(b) * cap;
  if (!kSortAll && (K < 0 || C <= K)) {
    if (t == 0) sel_count[b] = C;  // host checks C <= cap
    for (int i = t; i < C && i < cap; i += blockDim.x) {
      oi[i] = ci[i];
      os[i] = cs[i];
    }
    return;
  }
  int n = K;  // keys to sort
  if (kSortAll && C <= K) {
    for (int i = t; i < C; i += blockDim.x)
      keys[i] = (static_cast<unsigned long long>(~__float_as_uint(cs[i])) << 32) | static_cast<unsigned>(ci[i]);
    n = C;
  } else {
    // ---- radix select of the K-th largest score (scores > 0 -> float bits are order preserving)
    if (t == 0) {
      s_prefix = 0;
      s_remaining = K;
    }
    __syncthreads();
    for (int shift = 24; shift >= 0; shift -= 8) {
      if (t < 256) hist[t] = 0;
      __syncthreads();
      const unsigned prefix = s_prefix;
      const unsigned himask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
      for (int i = t; i < C; i += blockDim.x) {
        const unsigned u = __float_as_uint(cs[i]);
        if ((u & himask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (t == 0) {
        unsigned rem = s_remaining, d = 255;
        for (;; --d) {  // walk digits from large to small
          if (hist[d] >= rem) break;
          rem -= hist[d];
          if (d == 0) break;
        }
        s_prefix = prefix | (d << shift);
        s_remaining = rem;  // how many elements equal to the final threshold are still needed
      }
      __syncthreads();
    }
    const unsigned T = s_prefix;       // bit pattern of the K-th largest score
    const unsigned need_ties = s_remaining;
    if (t == 0) {
      s_ngreater = 0;
      s_tiepos = 0;
    }
    __syncthreads();
    // ---- gather: strictly greater first (any order, sorted below), then the first `need_ties` ties by index.
    // key = (~scorebits << 32) | pixel index : ascending key order == score desc, index asc
    for (int i = t; i < C; i += blockDim.x) {
      const unsigned u = __float_as_uint(cs[i]);
      if (u > T) {
        const unsigned pos = atomicAdd(&s_ngreater, 1u);
        keys[pos] = (static_cast<unsigned long long>(~u) << 32) | static_cast<unsigned>(ci[i]);
      }
    }
    __syncthreads();
    const unsigned G = s_ngreater;  // == K - need_ties
    // ties: candidates are stored in increasing pixel index, so rank among ties = number of earlier ties
    for (int base = 0; base < C; base += blockDim.x) {
      const int i = base + t;
      const bool tie = i < C && __float_as_uint(cs[i]) == T;
      // block-wide ordered rank via ballot + warp counts
      __shared__ unsigned wcnt[32];
      const unsigned bal = __ballot_sync(0xffffffffu, tie);
      if ((t & 31) == 0) wcnt[t >> 5] = __popc(bal);
      __syncthreads();
      unsigned before = s_tiepos;
      for (int wv = 0; wv < (t >> 5); ++wv) before += wcnt[wv];
      before += __popc(bal & ((1u << (t & 31)) - 1u));
      if (tie && before < need_ties)
        keys[G + before] = (static_cast<unsigned long long>(~T) << 32) | static_cast<unsigned>(ci[i]);
      __syncthreads();
      if (t == 0) {
        unsigned tot = 0;
        for (int wv = 0; wv < 32; ++wv) tot += wcnt[wv];
        s_tiepos += tot;
      }
      __syncthreads();
    }
  }
  // ---- bitonic sort of n keys padded to a power of two
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = n + t; i < P; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], c = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > c) == up) {
            keys[i] = c;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  for (int i = t; i < n; i += blockDim.x) {
    oi[i] = static_cast<int>(keys[i] & 0xffffffffull);
    os[i] = __uint_as_float(~static_cast<unsigned>(keys[i] >> 32));
  }
  if (t == 0) sel_count[b] = K;
}


// Sort-always selection with count C < K: slot C + j takes the j-th pixel (row-major) that is not a candidate, with score 0 (the NMS
// value torch.topk reports for it when the candidates are exactly the nonzero pixels, as in ALIKED's top-k mode).  Needs K <= HW.
__global__ void __launch_bounds__(256) topk_fill_kernel(const int* __restrict__ cand_idx, const int* __restrict__ cand_count,
                                                        int* __restrict__ sel_idx, float* __restrict__ sel_score, int HW, int K, int cap) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const int C = cand_count[b];
  if (j >= K - C) return;
  // candidates ascend, so ci[i] - i never decreases; the m candidates with ci[i] - i <= j are the ones before the j-th other pixel
  const int* ci = cand_idx + static_cast<size_t>(b) * HW;
  int lo = 0, hi = C;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ci[mid] - mid <= j) lo = mid + 1;
    else hi = mid;
  }
  sel_idx[static_cast<size_t>(b) * cap + C + j] = j + lo;
  sel_score[static_cast<size_t>(b) * cap + C + j] = 0.f;
}

// ------------------------------------------------------------------ grid-wide top-k (K > kMaxTopK)
// Same selection rule and output as sp_select_kernel, with every stage spread over a grid of CTAs per image:
//   1. radix select of the K-th largest score: four 8-bit digit passes, each a per-CTA shared histogram added into a [B][256] global
//      one, then topk_digit_kernel walks the digits (thread 0 of sp_select_kernel's walk) and keeps (prefix, ties still needed);
//   2. ordered gather: chunked count / scan / write keeps every candidate above the threshold and the first `needed` ties, in
//      ascending pixel index;
//   3. stable LSD radix sort of the kept ones on the inverted score bits (four 8-bit passes: per-CTA digit counts, per-image scan,
//      stable scatter), so that equal scores stay in ascending index order.  The last pass writes sel_idx / sel_score.
// The decisions (select or keep all, sort or not) are taken per image on the device; nothing waits for the host.
constexpr int kTopkThreads = 256;
constexpr int kTopkSelGrid = 64;   // histogram CTAs per image (grid-stride over the candidates)
constexpr int kSortTile = 2048;    // keys per CTA of a sort pass: 8 warps x 256, each warp a contiguous run
enum { kTkPrefix = 0, kTkNeed, kTkSelect, kTkSort, kTkState = 8 };  // per-image state words

// Device scratch of the grid-wide path for up to B images of HW pixels at top-K
struct TopkScratch {
  unsigned* hist = nullptr;         // [B][256] digit histogram of the running select pass
  unsigned* state = nullptr;        // [B][kTkState]
  int *chunk_cnt = nullptr, *gt_off = nullptr, *tie_off = nullptr;  // [B][ceil(HW / kChunk)] gather counts and offsets
  int* digit_off = nullptr;         // [B][ceil(K / kSortTile)][256] sort-pass digit counts, then offsets
  unsigned long long *keys0 = nullptr, *keys1 = nullptr;  // [B][K] ping-pong sort keys (~score bits << 32 | pixel index)
  int B = 0, HW = 0, K = 0;         // capacity
};

// element counts of TopkScratch's buffers: hist, state, one chunk array, digit_off, one key array
struct TopkSizes {
  size_t hist, state, chunks, digits, keys;
};
inline TopkSizes topk_sizes(int B, int HW, int K) {
  const size_t b = B;
  return {b * 256, b * kTkState, b * ceil_div(HW, kChunk), b * ceil_div(K, kSortTile) * 256, b * K};
}

__device__ __forceinline__ unsigned long long topk_key(unsigned u, int idx) {
  return (static_cast<unsigned long long>(~u) << 32) | static_cast<unsigned>(idx);
}

__global__ void __launch_bounds__(kTopkThreads) topk_init_kernel(const int* __restrict__ cand_count, int K, int sort_all,
                                                                 unsigned* __restrict__ hist, unsigned* __restrict__ state,
                                                                 int* __restrict__ sel_count) {
  const int b = blockIdx.x;
  hist[b * 256 + threadIdx.x] = 0u;
  if (threadIdx.x == 0) {
    const int C = cand_count[b], keep = min(C, K);
    unsigned* s = state + b * kTkState;
    s[kTkPrefix] = 0u;  // with no select pass every candidate (score > 0) is above the threshold 0
    s[kTkNeed] = K;
    s[kTkSelect] = C > K;
    s[kTkSort] = (C > K || sort_all) ? keep : 0;  // keys to sort; 0: the gather writes the output in row-major order
    sel_count[b] = sort_all ? K : keep;
  }
}

// one digit pass of the radix select: histogram of digit (u >> shift) & 255 over the candidates matching the prefix so far
__global__ void __launch_bounds__(kTopkThreads) topk_hist_kernel(const float* __restrict__ cand_score, const int* __restrict__ cand_count,
                                                                 const unsigned* __restrict__ state, unsigned* __restrict__ hist, int HW,
                                                                 int shift) {
  const int b = blockIdx.y, t = threadIdx.x, lane = t & 31;
  if (!state[b * kTkState + kTkSelect]) return;
  __shared__ unsigned h[256];
  h[t] = 0u;
  __syncthreads();
  const int C = cand_count[b];
  const float* cs = cand_score + static_cast<size_t>(b) * HW;
  const unsigned prefix = state[b * kTkState + kTkPrefix];
  const unsigned himask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
  for (int base = blockIdx.x * kTopkThreads; base < C; base += gridDim.x * kTopkThreads) {  // block-uniform trip count
    const int i = base + t;
    unsigned d = 0xffffffffu;
    if (i < C) {
      const unsigned u = __float_as_uint(cs[i]);
      if ((u & himask) == prefix) d = (u >> shift) & 255u;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);  // scores cluster in few digits: one shared atomic per digit and warp
    if (d != 0xffffffffu && lane == __ffs(peers) - 1) atomicAdd(&h[d], __popc(peers));
  }
  __syncthreads();
  if (h[t]) atomicAdd(&hist[b * 256 + t], h[t]);
}

__global__ void __launch_bounds__(kTopkThreads) topk_digit_kernel(unsigned* __restrict__ hist, unsigned* __restrict__ state, int shift) {
  const int b = blockIdx.x, t = threadIdx.x;
  unsigned* s = state + b * kTkState;
  if (!s[kTkSelect]) return;
  __shared__ unsigned h[256];
  h[t] = hist[b * 256 + t];
  hist[b * 256 + t] = 0u;  // ready for the next pass
  __syncthreads();
  if (t == 0) {
    unsigned rem = s[kTkNeed], d = 255;
    for (;; --d) {  // walk digits from large to small
      if (h[d] >= rem) break;
      rem -= h[d];
      if (d == 0) break;
    }
    s[kTkPrefix] |= d << shift;
    s[kTkNeed] = rem;  // after the last pass: how many candidates equal to the threshold are still needed
  }
}

// per chunk of kChunk candidates: (above threshold << 16) | (equal to threshold)
__global__ void __launch_bounds__(kTopkThreads) topk_gather_count_kernel(const float* __restrict__ cand_score,
                                                                         const int* __restrict__ cand_count,
                                                                         const unsigned* __restrict__ state, int* __restrict__ chunk_cnt,
                                                                         int HW, int nchunks) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int C = cand_count[b];
  if (chunk * kChunk >= C) return;
  const float* cs = cand_score + static_cast<size_t>(b) * HW;
  const unsigned T = state[b * kTkState + kTkPrefix];
  int cnt = 0;
  const int base = chunk * kChunk + threadIdx.x * 16;
  for (int i = 0; i < 16; ++i) {
    const int p = base + i;
    if (p < C) {
      const unsigned u = __float_as_uint(cs[p]);
      cnt += u > T ? 0x10000 : (u == T ? 1 : 0);
    }
  }
  __shared__ int red[kTopkThreads / 32];
#pragma unroll
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot = 0;
    for (int i = 0; i < kTopkThreads / 32; ++i) tot += red[i];
    chunk_cnt[b * nchunks + chunk] = tot;
  }
}

__global__ void topk_gather_scan_kernel(const int* __restrict__ chunk_cnt, const int* __restrict__ cand_count, int* __restrict__ gt_off,
                                        int* __restrict__ tie_off, int nchunks) {
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {  // a few hundred chunks at most: a serial scan, as sp_scan_kernel
    const int live = ceil_div(cand_count[b], kChunk);
    int gt = 0, tie = 0;
    for (int i = 0; i < live; ++i) {
      const int c = chunk_cnt[b * nchunks + i];
      gt_off[b * nchunks + i] = gt;
      tie_off[b * nchunks + i] = tie;
      gt += c >> 16;
      tie += c & 0xffff;
    }
  }
}

// writes the kept candidates of one chunk at their rank in index order: to the sort keys, or straight to the output when the image
// needs no sort (count <= K, not sort-always)
__global__ void __launch_bounds__(kTopkThreads) topk_gather_write_kernel(const int* __restrict__ cand_idx,
                                                                         const float* __restrict__ cand_score,
                                                                         const int* __restrict__ cand_count,
                                                                         const unsigned* __restrict__ state, const int* __restrict__ gt_off,
                                                                         const int* __restrict__ tie_off, unsigned long long* __restrict__ keys,
                                                                         int* __restrict__ sel_idx, float* __restrict__ sel_score, int HW,
                                                                         int K, int cap, int nchunks) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int C = cand_count[b];
  if (chunk * kChunk >= C) return;
  const unsigned* s = state + b * kTkState;
  const unsigned T = s[kTkPrefix], need = s[kTkNeed];
  const bool sort = s[kTkSort] != 0u;
  const int* ci = cand_idx + static_cast<size_t>(b) * HW;
  const float* cs = cand_score + static_cast<size_t>(b) * HW;
  const int base = chunk * kChunk + threadIdx.x * 16;
  unsigned u[16];
  int cnt = 0;
  for (int i = 0; i < 16; ++i) {
    const int p = base + i;
    u[i] = p < C ? __float_as_uint(cs[p]) : 0u;  // 0: neither above nor equal to a threshold of a positive score
    cnt += u[i] > T ? 0x10000 : (u[i] == T && p < C ? 1 : 0);
  }
  // block exclusive scan of the packed counts (each field at most kChunk)
  __shared__ int wsum[kTopkThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) wsum[wid] = inc;
  __syncthreads();
  int ex = inc - cnt;
  for (int i = 0; i < wid; ++i) ex += wsum[i];
  unsigned gt = gt_off[b * nchunks + chunk] + (ex >> 16), tie = tie_off[b * nchunks + chunk] + (ex & 0xffff);
  unsigned long long* ko = keys + static_cast<size_t>(b) * K;
  int* oi = sel_idx + static_cast<size_t>(b) * cap;
  float* os = sel_score + static_cast<size_t>(b) * cap;
  for (int i = 0; i < 16; ++i) {
    const int p = base + i;
    if (p >= C) break;
    unsigned pos;
    bool keep = false;
    if (u[i] > T) {
      keep = true;
      pos = gt + min(tie, need);  // kept before it: every earlier candidate above T and the first `need` earlier ties
      ++gt;
    } else if (u[i] == T) {
      keep = tie < need;
      pos = gt + tie;
      ++tie;
    }
    if (!keep) continue;
    if (sort) {
      ko[pos] = topk_key(u[i], ci[p]);
    } else {
      oi[pos] = ci[p];
      os[pos] = __uint_as_float(u[i]);
    }
  }
}

// One pass of the LSD sort on digit (key >> shift) & 255.  Each warp walks its contiguous 256 keys 32 at a time, in order; lanes with
// the same digit rank among themselves with __match_any_sync, so equal digits keep their input order (stable).  SCATTER false: the
// CTA's digit counts to digit_off.  SCATTER true: digit_off holds the CTA's first output slot per digit (topk_sort_scan_kernel).
template <bool SCATTER>
__global__ void __launch_bounds__(kTopkThreads) topk_sort_pass_kernel(const unsigned long long* __restrict__ src,
                                                                      unsigned long long* __restrict__ dst, int* __restrict__ sel_idx,
                                                                      float* __restrict__ sel_score, int* __restrict__ digit_off,
                                                                      const unsigned* __restrict__ state, int K, int cap, int nblk,
                                                                      int shift) {
  const int b = blockIdx.y, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int n = static_cast<int>(state[b * kTkState + kTkSort]);
  const int blk0 = blockIdx.x * kSortTile;
  if (blk0 >= n) return;
  __shared__ int wh[kTopkThreads / 32][256];  // per-warp digit counts, then per-warp running output slots
  for (int i = t; i < kTopkThreads / 32 * 256; i += kTopkThreads) (&wh[0][0])[i] = 0;
  __syncthreads();
  const unsigned long long* in = src + static_cast<size_t>(b) * K;
  const int seg = blk0 + w * (kSortTile / (kTopkThreads / 32));
  constexpr int kRounds = kSortTile / kTopkThreads;
  for (int r = 0; r < kRounds; ++r) {
    const int i = seg + r * 32 + lane;
    const unsigned d = i < n ? static_cast<unsigned>(in[i] >> shift) & 255u : 0xffffffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d != 0xffffffffu && lane == __ffs(peers) - 1) wh[w][d] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  int* off = digit_off + (static_cast<size_t>(b) * nblk + blockIdx.x) * 256;
  if (!SCATTER) {
    int tot = 0;
#pragma unroll
    for (int q = 0; q < kTopkThreads / 32; ++q) tot += wh[q][t];
    off[t] = tot;
    return;
  }
  {
    int run = off[t];
#pragma unroll
    for (int q = 0; q < kTopkThreads / 32; ++q) {
      const int c = wh[q][t];
      wh[q][t] = run;
      run += c;
    }
  }
  __syncthreads();
  const bool last = dst == nullptr;
  unsigned long long* out = last ? nullptr : dst + static_cast<size_t>(b) * K;
  int* oi = sel_idx + static_cast<size_t>(b) * cap;
  float* os = sel_score + static_cast<size_t>(b) * cap;
  const unsigned lt = (1u << lane) - 1u;
  for (int r = 0; r < kRounds; ++r) {
    const int i = seg + r * 32 + lane;
    const unsigned long long key = i < n ? in[i] : 0ull;
    const unsigned d = i < n ? static_cast<unsigned>(key >> shift) & 255u : 0xffffffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d != 0xffffffffu) {
      const int pos = wh[w][d] + __popc(peers & lt);
      if (last) {
        oi[pos] = static_cast<int>(key & 0xffffffffull);
        os[pos] = __uint_as_float(~static_cast<unsigned>(key >> 32));
      } else {
        out[pos] = key;
      }
    }
    __syncwarp();
    if (d != 0xffffffffu && lane == __ffs(peers) - 1) wh[w][d] += __popc(peers);
    __syncwarp();
  }
}

// digit_off [B][nblk][256]: per-CTA digit counts -> first output slot of each (CTA, digit), digits ascending, CTAs in order
__global__ void __launch_bounds__(256) topk_sort_scan_kernel(int* __restrict__ digit_off, const unsigned* __restrict__ state, int nblk) {
  const int b = blockIdx.x, d = threadIdx.x, lane = d & 31, w = d >> 5;
  const int n = static_cast<int>(state[b * kTkState + kTkSort]);
  if (n == 0) return;
  const int live = ceil_div(n, kSortTile);
  int* off = digit_off + static_cast<size_t>(b) * nblk * 256;
  int run = 0;
  for (int k = 0; k < live; ++k) {
    const int c = off[k * 256 + d];
    off[k * 256 + d] = run;
    run += c;
  }
  // exclusive scan of the digit totals
  __shared__ int ws[8];
  int inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) ws[w] = inc;
  __syncthreads();
  int base = inc - run;
  for (int q = 0; q < w; ++q) base += ws[q];
  for (int k = 0; k < live; ++k) off[k * 256 + d] += base;
}


// How simple_nms runs at radius r: kernel 2 = sp_nms2_kernel (bit masks), 1 = sp_nms_kernel (first cut); tile x tile outputs per CTA.
struct NmsPlan {
  int kernel, tile, threads, smem;
};

// ver 2: the bit-mask kernel for radii 1..5 and the first cut for the others (what production runs); 1: the first cut at every radius
constexpr int kNmsProductionVer = 2;
inline NmsPlan nms_plan(int r, int ver) {
  if (ver == 2 && r >= 1 && r <= 5) {
    static constexpr int smem2[5] = {Nms2<1>::kSmem, Nms2<2>::kSmem, Nms2<3>::kSmem, Nms2<4>::kSmem, Nms2<5>::kSmem};
    return {2, kNmsTile, Nms2<1>::kThreads, smem2[r - 1]};
  }
  // five S x S planes (S = tile + 10 r): four float, two byte masks.  64 x 64 outputs per CTA unless the 5r halo no longer fits
  auto smem = [r](int t) { return (t + 10 * r) * ((t + 10 * r) | 1) * static_cast<int>(4 * sizeof(float) + 2); };
  const int T = smem(kNmsTile) > kSmemOptin ? 32 : kNmsTile;
  return {1, T, 1024, smem(T)};
}

// launches simple_nms on a [B][H][W] score map with the kernel nms_plan(r, ver) picks (production: ver = kNmsProductionVer)
inline int launch_nms(dimb_ctx* ctx, cudaStream_t st, const float* scores, float* out, int B, int H, int W, int r, int ver) {
  const NmsPlan p = nms_plan(r, ver);
  if (p.kernel == 2) {
    dim3 grid2(ceil_div(W, kNmsTile), ceil_div(H, kNmsTile), B);
    auto launch2 = [&](auto kern) -> int {
      DIMB_TRY(dimb_func_smem(ctx, kern, p.smem));
      kern<<<grid2, p.threads, p.smem, st>>>(scores, out, H, W);
      return DIMB_OK;
    };
    switch (r) {
      case 1: DIMB_TRY(launch2(sp_nms2_kernel<1>)); break;
      case 2: DIMB_TRY(launch2(sp_nms2_kernel<2>)); break;
      case 3: DIMB_TRY(launch2(sp_nms2_kernel<3>)); break;
      case 4: DIMB_TRY(launch2(sp_nms2_kernel<4>)); break;
      default: DIMB_TRY(launch2(sp_nms2_kernel<5>)); break;
    }
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  }
  const int T = p.tile;
  dim3 grid(ceil_div(W, T), ceil_div(H, T), B);
  auto launch = [&](auto kern) -> int {
    DIMB_TRY(dimb_func_smem(ctx, kern, p.smem));
    kern<<<grid, p.threads, p.smem, st>>>(scores, out, H, W, r, T);
    return DIMB_OK;
  };
  switch (r) {  // the reference's configurations use 2/3 (pipelines), 4 (defaults) and 5 (tile preselection)
    case 2: DIMB_TRY(launch(sp_nms_kernel<2>)); break;
    case 3: DIMB_TRY(launch(sp_nms_kernel<3>)); break;
    case 4: DIMB_TRY(launch(sp_nms_kernel<4>)); break;
    case 5: DIMB_TRY(launch(sp_nms_kernel<5>)); break;
    default: DIMB_TRY(launch(sp_nms_kernel<-1>)); break;
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// Candidate buffers of B images of H x W: chunk_count / chunk_off [B][ceil(H W / kChunk)], cand_count [B], cand_idx / cand_score [B][H W]
struct CandBufs {
  int *chunk_count, *chunk_off, *cand_count, *cand_idx;
  float* cand_score;
};

// Pixels of nms with score > thr, at least `border` pixels inside the image: counted (cand_count) and, with `compact`, written in
// row-major order to cand_idx / cand_score.  thr_dev [B] (may be null): per-image thresholds read on the device, replacing thr.
inline int launch_candidates(dimb_ctx* ctx, cudaStream_t st, const float* nms, const CandBufs& c, int B, int H, int W, float thr,
                             int border, const float* thr_dev, bool compact) {
  const int nch = ceil_div(H * W, kChunk);
  sp_count_kernel<<<dim3(nch, B), 256, 0, st>>>(nms, c.chunk_count, H, W, thr, border, nch, thr_dev);
  DIMB_LAUNCH_CHECK(ctx);
  sp_scan_kernel<<<B, 32, 0, st>>>(c.chunk_count, c.chunk_off, c.cand_count, nch);
  DIMB_LAUNCH_CHECK(ctx);
  if (compact) {
    sp_compact_kernel<<<dim3(nch, B), 256, 0, st>>>(nms, c.chunk_off, c.cand_idx, c.cand_score, H, W, thr, border, nch, thr_dev);
    DIMB_LAUNCH_CHECK(ctx);
  }
  return DIMB_OK;
}

// Grows s to B images of HW pixels at top-K.  The buffers belong to the current owner (OwnerScope) of the context.
inline int topk_reserve(dimb_ctx* ctx, TopkScratch& s, int B, int HW, int K) {
  if (s.hist && B <= s.B && HW <= s.HW && K <= s.K) return DIMB_OK;
  for (void* p : {static_cast<void*>(s.hist), static_cast<void*>(s.state), static_cast<void*>(s.chunk_cnt), static_cast<void*>(s.gt_off),
                  static_cast<void*>(s.tie_off), static_cast<void*>(s.digit_off), static_cast<void*>(s.keys0), static_cast<void*>(s.keys1)})
    dimb_free(ctx, p);
  s = TopkScratch{};
  const TopkSizes z = topk_sizes(B, HW, K);
  DIMB_TRY(dimb_alloc_t(ctx, &s.hist, z.hist));
  DIMB_TRY(dimb_alloc_t(ctx, &s.state, z.state));
  DIMB_TRY(dimb_alloc_t(ctx, &s.chunk_cnt, z.chunks));
  DIMB_TRY(dimb_alloc_t(ctx, &s.gt_off, z.chunks));
  DIMB_TRY(dimb_alloc_t(ctx, &s.tie_off, z.chunks));
  DIMB_TRY(dimb_alloc_t(ctx, &s.digit_off, z.digits));
  DIMB_TRY(dimb_alloc_t(ctx, &s.keys0, z.keys, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s.keys1, z.keys, false));
  s.B = B, s.HW = HW, s.K = K;
  return DIMB_OK;
}

// Top-K of each image's candidates into sel_idx / sel_score [B][cap], counts to sel_count [B]; K < 0 keeps all (in row-major order).
// K <= kMaxTopK runs sp_select_kernel, larger K (or any K >= 1 with `grid`, for tests) the grid-wide path with scratch `tk`
// (topk_reserve'd for B, HW, K).  sort_all (1 <= K <= HW): ALIKED's top-k mode, see sp_select_kernel.
inline int launch_select(dimb_ctx* ctx, cudaStream_t st, const CandBufs& c, int* sel_idx, float* sel_score, int* sel_count, int B, int HW,
                         int K, int cap, TopkScratch* tk, bool sort_all, bool grid = false) {
  if (K <= kMaxTopK && !grid) {
    int P = 1;  // the bitonic sort runs on K keys padded to a power of two
    while (P < std::max(K, 1)) P <<= 1;
    const size_t smem = static_cast<size_t>(P) * sizeof(unsigned long long);
    auto kern = sort_all ? sp_select_kernel<true> : sp_select_kernel<false>;
    DIMB_TRY(dimb_func_smem(ctx, kern, static_cast<int>(smem)));
    kern<<<B, kSelThreads, smem, st>>>(c.cand_idx, c.cand_score, c.cand_count, sel_idx, sel_score, sel_count, HW, K, cap, P);
    DIMB_LAUNCH_CHECK(ctx);
  } else {
    if (!tk || B > tk->B || HW > tk->HW || K > tk->K) {
      dimb_set_error(ctx, "launch_select: top-k scratch smaller than the call");
      return DIMB_ERR_ARG;
    }
    const int nch = ceil_div(HW, kChunk), nblk = ceil_div(K, kSortTile);
    topk_init_kernel<<<B, kTopkThreads, 0, st>>>(c.cand_count, K, sort_all ? 1 : 0, tk->hist, tk->state, sel_count);
    DIMB_LAUNCH_CHECK(ctx);
    const dim3 hgrid(std::min(kTopkSelGrid, ceil_div(HW, kTopkThreads * 16)), B);
    for (int shift = 24; shift >= 0; shift -= 8) {
      topk_hist_kernel<<<hgrid, kTopkThreads, 0, st>>>(c.cand_score, c.cand_count, tk->state, tk->hist, HW, shift);
      DIMB_LAUNCH_CHECK(ctx);
      topk_digit_kernel<<<B, kTopkThreads, 0, st>>>(tk->hist, tk->state, shift);
      DIMB_LAUNCH_CHECK(ctx);
    }
    topk_gather_count_kernel<<<dim3(nch, B), kTopkThreads, 0, st>>>(c.cand_score, c.cand_count, tk->state, tk->chunk_cnt, HW, nch);
    DIMB_LAUNCH_CHECK(ctx);
    topk_gather_scan_kernel<<<B, 32, 0, st>>>(tk->chunk_cnt, c.cand_count, tk->gt_off, tk->tie_off, nch);
    DIMB_LAUNCH_CHECK(ctx);
    topk_gather_write_kernel<<<dim3(nch, B), kTopkThreads, 0, st>>>(c.cand_idx, c.cand_score, c.cand_count, tk->state, tk->gt_off,
                                                                    tk->tie_off, tk->keys0, sel_idx, sel_score, HW, K, cap, nch);
    DIMB_LAUNCH_CHECK(ctx);
    // keys0 -> keys1 -> keys0 -> keys1 -> sel_idx / sel_score
    const dim3 sgrid(nblk, B);
    for (int pass = 0; pass < 4; ++pass) {
      const unsigned long long* src = pass & 1 ? tk->keys1 : tk->keys0;
      unsigned long long* dst = pass == 3 ? nullptr : (pass & 1 ? tk->keys0 : tk->keys1);
      const int shift = 32 + 8 * pass;
      topk_sort_pass_kernel<false><<<sgrid, kTopkThreads, 0, st>>>(src, dst, sel_idx, sel_score, tk->digit_off, tk->state, K, cap, nblk, shift);
      DIMB_LAUNCH_CHECK(ctx);
      topk_sort_scan_kernel<<<B, 256, 0, st>>>(tk->digit_off, tk->state, nblk);
      DIMB_LAUNCH_CHECK(ctx);
      topk_sort_pass_kernel<true><<<sgrid, kTopkThreads, 0, st>>>(src, dst, sel_idx, sel_score, tk->digit_off, tk->state, K, cap, nblk, shift);
      DIMB_LAUNCH_CHECK(ctx);
    }
  }
  if (sort_all) {
    topk_fill_kernel<<<dim3(ceil_div(K, 256), B), 256, 0, st>>>(c.cand_idx, c.cand_count, sel_idx, sel_score, HW, K, cap);
    DIMB_LAUNCH_CHECK(ctx);
  }
  return DIMB_OK;
}

}  // namespace
