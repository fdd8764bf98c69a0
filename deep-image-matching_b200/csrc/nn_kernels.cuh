// nn_kernels.cuh - the brute-force NN engine of nn_match.cu: prep, the top-2 GEMM epilogues, merge and select kernels and nn_run,
// which drives them on 2P sides.  The three dimb_nn_match* entries (nn_match.cu) call nn_run, and the self-test library (selftest.cu,
// dimb_selftest_nn_*) calls the same pieces on caller-given descriptors and row statistics.  See nn_match.cu for the stages.
#pragma once
#include <algorithm>
#include <vector>

#include "gemm.cuh"

namespace {

// 128 x 128 output tiles: with register accumulators a 128 x 256 tile leaves the running top-2 epilogue too few registers
// (it spills), so the wider tile's halved A re-reads are not worth it
constexpr int kNnBN = 128;

// one side of the engine (dimb_feats_dev, resolved)
struct NNSideIn {
  const void* desc;  // (D, n) rows of pitch ld, float32 or float16
  const int* n;      // device count (rows = min(*n, n_cap)), or NULL: n_cap rows (the host-count entries)
  int n_cap, ld, f16, round_fp16;
};

__host__ __device__ inline bool nn_trivially_empty(int n0, int n1, int mode) {
  // kornia: empty inputs / fewer than two candidates for the ratio tests -> no match
  return n0 == 0 || n1 == 0 || (mode == DIMB_NN_SNN && n1 < 2) || (mode == DIMB_NN_SMNN && (n0 < 2 || n1 < 2));
}

__device__ __forceinline__ int nn_side_rows(const NNSideIn& s) { return s.n ? max(0, min(*s.n, s.n_cap)) : s.n_cap; }

// The largest squared distance whose float32 distance sqrt(max(s, 0)) equals that of s: 0 for s <= 0, else s or a few floats above it
// (sqrt halves relative spacings).  Out of line: nn_top2_chunk calls it only for a chunk whose two best squares nearly tie.
__device__ __noinline__ float nn_same_dist_max(float s) {
  if (s <= 0.f) return 0.f;
  const float r = sqrtf(s);
  for (;;) {
    const float up = __int_as_float(__float_as_int(s) + 1);
    if (sqrtf(up) != r) return s;
    s = up;
  }
}

// Running (best, second best, argbest) of one row over the 32 columns n..n+31 of a GEMM tile, written as the partial of chunk n / 32
// at pd1 / pd2 / pi1 [o].  Squared distances |a|^2 + |b|^2 - 2ab are compared as they are, which keeps the IEEE sqrt (8
// instructions) off the per-element path.  sqrt is monotone but not strictly: squared distances a few ulps apart can round to the
// same float distance (integers from 2^22 on, e.g. 4197200 and 4197201; floats at any size), and torch.cdist + min then keeps the
// earlier column, while the squared order keeps the smaller square.  Such a column lies within 2^-21 (relative) of the best, so
// when the second smallest square is that close, hi = the largest square with the best's distance is found, and if the second is
// within it the first column at or below hi becomes the best (the old best, the smallest square, is then the second).  The merge
// kernel compares the chunk partials in the sqrt domain again.
__device__ __forceinline__ void nn_top2_chunk(const float (&v)[32], float a2, const float* __restrict__ nb, int n, int n_cols,
                                              float* pd1, float* pd2, int* pi1, size_t o) {
  float d1 = INFINITY, d2 = INFINITY;
  int i1 = 0x7fffffff;
  const float4* nb4 = reinterpret_cast<const float4*>(nb + n);  // norms are padded to a multiple of 128 columns
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 b = __ldg(nb4 + q);
    const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = 4 * q + e;
      float d = fmaf(-2.f, v[j], a2 + bb[e]);
      if (n + j >= n_cols) d = INFINITY;
      if (d < d1) {
        d2 = d1;
        d1 = d;
        i1 = n + j;
      } else if (d < d2) {
        d2 = d;
      }
    }
  }
  if (d1 < INFINITY && d2 <= fmaxf(d1, 0.f) * (1.f + 0x1p-21f)) {
    const float hi = nn_same_dist_max(d1);
    if (d2 <= hi) {
      int first = i1;
#pragma unroll
      for (int q = 7; q >= 0; --q) {
        const float4 b = __ldg(nb4 + q);
        const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int e = 3; e >= 0; --e) {
          const int j = 4 * q + e;
          if (n + j < n_cols && fmaf(-2.f, v[j], a2 + bb[e]) <= hi) first = n + j;
        }
      }
      if (first != i1) {
        i1 = first;
        d2 = d1;
      }
    }
  }
  pd1[o] = d1;
  pd2[o] = d2;
  pi1[o] = i1;
}

// Top-2 epilogue of one pair with host counts (dimb_nn_match_dev / dimb_nn_match): the A and B maps start at the row side and its
// partner, the launch covers exactly the tiles of the counts, and the counts are kernel arguments.  The B panel is the same for
// every tile, so it may stay resident in shared memory.
struct EpiNNTop2 : EpiBase {
  const float *na, *nb;  // squared norms of A rows / B rows
  float *pd1, *pd2;      // [rows][chunks] best / second best SQUARED distance of each 32-column chunk
  int* pi1;              // [rows][chunks] argbest
  int n_rows, n_cols, chunks;
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float*) const {
    const int row = tc.m0 + r;
    if (row >= n_rows) return;
    nn_top2_chunk(v, na[row], nb, n, n_cols, pd1, pd2, pi1, static_cast<size_t>(row) * chunks + (n >> 5));
  }
};

// Top-2 epilogue of P pairs with device counts: rows of sides 2p + swap against their partner sides 2p + 1 - swap, both maps over
// all sides; row tiles at or past a side's live count, and pairs with an empty partner, are skipped on the device.
struct EpiNNTop2Batch : EpiBase {
  static constexpr bool kConstB = false;
  const float* norm;     // [2P][NPp] squared norms
  const int* n_live;     // [2P] live rows
  float *pd1, *pd2;      // [P][NPp][stride]
  int* pi1;
  int NPp, tps, swap, stride;  // tps: row tiles per pair in the launch
  __device__ int m0_of(int t) const { return ((t / tps) * 2 + swap) * NPp + (t % tps) * kTileM; }
  __device__ bool tile_active(const TileCoord& tc) const {
    const int side = tc.m0 / NPp;
    return tc.m0 - side * NPp < n_live[side] && tc.n0 < n_live[side ^ 1];
  }
  __device__ int b_row_offset(const TileCoord& tc) const { return ((tc.m0 / NPp) ^ 1) * NPp; }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float*) const {
    const int side = tc.m0 / NPp, row = tc.m0 - side * NPp + r;
    if (row >= n_live[side]) return;
    nn_top2_chunk(v, norm[tc.m0 + r], norm + (side ^ 1) * NPp, n, n_live[side ^ 1], pd1, pd2, pi1,
                  (static_cast<size_t>(side >> 1) * NPp + row) * stride + (n >> 5));
  }
};

// grid (NPp / 32, 2P), block (32, 8): (D,n) descriptors of every side -> [2P][NPp][Dp] fp16 hi (/ lo) + squared norms, transposing
// 32x32 tiles.  Dp = D rounded up to 64: the padding columns are zero, which changes no distance (any descriptor size works).  Rows
// past the live count get a zero norm (keeping the masked padded columns finite) and no hi / lo.  round_fp16 rounds float32 inputs
// to fp16 first (round to nearest even, the features.h5 cast).  any_lo is set when some value is not exactly fp16: only then does
// the GEMM need the lo planes.
__global__ void nn_prep_kernel(const NNSideIn* __restrict__ in, int mode, int D, int Dp, int NPp, __half* __restrict__ hi,
                               __half* __restrict__ lo, float* __restrict__ norm, int* __restrict__ n_live, int* __restrict__ any_lo) {
  __shared__ float tile[32][33];
  const int side = blockIdx.y, t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const NNSideIn si = in[side];
  const int na = nn_side_rows(in[side & ~1]), nb = nn_side_rows(in[side | 1]);
  const int n = nn_trivially_empty(na, nb, mode) ? 0 : ((side & 1) ? nb : na);
  if (blockIdx.x == 0 && tx == 0 && ty == 0) n_live[side] = n;
  const size_t r0 = static_cast<size_t>(side) * NPp;
  if (t0 >= n) {
    if (tx == 0)
      for (int k = ty; k < 32; k += 8) norm[r0 + t0 + k] = 0.f;
    return;
  }
  // row k = ty + 8 q of the tile (q = 0..3, unrolled so that acc stays in registers)
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  bool nz = false;
  for (int c0 = 0; c0 < Dp; c0 += 32) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = ty + 8 * q;
      float v = 0.f;
      if (t0 + tx < n && c0 + k < D) {
        const size_t o = static_cast<size_t>(c0 + k) * si.ld + t0 + tx;
        if (si.f16) {
          v = __half2float(static_cast<const __half*>(si.desc)[o]);
        } else {
          v = static_cast<const float*>(si.desc)[o];
          if (si.round_fp16) v = __half2float(__float2half_rn(v));
        }
      }
      tile[k][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = ty + 8 * q;
      const float v = tile[tx][k];  // token t0+k, channel c0+tx
      if (t0 + k < n) {
        __half h, l;
        split_f32(v, h, l);
        hi[(r0 + t0 + k) * Dp + c0 + tx] = h;
        if (lo) lo[(r0 + t0 + k) * Dp + c0 + tx] = l;
        nz |= __half2float(l) != 0.f;
      }
      float sq = v * v;
#pragma unroll
      for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      acc[q] += sq;
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (tx == 0) norm[r0 + t0 + ty + 8 * q] = acc[q];  // 0 on rows past n: their tile values are zero
  if (any_lo && __any_sync(0xffffffffu, nz) && tx == 0) atomicOr(any_lo, 1);
}

// warp per row of the sides 2p + swap (rows_pp rows per pair in the grid; rows past the live count exit): merge the chunk partials
// that hold a live column of the partner, chunks [0, ceil(n / 32)) -> best, second, arg (first index wins ties) at row side * NPp + row
// of d1 / d2 / i1.  The chunks past them in a 128-column tile are all +inf and would change no result.  The partials are squared
// distances, the comparison happens on the distances (clamp at 0, IEEE sqrt) like torch.cdist + min / topk.
__global__ void nn_merge_kernel(const float* __restrict__ pd1, const float* __restrict__ pd2, const int* __restrict__ pi1,
                                const int* __restrict__ n_live, int P, int NPp, int rows_pp, int swap, int stride, float* __restrict__ d1,
                                float* __restrict__ d2, int* __restrict__ i1) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= P * rows_pp) return;
  const int p = q / rows_pp, row = q - p * rows_pp, side = 2 * p + swap;
  if (row >= n_live[side]) return;
  const int chunks = ceil_div(n_live[side ^ 1], 32);
  const size_t base = (static_cast<size_t>(p) * NPp + row) * stride;
  float b1 = INFINITY, b2 = INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane; c < chunks; c += 32) {
    const size_t o = base + c;
    const float x1 = sqrtf(fmaxf(pd1[o], 0.f)), x2 = sqrtf(fmaxf(pd2[o], 0.f));
    const int xi = pi1[o];
    if (x1 < b1 || (x1 == b1 && xi < bi)) {
      b2 = fminf(b1, x2);
      b1 = x1;
      bi = xi;
    } else {
      b2 = fminf(b2, x1);
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float x1 = __shfl_xor_sync(0xffffffffu, b1, o), x2 = __shfl_xor_sync(0xffffffffu, b2, o);
    const int xi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (x1 < b1 || (x1 == b1 && xi < bi)) {
      b2 = fminf(b1, x2);
      b1 = x1;
      bi = xi;
    } else {
      b2 = fminf(b2, x1);
    }
  }
  if (lane == 0) {
    const size_t out = static_cast<size_t>(side) * NPp + row;
    d1[out] = b1;
    d2[out] = b2;
    i1[out] = bi;
  }
}

// one CTA per pair: apply the kornia mode logic to the row statistics of its sides (forward at side 2p, backward at side 2p + 1) and
// compact in ascending row order into the pair's [cap] rows; count = the full number of matches
__global__ void __launch_bounds__(1024)
nn_select_kernel(int mode, float th, const int* __restrict__ n_live, int NPp, const float* __restrict__ sd1, const float* __restrict__ sd2,
                 const int* __restrict__ si1, long long* __restrict__ idx_all, float* __restrict__ dist_all, int* __restrict__ count, int cap) {
  __shared__ int wsum[32];
  __shared__ int s_base;
  const int t = threadIdx.x, p = blockIdx.x;
  const int n0 = n_live[2 * p], n1 = n_live[2 * p + 1];
  const size_t f = static_cast<size_t>(2 * p) * NPp, b = f + NPp;
  const float *fd1 = sd1 + f, *fd2 = sd2 + f, *bd1 = sd1 + b, *bd2 = sd2 + b;
  const int *fi1 = si1 + f, *bi1 = si1 + b;
  long long* idx = idx_all + static_cast<size_t>(p) * cap * 2;
  float* dist = dist_all + static_cast<size_t>(p) * cap;
  if (t == 0) s_base = 0;
  __syncthreads();
  const int ms = min(n0, n1);
  const bool swapped = (mode == DIMB_NN_MNN) && (n0 > n1);  // kornia match_mnn iterates the smaller side
  const int iters = (mode == DIMB_NN_MNN) ? ms : n0;
  for (int base = 0; base < iters; base += blockDim.x) {
    const int i = base + t;
    bool valid = false;
    long long a = 0, bb = 0;
    float dv = 0.f;
    if (i < iters) {
      if (mode == DIMB_NN_NN) {
        valid = true, a = i, bb = fi1[i], dv = fd1[i];
      } else if (mode == DIMB_NN_MNN) {
        if (!swapped) {
          const int j = fi1[i];
          valid = bi1[j] == i, a = i, bb = j, dv = fd1[i];
        } else {
          const int j = bi1[i];  // i indexes desc2
          valid = fi1[j] == i, a = j, bb = i, dv = bd1[i];
        }
      } else if (mode == DIMB_NN_SNN) {
        const float ratio = fd1[i] / fd2[i];
        valid = ratio <= th, a = i, bb = fi1[i], dv = ratio;
      } else {  // SMNN
        const float rf = fd1[i] / fd2[i];
        const int j = fi1[i];
        const float rb = bd1[j] / bd2[j];
        valid = (rf <= th) && (rb <= th) && (bi1[j] == i);
        a = i, bb = j, dv = fmaxf(rf, rb);
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, valid);
    if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
    __syncthreads();
    int before = s_base;
    for (int wv = 0; wv < (t >> 5); ++wv) before += wsum[wv];
    before += __popc(bal & ((1u << (t & 31)) - 1u));
    if (valid && before < cap) {
      idx[2 * before] = a;
      idx[2 * before + 1] = bb;
      dist[before] = dv;
    }
    __syncthreads();
    if (t == 0) {
      int tot = 0;
      for (int wv = 0; wv < 32; ++wv) tot += wsum[wv];
      s_base += tot;
    }
    __syncthreads();
  }
  if (t == 0) count[p] = s_base;
}

// Launch geometry of one call: NPp rows per side; per direction (0: rows of sides 2p, 1: rows of sides 2p + 1) the row tiles per
// pair and the padded partner columns.  Device counts: every tile of NPp (dead ones are skipped on the device).  Host counts
// (P = 1): exactly the tiles of the counts.
struct NNShape {
  int P, NPp, tps[2], npad[2];
  bool host;  // the counts are host_n (P = 1): EpiNNTop2 with the counts as kernel arguments
  int hn[2];
};

NNShape nn_shape(int P, int max_cap, const int* host_n) {
  NNShape s;
  s.P = P;
  s.host = host_n != nullptr;
  s.hn[0] = host_n ? host_n[0] : 0;
  s.hn[1] = host_n ? host_n[1] : 0;
  s.NPp = std::max(round_up(max_cap, kNnBN), kNnBN);
  for (int d = 0; d < 2; ++d) {
    s.tps[d] = host_n ? ceil_div(host_n[d], kTileM) : s.NPp / kTileM;
    s.npad[d] = host_n ? round_up(host_n[d ^ 1], kNnBN) : s.NPp;
  }
  return s;
}

struct NNWork {  // grow-only scratch of one matching call (context slots: no cudaMalloc / cudaFree in steady state)
  __half *hi, *lo;  // [2P][NPp][Dp]; lo is NULL without the split
  float* norm;      // [2P][NPp]
  NNSideIn* sides;  // [2P]
  int* n_live;      // [2P]
  float *pd1, *pd2; // [P][NPp][NPp / 32] chunk partials, shared by the two directions
  int* pi1;
  float *d1, *d2;   // [2P][NPp] merged row statistics
  int *i1, *any_lo;
  CUtensorMap mA[2][2], mB[2][2];  // [direction][hi, lo]: host counts: the row side / its partner only; else all rows
  int Dp;
};

// slots 0..7 belong to the host-buffer entry (staging + outputs)
int nn_workspace(dimb_ctx* ctx, const NNShape& sh, int D, bool want_lo, NNWork* w) {
  int slot = 8;
  auto alloc = [&](void* p, size_t bytes) -> int { return dimb_scratch(ctx, slot++, bytes, reinterpret_cast<void**>(p)); };
  const int P = sh.P, NPp = sh.NPp, Dp = w->Dp = round_up(D, 64);
  const size_t rows = static_cast<size_t>(2 * P) * NPp, plane = rows * Dp * sizeof(__half);
  DIMB_TRY(alloc(&w->hi, plane));
  DIMB_TRY(alloc(&w->lo, want_lo ? plane : 256));
  if (!want_lo) w->lo = nullptr;
  DIMB_TRY(alloc(&w->norm, rows * sizeof(float)));
  DIMB_TRY(alloc(&w->sides, 2 * P * sizeof(NNSideIn)));
  DIMB_TRY(alloc(&w->n_live, 2 * P * sizeof(int)));
  const size_t part = static_cast<size_t>(P) * NPp * (NPp / 32);
  DIMB_TRY(alloc(&w->pd1, part * sizeof(float)));
  DIMB_TRY(alloc(&w->pd2, part * sizeof(float)));
  DIMB_TRY(alloc(&w->pi1, part * sizeof(int)));
  DIMB_TRY(alloc(&w->d1, rows * sizeof(float)));
  DIMB_TRY(alloc(&w->d2, rows * sizeof(float)));
  DIMB_TRY(alloc(&w->i1, rows * sizeof(int)));
  DIMB_TRY(alloc(&w->any_lo, sizeof(int)));
  __half* planes[2] = {w->hi, want_lo ? w->lo : w->hi};
  for (int d = 0; d < 2; ++d)
    for (int pl = 0; pl < 2; ++pl) {
      __half* a = planes[pl] + (sh.host ? static_cast<size_t>(d) * NPp * Dp : 0);
      __half* b = planes[pl] + (sh.host ? static_cast<size_t>(d ^ 1) * NPp * Dp : 0);
      const size_t r = sh.host ? NPp : rows;
      DIMB_TRY(dimb_tmap_2d(ctx, &w->mA[d][pl], a, r, Dp, Dp, kTileM));
      DIMB_TRY(dimb_tmap_2d(ctx, &w->mB[d][pl], b, r, Dp, Dp, kNnBN));  // as B operand: boxes of kNnBN rows
    }
  return DIMB_OK;
}

// rows of sides 2p + d against sides 2p + 1 - d: top-2 GEMM of every pair, then the merge
int nn_direction(dimb_ctx* ctx, cudaStream_t st, const NNWork& w, const NNShape& sh, int d, bool split) {
  const TcOperands ops{w.mA[d][0], w.mA[d][1], w.mB[d][0], w.mB[d][1]};
  const int m_tiles = sh.P * sh.tps[d], stride = sh.npad[d] / 32;
  GemmArgs g{};
  g.num_kb = w.Dp / 64;
  g.M = sh.host ? sh.hn[d] : 2 * sh.P * sh.NPp;
  g.N = sh.npad[d];
  // descriptors that are exactly fp16 (everything read back from features.h5 is) have zero lo planes: ONE MMA per product
  // gives exact products (the fp32 accumulation rounds either way), and (host counts) the 256-descriptor B panel (128 KB)
  // stays resident in shared memory while the A tiles stream
  if (sh.host) {
    EpiNNTop2 e;
    e.na = w.norm + static_cast<size_t>(d) * sh.NPp;
    e.nb = w.norm + static_cast<size_t>(d ^ 1) * sh.NPp;
    e.pd1 = w.pd1;
    e.pd2 = w.pd2;
    e.pi1 = w.pi1;
    e.n_rows = sh.hn[d];
    e.n_cols = sh.hn[d ^ 1];
    e.chunks = stride;
    DIMB_TRY((launch_gemm<kNnBN, false>(ctx, st, ops, g, e, m_tiles, sh.npad[d], "nn.top2_gemm", split ? 1 : 0)));
  } else {
    EpiNNTop2Batch e;
    e.norm = w.norm;
    e.n_live = w.n_live;
    e.pd1 = w.pd1;
    e.pd2 = w.pd2;
    e.pi1 = w.pi1;
    e.NPp = sh.NPp;
    e.tps = sh.tps[d];
    e.swap = d;
    e.stride = stride;
    DIMB_TRY((launch_gemm<kNnBN, false>(ctx, st, ops, g, e, m_tiles, sh.npad[d], "nn.top2_gemm", split ? 1 : 0)));
  }
  ProfScope prof(ctx, st, "nn.merge");
  const int rows_pp = sh.tps[d] * kTileM;
  nn_merge_kernel<<<ceil_div(sh.P * rows_pp, 8), 256, 0, st>>>(w.pd1, w.pd2, w.pi1, w.n_live, sh.P, sh.NPp, rows_pp, d, stride, w.d1, w.d2,
                                                               w.i1);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// The engine on 2P sides.  split: 1 / 0 = three / one MMA per product; -1 = decide from the prepared operands (one host
// synchronise: the host entry's check for descriptors that are exactly fp16).
int nn_run(dimb_ctx* ctx, cudaStream_t st, const std::vector<NNSideIn>& sides, const NNShape& sh, int D, int mode, float th, int split,
           long long* d_idx, float* d_dist, int* d_n, int cap) {
  NNWork w;
  DIMB_TRY(nn_workspace(ctx, sh, D, split != 0, &w));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(w.sides, sides.data(), sides.size() * sizeof(NNSideIn), cudaMemcpyHostToDevice, st));
  {
    ProfScope prof(ctx, st, "nn.prep");
    if (split < 0) DIMB_CUDA_OK(ctx, cudaMemsetAsync(w.any_lo, 0, sizeof(int), st));
    nn_prep_kernel<<<dim3(sh.NPp / 32, 2 * sh.P), dim3(32, 8), 0, st>>>(w.sides, mode, D, w.Dp, sh.NPp, w.hi, w.lo, w.norm, w.n_live,
                                                                         split < 0 ? w.any_lo : nullptr);
    DIMB_LAUNCH_CHECK(ctx);
  }
  if (split < 0) {
    int any_lo = 0;
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(&any_lo, w.any_lo, sizeof(int), cudaMemcpyDeviceToHost, st));
    DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
    split = any_lo != 0;
  }
  DIMB_TRY(nn_direction(ctx, st, w, sh, 0, split));
  if (mode == DIMB_NN_MNN || mode == DIMB_NN_SMNN) DIMB_TRY(nn_direction(ctx, st, w, sh, 1, split));
  ProfScope prof(ctx, st, "nn.select");
  nn_select_kernel<<<sh.P, 1024, 0, st>>>(mode, th, w.n_live, sh.NPp, w.d1, w.d2, w.i1, d_idx, d_dist, d_n, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
