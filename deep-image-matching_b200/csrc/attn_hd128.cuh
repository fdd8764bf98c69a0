// attn_hd128.cuh - tensor-core flash attention for head dims 65..128 (LighterGlue: one head of 96), used by the shape-generic
// LightGlue path (lightglue_generic.cu).  Attention is 93 % of LighterGlue's arithmetic (19.3 of 20.7 GMAC per 2048 x 2048 pair); the
// linears stay on the plain fp32 kernels.
//
// The kernel is attention.cuh's with the head dim padded to 128 (zero columns): Q / K tiles are two SWIZZLE_128B atoms side by side,
// the V^T tile has 128 rows.  S sides share one set of buffers: side s owns fp32 rows [s NP, (s + 1) NP) and packed rows
// [s h NPp, (s + 1) h NPp).  hd128_attend packs the fp32 activations of every running side (lgx_pack_rows_kernel / lgx_pack_vt_kernel)
// and runs the attention on them; the result is written as fp32 rows.  EXACT mode = fp16 hi / lo planes, three MMAs per product
// (fp32-class); FAST = hi plane only.
#pragma once
#include "attention.cuh"
#include "common.cuh"

namespace {

constexpr int kXHd = 128;   // padded head dim

struct AttnXArgs {
  int nq, nk;       // live queries / keys
  int NP;           // rows per head in the packed Q / K buffers, columns of the packed V^T buffer
  int hd;           // real head dim (<= 128)
  float scale;      // hd^-0.5
  float lazy;       // lazy-rescale threshold (log2 units)
  float* out;       // [nq][ldo] fp32, head h at columns h * hd
  int ldo;
};

// rows a layer kernel works on: none once the side's pair has stopped
__device__ __forceinline__ int live_rows(const int* nact, const int* stopped, int side) { return stopped[side >> 1] ? 0 : nact[side]; }

// fp32 rows [n][ld] (head h at columns h*hd) -> fp16 hi / lo planes [H][NP][128]; rows >= n and columns >= hd are zero
__device__ __forceinline__ void gx_pack_rows_one(const float* __restrict__ src, int ld, int n, int hd, int NP, __half* __restrict__ hi,
                                                 __half* __restrict__ lo, int row, int head, int c) {
  float v = 0.f;
  if (row < n && c < hd) v = src[static_cast<size_t>(row) * ld + head * hd + c];
  __half h, l;
  split_f32(v, h, l);
  const size_t o = (static_cast<size_t>(head) * NP + row) * kXHd + c;
  hi[o] = h;
  if (lo) lo[o] = l;
}

// fp32 rows [n][ld] -> transposed fp16 hi / lo planes [H][128][NP] (the K-major B operand of P V); columns >= n and rows >= hd are zero
__device__ __forceinline__ void gx_pack_vt_block(const float* __restrict__ src, int ld, int n, int hd, int NP, __half* __restrict__ hi,
                                                 __half* __restrict__ lo, int t0, int c0, int head) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;  // (32, 8)
  for (int k = ty; k < 32; k += 8) {
    const int tok = t0 + k, c = c0 + tx;
    tile[k][tx] = (tok < n && c < hd) ? src[static_cast<size_t>(tok) * ld + head * hd + c] : 0.f;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int c = c0 + k, tok = t0 + tx;
    __half h, l;
    split_f32(tile[tx][k], h, l);
    const size_t o = (static_cast<size_t>(head) * kXHd + c) * NP + tok;
    hi[o] = h;
    if (lo) lo[o] = l;
  }
}

// packed tensor-core operands of every running side: grid (NPp, h, S) rows, (NPp / 32, 4, h * S) V^T
__global__ void lgx_pack_rows_kernel(const float* __restrict__ src, int d, int hd, int NP, int NPp, __half* __restrict__ hi, __half* __restrict__ lo,
                                     const int* __restrict__ nact, const int* __restrict__ stopped) {
  const int side = blockIdx.z;
  if (stopped[side >> 1]) return;
  const size_t o = static_cast<size_t>(side) * gridDim.y * NPp * kXHd;
  gx_pack_rows_one(src + static_cast<size_t>(side) * NP * d, d, nact[side], hd, NPp, hi + o, lo ? lo + o : nullptr, blockIdx.x, blockIdx.y,
                   threadIdx.x);
}
__global__ void lgx_pack_vt_kernel(const float* __restrict__ src, int d, int hd, int h, int NP, int NPp, __half* __restrict__ hi,
                                   __half* __restrict__ lo, const int* __restrict__ nact, const int* __restrict__ stopped) {
  const int side = blockIdx.z / h, head = blockIdx.z - side * h;
  if (stopped[side >> 1]) return;
  const size_t o = static_cast<size_t>(side) * h * kXHd * NPp;
  gx_pack_vt_block(src + static_cast<size_t>(side) * NP * d, d, nact[side], hd, NPp, hi + o, lo ? lo + o : nullptr, blockIdx.x * 32,
                   blockIdx.y * 32, head);
}

struct AttnOutX {  // O rows of one head -> fp32 [nq][ldo], head h at columns h * hd; padding columns >= hd dropped
  float* out;
  int ldo, hd;
  __device__ void operator()(int row, int col, float x, float y) const {
    float* dst = out + static_cast<size_t>(row) * ldo + col;
    if (col < hd) dst[0] = x;
    if (col + 1 < hd) dst[1] = y;
  }
};

// grid (NPp / 128, h, S): the side's query rows against its own keys (cross 0) or its partner's (cross 1)
template <bool SPLIT>
__global__ void __launch_bounds__(kAttnThreads, 1)
lgx_attn_tc_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                   const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
                   const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, AttnXArgs a, int NP, int cross,
                   const int* __restrict__ nact, const int* __restrict__ stopped) {
  const int head = blockIdx.y, side = blockIdx.z, ks = cross ? side ^ 1 : side, h = gridDim.y, qbase = blockIdx.x * kAttnTile;
  const int nq = live_rows(nact, stopped, side);
  if (qbase >= nq) return;
  const AttnOutX out{a.out + (static_cast<size_t>(side) * NP + qbase) * a.ldo + head * a.hd, a.ldo, a.hd};
  attn_tile<kXHd, SPLIT>(&tmQh, &tmQl, &tmKh, &tmKl, &tmVh, &tmVl, (side * h + head) * a.NP + qbase, (ks * h + head) * a.NP,
                         (ks * h + head) * kXHd, nq - qbase, nact[ks], a.scale, a.lazy, out);
}

// The packed operands of up to S sides of d = h * hd columns, NP fp32 rows per side, NPp = NP rounded up to the query tile: Q / K rows
// [S][h][NPp][128], V^T [S][h][128][NPp], hi and lo planes (zero-initialised: pad rows / columns stay finite), and their tensor maps
// (Q box 128 rows, Q as keys and K box 64 rows, V^T box 128 rows)
struct Hd128Ops {
  int S, h, d, hd, NP, NPp;
  __half *q[2], *k[2], *vt[2];
  CUtensorMap mQ128[2], mQ64[2], mK64[2], mVt[2];
};

inline int hd128_maps(dimb_ctx* ctx, Hd128Ops& o) {
  const uint64_t rows = static_cast<uint64_t>(o.S) * o.h * o.NPp;
  for (int pl = 0; pl < 2; ++pl) {
    DIMB_TRY(dimb_tmap_2d(ctx, &o.mQ128[pl], o.q[pl], rows, kXHd, kXHd, kAttnTile));
    DIMB_TRY(dimb_tmap_2d(ctx, &o.mQ64[pl], o.q[pl], rows, kXHd, kXHd, kAttnBlk));
    DIMB_TRY(dimb_tmap_2d(ctx, &o.mK64[pl], o.k[pl], rows, kXHd, kXHd, kAttnBlk));
    DIMB_TRY(dimb_tmap_2d(ctx, &o.mVt[pl], o.vt[pl], static_cast<uint64_t>(o.S) * o.h * kXHd, o.NPp, o.NPp, kXHd));
  }
  return DIMB_OK;
}

// Attention of the first S <= o.S sides over fp32 rows q / k / v [S][NP][d] (live rows nact[side]; a stopped pair is skipped): packs q,
// k (self only) and v, then side s's queries attend to its own keys (cross 0) or to the q rows of side s ^ 1 (cross 1: the shared to_qk
// projection).  out [S][NP][d]: rows past a side's live count are not written.  lazy: rescale threshold in log2 units.
inline int hd128_attend(dimb_ctx* ctx, cudaStream_t st, const Hd128Ops& o, int S, const float* q, const float* k, const float* v, int cross,
                        const int* nact, const int* stopped, float lazy, float* out) {
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int h = o.h, d = o.d, hd = o.hd, NP = o.NP, NPp = o.NPp;
  lgx_pack_rows_kernel<<<dim3(NPp, h, S), kXHd, 0, st>>>(q, d, hd, NP, NPp, o.q[0], exact ? o.q[1] : nullptr, nact, stopped);
  DIMB_LAUNCH_CHECK(ctx);
  if (!cross) {
    lgx_pack_rows_kernel<<<dim3(NPp, h, S), kXHd, 0, st>>>(k, d, hd, NP, NPp, o.k[0], exact ? o.k[1] : nullptr, nact, stopped);
    DIMB_LAUNCH_CHECK(ctx);
  }
  lgx_pack_vt_kernel<<<dim3(NPp / 32, kXHd / 32, h * S), dim3(32, 8), 0, st>>>(v, d, hd, h, NP, NPp, o.vt[0], exact ? o.vt[1] : nullptr, nact,
                                                                               stopped);
  DIMB_LAUNCH_CHECK(ctx);
  AttnXArgs a;
  a.nq = 0, a.nk = 0, a.NP = NPp, a.hd = hd;
  a.scale = 1.f / sqrtf(static_cast<float>(hd));
  a.lazy = lazy;
  a.out = out, a.ldo = d;
  const dim3 grid(NPp / kAttnTile, h, S);
  const CUtensorMap* K = cross ? o.mQ64 : o.mK64;
  if (exact) {
    constexpr int smem = AttnGeom<kXHd, true>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, lgx_attn_tc_kernel<true>, smem));
    lgx_attn_tc_kernel<true><<<grid, kAttnThreads, smem, st>>>(o.mQ128[0], o.mQ128[1], K[0], K[1], o.mVt[0], o.mVt[1], a, NP, cross, nact, stopped);
  } else {
    constexpr int smem = AttnGeom<kXHd, false>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, lgx_attn_tc_kernel<false>, smem));
    lgx_attn_tc_kernel<false><<<grid, kAttnThreads, smem, st>>>(o.mQ128[0], o.mQ128[0], K[0], K[0], o.mVt[0], o.mVt[0], a, NP, cross, nact, stopped);
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
