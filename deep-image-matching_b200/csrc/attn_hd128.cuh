// attn_hd128.cuh - tensor-core flash attention for head dims 65..128 (LighterGlue: one head of 96), used by the shape-generic
// LightGlue path (lightglue_generic.cu).  Attention is 93 % of LighterGlue's arithmetic (19.3 of 20.7 GMAC per 2048 x 2048 pair); the
// linears stay on the plain fp32 kernels.
//
// The kernel is attention.cuh's with the head dim padded to 128 (zero columns): Q / K tiles are two SWIZZLE_128B atoms side by side,
// the V^T tile has 128 rows.  Inputs are packed by gx_pack_rows_kernel / gx_pack_vt_kernel from the fp32 activations of the generic
// path; the result is written as fp32 rows.  EXACT mode = fp16 hi / lo planes, three MMAs per product (fp32-class); FAST = hi plane only.
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
__global__ void gx_pack_rows_kernel(const float* __restrict__ src, int ld, int n, int hd, int NP, __half* __restrict__ hi,
                                    __half* __restrict__ lo) {
  gx_pack_rows_one(src, ld, n, hd, NP, hi, lo, blockIdx.x, blockIdx.y, threadIdx.x);  // 128 threads
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
__global__ void gx_pack_vt_kernel(const float* __restrict__ src, int ld, int n, int hd, int NP, __half* __restrict__ hi,
                                  __half* __restrict__ lo) {
  gx_pack_vt_block(src, ld, n, hd, NP, hi, lo, blockIdx.x * 32, blockIdx.y * 32, blockIdx.z);
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

// grid (ceil(nq / 128), H)
template <bool SPLIT>
__global__ void __launch_bounds__(kAttnThreads, 1)
gx_attn_tc_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                  const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
                  const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, AttnXArgs a) {
  const int head = blockIdx.y, qbase = blockIdx.x * kAttnTile;
  if (qbase >= a.nq) return;
  const AttnOutX out{a.out + static_cast<size_t>(qbase) * a.ldo + head * a.hd, a.ldo, a.hd};
  attn_tile<kXHd, SPLIT>(&tmQh, &tmQl, &tmKh, &tmKl, &tmVh, &tmVl, head * a.NP + qbase, head * a.NP, head * kXHd, a.nq - qbase, a.nk,
                         a.scale, a.lazy, out);
}

inline int launch_attn_hd128(dimb_ctx* ctx, cudaStream_t st, const CUtensorMap* Q /*[2] hi,lo, box 128 rows*/,
                             const CUtensorMap* K /*[2], box 64 rows*/, const CUtensorMap* V /*[2] V^T, box 128 rows*/, int heads,
                             const AttnXArgs& a, bool exact) {
  if (a.nq <= 0) return DIMB_OK;
  dim3 grid((a.nq + kAttnTile - 1) / kAttnTile, heads);
  if (exact) {
    constexpr int smem = AttnGeom<kXHd, true>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, gx_attn_tc_kernel<true>, smem));
    gx_attn_tc_kernel<true><<<grid, kAttnThreads, smem, st>>>(Q[0], Q[1], K[0], K[1], V[0], V[1], a);
  } else {
    constexpr int smem = AttnGeom<kXHd, false>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, gx_attn_tc_kernel<false>, smem));
    gx_attn_tc_kernel<false><<<grid, kAttnThreads, smem, st>>>(Q[0], Q[0], K[0], K[0], V[0], V[0], a);
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
