// lg_kernels.cuh - the tensor-core building blocks of a 256-dim / 4-head x 64 attentional matcher, shared by LightGlue
// (lightglue.cu) and SuperGlue (superglue.cu, same attention shape: models/superglue.py:96-152): the GEMM epilogues that produce the
// attention operands (q / k head-split with optional rotary, V^T), the message / residual epilogues on the [x | message] concat
// buffer, the final projection / similarity epilogues, and the launch of the flash-attention kernel (attention.cuh).
#pragma once
#include "attention.cuh"
#include "gemm.cuh"

namespace {

constexpr int kD = 256;    // descriptor_dim
constexpr int kHeads = 4;  // num_heads
constexpr int kHd = 64;    // head dim
constexpr int kBlkK = 64;  // keys per attention block

struct LgRows {  // device-side liveness of a 128-row tile
  const int* n_act;    // [S] live rows of each side (this layer's buffer parity)
  const int* stopped;  // [P] 0 = running, else 1-based stop layer
  int NP;
  __device__ bool active(int m0) const {
    const int side = m0 / NP;
    return stopped[side >> 1] == 0 && (m0 - side * NP) < n_act[side];
  }
};

// ------------------------------------------------------------------ GEMM epilogues
// Self-attention q,k: columns [q(4x64) | k(4x64)] (weights re-packed at load), rotary applied; cross: [qk(4x64)].
struct EpiQK : EpiBase {
  LgRows rows;
  const float* bias;           // [512] or [256]
  const float *cs, *sn;        // [R][32] rotary tables (unused for cross)
  __half *qh, *ql, *kh, *kl;   // [S][4][NP][64]
  int cross;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int which = n >> 8;  // 0 q (or qk), 1 k
    const int head = (n & 255) >> 6, d0 = n & 63;
    const int lane = r & 31, c4 = (lane & 7) * 4;
    // rotary factors of the eight rows this lane finishes: requested BEFORE the transpose (its __syncwarp is a scheduling fence for
    // loads), so their latency overlaps the shared-memory round trip instead of following it
    float2 rc[8], rs[8];
    if (!cross) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const size_t ro = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * 32 + ((d0 + c4) >> 1);
        rc[it] = __ldg(reinterpret_cast<const float2*>(cs + ro));
        rs[it] = __ldg(reinterpret_cast<const float2*>(sn + ro));
      }
    }
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + n + c4));
    float4 f[8];
    warp_transpose32(v, sc, f);  // lane -> 4 consecutive dims of row it*4 + lane/8: coalesced q / k stores
    __half* dh = which == 0 ? qh : kh;
    __half* dl = which == 0 ? ql : kl;
    const int side = tc.m0 / rows.NP;  // NP is a multiple of the 128-row tile: one side per tile, one division per chunk
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = tc.m0 + (r & ~31) + it * 4 + (lane >> 3), tok = row - side * rows.NP;
      float4 x = make_float4(f[it].x + b.x, f[it].y + b.y, f[it].z + b.z, f[it].w + b.w);
      if (!cross) {  // apply_cached_rotary_emb (lightglue.py:47-54): pairs (2i, 2i+1) share frequency i
        const float2 c = rc[it], s = rs[it];
        x = make_float4(x.x * c.x + (-x.y) * s.x, x.y * c.x + x.x * s.x, x.z * c.y + (-x.w) * s.y, x.w * c.y + x.z * s.y);
      }
      const size_t off = ((static_cast<size_t>(side) * kHeads + head) * rows.NP + tok) * kHd + d0 + c4;
      store_split4(dh + off, dl ? dl + off : nullptr, x);
    }
  }
};

// V projection with the operand roles swapped: D[dim][token] = Wv[dim][:] . x[token][:], so the accumulator tile IS a
// tile of V^T [side][head][dim][token] (the K-major B operand of the P V product) and its rows store coalesced.
struct EpiVT : EpiBase {
  LgRows rows;
  const float* bias;  // full projection bias; V rows start at w_row0
  __half *vth, *vtl;  // [S][4][64][NP]
  int w_row0;         // first weight row of the V block inside the stacked projection (512 self, 256 cross)
  __device__ int m0_of(int t) const { return w_row0 + t * kTileM; }
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.n0); }  // columns = tokens
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, tok_g = n + (lane & 7) * 4, side = tok_g / rows.NP, tok = tok_g - side * rows.NP;
    float bv[8];  // global loads BEFORE the transpose: its __syncwarp fences the scheduler, loads issued after it are exposed latency
#pragma unroll
    for (int it = 0; it < 8; ++it) bv[it] = __ldg(bias + tc.m0 + (r & ~31) + it * 4 + (lane >> 3));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int wrow = tc.m0 + (r & ~31) + it * 4 + (lane >> 3), dim = wrow - w_row0;  // 0..255 = head*64 + d
      const float b = bv[it];
      const size_t off = ((static_cast<size_t>(side) * kHeads) * kHd + dim) * rows.NP + tok;
      store_split4(vth + off, vtl ? vtl + off : nullptr, make_float4(f[it].x + b, f[it].y + b, f[it].z + b, f[it].w + b));
    }
  }
};

// out = acc + bias -> fp16 hi/lo at a column offset (message half of the concat buffer), live tiles only
struct EpiLgSplit : EpiBase {
  LgRows rows;
  __half *hi, *lo;
  const float* bias;
  int ldc, col_off;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const size_t off = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * ldc + col_off + col;
      store_split4(hi + off, lo ? lo + off : nullptr, make_float4(f[it].x + b.x, f[it].y + b.y, f[it].z + b.z, f[it].w + b.w));
    }
  }
};

// out = acc + bias -> fp32 (pre-LayerNorm activations)
struct EpiLgF32 : EpiBase {
  LgRows rows;
  float* out;
  const float* bias;
  int ldc;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it)
      *reinterpret_cast<float4*>(out + static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * ldc + col) =
          make_float4(f[it].x + b.x, f[it].y + b.y, f[it].z + b.z, f[it].w + b.w);
  }
};

// exact (erf) GELU; erf by Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7, an order below the fp32 noise of the FFN that follows) with
// hardware rcp / ex2: ~12 instructions instead of libdevice erff's ~30
__device__ __forceinline__ float lg_gelu(float y) {
  const float ax = fabsf(y) * 0.70710678118654752440f;
  const float tt = __frcp_rn(fmaf(0.3275911f, ax, 1.f));
  const float poly = tt * fmaf(tt, fmaf(tt, fmaf(tt, fmaf(tt, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  const float er = 1.f - poly * sm90::fast_exp2(-ax * ax * 1.4426950408889634f);
  return 0.5f * y * (1.f + copysignf(er, y));
}

// x = (residual ? x : 0) + acc + bias -> fp32 master and fp16 hi/lo (first half of the concat buffer)
struct EpiLgResidual : EpiBase {
  LgRows rows;
  float* x32;          // [R][256]
  __half *xh, *xl;     // [R][512]
  const float* bias;
  int residual;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col));
    float4 x[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {  // all residual loads in flight BEFORE the transpose (its __syncwarp would hold them back)
      const size_t row = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3));
      x[it] = residual ? *reinterpret_cast<const float4*>(x32 + row * kD + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const size_t row = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3));
      const float4 y = make_float4(x[it].x + (f[it].x + b.x), x[it].y + (f[it].y + b.y), x[it].z + (f[it].z + b.z), x[it].w + (f[it].w + b.w));
      *reinterpret_cast<float4*>(x32 + row * kD + col) = y;
      const size_t off = row * (2 * kD) + col;
      store_split4(xh + off, xl ? xl + off : nullptr, y);
    }
  }
};

// final_proj with per-pair layer weights: md = (acc + bias[layer]) / d^0.25
struct EpiFinalProj : EpiBase {
  static constexpr bool kConstB = false;
  const int* nf;       // [S] final live rows
  const int* layer;    // [P] layer index whose log_assignment is used
  __half *hi, *lo;     // [R][256]
  const float* bias;   // [L][256]
  int NP;
  __device__ bool tile_active(const TileCoord& tc) const {
    const int side = tc.m0 / NP;
    return (tc.m0 - side * NP) < nf[side];
  }
  __device__ int b_row_offset(const TileCoord& tc) const { return layer[(tc.m0 / NP) >> 1] * kD; }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + layer[(tc.m0 / NP) >> 1] * kD + col));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const size_t off = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * kD + col;
      // mdesc / d**.25, d = 256
      store_split4(hi + off, lo ? lo + off : nullptr,
                   make_float4((f[it].x + b.x) / 4.f, (f[it].y + b.y) / 4.f, (f[it].z + b.z) / 4.f, (f[it].w + b.w) / 4.f));
    }
  }
};

// similarity of pair p: A rows = side 2p, B rows = side 2p+1 of the same md buffer
struct EpiSim : EpiBase {
  static constexpr bool kConstB = false;
  const int* nf;
  float* sim;  // [P][NP][NP]
  int NP, tiles_per_side;
  int swap = 0;  // 1: rows = side 2p+1, columns = side 2p (the transposed matrix, for coalesced column sweeps)
  __device__ int m0_of(int t) const { return ((t / tiles_per_side) * 2 + swap) * NP + (t % tiles_per_side) * kTileM; }
  __device__ bool tile_active(const TileCoord& tc) const {
    const int side = tc.m0 / NP;
    return (tc.m0 - side * NP) < nf[side] && tc.n0 < nf[side ^ 1];
  }
  __device__ int b_row_offset(const TileCoord& tc) const { return ((tc.m0 / NP) ^ 1) * NP; }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    float4 f[8];
    warp_transpose32(v, sc, f);
    const int lane = r & 31, side = tc.m0 / NP, i0 = tc.m0 - side * NP + (r & ~31);
#pragma unroll
    for (int it = 0; it < 8; ++it)
      *reinterpret_cast<float4*>(sim + (static_cast<size_t>(side >> 1) * NP + i0 + it * 4 + (lane >> 3)) * NP + n + (lane & 7) * 4) = f[it];
  }
};


// ------------------------------------------------------------------ attention
struct AttnArgs {
  LgRows rows;
  int cross;          // kv side = side ^ 1, K read from the q buffers (shared to_qk projection)
  __half *ctx_h, *ctx_l;  // [R][256]
  float scale;        // hd^-0.5
  float lazy;         // O / l are rescaled only when a row maximum grows by more than 2^lazy over the reference it was scaled by
};

struct AttnOutLg {  // O rows of (side, head) -> fp16 hi / lo planes of the context buffer [R][256], head h at columns 64 h
  __half *h, *l;
  __device__ void operator()(int row, int col, float x, float y) const {
    __half2 hi, lo;
    split2_f32(x, y, hi, lo);
    *reinterpret_cast<__half2*>(h + static_cast<size_t>(row) * kD + col) = hi;
    if (l) *reinterpret_cast<__half2*>(l + static_cast<size_t>(row) * kD + col) = lo;
  }
};

// grid (NP / 128, heads, sides): one 128-row query tile of one head of one side per CTA
template <bool SPLIT>
__global__ void __launch_bounds__(kAttnThreads, 1)
lg_attn_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
               const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
               const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, AttnArgs a) {
  const int side = blockIdx.z, head = blockIdx.y, qbase = blockIdx.x * kAttnTile, NP = a.rows.NP;
  const int ks = a.cross ? (side ^ 1) : side;
  if (a.rows.stopped[side >> 1] != 0) return;
  const int nq = a.rows.n_act[side], nk = a.rows.n_act[ks];
  if (qbase >= nq) return;
  const size_t obase = (static_cast<size_t>(side) * NP + qbase) * kD + head * kHd;
  const AttnOutLg out{a.ctx_h + obase, a.ctx_l ? a.ctx_l + obase : nullptr};
  attn_tile<kHd, SPLIT>(&tmQh, &tmQl, &tmKh, &tmKl, &tmVh, &tmVl, (side * kHeads + head) * NP + qbase, (ks * kHeads + head) * NP,
                        (ks * kHeads + head) * kHd, nq - qbase, nk, a.scale, a.lazy, out);
}

// Launch of the tensor-core attention (grid.y = heads, grid.z = sides; grid.x is set here: one CTA per 128-row query tile).
inline int launch_lg_attention(dimb_ctx* ctx, cudaStream_t st, dim3 grid, const CUtensorMap* Q, const CUtensorMap* K, const CUtensorMap* V,
                               const AttnArgs& a, bool exact) {
  grid.x = ceil_div(a.rows.NP, kAttnTile);
  if (exact) {
    constexpr int smem = AttnGeom<kHd, true>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, lg_attn_kernel<true>, smem));
    lg_attn_kernel<true><<<grid, kAttnThreads, smem, st>>>(Q[0], Q[1], K[0], K[1], V[0], V[1], a);
  } else {
    constexpr int smem = AttnGeom<kHd, false>::kSmem;
    DIMB_TRY(dimb_func_smem(ctx, lg_attn_kernel<false>, smem));
    lg_attn_kernel<false><<<grid, kAttnThreads, smem, st>>>(Q[0], Q[0], K[0], K[0], V[0], V[0], a);
  }
  return DIMB_OK;
}

}  // namespace
