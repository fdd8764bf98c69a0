// lightglue.cu - LightGlue matching (dimb_lg_*), replacing LightGlueMatcher._match_pairs
// (reference matchers/lightglue.py:102-125) and thirdparty/LightGlue/lightglue/lightglue.py:424-579.
//
// Batch layout: P pairs = S = 2P "sides"; side s owns rows [s*NP, (s+1)*NP) of every token buffer
// (NP = max_kpts rounded up to 128, so 128-row MMA tiles never straddle two images).
// The whole forward pass is ONE fixed launch sequence with no host synchronisation: the number of live
// keypoints per side (n_act), the per-pair stop flag and the pruning maps live in device memory; kernels
// of later layers exit immediately for stopped pairs / pruned rows (reference: host `if` per layer,
// lightglue.py:499,503).  The token state ping-pongs between two buffers per layer because the
// per-layer tail (confidence -> stop test -> prune mask -> compaction) gathers rows.
//
// Per layer (all sides at once):
//   self : QKV GEMM (+rotary, head split, V transposed) -> flash attention -> out_proj GEMM -> FFN0 GEMM
//          -> LayerNorm+GELU -> FFN3 GEMM (+residual)
//   cross: [to_qk;to_v] GEMM -> flash attention against the other side -> to_out -> FFN0 -> LN+GELU -> FFN3
//   tail : token confidence + matchability, stop decision, prune compaction, gather
// Final : gather by stop parity -> final_proj GEMM (stacked per-layer weights) -> similarity GEMM per pair
//         -> row/col log-sum-exp -> row/col argmax of the log assignment -> mutual filter + threshold.
#include <algorithm>
#include <memory>
#include <cmath>
#include <cstring>

#include "gemm.cuh"
#include "lightglue_generic.cuh"

#include "lg_assign.cuh"
#include "lg_kernels.cuh"

namespace {

// ------------------------------------------------------------------ input preparation
struct SideIn {
  const float* kpts;
  const float* desc;
  const int* n;
  int n_cap, layout, ld;
  float size0, size1;
  int round_fp16;
  int f16;              // keypoints / descriptors are __half arrays (feature store blocks)
  const int* size_dev;  // device [H, W] (overrides size0 / size1)
  const float* size_f32;  // device float[2] (overrides size_dev / size0 / size1)
};

__device__ __forceinline__ float maybe_round(float v, int r16) { return r16 ? __half2float(__float2half_rn(v)) : v; }
// element i of a float32 or float16 array
__device__ __forceinline__ float ld_feat(const float* p, size_t i, int f16) {
  return f16 ? __half2float(reinterpret_cast<const __half*>(p)[i]) : p[i];
}

// grid (NP/32, S), block (32, 8): transposes descriptors, writes tokens, positional encoding, state reset.
// dst: fp32 x + hi/lo (din == d) or the input-projection operand (din != d).
__global__ void lg_prep_kernel(const SideIn* __restrict__ in, const float* __restrict__ Wr /*[32][2]*/, int din, int NP,
                               float* __restrict__ x32, __half* __restrict__ xh, __half* __restrict__ xl, int ldx,
                               float* __restrict__ cs, float* __restrict__ sn, int* __restrict__ ind, int* __restrict__ n_act,
                               int* __restrict__ n_orig, int* __restrict__ stopped, int* __restrict__ counter) {
  const int side = blockIdx.y, t0 = blockIdx.x * 32;
  const SideIn si = in[side];
  const int n = min(min(*si.n, si.n_cap), NP);
  if (blockIdx.x == 0 && threadIdx.x == 0 && threadIdx.y == 0) {
    n_act[side] = n;
    n_orig[side] = n;
    if ((side & 1) == 0) {
      stopped[side >> 1] = 0;
      counter[side >> 1] = 0;
    }
  }
  __shared__ float tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int c0 = 0; c0 < din; c0 += 32) {
    // read desc[c][tok] (layout 0) coalesced over tok, or desc[tok][c] (layout 1) coalesced over c
    for (int k = ty; k < 32; k += 8) {
      float v = 0.f;
      if (si.layout == 0) {
        const int c = c0 + k, tok = t0 + tx;
        if (tok < n) v = ld_feat(si.desc, static_cast<size_t>(c) * si.ld + tok, si.f16);
        tile[k][tx] = v;  // tile[c][tok]
      } else {
        const int tok = t0 + k, c = c0 + tx;
        if (tok < n) v = ld_feat(si.desc, static_cast<size_t>(tok) * si.ld + c, si.f16);
        tile[tx][k] = v;
      }
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {
      const int tok = t0 + k, c = c0 + tx;
      if (tok < n) {
        const float v = maybe_round(tile[tx][k], si.round_fp16);
        const size_t row = static_cast<size_t>(side) * NP + tok;
        if (x32) x32[row * kD + c] = v;
        __half h, l;
        split_f32(v, h, l);
        xh[row * ldx + c] = h;
        if (xl) xl[row * ldx + c] = l;
      }
    }
    __syncthreads();
  }
  // normalize_keypoints (lightglue.py:24-34) + LearnableFourierPositionalEncoding (:57-70)
  float sz0 = si.size_dev ? static_cast<float>(si.size_dev[0]) : si.size0, sz1 = si.size_dev ? static_cast<float>(si.size_dev[1]) : si.size1;
  if (si.size_f32) sz0 = si.size_f32[0], sz1 = si.size_f32[1];
  const float shift0 = sz0 / 2.f, shift1 = sz1 / 2.f, scale = fmaxf(sz0, sz1) / 2.f;
  for (int k = ty; k < 32; k += 8) {
    const int tok = t0 + k;
    if (tok >= n) continue;
    const float kx = (maybe_round(ld_feat(si.kpts, 2 * tok, si.f16), si.round_fp16) - shift0) / scale;
    const float ky = (maybe_round(ld_feat(si.kpts, 2 * tok + 1, si.f16), si.round_fp16) - shift1) / scale;
    const float proj = Wr[2 * tx] * kx + Wr[2 * tx + 1] * ky;
    const size_t row = static_cast<size_t>(side) * NP + tok;
    cs[row * 32 + tx] = cosf(proj);
    sn[row * 32 + tx] = sinf(proj);
    if (tx == 0) ind[row] = tok;
  }
}

// ------------------------------------------------------------------ LayerNorm(512) + GELU -> fp16 hi/lo; warp per row
// lane l owns columns 4*(32*i + l) .. +3 (i = 0..3): every load / store instruction covers a contiguous run.
__global__ void lg_ln_gelu_kernel(LgRows rows, const float* __restrict__ h1, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, __half* __restrict__ oh, __half* __restrict__ ol, int R) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= R) return;
  const int side = row / rows.NP;
  if (rows.stopped[side >> 1] != 0 || (row - side * rows.NP) >= rows.n_act[side]) return;
  const float4* x = reinterpret_cast<const float4*>(h1 + static_cast<size_t>(row) * 512);
  float4 v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = x[i * 32 + lane];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / 512.f;
  float q2 = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q2 += (a * a + b * b) + (c * c + d * d);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q2 += __shfl_xor_sync(0xffffffffu, q2, o);
  const float rstd = 1.f / sqrtf(q2 / 512.f + 1e-5f);
  auto act = [&](float t, float g, float b) { return lg_gelu((t - mean) * rstd * g + b); };
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c)), b = __ldg(reinterpret_cast<const float4*>(beta + c));
    const size_t off = static_cast<size_t>(row) * 512 + c;
    store_split4(oh + off, ol ? ol + off : nullptr, make_float4(act(v[i].x, g.x, b.x), act(v[i].y, g.y, b.y), act(v[i].z, g.z, b.z), act(v[i].w, g.w, b.w)));
  }
}

// warp per destination row: x32, x hi/lo (first half of the concat buffer), rotary tables, original index
__global__ void lg_gather_kernel(const int* __restrict__ n_next, const int* __restrict__ stopped, int layer, const int* __restrict__ map,
                                 int NP, int R, const float* __restrict__ x32s, float* __restrict__ x32d,
                                 const __half* __restrict__ xhs, __half* __restrict__ xhd, const __half* __restrict__ xls,
                                 __half* __restrict__ xld, const float* __restrict__ css, float* __restrict__ csd,
                                 const float* __restrict__ sns, float* __restrict__ snd, const int* __restrict__ inds,
                                 int* __restrict__ indd) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= R) return;
  const int side = row / NP, j = row - side * NP;
  const int stp = stopped[side >> 1];
  if (stp != 0 && stp != layer + 1) return;  // pairs that stopped earlier keep their final buffer untouched
  if (j >= n_next[side]) return;
  const size_t src = static_cast<size_t>(side) * NP + map[static_cast<size_t>(side) * NP + j], dst = row;
  reinterpret_cast<float4*>(x32d + dst * kD)[lane] = reinterpret_cast<const float4*>(x32s + src * kD)[lane];
  reinterpret_cast<float4*>(x32d + dst * kD)[lane + 32] = reinterpret_cast<const float4*>(x32s + src * kD)[lane + 32];
  reinterpret_cast<uint4*>(xhd + dst * 2 * kD)[lane] = reinterpret_cast<const uint4*>(xhs + src * 2 * kD)[lane];
  if (xls) reinterpret_cast<uint4*>(xld + dst * 2 * kD)[lane] = reinterpret_cast<const uint4*>(xls + src * 2 * kD)[lane];
  csd[dst * 32 + lane] = css[src * 32 + lane];
  snd[dst * 32 + lane] = sns[src * 32 + lane];
  if (lane == 0) indd[dst] = inds[src];
}

// ------------------------------------------------------------------ final stage
// one thread per pair: which buffer parity / layer holds the result
__global__ void lg_final_select_kernel(const int* __restrict__ stopped, const int* __restrict__ n_act0, const int* __restrict__ n_act1,
                                       int* __restrict__ nf, int* __restrict__ layer, int* __restrict__ parity, int P, int L,
                                       int adaptive) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int c = stopped[p];
  const int par = adaptive ? (c ? (c & 1) : ((L - 1) & 1)) : 0;  // fixed-work runs never leave buffer 0
  parity[p] = par;
  layer[p] = c ? c - 1 : L - 1;
  const int* na = par ? n_act1 : n_act0;
  nf[2 * p] = na[2 * p];
  nf[2 * p + 1] = na[2 * p + 1];
}

__device__ __forceinline__ float logsigmoidf_(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }

// warp per row: copy the final tokens into a fixed buffer and evaluate logsigmoid(matchability) once per token
__global__ void lg_final_gather_kernel(const int* __restrict__ nf, const int* __restrict__ layer, const int* __restrict__ parity,
                                       int NP, int R, const float* __restrict__ x32a, const float* __restrict__ x32b,
                                       const __half* __restrict__ xha, const __half* __restrict__ xhb, const __half* __restrict__ xla,
                                       const __half* __restrict__ xlb, const int* __restrict__ inda, const int* __restrict__ indb,
                                       __half* __restrict__ fh, __half* __restrict__ fl, int* __restrict__ indf,
                                       const float* __restrict__ wm /*[L][256]*/, const float* __restrict__ bm /*[L]*/,
                                       float* __restrict__ z, float* __restrict__ xf32) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= R) return;
  const int side = row / NP, j = row - side * NP, p = side >> 1;
  if (j >= nf[side]) return;
  const int par = parity[p], ly = layer[p];
  const float* x = (par ? x32b : x32a) + static_cast<size_t>(row) * kD;
  const __half* xh = (par ? xhb : xha) + static_cast<size_t>(row) * 2 * kD;
  reinterpret_cast<uint4*>(fh + static_cast<size_t>(row) * kD)[lane] = reinterpret_cast<const uint4*>(xh)[lane];
  if (fl) {
    const __half* xl = (par ? xlb : xla) + static_cast<size_t>(row) * 2 * kD;
    reinterpret_cast<uint4*>(fl + static_cast<size_t>(row) * kD)[lane] = reinterpret_cast<const uint4*>(xl)[lane];
  }
  float a = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float xv = x[lane * 8 + e];
    xf32[static_cast<size_t>(row) * kD + lane * 8 + e] = xv;
    a = fmaf(xv, wm[ly * kD + lane * 8 + e], a);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) {
    z[row] = logsigmoidf_(a + bm[ly]);  // the assignment only ever needs logsigmoid(z) (lightglue.py:250-252)
    indf[row] = (par ? indb : inda)[row];
  }
}

struct Lin {
  __half *wh = nullptr, *wl = nullptr;
  float* bias = nullptr;
  int n = 0, k = 0;
  CUtensorMap tmh, tml;
  CUtensorMap tmh256, tml256;  // 256-row boxes for the BN = 256 tile shape (n % 256 == 0 only)
  CUtensorMap tmh256k32, tml256k32;  // the same with 32-wide K boxes, SWIZZLE_64B (gemm.cuh CONV 3)
  bool has256 = false;
};

}  // namespace

struct dimb_lg {
  std::vector<void*> mem;  // device memory owned by this handle
  dimb_lgx* gen = nullptr;  // shape-generic fp32 implementation (lightglue_generic.cu) when the shape is not 256 / 4 heads
  dimb_ctx* ctx;
  dimb_lg_conf conf;
  int S, NP, R, L, din;
  // weights
  float* Wr;
  Lin inproj;
  struct Layer {
    Lin qkv_s, out_s, f0_s, f3_s, qkv_c, out_c, f0_c, f3_c;
    float *g_s, *b_s, *g_c, *b_c;
    float *wt, *wm;
    float bt, bm;
    float thr;
  };
  std::vector<Layer> layers;
  Lin fproj;         // stacked [L*256][256]
  float *wm_all, *bm_all;  // [L][256], [L]
  // state
  float *x32[2], *cs[2], *sn[2];
  __half *xh[2], *xl[2];
  int *ind[2], *n_act[2];
  int *n_orig, *stopped, *counter, *map;
  __half *xinh, *xinl;  // [R][din] when din != d
  __half *qh, *ql, *kh, *kl, *vth, *vtl, *ctxh, *ctxl, *h2h, *h2l, *fh, *fl, *mdh, *mdl;
  float *h1, *tok, *mat, *z, *xf32, *sim, *smax, *slog, *best;
  int *arg, *indf, *nf, *layer_of, *parity;
  SideIn* side_in;
  // tensor maps over the static buffers
  CUtensorMap m_x[2][2], m_ctx[2], m_h2[2], m_f[2], m_md[2], m_xin[2];
  CUtensorMap m_x32[2][2];  // the token buffers as 32-column boxes, SWIZZLE_64B (gemm.cuh CONV 3)
  CUtensorMap m_q128[2], m_q64[2], m_k64[2], m_vt[2];
  // host staging of the host API
  float *st_kpts = nullptr, *st_desc = nullptr, *o_ms = nullptr;
  int *st_n = nullptr, *o_nm = nullptr, *o_sl = nullptr;
  long long* o_m = nullptr;
  int o_cap = 0;
};

namespace {

int make_lin(dimb_ctx* ctx, Lin& l, const std::vector<float>& w, const std::vector<float>& b, int n, int k, int box) {
  l.n = n;
  l.k = k;
  std::vector<__half> h(w.size()), lo(w.size());
  for (size_t i = 0; i < w.size(); ++i) {
    h[i] = __float2half_rn(w[i]);
    lo[i] = __float2half_rn(w[i] - __half2float(h[i]));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &l.wh, w.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &l.wl, w.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &l.bias, b.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(l.wh, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(l.wl, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(l.bias, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_TRY(dimb_tmap_2d(ctx, &l.tmh, l.wh, n, k, k, box));
  DIMB_TRY(dimb_tmap_2d(ctx, &l.tml, l.wl, n, k, k, box));
  if (box == 128 && n % 256 == 0) {
    DIMB_TRY(dimb_tmap_2d(ctx, &l.tmh256, l.wh, n, k, k, 256));
    DIMB_TRY(dimb_tmap_2d(ctx, &l.tml256, l.wl, n, k, k, 256));
    DIMB_TRY(dimb_tmap_2d_sw64(ctx, &l.tmh256k32, l.wh, n, k, k, 256));
    DIMB_TRY(dimb_tmap_2d_sw64(ctx, &l.tml256k32, l.wl, n, k, k, 256));
    l.has256 = true;
  }
  return DIMB_OK;
}

int upload_f32(dimb_ctx* ctx, float** d, const float* src, size_t n) {
  DIMB_TRY(dimb_alloc_t(ctx, d, n, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*d, src, n * sizeof(float), cudaMemcpyHostToDevice));
  return DIMB_OK;
}

template <class Epi>
int lg_gemm(dimb_lg* lg, cudaStream_t st, const CUtensorMap* A /*[2] hi,lo*/, const Lin& w, const Epi& epi, int m_tiles, const char* tag,
            bool wide = false, const CUtensorMap* A32 = nullptr) {
  TcOperands ops;
  ops.Ah = A[0];
  ops.Al = A[1];
  ops.Bh = w.tmh;
  ops.Bl = w.tml;
  GemmArgs g{};
  g.num_kb = w.k / 64;
  g.M = lg->R;
  g.N = w.n;
  // 128 x 256 tiles (DIMB_BN256=1): per MMA k-step 30 KB of shared-memory traffic per 128 x 128 of output instead of 36 KB (the
  // 128 x 128 EXACT tile is bound by the shared-memory pipe - operand reads + TMA fill - at ~66 % of the tensor pipe)
  // (same-box A/B, 37 pairs: q/k projection 3.62 -> 3.07 ms, FFN0 4.66 -> 3.93 ms per step; no gain for the HBM-bound FFN3 and a loss
  // for the 256-wide out_proj, which stay on 128 x 128 tiles)
  if (wide && lg->ctx->bn256 && w.has256) {
    if (lg->ctx->k32 && A32) {  // four 48 KB stages instead of two 96 KB ones (gemm.cuh CONV 3)
      ops.Ah = A32[0], ops.Al = A32[1];
      ops.Bh = w.tmh256k32, ops.Bl = w.tml256k32;
      g.num_kb = w.k / 32;
      return launch_gemm<256, 3>(lg->ctx, st, ops, g, epi, m_tiles, w.n, tag);
    }
    ops.Bh = w.tmh256;
    ops.Bl = w.tml256;
    return launch_gemm<256, false>(lg->ctx, st, ops, g, epi, m_tiles, w.n, tag);
  }
  return launch_gemm<128, false>(lg->ctx, st, ops, g, epi, m_tiles, w.n, tag);
}

int run_attention(dimb_lg* lg, cudaStream_t st, const LgRows& rows, int cross, int S) {
  dimb_ctx* ctx = lg->ctx;
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  AttnArgs a;
  a.rows = rows;
  a.cross = cross;
  a.ctx_h = lg->ctxh;
  a.ctx_l = exact ? lg->ctxl : nullptr;
  a.scale = 0.125f;  // hd^-0.5
  a.lazy = ctx->attn_lazy;
  ProfScope prof(ctx, st, cross ? "lg.attn_cross" : "lg.attn_self");
  dim3 grid(ceil_div(lg->NP, 2 * kTileM), kHeads, S);
  const CUtensorMap* K = cross ? lg->m_q64 : lg->m_k64;
  DIMB_TRY(launch_lg_attention(ctx, st, grid, lg->m_q128, K, lg->m_vt, a, exact));
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace

extern "C" {

int dimb_lg_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* cf, dimb_lg** out) {
  if (!ctx || !weights || !cf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (cf->n_layers < 1 || cf->max_pairs < 1 || cf->max_kpts < 1 || cf->input_dim < 1) return DIMB_ERR_ARG;
  if (cf->descriptor_dim != kD || cf->num_heads != kHeads || cf->input_dim % 64 != 0) {
    // not the shape the tensor-core kernels are built for (e.g. LighterGlue: 96 / 1 head): shape-generic fp32 implementation
    dimb_lg* lg = new dimb_lg();
    lg->ctx = ctx;
    lg->conf = *cf;
    lg->S = 2 * cf->max_pairs, lg->NP = cf->max_kpts, lg->din = cf->input_dim;  // what dimb_lg_match's host staging reads
    const int rc = lgx_create(ctx, weights, n_floats, cf, &lg->gen);
    if (rc != DIMB_OK) {
      delete lg;
      return rc;
    }
    *out = lg;
    return DIMB_OK;
  }
  const int L = cf->n_layers, din = cf->input_dim, d = kD;
  size_t need = 32 * 2;
  if (din != d) need += static_cast<size_t>(d) * din + d;
  const size_t per_layer = (3 * d * d + 3 * d) + (d * d + d) + 2 * ((2 * d) * (2 * d) + 2 * d + 2 * (2 * d) + d * (2 * d) + d) +
                           3 * (d * d + d);
  need += per_layer * L + static_cast<size_t>(L) * (d + 1 + d * d + d) + static_cast<size_t>(L - 1) * (d + 1);
  if (n_floats != need) {
    dimb_set_error(ctx, "dimb_lg_create: weight blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(need));
    return DIMB_ERR_ARG;
  }
  dimb_lg* lg = new dimb_lg();
  lg->ctx = ctx;
  std::unique_ptr<dimb_lg, void (*)(dimb_lg*)> guard(lg, dimb_lg_destroy);  // a failed create releases what it built
  OwnerScope own(ctx, &lg->mem);
  lg->conf = *cf;
  lg->L = L;
  lg->din = din;
  lg->S = 2 * cf->max_pairs;
  lg->NP = round_up(cf->max_kpts, 128);
  lg->R = lg->S * lg->NP;
  const float* p = weights;
  auto take = [&](size_t n) {
    std::vector<float> v(p, p + n);
    p += n;
    return v;
  };
  DIMB_TRY(upload_f32(ctx, &lg->Wr, p, 64));
  p += 64;
  if (din != d) {
    auto w = take(static_cast<size_t>(d) * din);
    auto b = take(d);
    DIMB_TRY(make_lin(ctx, lg->inproj, w, b, d, din, 128));
  }
  lg->layers.resize(L);
  for (int i = 0; i < L; ++i) {
    auto& ly = lg->layers[i];
    {  // Wqkv rows are interleaved (head, dim, {q,k,v}) (lightglue.py:153): re-pack to [q | k | v], head-major
      auto w = take(static_cast<size_t>(3) * d * d);
      auto b = take(3 * d);
      std::vector<float> w2(w.size()), b2(b.size());
      for (int hh = 0; hh < kHeads; ++hh)
        for (int dd = 0; dd < kHd; ++dd)
          for (int t = 0; t < 3; ++t) {
            const int src = hh * 3 * kHd + dd * 3 + t, dst = t * d + hh * kHd + dd;
            memcpy(&w2[static_cast<size_t>(dst) * d], &w[static_cast<size_t>(src) * d], d * sizeof(float));
            b2[dst] = b[src];
          }
      DIMB_TRY(make_lin(ctx, ly.qkv_s, w2, b2, 3 * d, d, 128));
    }
    {
      auto w = take(static_cast<size_t>(d) * d);
      auto b = take(d);
      DIMB_TRY(make_lin(ctx, ly.out_s, w, b, d, d, 128));
    }
    auto ffn = [&](Lin& f0, float** g, float** be, Lin& f3) -> int {
      auto w0 = take(static_cast<size_t>(4) * d * d);
      auto b0 = take(2 * d);
      DIMB_TRY(make_lin(ctx, f0, w0, b0, 2 * d, 2 * d, 128));
      DIMB_TRY(upload_f32(ctx, g, p, 2 * d));
      p += 2 * d;
      DIMB_TRY(upload_f32(ctx, be, p, 2 * d));
      p += 2 * d;
      auto w3 = take(static_cast<size_t>(2) * d * d);
      auto b3 = take(d);
      DIMB_TRY(make_lin(ctx, f3, w3, b3, d, 2 * d, 128));
      return static_cast<int>(DIMB_OK);
    };
    DIMB_TRY(ffn(ly.f0_s, &ly.g_s, &ly.b_s, ly.f3_s));
    {  // cross: stack [to_qk ; to_v]
      auto wq = take(static_cast<size_t>(d) * d);
      auto bq = take(d);
      auto wv = take(static_cast<size_t>(d) * d);
      auto bv = take(d);
      wq.insert(wq.end(), wv.begin(), wv.end());
      bq.insert(bq.end(), bv.begin(), bv.end());
      DIMB_TRY(make_lin(ctx, ly.qkv_c, wq, bq, 2 * d, d, 128));
      auto wo = take(static_cast<size_t>(d) * d);
      auto bo = take(d);
      DIMB_TRY(make_lin(ctx, ly.out_c, wo, bo, d, d, 128));
    }
    DIMB_TRY(ffn(ly.f0_c, &ly.g_c, &ly.b_c, ly.f3_c));
    ly.thr = static_cast<float>(std::min(1.0, std::max(0.0, 0.8 + 0.1 * std::exp(-4.0 * i / L))));
  }
  {
    std::vector<float> wm(static_cast<size_t>(L) * d), bm(L), wf, bf;
    for (int i = 0; i < L; ++i) {
      memcpy(&wm[static_cast<size_t>(i) * d], p, d * sizeof(float));
      bm[i] = p[d];
      p += d + 1;
      auto w = take(static_cast<size_t>(d) * d);
      auto b = take(d);
      wf.insert(wf.end(), w.begin(), w.end());
      bf.insert(bf.end(), b.begin(), b.end());
    }
    DIMB_TRY(upload_f32(ctx, &lg->wm_all, wm.data(), wm.size()));
    DIMB_TRY(upload_f32(ctx, &lg->bm_all, bm.data(), bm.size()));
    DIMB_TRY(make_lin(ctx, lg->fproj, wf, bf, L * d, d, 128));
    for (int i = 0; i < L; ++i) {
      lg->layers[i].wm = lg->wm_all + static_cast<size_t>(i) * d;
      lg->layers[i].bm = bm[i];
    }
    for (int i = 0; i + 1 < L; ++i) {
      DIMB_TRY(upload_f32(ctx, &lg->layers[i].wt, p, d));
      lg->layers[i].bt = p[d];
      p += d + 1;
    }
    if (L >= 1) lg->layers[L - 1].wt = nullptr;
  }
  // ---- state buffers
  const size_t R = lg->R, NP = lg->NP, S = lg->S, P = cf->max_pairs;
  for (int b = 0; b < 2; ++b) {
    DIMB_TRY(dimb_alloc_t(ctx, &lg->x32[b], R * d));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->xh[b], R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->xl[b], R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->cs[b], R * 32));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->sn[b], R * 32));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->ind[b], R));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->n_act[b], S));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &lg->n_orig, S));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->stopped, P));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->counter, P));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->map, R));
  if (din != d) {
    DIMB_TRY(dimb_alloc_t(ctx, &lg->xinh, R * din));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->xinl, R * din));
  }
  for (__half** b : {&lg->qh, &lg->ql, &lg->kh, &lg->kl, &lg->vth, &lg->vtl, &lg->ctxh, &lg->ctxl, &lg->fh, &lg->fl, &lg->mdh, &lg->mdl})
    DIMB_TRY(dimb_alloc_t(ctx, b, R * d));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->h2h, R * 2 * d));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->h2l, R * 2 * d));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->h1, R * 2 * d));
  for (float** b : {&lg->tok, &lg->mat, &lg->z, &lg->smax, &lg->slog, &lg->best}) DIMB_TRY(dimb_alloc_t(ctx, b, R));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->xf32, R * d));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->sim, P * NP * NP));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->arg, R));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->indf, R));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->nf, S));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->layer_of, P));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->parity, P));
  DIMB_TRY(dimb_alloc_t(ctx, &lg->side_in, S));
  // ---- tensor maps
  for (int b = 0; b < 2; ++b) {
    DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_x[b][0], lg->xh[b], R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_x[b][1], lg->xl[b], R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d_sw64(ctx, &lg->m_x32[b][0], lg->xh[b], R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d_sw64(ctx, &lg->m_x32[b][1], lg->xl[b], R, 2 * d, 2 * d, kTileM));
  }
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_ctx[0], lg->ctxh, R, d, d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_ctx[1], lg->ctxl, R, d, d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_h2[0], lg->h2h, R, 2 * d, 2 * d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_h2[1], lg->h2l, R, 2 * d, 2 * d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_f[0], lg->fh, R, d, d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_f[1], lg->fl, R, d, d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_md[0], lg->mdh, R, d, d, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_md[1], lg->mdl, R, d, d, kTileM));
  if (din != d) {
    DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_xin[0], lg->xinh, R, din, din, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_xin[1], lg->xinl, R, din, din, kTileM));
  }
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_q128[0], lg->qh, S * kHeads * NP, kHd, kHd, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_q128[1], lg->ql, S * kHeads * NP, kHd, kHd, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_q64[0], lg->qh, S * kHeads * NP, kHd, kHd, kBlkK));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_q64[1], lg->ql, S * kHeads * NP, kHd, kHd, kBlkK));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_k64[0], lg->kh, S * kHeads * NP, kHd, kHd, kBlkK));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_k64[1], lg->kl, S * kHeads * NP, kHd, kHd, kBlkK));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_vt[0], lg->vth, S * kHeads * kHd, NP, NP, kHd));
  DIMB_TRY(dimb_tmap_2d(ctx, &lg->m_vt[1], lg->vtl, S * kHeads * kHd, NP, NP, kHd));
  *out = guard.release();
  return DIMB_OK;
}

void dimb_lg_destroy(dimb_lg* lg) {
  if (!lg) return;
  lgx_destroy(lg->gen);
  dimb_release(lg->ctx, lg->mem);
  delete lg;
}

int dimb_lg_match_dev(dimb_lg* lg, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches, float* d_mscores,
                      int* d_n_matches, int* d_stop_layer, int cap, void* stream) {
  if (!lg || !f0 || !f1 || P < 1 || P > lg->conf.max_pairs || cap < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = lg->ctx;
  if (lg->gen) return lgx_match_dev(lg->gen, P, f0, f1, d_matches, d_mscores, d_n_matches, d_stop_layer, cap, static_cast<cudaStream_t>(stream));
  OwnerScope own(ctx, &lg->mem);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dimb_lg_conf& cf = lg->conf;
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int S = 2 * P, NP = lg->NP, L = lg->L, d = kD, din = lg->din;
  const int R = S * NP;  // rows of the sides in use (prefix of the buffers)
  const int m_tiles = R / kTileM;
  std::vector<SideIn> hin(S);
  for (int p = 0; p < P; ++p)
    for (int sd = 0; sd < 2; ++sd) {
      const dimb_feats_dev& f = sd ? f1[p] : f0[p];
      SideIn& s = hin[2 * p + sd];
      s.kpts = f.keypoints;
      s.desc = f.descriptors;
      s.n = f.n;
      s.n_cap = f.n_cap;
      s.layout = f.desc_layout;
      s.ld = f.desc_ld ? f.desc_ld : (f.desc_layout == 0 ? f.n_cap : din);
      s.size0 = f.size0;
      s.size1 = f.size1;
      s.round_fp16 = f.round_fp16;
      s.f16 = f.f16;
      s.size_dev = f.size_dev;
      s.size_f32 = f.size_f32_dev;
      if (f.n_cap > NP) {
        dimb_set_error(ctx, "dimb_lg_match: more keypoints than max_kpts given at create time");
        return DIMB_ERR_ARG;
      }
    }
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(lg->side_in, hin.data(), S * sizeof(SideIn), cudaMemcpyHostToDevice, st));
  const int do_stop = cf.depth_confidence > 0, do_prune = cf.width_confidence > 0;
  const bool adaptive = do_stop || do_prune;
  const float depth_conf = static_cast<float>(cf.depth_confidence);
  const float keep_thr = static_cast<float>(1.0 - cf.width_confidence);
  const float filt = static_cast<float>(cf.filter_threshold);

  // ---- prepare tokens
  if (din == d) {
    lg_prep_kernel<<<dim3(NP / 32, S), dim3(32, 8), 0, st>>>(lg->side_in, lg->Wr, din, NP, lg->x32[0], lg->xh[0],
                                                            exact ? lg->xl[0] : nullptr, 2 * d, lg->cs[0], lg->sn[0], lg->ind[0],
                                                            lg->n_act[0], lg->n_orig, lg->stopped, lg->counter);
    DIMB_LAUNCH_CHECK(ctx);
  } else {
    lg_prep_kernel<<<dim3(NP / 32, S), dim3(32, 8), 0, st>>>(lg->side_in, lg->Wr, din, NP, nullptr, lg->xinh,
                                                            exact ? lg->xinl : nullptr, din, lg->cs[0], lg->sn[0], lg->ind[0],
                                                            lg->n_act[0], lg->n_orig, lg->stopped, lg->counter);
    DIMB_LAUNCH_CHECK(ctx);
    EpiLgResidual e;
    e.rows = LgRows{lg->n_act[0], lg->stopped, NP};
    e.x32 = lg->x32[0];
    e.xh = lg->xh[0];
    e.xl = exact ? lg->xl[0] : nullptr;
    e.bias = lg->inproj.bias;
    e.residual = 0;
    DIMB_TRY(lg_gemm(lg, st, lg->m_xin, lg->inproj, e, m_tiles, "lg.input_proj"));
  }

  for (int i = 0; i < L; ++i) {
    // adaptive runs ping-pong the token buffers through the per-layer pruning gather; fixed-work runs (no early stop, no
    // pruning) have nothing to decide or to move, so they stay in buffer 0 and skip the confidence / decide / gather kernels
    const int cur = adaptive ? (i & 1) : 0, nxt = cur ^ 1;
    auto& ly = lg->layers[i];
    const LgRows rows{lg->n_act[cur], lg->stopped, NP};
    for (int blk = 0; blk < 2; ++blk) {  // 0 = self, 1 = cross
      const Lin& qkv = blk ? ly.qkv_c : ly.qkv_s;
      const Lin& outp = blk ? ly.out_c : ly.out_s;
      const Lin& f0 = blk ? ly.f0_c : ly.f0_s;
      const Lin& f3 = blk ? ly.f3_c : ly.f3_s;
      {
        EpiQK e;
        e.rows = rows;
        e.bias = qkv.bias;
        e.cs = lg->cs[cur];
        e.sn = lg->sn[cur];
        e.qh = lg->qh;
        e.ql = exact ? lg->ql : nullptr;
        e.kh = lg->kh;
        e.kl = exact ? lg->kl : nullptr;
        e.cross = blk;
        // q,k (self) or qk (cross): the first 512 / 256 rows of the stacked projection
        TcOperands ops;
        ops.Ah = lg->m_x[cur][0];
        ops.Al = lg->m_x[cur][1];
        ops.Bh = qkv.tmh;
        ops.Bl = qkv.tml;
        GemmArgs g{};
        g.num_kb = d / 64;
        g.M = lg->R;
        g.N = blk ? d : 2 * d;
        if (ctx->bn256 && qkv.has256 && ctx->k32) {
          ops.Ah = lg->m_x32[cur][0], ops.Al = lg->m_x32[cur][1];
          ops.Bh = qkv.tmh256k32, ops.Bl = qkv.tml256k32;
          g.num_kb = d / 32;
          DIMB_TRY((launch_gemm<256, 3>(ctx, st, ops, g, e, m_tiles, blk ? d : 2 * d, "lg.qk")));
        } else if (ctx->bn256 && qkv.has256) {
          ops.Bh = qkv.tmh256;
          ops.Bl = qkv.tml256;
          DIMB_TRY((launch_gemm<256, false>(ctx, st, ops, g, e, m_tiles, blk ? d : 2 * d, "lg.qk")));
        } else {
          DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, m_tiles, blk ? d : 2 * d, "lg.qk")));
        }
      }
      {
        EpiVT e;
        e.rows = rows;
        e.bias = qkv.bias;
        e.vth = lg->vth;
        e.vtl = exact ? lg->vtl : nullptr;
        e.w_row0 = blk ? d : 2 * d;
        // swapped roles: A = V rows of the projection weights (2 tiles of 128 dims), B = the token rows
        TcOperands ops;
        ops.Ah = qkv.tmh;
        ops.Al = qkv.tml;
        ops.Bh = lg->m_x[cur][0];
        ops.Bl = lg->m_x[cur][1];
        GemmArgs g{};
        g.num_kb = d / 64;
        g.M = qkv.n;
        g.N = R;
        DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, 2, R, "lg.vT")));
      }
      DIMB_TRY(run_attention(lg, st, rows, blk, S));
      {
        EpiLgSplit e;
        e.rows = rows;
        e.hi = lg->xh[cur];
        e.lo = exact ? lg->xl[cur] : nullptr;
        e.bias = outp.bias;
        e.ldc = 2 * d;
        e.col_off = d;
        DIMB_TRY(lg_gemm(lg, st, lg->m_ctx, outp, e, m_tiles, "lg.out_proj"));
      }
      {
        EpiLgF32 e;
        e.rows = rows;
        e.out = lg->h1;
        e.bias = f0.bias;
        e.ldc = 2 * d;
        DIMB_TRY(lg_gemm(lg, st, lg->m_x[cur], f0, e, m_tiles, "lg.ffn0", true, lg->m_x32[cur]));
      }
      {
        ProfScope prof_ln(ctx, st, "lg.ln_gelu");
        lg_ln_gelu_kernel<<<ceil_div(R * 32, 256), 256, 0, st>>>(rows, lg->h1, blk ? ly.g_c : ly.g_s, blk ? ly.b_c : ly.b_s, lg->h2h,
                                                                  exact ? lg->h2l : nullptr, R);
        DIMB_LAUNCH_CHECK(ctx);
      }
      {
        EpiLgResidual e;
        e.rows = rows;
        e.x32 = lg->x32[cur];
        e.xh = lg->xh[cur];
        e.xl = exact ? lg->xl[cur] : nullptr;
        e.bias = f3.bias;
        e.residual = 1;
        DIMB_TRY(lg_gemm(lg, st, lg->m_h2, f3, e, m_tiles, "lg.ffn3"));
      }
    }
    if (i == L - 1 || !adaptive) continue;  // no early stopping or adaptive width at the last layer (lightglue.py:494)
    ProfScope prof_tail(ctx, st, "lg.tail");
    DIMB_TRY(launch_lg_tail(ctx, st, P, rows, lg->x32[cur], ly.wt, ly.bt, ly.wm, ly.bm, lg->tok, lg->mat, lg->n_act[nxt], lg->n_orig,
                            lg->stopped, lg->counter, lg->map, i, ly.thr, depth_conf, keep_thr, do_stop, do_prune, cf.prune_min_kpts));
    lg_gather_kernel<<<ceil_div(R * 32, 256), 256, 0, st>>>(lg->n_act[nxt], lg->stopped, i, lg->map, NP, R, lg->x32[cur], lg->x32[nxt],
                                                             lg->xh[cur], lg->xh[nxt], exact ? lg->xl[cur] : nullptr, lg->xl[nxt],
                                                             lg->cs[cur], lg->cs[nxt], lg->sn[cur], lg->sn[nxt], lg->ind[cur],
                                                             lg->ind[nxt]);
    DIMB_LAUNCH_CHECK(ctx);
  }

  // ---- assignment
  lg_final_select_kernel<<<ceil_div(P, 128), 128, 0, st>>>(lg->stopped, lg->n_act[0], lg->n_act[1], lg->nf, lg->layer_of, lg->parity,
                                                           P, L, adaptive ? 1 : 0);
  DIMB_LAUNCH_CHECK(ctx);
  lg_final_gather_kernel<<<ceil_div(R * 32, 256), 256, 0, st>>>(lg->nf, lg->layer_of, lg->parity, NP, R, lg->x32[0], lg->x32[1],
                                                                 lg->xh[0], lg->xh[1], lg->xl[0], lg->xl[1], lg->ind[0], lg->ind[1],
                                                                 lg->fh, exact ? lg->fl : nullptr, lg->indf, lg->wm_all, lg->bm_all,
                                                                 lg->z, lg->xf32);
  DIMB_LAUNCH_CHECK(ctx);
  {
    EpiFinalProj e;
    e.nf = lg->nf;
    e.layer = lg->layer_of;
    e.hi = lg->mdh;
    e.lo = exact ? lg->mdl : nullptr;
    e.bias = lg->fproj.bias;
    e.NP = NP;
    TcOperands ops;
    ops.Ah = lg->m_f[0];
    ops.Al = lg->m_f[1];
    ops.Bh = lg->fproj.tmh;
    ops.Bl = lg->fproj.tml;
    GemmArgs g{};
    g.num_kb = d / 64;
    g.M = R;
    g.N = L * d;  // B rows: the stacked projections of all L layers, b_row_offset picks a pair's layer
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, m_tiles, d, "lg.final_proj")));
  }
  {
    EpiSim e;
    e.nf = lg->nf;
    e.sim = lg->sim;
    e.NP = NP;
    e.tiles_per_side = NP / kTileM;
    TcOperands ops;
    ops.Ah = lg->m_md[0];
    ops.Al = lg->m_md[1];
    ops.Bh = lg->m_md[0];
    ops.Bl = lg->m_md[1];
    GemmArgs g{};
    g.num_kb = d / 64;
    g.M = R;
    g.N = R;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, P * (NP / kTileM), NP, "lg.sim")));
  }
  ProfScope prof_asg(ctx, st, "lg.assign_reduce");
  return launch_lg_assign(ctx, st, P, NP, lg->sim, lg->nf, lg->n_orig, lg->layer_of, lg->z, lg->indf, filt, lg->smax, lg->slog, lg->best,
                          lg->arg, reinterpret_cast<long long*>(d_matches), d_mscores, d_n_matches, d_stop_layer, cap);
}

int dimb_lg_match(dimb_lg* lg, int P, const dimb_feats* f0, const dimb_feats* f1, int64_t* matches, float* mscores, int* n_matches,
                  int* stop_layer, int cap) {
  if (!lg || !f0 || !f1 || !matches || !mscores || !n_matches || !stop_layer || P < 1 || P > lg->conf.max_pairs) return DIMB_ERR_ARG;
  dimb_ctx* ctx = lg->ctx;
  OwnerScope own(ctx, &lg->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int S = 2 * P, NP = lg->NP, din = lg->din;
  if (!lg->st_kpts) {
    const size_t SS = lg->S;
    DIMB_TRY(dimb_alloc_t(ctx, &lg->st_kpts, SS * NP * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->st_desc, SS * NP * din));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->st_n, SS));
  }
  if (lg->o_cap < cap) {
    const size_t PP = lg->conf.max_pairs;
    for (void* old : {static_cast<void*>(lg->o_m), static_cast<void*>(lg->o_ms), static_cast<void*>(lg->o_nm), static_cast<void*>(lg->o_sl)})
      dimb_free(ctx, old);
    DIMB_TRY(dimb_alloc_t(ctx, &lg->o_m, PP * cap * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->o_ms, PP * cap));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->o_nm, PP));
    DIMB_TRY(dimb_alloc_t(ctx, &lg->o_sl, PP));
    lg->o_cap = cap;
  }
  cudaStream_t st = 0;
  std::vector<dimb_feats_dev> d0(P), d1(P);
  std::vector<int> ns(S);
  for (int p = 0; p < P; ++p)
    for (int sd = 0; sd < 2; ++sd) {
      const dimb_feats& f = sd ? f1[p] : f0[p];
      const int s = 2 * p + sd;
      if (f.n < 0 || f.n > NP || (f.n > 0 && (!f.keypoints || !f.descriptors))) {
        dimb_set_error(ctx, "dimb_lg_match: invalid feature set (n out of range for the workspace?)");
        return DIMB_ERR_ARG;
      }
      dimb_feats_dev& o = sd ? d1[p] : d0[p];
      float* dk = lg->st_kpts + static_cast<size_t>(s) * NP * 2;
      float* dd = lg->st_desc + static_cast<size_t>(s) * NP * din;
      const int ld = f.desc_ld ? f.desc_ld : (f.desc_layout == 0 ? f.n : din);
      if (f.n > 0) {
        DIMB_CUDA_OK(ctx, cudaMemcpyAsync(dk, f.keypoints, static_cast<size_t>(f.n) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
        if (f.desc_layout == 0)
          DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(dd, static_cast<size_t>(NP) * sizeof(float), f.descriptors, static_cast<size_t>(ld) * sizeof(float),
                                              static_cast<size_t>(f.n) * sizeof(float), din, cudaMemcpyHostToDevice, st));
        else
          DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(dd, static_cast<size_t>(din) * sizeof(float), f.descriptors, static_cast<size_t>(ld) * sizeof(float),
                                              static_cast<size_t>(din) * sizeof(float), f.n, cudaMemcpyHostToDevice, st));
      }
      ns[s] = f.n;
      o.keypoints = dk;
      o.descriptors = dd;
      o.n = lg->st_n + s;
      o.n_cap = f.n;
      o.desc_layout = f.desc_layout;
      o.desc_ld = f.desc_layout == 0 ? NP : din;
      o.round_fp16 = 0;
      if (f.has_size) {
        o.size0 = f.size0;
        o.size1 = f.size1;
      } else {  // size = 1 + kpts.max(-2) - kpts.min(-2)   (lightglue.py:26-27)
        float mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
        for (int k = 0; k < f.n; ++k) {
          mn0 = std::min(mn0, f.keypoints[2 * k]);
          mx0 = std::max(mx0, f.keypoints[2 * k]);
          mn1 = std::min(mn1, f.keypoints[2 * k + 1]);
          mx1 = std::max(mx1, f.keypoints[2 * k + 1]);
        }
        o.size0 = f.n ? 1.f + mx0 - mn0 : 1.f;
        o.size1 = f.n ? 1.f + mx1 - mn1 : 1.f;
      }
    }
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(lg->st_n, ns.data(), S * sizeof(int), cudaMemcpyHostToDevice, st));
  DIMB_TRY(dimb_lg_match_dev(lg, P, d0.data(), d1.data(), reinterpret_cast<int64_t*>(lg->o_m), lg->o_ms, lg->o_nm, lg->o_sl, cap, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(n_matches, lg->o_nm, P * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(stop_layer, lg->o_sl, P * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(matches, lg->o_m, static_cast<size_t>(P) * cap * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(mscores, lg->o_ms, static_cast<size_t>(P) * cap * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  for (int p = 0; p < P; ++p) {
    if (ns[2 * p] == 0 || ns[2 * p + 1] == 0) {  // "no keypoints" early return (lightglue.py:518-538): stop = 1
      n_matches[p] = 0;
      stop_layer[p] = 1;
    }
    if (n_matches[p] > cap) {
      dimb_set_error(ctx, "dimb_lg_match: more matches than cap");
      return DIMB_ERR_CAPACITY;
    }
  }
  return DIMB_OK;
}

int dimb_lg_debug_read(dimb_lg* lg, int which, int side, float* out, size_t n_floats) {
  if (!lg || !out || lg->gen || side < 0 || side >= lg->S) return DIMB_ERR_ARG;
  dimb_ctx* ctx = lg->ctx;
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  const size_t NP = lg->NP;
  if (which == 0) {  // final fp32 descriptors [NP][256]
    if (n_floats < NP * kD) return DIMB_ERR_ARG;
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, lg->xf32 + static_cast<size_t>(side) * NP * kD, NP * kD * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  if (which == 1) {  // similarity matrix of pair side/2 [NP][NP]
    if (n_floats < NP * NP) return DIMB_ERR_ARG;
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, lg->sim + static_cast<size_t>(side >> 1) * NP * NP, NP * NP * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  if (which == 2) {  // x32 of buffer 0 (state after an even number of gathers) [NP][256]
    if (n_floats < NP * kD) return DIMB_ERR_ARG;
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, lg->x32[0] + static_cast<size_t>(side) * NP * kD, NP * kD * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  return DIMB_ERR_ARG;
}

}  // extern "C"
