// superglue.cu - SuperGlue matching (dimb_sg_*), replacing SuperGlueMatcher._match_pairs
// (reference src/deep_image_matching/matchers/superglue.py:75-106, adapter features_2_sg :8-41) and the model it drives
// (thirdparty/SuperGluePretrainedNetwork/models/superglue.py:51-305: keypoint encoder :73-84, attentional GNN :96-152,
// log-space Sinkhorn :155-187, mutual-max matching :278-296).
//
// One batched engine (dimb_sg_match_dev) serves P pairs = S = 2P sides per call with no host synchronisation; side s owns rows
// [s * NPt, (s + 1) * NPt) of every token buffer (NPt = max_kpts rounded up to 128), as in lightglue.cu.  Keypoint counts, the
// per-pair Sinkhorn constants and the outputs stay on the device:
//   input    : one kernel over all sides reads float32 / float16 keypoints, descriptors and scores (optional fp16 rounding), writes
//              the token-major descriptors and the keypoint encoder's input (normalised x, y, score); padded rows are zero
//   encoder  : 3 -> 32 -> 64 -> 128 -> 256 -> 256 on the plain fp32 tile of generic_kernels.cuh, one launch per layer over all sides
//              (0.2 GMAC per side), rows past n skipped
//   GNN      : SuperGlue's attention shape is 256 / 4 heads x 64 - the shape of LightGlue's tensor-core kernels - so the 18 layers run
//              on the shared building blocks of lg_kernels.cuh: per layer ONE q|k GEMM (EpiQK without rotary), the V^T GEMM, the
//              flash-attention kernel (self: keys of the same side, cross: keys and values of the other side), merge -> message half of
//              the [x | message] buffer, MLP0 with the eval-mode BatchNorm folded in and a ReLU / hi-lo-split epilogue, MLP3 + residual;
//              then final_proj and the score block of every pair (and its transpose) as wgmma GEMMs
//   Sinkhorn : 100 log-space sweeps with the dustbin row / column kept virtual; one launch per half step serves a wave of pairs
//              whose two score blocks fit in L2 together, so each sweep reads L2 rather than HBM (DESIGN.md section 3)
//   matches  : row / column max and first argmax of the log assignment, then one CTA per pair for the mutual check, the threshold
//              and the ordered compaction into the [P][cap] tables of dimb_lg_match_dev
// Done once at create time: BatchNorm folding, and the reference's (dim, heads)-interleaved channel order of `view(b, dim, heads, n)`
// (:111-113) permuted to head-major.  dimb_sg_match stages one host pair and runs the same engine with P = 1.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "generic_kernels.cuh"
#include "lg_kernels.cuh"
#include "sg_assign.cuh"

namespace {

constexpr int kSgD = 256, kSgHeads = 4, kSgHd = 64;

// ---------------------------------------------------------------- tensor-core path helpers
// out = relu(acc + bias) -> fp16 hi/lo planes (MLP0 with the BatchNorm folded into weights and bias), live tiles only
struct EpiSgReluSplit : EpiBase {
  LgRows rows;
  __half *hi, *lo;
  const float* bias;
  int ldc;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const size_t off = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * ldc + col;
      store_split4(hi + off, lo ? lo + off : nullptr,
                   make_float4(fmaxf(f[it].x + b.x, 0.f), fmaxf(f[it].y + b.y, 0.f), fmaxf(f[it].z + b.z, 0.f), fmaxf(f[it].w + b.w, 0.f)));
    }
  }
};

// one side of the batched engine (dimb_sg_feats_dev, resolved)
struct SgSideIn {
  const void *kpts, *desc, *scores;
  const int* n;
  int n_cap, ld, f16, round_fp16, height, width;
  const int* size_dev;
};

// element i of a float32 or float16 array, float32 values optionally rounded to fp16 (the features.h5 round trip)
__device__ __forceinline__ float sg_ld(const void* p, size_t i, int f16, int r16) {
  if (f16) return __half2float(static_cast<const __half*>(p)[i]);
  const float v = static_cast<const float*>(p)[i];
  return r16 ? __half2float(__float2half_rn(v)) : v;
}

// live keypoints of side `side`: 0 for both sides of a pair with an empty side (the "no keypoints" return, superglue.py:248-256),
// so that no later kernel does any work for that pair
__device__ __forceinline__ int sg_side_n(const SgSideIn* in, int side, int NPs) {
  const SgSideIn &a = in[side], &b = in[side ^ 1];
  const int na = min(min(*a.n, a.n_cap), NPs), nb = min(min(*b.n, b.n_cap), NPs);
  return (na <= 0 || nb <= 0) ? 0 : na;
}

// grid (ceil(NPs / 32), S), block (32, 8).  FeaturesDict inputs of every side -> descriptors token-major in dst rows
// [side * NPs, (side + 1) * NPs) (pitch ldd, 32 x 32 tile transpose) and the keypoint encoder's input enc_in [row][3] = (normalised x,
// normalised y, score) (normalize_keypoints, superglue.py:63-70); padded rows are zero.  Block 0 of every side records the live
// count, and for even sides the pair's Sinkhorn constants pc[p] = {norm = -log(m + n), log n, log m} (:177-181).
__global__ void sg_input_kernel(const SgSideIn* __restrict__ in, int NPs, float* __restrict__ dst, int ldd, float* __restrict__ enc_in,
                                int* __restrict__ n_act, int* __restrict__ stopped, float* __restrict__ pc) {
  const int side = blockIdx.y, t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const SgSideIn si = in[side];
  const int n = sg_side_n(in, side, NPs);
  if (blockIdx.x == 0 && tx == 0 && ty == 0) {
    n_act[side] = n;
    if ((side & 1) == 0) {
      const int nb = sg_side_n(in, side + 1, NPs);
      stopped[side >> 1] = 0;  // SuperGlue has no early exit
      sg_pair_consts(n, nb, pc + 4 * (side >> 1));
    }
  }
  __shared__ float tile[32][33];
  for (int c0 = 0; c0 < kSgD; c0 += 32) {
    for (int k = ty; k < 32; k += 8) {
      const int tok = t0 + tx;
      tile[k][tx] = tok < n ? sg_ld(si.desc, static_cast<size_t>(c0 + k) * si.ld + tok, si.f16, si.round_fp16) : 0.f;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8)
      if (t0 + k < NPs) dst[(static_cast<size_t>(side) * NPs + t0 + k) * ldd + c0 + tx] = tile[tx][k];
    __syncthreads();
  }
  const int tok = t0 + tx;
  if (ty != 0 || tok >= NPs) return;
  float* e = enc_in + (static_cast<size_t>(side) * NPs + tok) * 3;
  if (tok >= n) {
    e[0] = e[1] = e[2] = 0.f;
    return;
  }
  const int H = si.size_dev ? si.size_dev[0] : si.height, W = si.size_dev ? si.size_dev[1] : si.width;
  const float cx = static_cast<float>(W) / 2.f, cy = static_cast<float>(H) / 2.f, sc = static_cast<float>(max(W, H)) * 0.7f;
  e[0] = (sg_ld(si.kpts, 2 * static_cast<size_t>(tok), si.f16, si.round_fp16) - cx) / sc;
  e[1] = (sg_ld(si.kpts, 2 * static_cast<size_t>(tok) + 1, si.f16, si.round_fp16) - cy) / sc;
  e[2] = sg_ld(si.scores, tok, si.f16, si.round_fp16);
}

// one keypoint-encoder layer over all sides: grid (ceil(N / 64), ceil(NPs / 64), S); rows past n_act[side] are neither read nor written
__global__ void __launch_bounds__(256) sg_enc_linear_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ C, int ldc, int N, int K,
                                                            int NPs, const int* __restrict__ n_act, int relu, int resid) {
  const int side = blockIdx.z, M = n_act[side], m0 = blockIdx.y * 64;
  if (m0 >= M) return;
  const size_t r0 = static_cast<size_t>(side) * NPs;
  float* c = C + r0 * ldc;
  gx_linear_tile(A + r0 * lda, lda, W, K, bias, c, ldc, M, N, K, 1.f, resid ? c : nullptr, ldc, relu, m0);
}

// fp32 token state -> fp16 hi/lo first half of the [x | message] concat buffer, one 256-thread block per row (padded rows included)
__global__ void sg_pack_kernel(const float* __restrict__ x32, __half* __restrict__ xh, __half* __restrict__ xl) {
  const size_t row = blockIdx.x;
  const int c = threadIdx.x;
  __half h, l;
  split_f32(x32[row * kSgD + c], h, l);
  xh[row * 2 * kSgD + c] = h;
  if (xl) xl[row * 2 * kSgD + c] = l;
}

struct SgLin {
  float *w = nullptr, *b = nullptr;
  int n = 0, k = 0;
};
struct SgTcLin {  // fp16 hi/lo planes [n][k] + fp32 bias + TMA maps (boxes of 128 rows)
  __half *wh = nullptr, *wl = nullptr;
  float* bias = nullptr;
  int n = 0, k = 0;
  CUtensorMap tmh, tml;
};
struct SgTcLayer {
  SgTcLin qkv, merge, mlp0, mlp3;  // qkv = [Wq ; Wk ; Wv] stacked (768 x 256), head-major rows
};

}  // namespace

struct dimb_sg {
  dimb_ctx* ctx;
  std::vector<void*> mem;
  dimb_sg_conf conf;
  int NP, L, max_pairs;
  std::vector<int> cross;  // per GNN layer: 1 = cross, 0 = self
  SgLin kenc[5];
  float* bin_score;
  // ---- batched engine (side s = rows [s * NPt, (s + 1) * NPt) of every token buffer, NPt = NP rounded up to 128)
  int NPt = 0, vld = 0, wave = 1;  // vld: pitch of the per-pair u / v vectors; wave: pairs per Sinkhorn launch (L2-resident blocks)
  std::vector<SgTcLayer> tc;
  SgTcLin tc_final;
  SgSideIn* side_in = nullptr;  // [2 * max_pairs]
  float *x32 = nullptr, *enc_in = nullptr;
  __half *xh, *xl, *qh, *ql, *kh, *kl, *vth, *vtl, *ctxh, *ctxl, *h2h, *h2l, *mdh, *mdl;
  float *sim = nullptr, *simT = nullptr;  // [P][NPt][NPt] score blocks and their transposes (both sweeps of a Sinkhorn iteration read rows)
  int *n_act = nullptr, *stopped = nullptr;
  float *pc = nullptr, *uu = nullptr, *vv = nullptr, *best0 = nullptr;  // pc [P][4] Sinkhorn constants, uu / vv [P][vld]
  int *arg0 = nullptr, *arg1 = nullptr;                                 // best0 / arg0 / arg1 [P][NPt]
  CUtensorMap m_x[2], m_ctx[2], m_h2[2], m_md[2], m_q128[2], m_k64[2], m_vt[2];
  // ---- host entry: staging of one host pair, output tables
  float *st_kp = nullptr, *st_sc = nullptr, *st_desc = nullptr;
  int* st_n = nullptr;
  int64_t* o_m = nullptr;
  float* o_ms = nullptr;
  int* o_nm = nullptr;
  int o_cap = 0;
};

namespace {

// host-side weight preparation: 1x1 conv [n][k] (+ optional eval BatchNorm folded in), optional row / column permutations
struct HostLin {
  std::vector<float> w, b;
  int n, k;
};
HostLin take_conv(const float*& p, int n, int k) {
  HostLin l;
  l.n = n, l.k = k;
  l.w.assign(p, p + static_cast<size_t>(n) * k);
  p += static_cast<size_t>(n) * k;
  l.b.assign(p, p + n);
  p += n;
  return l;
}
void fold_bn(HostLin& l, const float*& p) {  // gamma, beta, running_mean, running_var (eps 1e-5)
  const float *g = p, *be = p + l.n, *mu = p + 2 * l.n, *var = p + 3 * l.n;
  for (int o = 0; o < l.n; ++o) {
    const float a = g[o] / std::sqrt(var[o] + 1e-5f);
    for (int c = 0; c < l.k; ++c) l.w[static_cast<size_t>(o) * l.k + c] *= a;
    l.b[o] = a * (l.b[o] - mu[o]) + be[o];
  }
  p += 4 * l.n;
}
inline int head_major(int c) { return (c % kSgHeads) * kSgHd + c / kSgHeads; }  // reference channel d * heads + h -> h * 64 + d
void permute_rows(HostLin& l) {
  HostLin o = l;
  for (int c = 0; c < l.n; ++c) {
    std::memcpy(&o.w[static_cast<size_t>(head_major(c)) * l.k], &l.w[static_cast<size_t>(c) * l.k], l.k * sizeof(float));
    o.b[head_major(c)] = l.b[c];
  }
  l = o;
}
void permute_cols(HostLin& l) {
  HostLin o = l;
  for (int r = 0; r < l.n; ++r)
    for (int c = 0; c < l.k; ++c) o.w[static_cast<size_t>(r) * l.k + head_major(c)] = l.w[static_cast<size_t>(r) * l.k + c];
  l = o;
}
int upload_tc(dimb_ctx* ctx, SgTcLin& d, const HostLin& h) {
  d.n = h.n, d.k = h.k;
  std::vector<__half> hi(h.w.size()), lo(h.w.size());
  for (size_t i = 0; i < h.w.size(); ++i) {
    hi[i] = __float2half_rn(h.w[i]);
    lo[i] = __float2half_rn(h.w[i] - __half2float(hi[i]));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &d.wh, hi.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.wl, lo.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.bias, h.b.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.wh, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.wl, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.bias, h.b.data(), h.b.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_TRY(dimb_tmap_2d(ctx, &d.tmh, d.wh, h.n, h.k, h.k, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &d.tml, d.wl, h.n, h.k, h.k, 128));
  return DIMB_OK;
}
int upload(dimb_ctx* ctx, SgLin& d, const HostLin& h) {
  d.n = h.n, d.k = h.k;
  DIMB_TRY(dimb_alloc_t(ctx, &d.w, h.w.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.b, h.b.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.w, h.w.data(), h.w.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.b, h.b.data(), h.b.size() * sizeof(float), cudaMemcpyHostToDevice));
  return DIMB_OK;
}

// one GEMM over the token rows of all S sides: C = A [S * NPt][K] * W^T on the wgmma kernel of gemm.cuh with epilogue `epi`
template <class Epi>
int sg_tc_gemm(dimb_sg* g, cudaStream_t st, int S, const CUtensorMap* A, const SgTcLin& w, int n_out, const Epi& epi, const char* tag) {
  TcOperands ops;
  ops.Ah = A[0];
  ops.Al = A[1];
  ops.Bh = w.tmh;
  ops.Bl = w.tml;
  GemmArgs ga{};
  ga.num_kb = w.k / 64;
  ga.M = S * g->NPt;
  ga.N = n_out;
  return launch_gemm<128, false>(g->ctx, st, ops, ga, epi, S * g->NPt / kTileM, n_out, tag);
}

// keypoint encoder of S sides (rows of NPs per side; enc_in written by sg_input_kernel): dst rows += MLP(enc_in) (:73-84).  Its fp32
// scratch lives in the MLP hidden buffers h2h / h2l, which the GNN only uses afterwards.
int sg_encoder(dimb_sg* g, cudaStream_t st, int S, int NPs, float* dst, int ldd) {
  dimb_ctx* ctx = g->ctx;
  ProfScope prof(ctx, st, "sg.encoder");
  float *a = g->enc_in, *b = reinterpret_cast<float*>(g->h2h), *spare = reinterpret_cast<float*>(g->h2l);
  int lda = 3;
  for (int i = 0; i < 5; ++i) {
    const SgLin& l = g->kenc[i];
    const bool last = i == 4;  // no BN / ReLU; desc = desc + kenc(...)
    dim3 grid(ceil_div(l.n, 64), ceil_div(NPs, 64), S);
    sg_enc_linear_kernel<<<grid, 256, 0, st>>>(a, lda, l.w, l.b, last ? dst : b, last ? ldd : l.n, l.n, l.k, NPs, g->n_act, last ? 0 : 1,
                                               last ? 1 : 0);
    DIMB_LAUNCH_CHECK(ctx);
    a = b;
    std::swap(b, spare);
    lda = l.n;
  }
  return DIMB_OK;
}

// encoded descriptors (g->x32 / g->xh / g->xl of S = 2P sides) -> 18 GNN layers, final projection and the score blocks of the P pairs
// (g->sim and its transpose g->simT) on the tensor-core kernels.  Both sides advance together from the OLD descriptors, as the
// reference does (superglue.py:147-151).  Live rows come from g->n_act (device).
int sg_gnn_tc(dimb_sg* g, cudaStream_t st, int P) {
  dimb_ctx* ctx = g->ctx;
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int NPt = g->NPt, d = kSgD, S = 2 * P, R = S * NPt;
  const LgRows rows{g->n_act, g->stopped, NPt};
  for (int i = 0; i < g->L; ++i) {
    const SgTcLayer& ly = g->tc[i];
    {  // q | k for every token of every side (no rotary: EpiQK's cross flag only switches the rotation off)
      EpiQK e;
      e.rows = rows;
      e.bias = ly.qkv.bias;
      e.cs = e.sn = nullptr;
      e.qh = g->qh, e.ql = exact ? g->ql : nullptr, e.kh = g->kh, e.kl = exact ? g->kl : nullptr;
      e.cross = 1;
      DIMB_TRY(sg_tc_gemm(g, st, S, g->m_x, ly.qkv, 2 * d, e, "sg.qk"));
    }
    {  // V^T: weights as the A operand (rows 512..767 of the stacked projection), tokens as B
      EpiVT e;
      e.rows = rows;
      e.bias = ly.qkv.bias;
      e.vth = g->vth, e.vtl = exact ? g->vtl : nullptr;
      e.w_row0 = 2 * d;
      TcOperands ops;
      ops.Ah = ly.qkv.tmh, ops.Al = ly.qkv.tml, ops.Bh = g->m_x[0], ops.Bl = g->m_x[1];
      GemmArgs ga{};
      ga.num_kb = d / 64;
      ga.M = ly.qkv.n, ga.N = R;
      DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, 2, R, "sg.vT")));
    }
    {  // attention: self layers attend to their own side, cross layers to the keys AND values of the other side
      AttnArgs a;
      a.rows = rows;
      a.cross = g->cross[i];
      a.ctx_h = g->ctxh, a.ctx_l = exact ? g->ctxl : nullptr;
      a.scale = 0.125f;
      a.lazy = ctx->attn_lazy;
      ProfScope prof(ctx, st, "sg.attention");
      dim3 grid(ceil_div(NPt, 2 * kTileM), kHeads, S);
      DIMB_TRY(launch_lg_attention(ctx, st, grid, g->m_q128, g->m_k64, g->m_vt, a, exact));
      DIMB_LAUNCH_CHECK(ctx);
    }
    {  // merge -> message half of [x | message]
      EpiLgSplit e;
      e.rows = rows;
      e.hi = g->xh, e.lo = exact ? g->xl : nullptr;
      e.bias = ly.merge.bias;
      e.ldc = 2 * d, e.col_off = d;
      DIMB_TRY(sg_tc_gemm(g, st, S, g->m_ctx, ly.merge, d, e, "sg.merge"));
    }
    {  // MLP0 (BatchNorm folded) + ReLU
      EpiSgReluSplit e;
      e.rows = rows;
      e.hi = g->h2h, e.lo = exact ? g->h2l : nullptr;
      e.bias = ly.mlp0.bias;
      e.ldc = 2 * d;
      DIMB_TRY(sg_tc_gemm(g, st, S, g->m_x, ly.mlp0, 2 * d, e, "sg.mlp0"));
    }
    {  // x += MLP3(...)
      EpiLgResidual e;
      e.rows = rows;
      e.x32 = g->x32;
      e.xh = g->xh, e.xl = exact ? g->xl : nullptr;
      e.bias = ly.mlp3.bias;
      e.residual = 1;
      DIMB_TRY(sg_tc_gemm(g, st, S, g->m_h2, ly.mlp3, d, e, "sg.mlp3"));
    }
  }
  {  // mdesc = final_proj(x) / 256^0.25 on each side, so that the score block is mdesc0 . mdesc1^T / sqrt(256) (:262-265)
    EpiStoreSplit e;
    e.hi = g->mdh, e.lo = exact ? g->mdl : nullptr;
    e.bias = g->tc_final.bias;
    e.ldc = d, e.col_off = 0, e.n_valid = d, e.m_valid = R;
    e.scale = 0.25f;
    DIMB_TRY(sg_tc_gemm(g, st, S, g->m_x, g->tc_final, d, e, "sg.final_proj"));
  }
  {
    EpiSim e;
    e.nf = g->n_act;
    e.sim = g->sim;
    e.NP = NPt;
    e.tiles_per_side = NPt / kTileM;
    TcOperands ops;
    ops.Ah = g->m_md[0], ops.Al = g->m_md[1], ops.Bh = g->m_md[0], ops.Bl = g->m_md[1];
    GemmArgs ga{};
    ga.num_kb = d / 64;
    ga.M = R, ga.N = R;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, P * (NPt / kTileM), NPt, "sg.scores")));
    e.sim = g->simT;  // the same products with the operand roles swapped: scores^T, so that the column sweeps of Sinkhorn read rows
    e.swap = 1;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, P * (NPt / kTileM), NPt, "sg.scores")));
  }
  return DIMB_OK;
}

// row / column max and first argmax of the log assignment (score blocks Z of pitch ld, pairs pstride apart) and the match tables
int sg_matches(dimb_sg* g, cudaStream_t st, int P, const float* Z, int ld, size_t pstride, int NPs, int64_t* d_matches, float* d_mscores,
               int* d_n_matches, int cap) {
  dimb_ctx* ctx = g->ctx;
  ProfScope prof(ctx, st, "sg.matches");
  return launch_sg_matches(ctx, st, P, Z, ld, pstride, NPs, g->n_act, g->uu, g->vv, g->vld, g->pc, g->conf.match_threshold, g->best0, g->arg0,
                           g->arg1, reinterpret_cast<long long*>(d_matches), d_mscores, d_n_matches, cap);
}

}  // namespace

extern "C" {

size_t dimb_sg_weight_count(int n_layers) {
  const size_t d = kSgD;
  size_t n = 0;
  const int ch[6] = {3, 32, 64, 128, 256, 256};
  for (int i = 0; i < 5; ++i) n += static_cast<size_t>(ch[i + 1]) * ch[i] + ch[i + 1] + (i < 4 ? 4 * ch[i + 1] : 0);
  n += static_cast<size_t>(n_layers) * (4 * (d * d + d) + (2 * d * 2 * d + 2 * d) + 4 * 2 * d + (d * 2 * d + d));
  return n + d * d + d + 1;
}

int dimb_sg_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_sg_conf* conf, dimb_sg** out) {
  if (!ctx || !weights || !conf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  if (conf->n_layers < 1 || conf->n_layers > 64 || conf->max_kpts < 1 || conf->sinkhorn_iterations < 0 || conf->max_pairs < 0)
    return DIMB_ERR_ARG;
  if (n_floats != dimb_sg_weight_count(conf->n_layers)) {
    dimb_set_error(ctx, "dimb_sg_create: weight blob has " + std::to_string(n_floats) + " floats, expected " +
                            std::to_string(dimb_sg_weight_count(conf->n_layers)));
    return DIMB_ERR_ARG;
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  dimb_sg* g = new dimb_sg();
  g->ctx = ctx;
  std::unique_ptr<dimb_sg, void (*)(dimb_sg*)> guard(g, dimb_sg_destroy);
  OwnerScope own(ctx, &g->mem);
  g->conf = *conf;
  g->L = conf->n_layers;
  g->NP = conf->max_kpts;
  g->max_pairs = conf->max_pairs ? conf->max_pairs : 1;
  for (int i = 0; i < g->L; ++i) g->cross.push_back((conf->cross_mask >> i) & 1ull ? 1 : 0);
  const float* p = weights;
  const int ch[6] = {3, 32, 64, 128, 256, 256};
  for (int i = 0; i < 5; ++i) {
    HostLin l = take_conv(p, ch[i + 1], ch[i]);
    if (i < 4) fold_bn(l, p);
    DIMB_TRY(upload(ctx, g->kenc[i], l));
  }
  g->tc.resize(g->L);
  for (int i = 0; i < g->L; ++i) {  // state_dict order: attn.merge, attn.proj.0/1/2, mlp.0, mlp.1 (BN), mlp.3
    HostLin merge = take_conv(p, kSgD, kSgD), q = take_conv(p, kSgD, kSgD), k = take_conv(p, kSgD, kSgD), v = take_conv(p, kSgD, kSgD);
    HostLin m0 = take_conv(p, 2 * kSgD, 2 * kSgD);
    fold_bn(m0, p);
    HostLin m3 = take_conv(p, kSgD, 2 * kSgD);
    permute_rows(q), permute_rows(k), permute_rows(v), permute_cols(merge);
    HostLin qkv = q;
    qkv.n = 3 * kSgD;
    qkv.w.insert(qkv.w.end(), k.w.begin(), k.w.end());
    qkv.w.insert(qkv.w.end(), v.w.begin(), v.w.end());
    qkv.b.insert(qkv.b.end(), k.b.begin(), k.b.end());
    qkv.b.insert(qkv.b.end(), v.b.begin(), v.b.end());
    SgTcLayer& t = g->tc[i];
    DIMB_TRY(upload_tc(ctx, t.qkv, qkv));
    DIMB_TRY(upload_tc(ctx, t.merge, merge));
    DIMB_TRY(upload_tc(ctx, t.mlp0, m0));
    DIMB_TRY(upload_tc(ctx, t.mlp3, m3));
  }
  DIMB_TRY(upload_tc(ctx, g->tc_final, take_conv(p, kSgD, kSgD)));
  DIMB_TRY(dimb_alloc_t(ctx, &g->bin_score, 1, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(g->bin_score, p, sizeof(float), cudaMemcpyHostToDevice));
  const size_t NP = g->NP, PP = g->max_pairs, d = kSgD;
  {  // host entry: staging of one pair, outputs
    DIMB_TRY(dimb_alloc_t(ctx, &g->st_kp, 2 * NP * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &g->st_sc, 2 * NP));
    DIMB_TRY(dimb_alloc_t(ctx, &g->st_desc, 2 * d * NP));
    DIMB_TRY(dimb_alloc_t(ctx, &g->st_n, 2));
    DIMB_TRY(dimb_alloc_t(ctx, &g->o_nm, 1));
  }
  {  // batched engine
    const size_t NPt = round_up(g->NP, 128), S = 2 * PP, R = S * NPt;
    g->NPt = static_cast<int>(NPt);
    g->vld = static_cast<int>(NPt) + 1;
    // Sinkhorn waves: as many pairs per launch as keep their sim + simT blocks (at capacity) within 3/4 of L2
    int l2 = 0;
    DIMB_CUDA_OK(ctx, cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, ctx->device));
    g->wave = std::max<int>(1, static_cast<int>(static_cast<size_t>(l2) * 3 / 4 / (2 * NPt * NPt * sizeof(float))));
    DIMB_TRY(dimb_alloc_t(ctx, &g->side_in, S));
    DIMB_TRY(dimb_alloc_t(ctx, &g->x32, R * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->enc_in, R * 3));
    DIMB_TRY(dimb_alloc_t(ctx, &g->xh, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->xl, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->h2h, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->h2l, R * 2 * d));
    for (__half** b : {&g->qh, &g->ql, &g->kh, &g->kl, &g->vth, &g->vtl, &g->ctxh, &g->ctxl, &g->mdh, &g->mdl}) DIMB_TRY(dimb_alloc_t(ctx, b, R * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->sim, PP * NPt * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->simT, PP * NPt * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->n_act, S));
    DIMB_TRY(dimb_alloc_t(ctx, &g->stopped, PP));
    DIMB_TRY(dimb_alloc_t(ctx, &g->pc, 4 * PP));
    DIMB_TRY(dimb_alloc_t(ctx, &g->uu, PP * g->vld));
    DIMB_TRY(dimb_alloc_t(ctx, &g->vv, PP * g->vld));
    DIMB_TRY(dimb_alloc_t(ctx, &g->best0, PP * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->arg0, PP * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->arg1, PP * NPt));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_x[0], g->xh, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_x[1], g->xl, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_h2[0], g->h2h, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_h2[1], g->h2l, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_ctx[0], g->ctxh, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_ctx[1], g->ctxl, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_md[0], g->mdh, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_md[1], g->mdl, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_q128[0], g->qh, S * kHeads * NPt, kHd, kHd, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_q128[1], g->ql, S * kHeads * NPt, kHd, kHd, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_k64[0], g->kh, S * kHeads * NPt, kHd, kHd, kBlkK));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_k64[1], g->kl, S * kHeads * NPt, kHd, kHd, kBlkK));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_vt[0], g->vth, S * kHeads * kHd, NPt, NPt, kHd));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_vt[1], g->vtl, S * kHeads * kHd, NPt, NPt, kHd));
  }
  *out = guard.release();
  return DIMB_OK;
}

void dimb_sg_destroy(dimb_sg* g) {
  if (!g) return;
  dimb_release(g->ctx, g->mem);
  delete g;
}

int dimb_sg_match_dev(dimb_sg* g, int P, const dimb_sg_feats_dev* f0, const dimb_sg_feats_dev* f1, int64_t* d_matches, float* d_mscores,
                      int* d_n_matches, int cap, void* stream) {
  if (!g || !f0 || !f1 || !d_matches || !d_mscores || !d_n_matches || P < 1 || P > g->max_pairs || cap < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = g->ctx;
  const int S = 2 * P, NPt = g->NPt;
  std::vector<SgSideIn> hin(S);
  for (int p = 0; p < P; ++p)
    for (int sd = 0; sd < 2; ++sd) {
      const dimb_sg_feats_dev& f = sd ? f1[p] : f0[p];
      if (!f.keypoints || !f.descriptors || !f.scores || !f.n || f.n_cap < 0 || f.n_cap > g->NP) {
        dimb_set_error(ctx, "dimb_sg_match_dev: pair " + std::to_string(p) + " side " + std::to_string(sd) +
                                ": NULL keypoints / descriptors / scores / n, or n_cap above max_kpts");
        return DIMB_ERR_ARG;
      }
      hin[2 * p + sd] = SgSideIn{f.keypoints, f.descriptors, f.scores, f.n, f.n_cap, f.desc_ld ? f.desc_ld : f.n_cap, f.f16, f.round_fp16,
                                 f.height, f.width, f.size_dev};
    }
  OwnerScope own(ctx, &g->mem);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->side_in, hin.data(), S * sizeof(SgSideIn), cudaMemcpyHostToDevice, st));
  {
    ProfScope prof(ctx, st, "sg.input");
    sg_input_kernel<<<dim3(NPt / 32, S), dim3(32, 8), 0, st>>>(g->side_in, NPt, g->x32, kSgD, g->enc_in, g->n_act, g->stopped, g->pc);
    DIMB_LAUNCH_CHECK(ctx);
  }
  DIMB_TRY(sg_encoder(g, st, S, NPt, g->x32, kSgD));
  {
    ProfScope prof(ctx, st, "sg.input");
    sg_pack_kernel<<<S * NPt, kSgD, 0, st>>>(g->x32, g->xh, ctx->precision == DIMB_PRECISION_EXACT ? g->xl : nullptr);
    DIMB_LAUNCH_CHECK(ctx);
  }
  DIMB_TRY(sg_gnn_tc(g, st, P));
  {  // wave by wave: all iterations of a wave run while its score blocks are L2-resident
    ProfScope prof(ctx, st, "sg.sinkhorn");
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->uu, 0, static_cast<size_t>(P) * g->vld * sizeof(float), st));
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->vv, 0, static_cast<size_t>(P) * g->vld * sizeof(float), st));
    DIMB_TRY(launch_sg_sinkhorn(ctx, st, P, g->wave, 2 * g->conf.sinkhorn_iterations, g->sim, g->simT, NPt, g->n_act, g->bin_score, g->uu,
                                g->vv, g->vld, g->pc));
  }
  return sg_matches(g, st, P, g->sim, NPt, static_cast<size_t>(NPt) * NPt, NPt, d_matches, d_mscores, d_n_matches, cap);
}

// One pair.  Outputs (host): matches [cap][2] int64 ascending in column 0 (correspondence_matrix_from_matches0, superglue.py:44-52),
// mscores [cap] (matching_scores0 of the matched rows), n_matches.  Stages the pair and runs dimb_sg_match_dev with P = 1.
int dimb_sg_match(dimb_sg* g, const dimb_sg_feats* f0, const dimb_sg_feats* f1, int64_t* matches, float* mscores, int* n_matches, int cap) {
  if (!g || !f0 || !f1 || !matches || !mscores || !n_matches || cap < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = g->ctx;
  OwnerScope own(ctx, &g->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = 0;
  const dimb_sg_feats* F[2] = {f0, f1};
  const int n[2] = {f0->n, f1->n}, NP = g->NP, d = kSgD;
  *n_matches = 0;
  if (n[0] > NP || n[1] > NP || n[0] < 0 || n[1] < 0) {
    dimb_set_error(ctx, "dimb_sg_match: more keypoints than max_kpts");
    return DIMB_ERR_ARG;
  }
  if (n[0] == 0 || n[1] == 0) return DIMB_OK;  // "no keypoints" return of the reference (superglue.py:248-256): everything unmatched
  if (g->o_cap < cap) {
    dimb_free(ctx, g->o_m);
    dimb_free(ctx, g->o_ms);
    DIMB_TRY(dimb_alloc_t(ctx, &g->o_m, static_cast<size_t>(cap) * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &g->o_ms, static_cast<size_t>(cap)));
    g->o_cap = cap;
  }
  dimb_sg_feats_dev df[2];
  for (int s = 0; s < 2; ++s) {
    const dimb_sg_feats& f = *F[s];
    float* kp = g->st_kp + static_cast<size_t>(s) * NP * 2;
    float* sc = g->st_sc + static_cast<size_t>(s) * NP;
    float* de = g->st_desc + static_cast<size_t>(s) * d * NP;
    const int ld = f.desc_ld ? f.desc_ld : f.n;
    DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(de, static_cast<size_t>(NP) * sizeof(float), f.descriptors, static_cast<size_t>(ld) * sizeof(float),
                                        static_cast<size_t>(n[s]) * sizeof(float), d, cudaMemcpyHostToDevice, st));
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(kp, f.keypoints, static_cast<size_t>(n[s]) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(sc, f.scores, static_cast<size_t>(n[s]) * sizeof(float), cudaMemcpyHostToDevice, st));
    df[s] = dimb_sg_feats_dev{kp, de, sc, g->st_n + s, n[s], NP, 0, 0, f.height, f.width, nullptr};
  }
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->st_n, n, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
  DIMB_TRY(dimb_sg_match_dev(g, 1, &df[0], &df[1], g->o_m, g->o_ms, g->o_nm, cap, st));
  int cnt = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(&cnt, g->o_nm, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  const int rows = std::min(cnt, cap);
  DIMB_CUDA_OK(ctx, cudaMemcpy(matches, g->o_m, static_cast<size_t>(rows) * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost));
  DIMB_CUDA_OK(ctx, cudaMemcpy(mscores, g->o_ms, static_cast<size_t>(rows) * sizeof(float), cudaMemcpyDeviceToHost));
  *n_matches = cnt;
  if (cnt > cap) {
    dimb_set_error(ctx, "dimb_sg_match: more matches than cap");
    return DIMB_ERR_CAPACITY;
  }
  return DIMB_OK;
}

}  // extern "C"
