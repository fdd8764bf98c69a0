// lightglue_generic.cu - LightGlue for shapes other than (descriptor_dim 256, 4 heads x 64), i.e. the LighterGlue
// checkpoint the reference ships (thirdparty/accelerated_features/modules/lighterglue.py:12-27: descriptor_dim 96,
// one head, 6 layers, input_dim 64; matcher plugin src/deep_image_matching/matchers/lighterglue.py:78-262).
// Same algorithm as lightglue.cu (thirdparty/LightGlue/lightglue/lightglue.py:24-610) in plain fp32 on the CUDA cores:
// the tensor-core kernels of lightglue.cu are specialised for head dim 64 / model dim 256 (registers and shared-memory budgets of
// the attention kernel), this file trades speed for generality.  Control flow (early stop, pruning) is decided on the host
// from per-token confidences copied back once per layer - exactly the synchronisation points of the reference
// (lightglue.py:499,503).  One pair at a time.
//
// lgx_match_dev is the batched, device-resident form of the same arithmetic (dimb_lg_match_dev for these shapes): the 2P sides
// of P pairs share one set of token buffers (side s owns rows [s*NP, (s+1)*NP)), every layer's linears, rotary, attention,
// LayerNorm/GELU and row dots run as one launch over all sides, and the live counts, stop layers and pruning maps stay on the
// device.  Each row goes through the same per-element operations as in lgx_match_pair (the kernels share their bodies), so the
// two entries agree bit for bit; the host std::exp of the confidences and of filter_matches' exp(max) is reproduced on the device
// by glibc_expf below.
#include <algorithm>
#include <memory>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include "generic_kernels.cuh"
#include "attn_hd128.cuh"
#include "lightglue_generic.cuh"

namespace {

struct Lin {
  float *w = nullptr, *b = nullptr;
  int n = 0, k = 0;
};
struct Block {
  Lin qkv, to_qk, to_v, out, ffn0, ffn3;
  float *ln_g = nullptr, *ln_b = nullptr;
};

}  // namespace

struct dimb_lgx {
  dimb_ctx* ctx;
  std::vector<void*> mem;
  dimb_lg_conf conf;
  int d, h, hd, din, L, NP;
  float* Wr;
  Lin input_proj;
  std::vector<Block> self_, cross_;
  std::vector<Lin> matchab, final_proj, token;
  // per-side state (2 sides): cat [NP][2d] = [x | message], encodings [2][NP][hd], ping-pong copies for the pruning gather
  float *cat[2][2], *enc[2][2];
  float *desc_in, *kpts, *qkv[2], *q[2], *k[2], *v[2], *hid[2], *hid2[2], *md[2], *zt[2], *sim, *rlse, *clse, *best0, *best1;
  // the two sides of a pair run on two streams (their kernels are small: one side fills a fraction of the SMs); evPack[s]: the packed
  // q / v of side s are written (the other side's cross attention reads them), evAttn[s]: side s's cross attention has read them
  cudaStream_t sst[2] = {nullptr, nullptr};
  cudaEvent_t evPack[2] = {nullptr, nullptr}, evAttn[2] = {nullptr, nullptr};
  int *arg0, *arg1, *idx;
  // tensor-core attention (attn_hd128.cuh) for head dims 65..128: packed fp16 hi / lo operands per side and their tensor maps
  bool tc_attn = false;
  int NPp = 0;                       // max_kpts rounded up to the 128-row query tile
  __half *qp[2][2], *kp[2][2], *vt[2][2];  // [side][plane]: Q / K rows [h][NPp][128], V^T [h][128][NPp]
  CUtensorMap mQ128[2][2], mQ64[2][2], mK64[2][2], mVt[2][2];
  // batched device path (lgx_match_dev): buffers for conf.max_pairs pairs, allocated by its first call
  struct Batch {
    bool ready = false;
    float *cat[2], *enc[2], *kp, *qkv, *q, *k, *v, *hid, *hid2, *xf, *md, *zt, *zm, *sim, *rlse, *clse, *best0;
    int *ind[2], *nact[2], *n_orig, *stopped, *idx, *indf, *nf, *layer, *parity, *arg0;
    void* in;                               // SideInX [2P]
    const float** tab;                      // [4][L]: final_proj w, b, matchability w, b (the final stage picks a pair's layer)
    __half *qp[2], *kp16[2], *vt[2];        // [plane]: all sides, Q / K rows [S][h][NPp][128], V^T [S][h][128][NPp]
    CUtensorMap mQ128[2], mQ64[2], mK64[2], mVt[2];
  } b;
};

namespace {

int linear(dimb_lgx* g, cudaStream_t st, const float* A, int lda, const Lin& l, float* C, int ldc, int M, float scale = 1.f,
           const float* resid = nullptr, int ldr = 0) {
  if (M <= 0) return DIMB_OK;
  dim3 grid(ceil_div(l.n, 64), ceil_div(M, 64));
  gx_linear_kernel<<<grid, 256, 0, st>>>(A, lda, l.w, l.k, l.b, C, ldc, M, l.n, l.k, scale, resid, ldr, 0);
  DIMB_LAUNCH_CHECK(g->ctx);
  return DIMB_OK;
}

// fp32 activations -> the packed fp16 hi / lo operands of the tensor-core attention (side s): what = 0 q, 1 k, 2 v
int pack_tc(dimb_lgx* g, cudaStream_t st, int s, int what, const float* src, int n) {
  const bool exact = g->ctx->precision == DIMB_PRECISION_EXACT;
  if (what == 2) {
    gx_pack_vt_kernel<<<dim3(g->NPp / 32, kXHd / 32, g->h), dim3(32, 8), 0, st>>>(src, g->d, n, g->hd, g->NPp, g->vt[s][0], exact ? g->vt[s][1] : nullptr);
  } else {
    __half** dst = what == 0 ? g->qp[s] : g->kp[s];
    gx_pack_rows_kernel<<<dim3(g->NPp, g->h), kXHd, 0, st>>>(src, g->d, n, g->hd, g->NPp, dst[0], exact ? dst[1] : nullptr);
  }
  DIMB_LAUNCH_CHECK(g->ctx);
  return DIMB_OK;
}

// tensor-core attention of side qs against the keys / values of side ks; cross: the keys are the packed q of side ks (shared to_qk)
int attention_tc(dimb_lgx* g, cudaStream_t st, int qs, int ks, bool cross, int nq, int nk, float* out, int ldo) {
  AttnXArgs a;
  a.nq = nq, a.nk = nk, a.NP = g->NPp, a.hd = g->hd;
  a.scale = 1.f / sqrtf(static_cast<float>(g->hd));
  a.lazy = g->ctx->attn_lazy;
  a.out = out, a.ldo = ldo;
  ProfScope prof(g->ctx, st, "lgx.attn_tc");
  return launch_attn_hd128(g->ctx, st, g->mQ128[qs], cross ? g->mQ64[ks] : g->mK64[ks], g->mVt[ks], g->h, a,
                           g->ctx->precision == DIMB_PRECISION_EXACT);
}

int attention(dimb_lgx* g, cudaStream_t st, const float* q, const float* k, const float* v, int nq, int nk, float* out, int ldo) {
  if (nq <= 0) return DIMB_OK;
  dim3 grid(ceil_div(nq, 8), g->h);
  if (g->hd <= 32)
    gx_attention_kernel<32><<<grid, 256, 0, st>>>(q, k, v, nq, nk, g->d, g->hd, out, ldo);
  else if (g->hd <= 64)
    gx_attention_kernel<64><<<grid, 256, 0, st>>>(q, k, v, nq, nk, g->d, g->hd, out, ldo);
  else if (g->hd <= 96)
    gx_attention_kernel<96><<<grid, 256, 0, st>>>(q, k, v, nq, nk, g->d, g->hd, out, ldo);
  else
    gx_attention_kernel<128><<<grid, 256, 0, st>>>(q, k, v, nq, nk, g->d, g->hd, out, ldo);
  DIMB_LAUNCH_CHECK(g->ctx);
  return DIMB_OK;
}

// x <- x + ffn3(gelu(ln(ffn0([x | msg]))))  on cat [n][2d]   (lightglue.py:135-143 / 176-184)
int ffn(dimb_lgx* g, cudaStream_t st, int side, float* cat, int n, const Block& b) {
  if (n <= 0) return DIMB_OK;
  const int d = g->d;
  DIMB_TRY(linear(g, st, cat, 2 * d, b.ffn0, g->hid[side], 2 * d, n));
  gx_ln_gelu_kernel<<<ceil_div(n * 32, 256), 256, 0, st>>>(g->hid[side], n, 2 * d, b.ln_g, b.ln_b, g->hid2[side]);
  DIMB_LAUNCH_CHECK(g->ctx);
  return linear(g, st, g->hid2[side], 2 * d, b.ffn3, cat, 2 * d, n, 1.f, cat, 2 * d);
}

float conf_threshold(int i, int L) {  // lightglue.py:581-584
  return static_cast<float>(std::min(std::max(0.8 + 0.1 * std::exp(-4.0 * i / L), 0.0), 1.0));
}

}  // namespace

int lgx_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* cf, dimb_lgx** out) {
  *out = nullptr;
  const int d = cf->descriptor_dim, h = cf->num_heads, L = cf->n_layers, din = cf->input_dim;
  if (d < 2 || h < 1 || d % h != 0 || (d / h) % 2 != 0 || d / h > 128 || d > 1024 || L < 1 || din < 1 || cf->max_kpts < 1) {
    dimb_set_error(ctx, "dimb_lg_create: unsupported LightGlue shape (head dim must be even and <= 128)");
    return DIMB_ERR_UNSUPPORTED;
  }
  const int hd = d / h;
  size_t need = static_cast<size_t>(hd / 2) * 2;
  if (din != d) need += static_cast<size_t>(d) * din + d;
  const size_t per_layer = (3 * d * d + 3 * d) + (d * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d)  // self
                           + 3 * (static_cast<size_t>(d) * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d);  // cross
  need += per_layer * L + static_cast<size_t>(L) * (d + 1 + d * d + d) + static_cast<size_t>(L - 1) * (d + 1);
  if (n_floats != need) {
    dimb_set_error(ctx, "dimb_lg_create: weight blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(need));
    return DIMB_ERR_ARG;
  }
  dimb_lgx* g = new dimb_lgx();
  g->ctx = ctx;
  std::unique_ptr<dimb_lgx, void (*)(dimb_lgx*)> guard(g, lgx_destroy);  // a failed create releases what it built
  OwnerScope own(ctx, &g->mem);
  g->conf = *cf;
  g->d = d, g->h = h, g->hd = hd, g->din = din, g->L = L;
  g->NP = cf->max_kpts;
  const float* p = weights;
  auto up = [&](float** dst, size_t n) -> int {
    DIMB_TRY(dimb_alloc_t(ctx, dst, n, false));
    DIMB_CUDA_OK(ctx, cudaMemcpy(*dst, p, n * sizeof(float), cudaMemcpyHostToDevice));
    p += n;
    return static_cast<int>(DIMB_OK);
  };
  auto lin = [&](Lin& l, int n, int k) -> int {
    l.n = n, l.k = k;
    DIMB_TRY(up(&l.w, static_cast<size_t>(n) * k));
    return up(&l.b, n);
  };
  DIMB_TRY(up(&g->Wr, static_cast<size_t>(hd / 2) * 2));
  if (din != d) DIMB_TRY(lin(g->input_proj, d, din));
  g->self_.resize(L), g->cross_.resize(L);
  for (int i = 0; i < L; ++i) {
    Block& s = g->self_[i];
    DIMB_TRY(lin(s.qkv, 3 * d, d));
    DIMB_TRY(lin(s.out, d, d));
    DIMB_TRY(lin(s.ffn0, 2 * d, 2 * d));
    DIMB_TRY(up(&s.ln_g, 2 * d));
    DIMB_TRY(up(&s.ln_b, 2 * d));
    DIMB_TRY(lin(s.ffn3, d, 2 * d));
    Block& c = g->cross_[i];
    DIMB_TRY(lin(c.to_qk, d, d));
    DIMB_TRY(lin(c.to_v, d, d));
    DIMB_TRY(lin(c.out, d, d));
    DIMB_TRY(lin(c.ffn0, 2 * d, 2 * d));
    DIMB_TRY(up(&c.ln_g, 2 * d));
    DIMB_TRY(up(&c.ln_b, 2 * d));
    DIMB_TRY(lin(c.ffn3, d, 2 * d));
  }
  g->matchab.resize(L), g->final_proj.resize(L), g->token.resize(std::max(L - 1, 0));
  for (int i = 0; i < L; ++i) {
    DIMB_TRY(lin(g->matchab[i], 1, d));
    DIMB_TRY(lin(g->final_proj[i], d, d));
  }
  for (int i = 0; i < L - 1; ++i) DIMB_TRY(lin(g->token[i], 1, d));
  const size_t NP = g->NP;
  for (int s = 0; s < 2; ++s)
    for (int b = 0; b < 2; ++b) {
      DIMB_TRY(dimb_alloc_t(ctx, &g->cat[s][b], NP * 2 * d));
      DIMB_TRY(dimb_alloc_t(ctx, &g->enc[s][b], 2 * NP * hd));
    }
  DIMB_TRY(dimb_alloc_t(ctx, &g->desc_in, NP * std::max(din, d)));
  DIMB_TRY(dimb_alloc_t(ctx, &g->kpts, NP * 2));
  for (int s = 0; s < 2; ++s) {
    DIMB_TRY(dimb_alloc_t(ctx, &g->qkv[s], NP * 3 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->hid[s], NP * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->hid2[s], NP * 2 * d));
    DIMB_CUDA_OK(ctx, cudaStreamCreateWithFlags(&g->sst[s], cudaStreamNonBlocking));
    DIMB_CUDA_OK(ctx, cudaEventCreateWithFlags(&g->evPack[s], cudaEventDisableTiming));
    DIMB_CUDA_OK(ctx, cudaEventCreateWithFlags(&g->evAttn[s], cudaEventDisableTiming));
  }
  for (int s = 0; s < 2; ++s) {
    DIMB_TRY(dimb_alloc_t(ctx, &g->q[s], NP * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->k[s], NP * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->v[s], NP * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->md[s], NP * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->zt[s], NP * 2));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &g->sim, NP * NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->rlse, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->clse, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->best0, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->best1, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->arg0, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->arg1, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->idx, NP));
  // head dims 65..128 (LighterGlue: 96): attention on the tensor cores (attn_hd128.cuh); other head dims run the fp32 kernel
  g->tc_attn = hd > 64 && hd <= kXHd;
  if (g->tc_attn) {
    g->NPp = (g->NP + kAttnTile - 1) / kAttnTile * kAttnTile;
    const size_t rows = static_cast<size_t>(h) * g->NPp, nel = rows * kXHd;
    for (int s = 0; s < 2; ++s)
      for (int pl = 0; pl < 2; ++pl) {
        DIMB_TRY(dimb_alloc_t(ctx, &g->qp[s][pl], nel));  // zero-initialised: pad rows / columns stay finite
        DIMB_TRY(dimb_alloc_t(ctx, &g->kp[s][pl], nel));
        DIMB_TRY(dimb_alloc_t(ctx, &g->vt[s][pl], nel));
        DIMB_TRY(dimb_tmap_2d(ctx, &g->mQ128[s][pl], g->qp[s][pl], rows, kXHd, kXHd, kAttnTile));
        DIMB_TRY(dimb_tmap_2d(ctx, &g->mQ64[s][pl], g->qp[s][pl], rows, kXHd, kXHd, kAttnBlk));
        DIMB_TRY(dimb_tmap_2d(ctx, &g->mK64[s][pl], g->kp[s][pl], rows, kXHd, kXHd, kAttnBlk));
        DIMB_TRY(dimb_tmap_2d(ctx, &g->mVt[s][pl], g->vt[s][pl], static_cast<uint64_t>(h) * kXHd, g->NPp, g->NPp, kXHd));
      }
  }
  *out = guard.release();
  return DIMB_OK;
}

void lgx_destroy(dimb_lgx* g) {
  if (!g) return;
  for (int s = 0; s < 2; ++s) {
    if (g->sst[s]) cudaStreamDestroy(g->sst[s]);
    if (g->evPack[s]) cudaEventDestroy(g->evPack[s]);
    if (g->evAttn[s]) cudaEventDestroy(g->evAttn[s]);
  }
  dimb_release(g->ctx, g->mem);
  delete g;
}

// one pair; outputs as dimb_lg_match
static int lgx_match_pair(dimb_lgx* g, const dimb_feats& f0, const dimb_feats& f1, int64_t* matches, float* mscores, int* n_matches,
                          int* stop_layer, int cap) {
  dimb_ctx* ctx = g->ctx;
  cudaStream_t st = 0;
  const int d = g->d, hd = g->hd, L = g->L, din = g->din, NP = g->NP;
  const dimb_lg_conf& cf = g->conf;
  const dimb_feats* F[2] = {&f0, &f1};
  int n[2] = {f0.n, f1.n};
  *n_matches = 0;
  if (n[0] > NP || n[1] > NP) {
    dimb_set_error(ctx, "dimb_lg_match: more keypoints than max_kpts");
    return DIMB_ERR_ARG;
  }
  if (n[0] == 0 || n[1] == 0) {  // "no keypoints" return of the reference (lightglue.py:518-538): stop = 1
    *stop_layer = 1;
    return DIMB_OK;
  }
  int cur[2] = {0, 0};  // which ping-pong copy holds the live state of each side
  std::vector<int> ind[2];
  for (int s = 0; s < 2; ++s) {
    const dimb_feats& f = *F[s];
    ind[s].resize(n[s]);
    std::iota(ind[s].begin(), ind[s].end(), 0);
    // descriptors -> [n][din] on the device (layout 0 = (D,N): transpose on the host, this is not a tuned path)
    std::vector<float> tmp;
    const float* src = f.descriptors;
    if (f.desc_layout == 0) {
      const int ld = f.desc_ld ? f.desc_ld : f.n;
      tmp.resize(static_cast<size_t>(n[s]) * din);
      for (int c = 0; c < din; ++c)
        for (int i = 0; i < n[s]; ++i) tmp[static_cast<size_t>(i) * din + c] = f.descriptors[static_cast<size_t>(c) * ld + i];
      src = tmp.data();
    } else if (f.desc_ld && f.desc_ld != din) {
      tmp.resize(static_cast<size_t>(n[s]) * din);
      for (int i = 0; i < n[s]; ++i) std::memcpy(&tmp[static_cast<size_t>(i) * din], f.descriptors + static_cast<size_t>(i) * f.desc_ld, din * sizeof(float));
      src = tmp.data();
    }
    DIMB_CUDA_OK(ctx, cudaMemcpy(g->desc_in, src, static_cast<size_t>(n[s]) * din * sizeof(float), cudaMemcpyHostToDevice));
    DIMB_CUDA_OK(ctx, cudaMemcpy(g->kpts, f.keypoints, static_cast<size_t>(n[s]) * 2 * sizeof(float), cudaMemcpyHostToDevice));
    float s0 = f.size0, s1 = f.size1;
    if (!f.has_size) {  // size = 1 + kpts.max(-2) - kpts.min(-2)   (lightglue.py:26-27)
      float mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
      for (int i = 0; i < n[s]; ++i) {
        mn0 = std::min(mn0, f.keypoints[2 * i]), mx0 = std::max(mx0, f.keypoints[2 * i]);
        mn1 = std::min(mn1, f.keypoints[2 * i + 1]), mx1 = std::max(mx1, f.keypoints[2 * i + 1]);
      }
      s0 = 1.f + mx0 - mn0, s1 = 1.f + mx1 - mn1;
    }
    gx_posenc_kernel<<<n[s], std::max(32, hd / 2), 0, st>>>(g->kpts, n[s], s0, s1, g->Wr, hd, g->enc[s][0], NP);
    DIMB_LAUNCH_CHECK(ctx);
    if (din != d) {
      DIMB_TRY(linear(g, st, g->desc_in, din, g->input_proj, g->cat[s][0], 2 * d, n[s]));
    } else {
      DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(g->cat[s][0], 2 * d * sizeof(float), g->desc_in, d * sizeof(float), d * sizeof(float), n[s],
                                          cudaMemcpyDeviceToDevice, st));
    }
    DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));  // desc_in / kpts are reused by the other side
  }
  const bool do_stop = cf.depth_confidence > 0, do_prune = cf.width_confidence > 0;
  const bool tc = g->tc_attn;
  const int m_total = n[0] + n[1];
  std::vector<float> tok[2], sc;
  bool have_tok = false;
  int i = 0;
  for (i = 0; i < L; ++i) {
    if (n[0] == 0 || n[1] == 0) break;
    const Block &sb = g->self_[i], &cb = g->cross_[i];
    for (int s = 0; s < 2; ++s) {  // self block (lightglue.py:146-159), side s on its own stream
      cudaStream_t ss = g->sst[s];
      float* cat = g->cat[s][cur[s]];
      DIMB_TRY(linear(g, ss, cat, 2 * d, sb.qkv, g->qkv[s], 3 * d, n[s]));
      // the other side's cross attention of the previous layer has read our q / v (fp32 buffers or their packed copies)
      if (i > 0) DIMB_CUDA_OK(ctx, cudaStreamWaitEvent(ss, g->evAttn[1 - s], 0));
      gx_qkv_rotary_kernel<<<n[s], std::max(32, d / 2), 0, ss>>>(g->qkv[s], n[s], d, hd, g->enc[s][cur[s]], NP, g->q[s], g->k[s], g->v[s]);
      DIMB_LAUNCH_CHECK(ctx);
      if (tc) {
        DIMB_TRY(pack_tc(g, ss, s, 0, g->q[s], n[s]));
        DIMB_TRY(pack_tc(g, ss, s, 1, g->k[s], n[s]));
        DIMB_TRY(pack_tc(g, ss, s, 2, g->v[s], n[s]));
        DIMB_TRY(attention_tc(g, ss, s, s, false, n[s], n[s], g->hid[s], d));
      } else {
        DIMB_TRY(attention(g, ss, g->q[s], g->k[s], g->v[s], n[s], n[s], g->hid[s], d));
      }
      DIMB_TRY(linear(g, ss, g->hid[s], d, sb.out, cat + d, 2 * d, n[s]));
      DIMB_TRY(ffn(g, ss, s, cat, n[s], sb));
    }
    for (int s = 0; s < 2; ++s) {  // cross block (lightglue.py:186-211): shared q/k projection, v projection
      cudaStream_t ss = g->sst[s];
      float* cat = g->cat[s][cur[s]];
      DIMB_TRY(linear(g, ss, cat, 2 * d, cb.to_qk, g->q[s], d, n[s]));
      DIMB_TRY(linear(g, ss, cat, 2 * d, cb.to_v, g->v[s], d, n[s]));
      if (tc) {
        DIMB_TRY(pack_tc(g, ss, s, 0, g->q[s], n[s]));
        DIMB_TRY(pack_tc(g, ss, s, 2, g->v[s], n[s]));
      }
      DIMB_CUDA_OK(ctx, cudaEventRecord(g->evPack[s], ss));
    }
    for (int s = 0; s < 2; ++s) {
      cudaStream_t ss = g->sst[s];
      float* cat = g->cat[s][cur[s]];
      DIMB_CUDA_OK(ctx, cudaStreamWaitEvent(ss, g->evPack[1 - s], 0));  // keys / values of the other side are in place
      if (tc)
        DIMB_TRY(attention_tc(g, ss, s, 1 - s, true, n[s], n[1 - s], g->hid[s], d));
      else
        DIMB_TRY(attention(g, ss, g->q[s], g->q[1 - s], g->v[1 - s], n[s], n[1 - s], g->hid[s], d));
      DIMB_CUDA_OK(ctx, cudaEventRecord(g->evAttn[s], ss));
      DIMB_TRY(linear(g, ss, g->hid[s], d, cb.out, cat + d, 2 * d, n[s]));
      DIMB_TRY(ffn(g, ss, s, cat, n[s], cb));
    }
    if (i == L - 1) continue;
    if (do_stop) {  // token confidence + check_if_stop (lightglue.py:73-83, 593-604)
      const float thr = conf_threshold(i, L);
      int below = 0;
      for (int s = 0; s < 2; ++s) {
        gx_rowdot_kernel<<<ceil_div(n[s] * 32, 256), 256, 0, g->sst[s]>>>(g->cat[s][cur[s]], 2 * d, n[s], d, g->token[i].w, g->token[i].b, g->zt[s]);
        DIMB_LAUNCH_CHECK(ctx);
        tok[s].resize(n[s]);
        DIMB_CUDA_OK(ctx, cudaMemcpyAsync(tok[s].data(), g->zt[s], n[s] * sizeof(float), cudaMemcpyDeviceToHost, g->sst[s]));
      }
      DIMB_CUDA_OK(ctx, cudaStreamSynchronize(g->sst[0]));
      DIMB_CUDA_OK(ctx, cudaStreamSynchronize(g->sst[1]));
      for (int s = 0; s < 2; ++s)
        for (float& z : tok[s]) {
          z = 1.f / (1.f + std::exp(-z));
          below += z < thr;
        }
      have_tok = true;
      const float ratio = 1.0f - static_cast<float>(below) / static_cast<float>(m_total);
      if (ratio > static_cast<float>(cf.depth_confidence)) break;
    }
    for (int s = 0; s < 2 && do_prune; ++s) {  // pruning (lightglue.py:481-516, 586-591)
      if (n[s] <= cf.prune_min_kpts) continue;
      cudaStream_t ss = g->sst[s];
      gx_rowdot_kernel<<<ceil_div(n[s] * 32, 256), 256, 0, ss>>>(g->cat[s][cur[s]], 2 * d, n[s], d, g->matchab[i].w, g->matchab[i].b, g->zt[s]);
      DIMB_LAUNCH_CHECK(ctx);
      sc.resize(n[s]);
      DIMB_CUDA_OK(ctx, cudaMemcpyAsync(sc.data(), g->zt[s], n[s] * sizeof(float), cudaMemcpyDeviceToHost, ss));
      DIMB_CUDA_OK(ctx, cudaStreamSynchronize(ss));
      const float thr = conf_threshold(i, L), keep_thr = static_cast<float>(1.0 - cf.width_confidence);
      std::vector<int> kidx;
      for (int j = 0; j < n[s]; ++j) {
        bool keep = 1.f / (1.f + std::exp(-sc[j])) > keep_thr;
        if (have_tok) keep = keep || tok[s][j] <= thr;
        if (keep) kidx.push_back(j);
      }
      const int nn = static_cast<int>(kidx.size());
      if (nn) {
        DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->idx, kidx.data(), nn * sizeof(int), cudaMemcpyHostToDevice, ss));
        gx_gather_kernel<<<nn, 128, 0, ss>>>(g->cat[s][cur[s]], g->cat[s][1 - cur[s]], 2 * d, d, g->enc[s][cur[s]], g->enc[s][1 - cur[s]], hd,
                                              NP, g->idx, nn);
        DIMB_LAUNCH_CHECK(ctx);
        DIMB_CUDA_OK(ctx, cudaStreamSynchronize(ss));
      }
      std::vector<int> ni(nn);
      for (int j = 0; j < nn; ++j) ni[j] = ind[s][kidx[j]];
      ind[s].swap(ni);
      if (have_tok) {
        std::vector<float> nt(nn);
        for (int j = 0; j < nn; ++j) nt[j] = tok[s][kidx[j]];
        tok[s].swap(nt);
      }
      cur[s] = 1 - cur[s];
      n[s] = nn;
    }
  }
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(g->sst[0]));  // join the two side streams: the assignment below runs on the default stream
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(g->sst[1]));
  *stop_layer = std::min(i, L - 1) + 1;
  if (n[0] == 0 || n[1] == 0) return DIMB_OK;
  const int li = std::min(i, L - 1);
  // ---- assignment (lightglue.py:246-275) and filter_matches (:281-297)
  const float inv = 1.f / std::pow(static_cast<float>(d), 0.25f);
  for (int s = 0; s < 2; ++s) {
    DIMB_TRY(linear(g, st, g->cat[s][cur[s]], 2 * d, g->final_proj[li], g->md[s], d, n[s], inv));
    gx_rowdot_kernel<<<ceil_div(n[s] * 32, 256), 256, 0, st>>>(g->cat[s][cur[s]], 2 * d, n[s], d, g->matchab[li].w, g->matchab[li].b, g->zt[s]);
    DIMB_LAUNCH_CHECK(ctx);
  }
  {
    dim3 grid(ceil_div(n[1], 64), ceil_div(n[0], 64));
    gx_linear_kernel<<<grid, 256, 0, st>>>(g->md[0], d, g->md[1], d, nullptr, g->sim, NP, n[0], n[1], d, 1.f, nullptr, 0, 0);
    DIMB_LAUNCH_CHECK(ctx);
  }
  gx_lse_kernel<<<ceil_div(n[0] * 32, 256), 256, 0, st>>>(g->sim, NP, n[0], n[1], 0, g->rlse);
  DIMB_LAUNCH_CHECK(ctx);
  gx_lse_kernel<<<ceil_div(n[1] * 32, 256), 256, 0, st>>>(g->sim, NP, n[0], n[1], 1, g->clse);
  DIMB_LAUNCH_CHECK(ctx);
  gx_argmax_kernel<<<ceil_div(n[0] * 32, 256), 256, 0, st>>>(g->sim, NP, n[0], n[1], g->rlse, g->clse, g->zt[0], g->zt[1], 0, g->best0, g->arg0);
  DIMB_LAUNCH_CHECK(ctx);
  gx_argmax_kernel<<<ceil_div(n[1] * 32, 256), 256, 0, st>>>(g->sim, NP, n[0], n[1], g->rlse, g->clse, g->zt[0], g->zt[1], 1, g->best1, g->arg1);
  DIMB_LAUNCH_CHECK(ctx);
  std::vector<float> b0(n[0]);
  std::vector<int> a0(n[0]), a1(n[1]);
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(b0.data(), g->best0, n[0] * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(a0.data(), g->arg0, n[0] * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(a1.data(), g->arg1, n[1] * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  const int cnt = lgx_filter(n[0], n[1], b0.data(), a0.data(), a1.data(), ind[0].data(), ind[1].data(),
                             static_cast<float>(cf.filter_threshold), matches, mscores, cap);
  *n_matches = cnt;
  if (cnt > cap) {
    dimb_set_error(ctx, "dimb_lg_match: more matches than cap");
    return DIMB_ERR_CAPACITY;
  }
  return DIMB_OK;
}

int lgx_match(dimb_lgx* g, int P, const dimb_feats* f0, const dimb_feats* f1, int64_t* matches, float* mscores, int* n_matches,
              int* stop_layer, int cap) {
  dimb_ctx* ctx = g->ctx;
  OwnerScope own(ctx, &g->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  for (int p = 0; p < P; ++p)
    DIMB_TRY(lgx_match_pair(g, f0[p], f1[p], matches + static_cast<size_t>(p) * cap * 2, mscores + static_cast<size_t>(p) * cap, n_matches + p,
                            stop_layer + p, cap));
  return DIMB_OK;
}

// ==================================================================== batched device path (lgx_match_dev)
namespace {

// glibc's expf (sysdeps/ieee754/flt-32/e_expf.c, the FMA build x86-64 CPUs with FMA run): exp(x) = 2^(k/32) * 2^(r/32) with
// k = round(x * 32 / ln 2), 2^(k/32) from a 32-entry table and 2^(r/32) a cubic, all in double.  The host path calls std::exp(float);
// this reproduces it bit for bit (checked against glibc 2.39 over every float with |x| < 87), which plain (float)exp((double)x)
// does not (it is correctly rounded, glibc is not quite: 0.502 ulp).
__constant__ unsigned long long kExp2fTab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, 0x3fef72b83c7d517bull, 0x3fef54873168b9aaull,
    0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, 0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, 0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull,
    0x3feea11473eb0187ull, 0x3feea589994cce13ull, 0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, 0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full,
    0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

__device__ __forceinline__ float glibc_expf(float x) {
  if (x != x) return x + x;
  if (x > 0x1.62e42ep6f) return INFINITY;
  if (x < -0x1.9fe368p6f) return 0.f;
  const double inv_ln2_n = 0x1.71547652b82fep+0 * 32, shift = 0x1.8p+52;
  const double c0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, c1 = 0x1.ebfce50fac4f3p-3 / 32 / 32, c2 = 0x1.62e42ff0c52d6p-1 / 32;
  const double xd = static_cast<double>(x);
  double kd = __fma_rn(inv_ln2_n, xd, shift);
  const unsigned long long ki = static_cast<unsigned long long>(__double_as_longlong(kd));
  kd = __dsub_rn(kd, shift);
  const double r = __fma_rn(inv_ln2_n, xd, -kd);
  const unsigned long long t = kExp2fTab[ki % 32] + (ki << 47);
  const double s = __longlong_as_double(static_cast<long long>(t));
  const double z = __fma_rn(c0, r, c1), r2 = __dmul_rn(r, r);
  double y = __fma_rn(c2, r, 1.0);
  y = __fma_rn(z, r2, y);
  return __double2float_rn(__dmul_rn(y, s));
}
// the host's 1.f / (1.f + std::exp(-z))
__device__ __forceinline__ float host_sigmoid(float z) { return __fdiv_rn(1.f, __fadd_rn(1.f, glibc_expf(-z))); }

struct SideInX {  // one side's dimb_feats_dev as the kernels read it
  const void* kpts;
  const void* desc;
  const int* n;
  int n_cap, layout, ld;
  float size0, size1;
  int round_fp16, f16;
  const int* size_dev;
  const float* size_f32;
};

__device__ __forceinline__ float feat_at(const void* p, size_t i, int f16, int r16) {
  const float v = f16 ? __half2float(static_cast<const __half*>(p)[i]) : static_cast<const float*>(p)[i];
  return r16 ? __half2float(__float2half_rn(v)) : v;
}
__device__ __forceinline__ int side_rows(const SideInX& si, int NP) { return min(min(*si.n, si.n_cap), NP); }
// rows a layer kernel works on: none once the side's pair has stopped
__device__ __forceinline__ int live_rows(const int* nact, const int* stopped, int side) { return stopped[side >> 1] ? 0 : nact[side]; }

// grid (ceil(NP / 32), S), block (32, 8): descriptors -> x rows [S][NP][ldx] (fp32, transposed from (D,n)), keypoints -> kp [S][NP][2],
// identity original indices, live counts; a pair with an empty side is stopped at once (stop 1, no matches: lightglue.py:518-538)
__global__ void lgx_prep_kernel(const SideInX* __restrict__ in, int din, int NP, float* __restrict__ x, int ldx, float* __restrict__ kp,
                                int* __restrict__ ind, int* __restrict__ nact, int* __restrict__ n_orig, int* __restrict__ stopped) {
  const int side = blockIdx.y, t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const SideInX si = in[side];
  const int n = side_rows(si, NP);
  if (blockIdx.x == 0 && tx == 0 && ty == 0) {
    nact[side] = n;
    n_orig[side] = n;
    if ((side & 1) == 0) stopped[side >> 1] = (n == 0 || side_rows(in[side + 1], NP) == 0) ? 1 : 0;
  }
  if (t0 >= n) return;
  __shared__ float tile[32][33];
  for (int c0 = 0; c0 < din; c0 += 32) {
    for (int k = ty; k < 32; k += 8) {
      if (si.layout == 0) {  // desc[c][tok], coalesced over tok
        const int c = c0 + k, tok = t0 + tx;
        tile[k][tx] = (tok < n && c < din) ? feat_at(si.desc, static_cast<size_t>(c) * si.ld + tok, si.f16, si.round_fp16) : 0.f;
      } else {  // desc[tok][c], coalesced over c
        const int tok = t0 + k, c = c0 + tx;
        tile[tx][k] = (tok < n && c < din) ? feat_at(si.desc, static_cast<size_t>(tok) * si.ld + c, si.f16, si.round_fp16) : 0.f;
      }
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {
      const int tok = t0 + k, c = c0 + tx;
      if (tok < n && c < din) x[(static_cast<size_t>(side) * NP + tok) * ldx + c] = tile[tx][k];
    }
    __syncthreads();
  }
  for (int k = ty; k < 32; k += 8) {
    const int tok = t0 + k;
    if (tok >= n || tx >= 2) continue;
    const size_t row = static_cast<size_t>(side) * NP + tok;
    kp[row * 2 + tx] = feat_at(si.kpts, 2 * static_cast<size_t>(tok) + tx, si.f16, si.round_fp16);
    if (tx == 0) ind[row] = tok;
  }
}

// block (1024) per side: the normalisation size (given, or the keypoints' own extent (1 + max) - min as lgx_match_pair computes it
// on the host) and the positional encoding of every live row
__global__ void __launch_bounds__(1024) lgx_posenc_kernel(const SideInX* __restrict__ in, const float* __restrict__ kp, const int* __restrict__ nact,
                                                          int NP, const float* __restrict__ Wr, int hd, float* __restrict__ enc) {
  const int side = blockIdx.x, n = nact[side];
  if (n == 0) return;
  const SideInX si = in[side];
  const float* k = kp + static_cast<size_t>(side) * NP * 2;
  float s0 = si.size0, s1 = si.size1;
  if (si.size_f32) {
    s0 = si.size_f32[0], s1 = si.size_f32[1];
  } else if (si.size_dev) {
    s0 = static_cast<float>(si.size_dev[0]), s1 = static_cast<float>(si.size_dev[1]);
  } else if (s0 == 0.f && s1 == 0.f) {
    __shared__ float red[4][32];
    float v[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};  // min x, min y, max x, max y
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      v[0] = fminf(v[0], k[2 * i]), v[1] = fminf(v[1], k[2 * i + 1]);
      v[2] = fmaxf(v[2], k[2 * i]), v[3] = fmaxf(v[3], k[2 * i + 1]);
    }
#pragma unroll
    for (int of = 16; of; of >>= 1)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float o = __shfl_xor_sync(0xffffffffu, v[j], of);
        v[j] = j < 2 ? fminf(v[j], o) : fmaxf(v[j], o);
      }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0)
      for (int j = 0; j < 4; ++j) red[j][w] = v[j];
    __syncthreads();
    for (int j = 0; j < 4; ++j) {
      float r = red[j][0];
      for (int q = 1; q < nw; ++q) r = j < 2 ? fminf(r, red[j][q]) : fmaxf(r, red[j][q]);
      v[j] = r;
    }
    s0 = __fsub_rn(__fadd_rn(1.f, v[2]), v[0]), s1 = __fsub_rn(__fadd_rn(1.f, v[3]), v[1]);
  }
  const int nf = hd / 2;
  float* e = enc + static_cast<size_t>(side) * 2 * NP * hd;
  for (int t = threadIdx.x; t < n * nf; t += blockDim.x) gx_posenc_one(k, t / nf, t % nf, s0, s1, Wr, hd, e, NP);
}

// C rows of every side = A rows . W^T (+ bias, * scale, + resid); grid (ceil(N / 64), ceil(NP / 64), S).  gate: only the live rows of
// running pairs, else all nact rows.  wtab / btab (per layer) + layer (per pair): the weights of the layer each pair ended at.
__global__ void __launch_bounds__(256) lgx_linear_kernel(const float* __restrict__ A, int lda, size_t sA, const float* __restrict__ W,
                                                         const float* __restrict__ bias, float* __restrict__ C, int ldc, size_t sC, int N, int K,
                                                         float scale, const float* __restrict__ resid, const int* __restrict__ nact,
                                                         const int* __restrict__ stopped, int gate, const float* const* __restrict__ wtab,
                                                         const float* const* __restrict__ btab, const int* __restrict__ layer) {
  const int side = blockIdx.z, m0 = blockIdx.y * 64;
  const int M = gate ? live_rows(nact, stopped, side) : nact[side];
  if (m0 >= M) return;
  if (wtab) W = wtab[layer[side >> 1]], bias = btab[layer[side >> 1]];
  gx_linear_tile(A + side * sA, lda, W, K, bias, C + side * sC, ldc, M, N, K, scale, resid ? resid + side * sC : nullptr, ldc, 0, m0);
}

// z[side][row] = x[side][row] . w + b over the rows of every side; warp per row (wtab / btab / layer as lgx_linear_kernel)
__global__ void lgx_rowdot_kernel(const float* __restrict__ x, int ldx, int n, int NP, const float* __restrict__ w, const float* __restrict__ b,
                                  float* __restrict__ z, const int* __restrict__ nact, const int* __restrict__ stopped, int gate,
                                  const float* const* __restrict__ wtab, const float* const* __restrict__ btab, const int* __restrict__ layer,
                                  int S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int side = row / NP, j = row - side * NP;
  if (side >= S || j >= (gate ? live_rows(nact, stopped, side) : nact[side])) return;
  if (wtab) w = wtab[layer[side >> 1]], b = btab[layer[side >> 1]];
  gx_rowdot_row(x + static_cast<size_t>(side) * NP * ldx, ldx, j, lane, n, w, b, z + static_cast<size_t>(side) * NP);
}

// grid (NP, S), block max(32, d / 2)
__global__ void lgx_qkv_rotary_kernel(const float* __restrict__ qkv, int d, int hd, const float* __restrict__ enc, int NP, float* __restrict__ q,
                                      float* __restrict__ k, float* __restrict__ v, const int* __restrict__ nact, const int* __restrict__ stopped) {
  const int side = blockIdx.y, i = blockIdx.x, c = threadIdx.x * 2;
  if (i >= live_rows(nact, stopped, side) || c >= d) return;
  const size_t o = static_cast<size_t>(side) * NP * d;
  gx_qkv_rotary_one(qkv + 3 * o, i, c, d, hd, enc + static_cast<size_t>(side) * 2 * NP * hd, NP, q + o, k + o, v + o);
}

// grid (ceil(NP / 8), h, S): side s attends to its own keys (self) or to those of its partner s ^ 1 (cross)
template <int HDP>
__global__ void __launch_bounds__(256) lgx_attention_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                            int NP, int d, int hd, int cross, float* __restrict__ out, const int* __restrict__ nact,
                                                            const int* __restrict__ stopped) {
  const int side = blockIdx.z, ks = cross ? side ^ 1 : side;
  const int nq = live_rows(nact, stopped, side);
  if (static_cast<int>(blockIdx.x) * 8 >= nq) return;
  const size_t so = static_cast<size_t>(side) * NP * d, ko = static_cast<size_t>(ks) * NP * d;
  gx_attention_block<HDP>(q + so, k + ko, v + ko, nq, nact[ks], d, hd, out + so, d, blockIdx.x, blockIdx.y);
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

// grid (NPp / 128, h, S): attn_hd128's kernel with the side's rows of the all-sides operand maps
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

__global__ void lgx_ln_gelu_kernel(const float* __restrict__ x, int n, int NP, const float* __restrict__ g, const float* __restrict__ b,
                                   float* __restrict__ y, const int* __restrict__ nact, const int* __restrict__ stopped, int S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int side = row / NP, j = row - side * NP;
  if (side >= S || j >= live_rows(nact, stopped, side)) return;
  gx_ln_gelu_row(x, row, lane, n, g, b, y);
}

// block (1024) per running pair, after layer i < L - 1: token confidences, the stop test (lightglue.py:593-604), and per side the
// pruning mask (:586-591) compacted in row order into idx (ballot + block prefix; identity when the side is not pruned).  A pair that
// stops keeps stopped = i + 1; one that prunes a side to nothing stops as lgx_match_pair's next layer would, at min(i + 1, L - 1) + 1.
__global__ void __launch_bounds__(1024) lgx_decide_kernel(int i, int L, int NP, const float* __restrict__ ztok, const float* __restrict__ zmat,
                                                          const int* __restrict__ nact, int* __restrict__ nnext, const int* __restrict__ n_orig,
                                                          int* __restrict__ stopped, int* __restrict__ idx, float thr, float depth_conf,
                                                          float keep_thr, int do_stop, int do_prune, int prune_min) {
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (stopped[p]) return;
  __shared__ int below, wsum[32], total;
  if (do_stop) {
    if (tid == 0) below = 0;
    __syncthreads();
    int cnt = 0;
    for (int sd = 0; sd < 2; ++sd) {
      const int s = 2 * p + sd;
      for (int j = tid; j < nact[s]; j += blockDim.x) cnt += host_sigmoid(ztok[static_cast<size_t>(s) * NP + j]) < thr;
    }
    atomicAdd(&below, cnt);
    __syncthreads();
    const float ratio = __fsub_rn(1.0f, __fdiv_rn(static_cast<float>(below), static_cast<float>(n_orig[2 * p] + n_orig[2 * p + 1])));
    if (ratio > depth_conf) {
      if (tid == 0) stopped[p] = i + 1;
      return;
    }
  }
  int empty = 0;
  for (int sd = 0; sd < 2; ++sd) {
    const int s = 2 * p + sd, n = nact[s];
    const size_t o = static_cast<size_t>(s) * NP;
    const bool prune = do_prune && n > prune_min;
    int base = 0;
    for (int j0 = 0; j0 < n; j0 += blockDim.x) {
      const int j = j0 + tid;
      bool keep = j < n;
      if (keep && prune) {
        keep = host_sigmoid(zmat[o + j]) > keep_thr;
        if (do_stop) keep = keep || host_sigmoid(ztok[o + j]) <= thr;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) wsum[w] = __popc(bal);
      __syncthreads();
      if (w == 0) {
        const int nw = blockDim.x >> 5;
        int v = lane < nw ? wsum[lane] : 0, incl = v;
#pragma unroll
        for (int of = 1; of < 32; of <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, of);
          if (lane >= of) incl += t;
        }
        if (lane < nw) wsum[lane] = incl - v;
        if (lane == 31) total = incl;
      }
      __syncthreads();
      if (keep) idx[o + base + wsum[w] + __popc(bal & ((1u << lane) - 1u))] = j;
      base += total;
      __syncthreads();
    }
    if (tid == 0) nnext[s] = base;
    empty |= base == 0;
  }
  if (tid == 0 && empty) stopped[p] = min(i + 1, L - 1) + 1;
}

// grid (NP, S), block 128: the rows kept by lgx_decide_kernel into the other ping-pong buffer (state x, both encoding halves, original
// index), for the pairs still running after layer i and those that have just pruned a side to nothing
__global__ void lgx_gather_kernel(int i, const int* __restrict__ stopped, const int* __restrict__ nnext, const int* __restrict__ idx, int NP,
                                  int d, int hd, const float* __restrict__ xs, float* __restrict__ xd, const float* __restrict__ es,
                                  float* __restrict__ ed, const int* __restrict__ is, int* __restrict__ id) {
  const int side = blockIdx.y, j = blockIdx.x, st = stopped[side >> 1];
  if ((st != 0 && st <= i + 1) || j >= nnext[side]) return;
  const size_t base = static_cast<size_t>(side) * NP, src = base + idx[base + j], dst = base + j;
  for (int c = threadIdx.x; c < d; c += blockDim.x) xd[dst * 2 * d + c] = xs[src * 2 * d + c];
  const size_t eb = static_cast<size_t>(side) * 2 * NP * hd;
  const size_t es0 = eb + (src - base) * hd, ed0 = eb + static_cast<size_t>(j) * hd, half = static_cast<size_t>(NP) * hd;
  for (int c = threadIdx.x; c < hd; c += blockDim.x) {
    ed[ed0 + c] = es[es0 + c];
    ed[ed0 + half + c] = es[es0 + half + c];
  }
  if (threadIdx.x == 0) id[dst] = is[src];
}

// thread per pair: the layer a pair ended at (its stop layer, or the last) and the ping-pong buffer holding its state
__global__ void lgx_final_select_kernel(const int* __restrict__ stopped, const int* __restrict__ nact0, const int* __restrict__ nact1,
                                        int* __restrict__ nf, int* __restrict__ layer, int* __restrict__ parity, int P, int L, int adaptive) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int st = stopped[p];
  const int par = adaptive ? ((st ? st - 1 : L - 1) & 1) : 0;
  parity[p] = par;
  layer[p] = st ? st - 1 : L - 1;
  const int* na = par ? nact1 : nact0;
  nf[2 * p] = na[2 * p];
  nf[2 * p + 1] = na[2 * p + 1];
}

// grid (NP, S), block 128: the final state x and original indices of every side into fixed buffers
__global__ void lgx_final_gather_kernel(const int* __restrict__ nf, const int* __restrict__ parity, int NP, int d, const float* __restrict__ x0,
                                        const float* __restrict__ x1, const int* __restrict__ i0, const int* __restrict__ i1, float* __restrict__ xf,
                                        int* __restrict__ indf) {
  const int side = blockIdx.y, j = blockIdx.x;
  if (j >= nf[side]) return;
  const int par = parity[side >> 1];
  const size_t row = static_cast<size_t>(side) * NP + j;
  const float* x = (par ? x1 : x0) + row * 2 * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) xf[row * d + c] = x[c];
  if (threadIdx.x == 0) indf[row] = (par ? i1 : i0)[row];
}

// grid (ceil(NP / 64), ceil(NP / 64), P): sim of pair p [n0][n1] (row stride NP) = md0 . md1^T
__global__ void __launch_bounds__(256) lgx_sim_kernel(const float* __restrict__ md, int d, int NP, const int* __restrict__ nf, float* __restrict__ sim) {
  const int p = blockIdx.z, n0 = nf[2 * p], n1 = nf[2 * p + 1], m0 = blockIdx.y * 64;
  if (m0 >= n0 || static_cast<int>(blockIdx.x) * 64 >= n1) return;
  const size_t o = static_cast<size_t>(2 * p) * NP * d;
  gx_linear_tile(md + o, d, md + o + static_cast<size_t>(NP) * d, d, nullptr, sim + static_cast<size_t>(p) * NP * NP, NP, n0, n1, d, 1.f, nullptr,
                 0, 0, m0);
}

// warp per (pair, row or column): log-sum-exp (what = 0) or maximum / first argmax of the log assignment (what = 1), dir 0 rows, 1 columns
__global__ void lgx_assign_kernel(int what, int dir, const float* __restrict__ sim, int NP, const int* __restrict__ nf,
                                  float* __restrict__ rlse, float* __restrict__ clse, const float* __restrict__ z, float* __restrict__ best,
                                  int* __restrict__ arg, int P) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int p = gw / NP, i = gw - p * NP;
  if (p >= P) return;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  if (m == 0 || n == 0 || i >= (dir == 0 ? m : n)) return;
  const float* s = sim + static_cast<size_t>(p) * NP * NP;
  const size_t o = static_cast<size_t>(p) * NP;
  if (what == 0) {
    gx_lse_one(s, NP, m, n, dir, (dir == 0 ? rlse : clse) + o, i, lane);
  } else {
    gx_argmax_one(s, NP, m, n, rlse + o, clse + o, z + 2 * o, z + 2 * o + NP, dir, best + 2 * o + (dir ? NP : 0), arg + 2 * o + (dir ? NP : 0),
                  i, lane);
  }
}

// block (1024) per pair: lgx_filter on the device - mutual argmax, exp(max) > th, matches in row order (first cap written, full count
// reported) - and the stop layer (1 for a pair with an empty side)
__global__ void __launch_bounds__(1024) lgx_filter_kernel(const int* __restrict__ nf, const int* __restrict__ stopped, int L, int NP,
                                                          const float* __restrict__ best, const int* __restrict__ arg, const int* __restrict__ indf,
                                                          float th, long long* __restrict__ matches, float* __restrict__ mscores,
                                                          int* __restrict__ n_matches, int* __restrict__ stop_layer, int cap) {
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int st = stopped[p], n0 = nf[2 * p], n1 = nf[2 * p + 1];
  const bool run = n0 > 0 && n1 > 0;
  __shared__ int wsum[32], total;
  const size_t o = static_cast<size_t>(2 * p) * NP;
  const float* b0 = best + o;
  const int *a0 = arg + o, *a1 = arg + o + NP;
  int base = 0;
  for (int r0 = 0; run && r0 < n0; r0 += blockDim.x) {
    const int r = r0 + tid;
    int c = -1;
    float e = 0.f;
    bool ok = false;
    if (r < n0) {
      c = a0[r];
      if (c >= 0 && c < n1 && a1[c] == r) {
        e = glibc_expf(b0[r]);
        ok = e > th;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    if (w == 0) {
      const int nw = blockDim.x >> 5;
      int v = lane < nw ? wsum[lane] : 0, incl = v;
#pragma unroll
      for (int of = 1; of < 32; of <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, of);
        if (lane >= of) incl += t;
      }
      if (lane < nw) wsum[lane] = incl - v;
      if (lane == 31) total = incl;
    }
    __syncthreads();
    const int pos = base + wsum[w] + __popc(bal & ((1u << lane) - 1u));
    if (ok && pos < cap) {
      const size_t q = static_cast<size_t>(p) * cap + pos;
      matches[2 * q] = indf[o + r];
      matches[2 * q + 1] = indf[o + NP + c];
      mscores[q] = e;
    }
    base += total;
    __syncthreads();
  }
  if (tid == 0) {
    n_matches[p] = base;
    stop_layer[p] = st ? st : L;
  }
}

int grow_batch(dimb_lgx* g) {
  dimb_ctx* ctx = g->ctx;
  auto& b = g->b;
  const size_t P = g->conf.max_pairs, S = 2 * P, NP = g->NP, d = g->d, hd = g->hd, R = S * NP;
  for (int k = 0; k < 2; ++k) {
    DIMB_TRY(dimb_alloc_t(ctx, &b.cat[k], R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &b.enc[k], R * 2 * hd));
    DIMB_TRY(dimb_alloc_t(ctx, &b.ind[k], R));
    DIMB_TRY(dimb_alloc_t(ctx, &b.nact[k], S));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &b.kp, R * 2));
  DIMB_TRY(dimb_alloc_t(ctx, &b.qkv, R * 3 * d));
  for (float** p : {&b.q, &b.k, &b.v, &b.xf, &b.md}) DIMB_TRY(dimb_alloc_t(ctx, p, R * d));
  DIMB_TRY(dimb_alloc_t(ctx, &b.hid, R * 2 * d));
  DIMB_TRY(dimb_alloc_t(ctx, &b.hid2, R * std::max<size_t>(2 * d, g->din)));  // also the input-projection operand
  for (float** p : {&b.zt, &b.zm, &b.best0}) DIMB_TRY(dimb_alloc_t(ctx, p, R));
  for (float** p : {&b.rlse, &b.clse}) DIMB_TRY(dimb_alloc_t(ctx, p, P * NP));
  DIMB_TRY(dimb_alloc_t(ctx, &b.sim, P * NP * NP));
  for (int** p : {&b.idx, &b.indf, &b.arg0}) DIMB_TRY(dimb_alloc_t(ctx, p, R));
  for (int** p : {&b.n_orig, &b.nf}) DIMB_TRY(dimb_alloc_t(ctx, p, S));
  for (int** p : {&b.stopped, &b.layer, &b.parity}) DIMB_TRY(dimb_alloc_t(ctx, p, P));
  DIMB_TRY(dimb_alloc(ctx, &b.in, S * sizeof(SideInX)));
  const int L = g->L;
  std::vector<const float*> tab(4 * static_cast<size_t>(L));
  for (int i = 0; i < L; ++i) {
    tab[i] = g->final_proj[i].w, tab[L + i] = g->final_proj[i].b;
    tab[2 * L + i] = g->matchab[i].w, tab[3 * L + i] = g->matchab[i].b;
  }
  DIMB_TRY(dimb_alloc(ctx, reinterpret_cast<void**>(&b.tab), tab.size() * sizeof(float*)));
  DIMB_CUDA_OK(ctx, cudaMemcpy(b.tab, tab.data(), tab.size() * sizeof(float*), cudaMemcpyHostToDevice));
  if (g->tc_attn) {
    const size_t rows = S * g->h * g->NPp, nel = rows * kXHd;
    for (int pl = 0; pl < 2; ++pl) {
      DIMB_TRY(dimb_alloc_t(ctx, &b.qp[pl], nel));
      DIMB_TRY(dimb_alloc_t(ctx, &b.kp16[pl], nel));
      DIMB_TRY(dimb_alloc_t(ctx, &b.vt[pl], nel));
      DIMB_TRY(dimb_tmap_2d(ctx, &b.mQ128[pl], b.qp[pl], rows, kXHd, kXHd, kAttnTile));
      DIMB_TRY(dimb_tmap_2d(ctx, &b.mQ64[pl], b.qp[pl], rows, kXHd, kXHd, kAttnBlk));
      DIMB_TRY(dimb_tmap_2d(ctx, &b.mK64[pl], b.kp16[pl], rows, kXHd, kXHd, kAttnBlk));
      DIMB_TRY(dimb_tmap_2d(ctx, &b.mVt[pl], b.vt[pl], S * g->h * kXHd, g->NPp, g->NPp, kXHd));
    }
  }
  b.ready = true;
  return DIMB_OK;
}

}  // namespace

int lgx_match_dev(dimb_lgx* g, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches, float* d_mscores, int* d_n_matches,
                  int* d_stop_layer, int cap, cudaStream_t st) {
  dimb_ctx* ctx = g->ctx;
  const dimb_lg_conf& cf = g->conf;
  const int d = g->d, hd = g->hd, h = g->h, L = g->L, din = g->din, NP = g->NP, S = 2 * P;
  if (!d_matches || !d_mscores || !d_n_matches || !d_stop_layer || P < 1 || P > cf.max_pairs || cap < 1) return DIMB_ERR_ARG;
  std::vector<SideInX> hin(S);
  for (int s = 0; s < S; ++s) {
    const dimb_feats_dev& f = (s & 1) ? f1[s >> 1] : f0[s >> 1];
    if (f.n_cap < 0 || f.n_cap > NP || !f.n || (f.n_cap > 0 && (!f.keypoints || !f.descriptors)) || (f.desc_layout != 0 && f.desc_layout != 1)) {
      dimb_set_error(ctx, "dimb_lg_match_dev: invalid feature set (n_cap above max_kpts, NULL pointer or unknown layout)");
      return DIMB_ERR_ARG;
    }
    SideInX& o = hin[s];
    o.kpts = f.keypoints, o.desc = f.descriptors, o.n = f.n, o.n_cap = f.n_cap, o.layout = f.desc_layout;
    o.ld = f.desc_ld ? f.desc_ld : (f.desc_layout == 0 ? f.n_cap : din);
    o.size0 = f.size0, o.size1 = f.size1, o.round_fp16 = f.round_fp16, o.f16 = f.f16, o.size_dev = f.size_dev, o.size_f32 = f.size_f32_dev;
  }
  OwnerScope own(ctx, &g->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (!g->b.ready) DIMB_TRY(grow_batch(g));
  auto& b = g->b;
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT, tc = g->tc_attn;
  const int do_stop = cf.depth_confidence > 0, do_prune = cf.width_confidence > 0, adaptive = do_stop || do_prune;
  const size_t sRow2 = static_cast<size_t>(NP) * 2 * d, sRow = static_cast<size_t>(NP) * d;
  const int* const stp = b.stopped;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(b.in, hin.data(), S * sizeof(SideInX), cudaMemcpyHostToDevice, st));
  auto lin = [&](const float* A, int lda, size_t sA, const Lin& l, float* C, int ldc, size_t sC, const int* nact, bool resid) -> int {
    lgx_linear_kernel<<<dim3(ceil_div(l.n, 64), ceil_div(NP, 64), S), 256, 0, st>>>(A, lda, sA, l.w, l.b, C, ldc, sC, l.n, l.k, 1.f,
                                                                                    resid ? C : nullptr, nact, stp, 1, nullptr, nullptr, nullptr);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  const int rows_grid = ceil_div(S * NP * 32, 256);
  {  // ---- inputs, input projection, positional encoding
    ProfScope prof(ctx, st, "lgx.prep");
    const SideInX* in = static_cast<const SideInX*>(b.in);
    float* x = din != d ? b.hid2 : b.cat[0];
    lgx_prep_kernel<<<dim3(ceil_div(NP, 32), S), dim3(32, 8), 0, st>>>(in, din, NP, x, din != d ? din : 2 * d, b.kp, b.ind[0], b.nact[0], b.n_orig,
                                                                         b.stopped);
    DIMB_LAUNCH_CHECK(ctx);
    if (din != d) DIMB_TRY(lin(b.hid2, din, static_cast<size_t>(NP) * din, g->input_proj, b.cat[0], 2 * d, sRow2, b.nact[0], false));
    lgx_posenc_kernel<<<S, 1024, 0, st>>>(in, b.kp, b.nact[0], NP, g->Wr, hd, b.enc[0]);
    DIMB_LAUNCH_CHECK(ctx);
  }
  auto attend = [&](const float* q, const float* k, const float* v, int cross, const int* nact) -> int {
    if (tc) {
      AttnXArgs a;
      a.nq = 0, a.nk = 0, a.NP = g->NPp, a.hd = hd;
      a.scale = 1.f / sqrtf(static_cast<float>(hd));
      a.lazy = ctx->attn_lazy;
      a.out = b.hid, a.ldo = d;
      ProfScope prof(ctx, st, "lgx.attn_tc");
      const dim3 grid(g->NPp / kAttnTile, h, S);
      const CUtensorMap* K = cross ? b.mQ64 : b.mK64;
      if (exact) {
        constexpr int smem = AttnGeom<kXHd, true>::kSmem;
        DIMB_TRY(dimb_func_smem(ctx, lgx_attn_tc_kernel<true>, smem));
        lgx_attn_tc_kernel<true><<<grid, kAttnThreads, smem, st>>>(b.mQ128[0], b.mQ128[1], K[0], K[1], b.mVt[0], b.mVt[1], a, NP, cross, nact, stp);
      } else {
        constexpr int smem = AttnGeom<kXHd, false>::kSmem;
        DIMB_TRY(dimb_func_smem(ctx, lgx_attn_tc_kernel<false>, smem));
        lgx_attn_tc_kernel<false><<<grid, kAttnThreads, smem, st>>>(b.mQ128[0], b.mQ128[0], K[0], K[0], b.mVt[0], b.mVt[0], a, NP, cross, nact, stp);
      }
      DIMB_LAUNCH_CHECK(ctx);
      return DIMB_OK;
    }
    ProfScope prof(ctx, st, "lgx.attn");
    const dim3 grid(ceil_div(NP, 8), h, S);
    if (hd <= 32)
      lgx_attention_kernel<32><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, b.hid, nact, stp);
    else if (hd <= 64)
      lgx_attention_kernel<64><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, b.hid, nact, stp);
    else if (hd <= 96)
      lgx_attention_kernel<96><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, b.hid, nact, stp);
    else
      lgx_attention_kernel<128><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, b.hid, nact, stp);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  auto pack = [&](int what, const float* src, const int* nact) -> int {  // 0 q, 1 k, 2 v
    if (what == 2) {
      lgx_pack_vt_kernel<<<dim3(g->NPp / 32, kXHd / 32, h * S), dim3(32, 8), 0, st>>>(src, d, hd, h, NP, g->NPp, b.vt[0], exact ? b.vt[1] : nullptr,
                                                                                     nact, stp);
    } else {
      __half** dst = what == 0 ? b.qp : b.kp16;
      lgx_pack_rows_kernel<<<dim3(g->NPp, h, S), kXHd, 0, st>>>(src, d, hd, NP, g->NPp, dst[0], exact ? dst[1] : nullptr, nact, stp);
    }
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  auto ffn = [&](float* cat, const Block& bl, const int* nact) -> int {
    DIMB_TRY(lin(cat, 2 * d, sRow2, bl.ffn0, b.hid, 2 * d, sRow2, nact, false));
    lgx_ln_gelu_kernel<<<rows_grid, 256, 0, st>>>(b.hid, 2 * d, NP, bl.ln_g, bl.ln_b, b.hid2, nact, stp, S);
    DIMB_LAUNCH_CHECK(ctx);
    return lin(b.hid2, 2 * d, sRow2, bl.ffn3, cat, 2 * d, sRow2, nact, true);
  };
  for (int i = 0; i < L; ++i) {
    const int cur = adaptive ? (i & 1) : 0, nxt = cur ^ 1;
    float* cat = b.cat[cur];
    const int* nact = b.nact[cur];
    const Block &sb = g->self_[i], &cb = g->cross_[i];
    {
      ProfScope prof(ctx, st, "lgx.self");
      DIMB_TRY(lin(cat, 2 * d, sRow2, sb.qkv, b.qkv, 3 * d, 3 * sRow, nact, false));
      lgx_qkv_rotary_kernel<<<dim3(NP, S), std::max(32, d / 2), 0, st>>>(b.qkv, d, hd, b.enc[cur], NP, b.q, b.k, b.v, nact, stp);
      DIMB_LAUNCH_CHECK(ctx);
      if (tc) {
        DIMB_TRY(pack(0, b.q, nact));
        DIMB_TRY(pack(1, b.k, nact));
        DIMB_TRY(pack(2, b.v, nact));
      }
    }
    DIMB_TRY(attend(b.q, b.k, b.v, 0, nact));
    {
      ProfScope prof(ctx, st, "lgx.self");
      DIMB_TRY(lin(b.hid, d, sRow, sb.out, cat + d, 2 * d, sRow2, nact, false));
      DIMB_TRY(ffn(cat, sb, nact));
    }
    {
      ProfScope prof(ctx, st, "lgx.cross");
      DIMB_TRY(lin(cat, 2 * d, sRow2, cb.to_qk, b.q, d, sRow, nact, false));
      DIMB_TRY(lin(cat, 2 * d, sRow2, cb.to_v, b.v, d, sRow, nact, false));
      if (tc) {
        DIMB_TRY(pack(0, b.q, nact));
        DIMB_TRY(pack(2, b.v, nact));
      }
    }
    DIMB_TRY(attend(b.q, b.q, b.v, 1, nact));
    {
      ProfScope prof(ctx, st, "lgx.cross");
      DIMB_TRY(lin(b.hid, d, sRow, cb.out, cat + d, 2 * d, sRow2, nact, false));
      DIMB_TRY(ffn(cat, cb, nact));
    }
    if (i == L - 1 || !adaptive) continue;  // nothing to decide after the last layer, nor in a fixed-work run
    ProfScope prof(ctx, st, "lgx.tail");
    if (do_stop) {
      lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(cat, 2 * d, d, NP, g->token[i].w, g->token[i].b, b.zt, nact, stp, 1, nullptr, nullptr, nullptr, S);
      DIMB_LAUNCH_CHECK(ctx);
    }
    if (do_prune) {
      lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(cat, 2 * d, d, NP, g->matchab[i].w, g->matchab[i].b, b.zm, nact, stp, 1, nullptr, nullptr, nullptr,
                                                   S);
      DIMB_LAUNCH_CHECK(ctx);
    }
    lgx_decide_kernel<<<P, 1024, 0, st>>>(i, L, NP, b.zt, b.zm, nact, b.nact[nxt], b.n_orig, b.stopped, b.idx, conf_threshold(i, L),
                                          static_cast<float>(cf.depth_confidence), static_cast<float>(1.0 - cf.width_confidence), do_stop, do_prune,
                                          cf.prune_min_kpts);
    DIMB_LAUNCH_CHECK(ctx);
    lgx_gather_kernel<<<dim3(NP, S), 128, 0, st>>>(i, b.stopped, b.nact[nxt], b.idx, NP, d, hd, cat, b.cat[nxt], b.enc[cur], b.enc[nxt], b.ind[cur],
                                                   b.ind[nxt]);
    DIMB_LAUNCH_CHECK(ctx);
  }
  // ---- assignment (lightglue.py:246-275) and filter_matches (:281-297), per pair at the layer it ended at
  ProfScope prof(ctx, st, "lgx.assign");
  lgx_final_select_kernel<<<ceil_div(P, 128), 128, 0, st>>>(b.stopped, b.nact[0], b.nact[1], b.nf, b.layer, b.parity, P, L, adaptive);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_final_gather_kernel<<<dim3(NP, S), 128, 0, st>>>(b.nf, b.parity, NP, d, b.cat[0], b.cat[1], b.ind[0], b.ind[1], b.xf, b.indf);
  DIMB_LAUNCH_CHECK(ctx);
  const float inv = 1.f / std::pow(static_cast<float>(d), 0.25f);
  lgx_linear_kernel<<<dim3(ceil_div(d, 64), ceil_div(NP, 64), S), 256, 0, st>>>(b.xf, d, sRow, nullptr, nullptr, b.md, d, sRow, d, d, inv, nullptr,
                                                                                b.nf, b.stopped, 0, b.tab, b.tab + L, b.layer);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(b.xf, d, d, NP, nullptr, nullptr, b.zt, b.nf, b.stopped, 0, b.tab + 2 * L, b.tab + 3 * L, b.layer, S);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_sim_kernel<<<dim3(ceil_div(NP, 64), ceil_div(NP, 64), P), 256, 0, st>>>(b.md, d, NP, b.nf, b.sim);
  DIMB_LAUNCH_CHECK(ctx);
  const int pair_rows = ceil_div(P * NP * 32, 256);
  for (int what = 0; what < 2; ++what)
    for (int dir = 0; dir < 2; ++dir) {
      lgx_assign_kernel<<<pair_rows, 256, 0, st>>>(what, dir, b.sim, NP, b.nf, b.rlse, b.clse, b.zt, b.best0, b.arg0, P);
      DIMB_LAUNCH_CHECK(ctx);
    }
  lgx_filter_kernel<<<P, 1024, 0, st>>>(b.nf, b.stopped, L, NP, b.best0, b.arg0, b.indf, static_cast<float>(cf.filter_threshold),
                                        reinterpret_cast<long long*>(d_matches), d_mscores, d_n_matches, d_stop_layer, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
