// lightglue_generic.cu - LightGlue for shapes other than (descriptor_dim 256, 4 heads x 64), i.e. the LighterGlue
// checkpoint the reference ships (thirdparty/accelerated_features/modules/lighterglue.py:12-27: descriptor_dim 96,
// one head, 6 layers, input_dim 64; matcher plugin src/deep_image_matching/matchers/lighterglue.py:78-262).
// Same algorithm as lightglue.cu (thirdparty/LightGlue/lightglue/lightglue.py:24-610) in plain fp32 on the CUDA cores:
// the tensor-core kernels of lightglue.cu are specialised for head dim 64 / model dim 256 (registers and shared-memory budgets of
// the attention kernel), this file trades speed for generality.  Control flow (early stop, pruning) is decided on the host
// from per-token confidences copied back once per layer - exactly the synchronisation points of the reference
// (lightglue.py:499,503).  One pair at a time.
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
