// aliked.cu - ALIKED extraction (dimb_aliked_*), replacing AlikedExtractor._extract
// (reference extractors/aliked.py:45-64) and the LightGlue port of ALIKED it drives
// (thirdparty/LightGlue/lightglue/aliked.py:560-693; DKD :92-244; SDDH :452-558; DeformableConv2d :274-330).
//
// ALIKED-n16 is a small network (677 k parameters, 16..128 channels): its cost in the reference is memory traffic
// and launch overhead, not FLOPs (SURVEY 8a A1).  Everything here is fp32 on the CUDA cores - exact parity with
// the fp32 graph up to summation order - in planar NCHW layout:
//   al_pad_kernel            /255 + replicate pad to a multiple of 32 (InputPadder)
//   al_conv3x3_kernel        3x3 conv + folded eval-mode BatchNorm + SELU / residual (blocks 1-2, score head)
//   al_conv1x1_kernel        laterals, downsample shortcuts, score_head.0
//   al_deform_conv_kernel    torchvision.ops.deform_conv2d semantics (blocks 3-4): offsets from a 3x3 conv, clamped
//   al_avgpool_kernel, al_aggregate_kernel (bilinear x2/x8/x32, align_corners=True, concat), al_normalize_kernel
//   detect.cuh               simple_nms, threshold + border compaction, n_limit / top-k selection (shared with SuperPoint)
//   al_dkd_refine_kernel     soft-argmax (T = 0.1) sub-pixel keypoints, score dispersity, bilinear score
//   al_sddh_*                deformable descriptor head: offsets + sampling kernels, two tensor-core GEMMs (gemm.cuh)
// The kernels, their launch helpers and the host weight transforms live in aliked_kernels.cuh, shared with the self-test library.
#include <algorithm>
#include <memory>
#include <cmath>
#include <cstring>
#include <vector>

#include "aliked_kernels.cuh"
#include "detect.cuh"

struct dimb_aliked {
  std::vector<void*> mem;  // device memory owned by this handle
  dimb_ctx* ctx;
  dimb_aliked_conf conf;
  // weights (device)
  BnConv b1c1, b1c2, b2c1, b2c2, b3c1, b3c2, b4c1, b4c2;  // 3x3 (regular or the regular part of a DCN), BN folded as alpha/beta
  float *b2dw, *b2db, *b3dw, *b3db, *b4dw, *b4db;          // 1x1 downsample shortcuts
  float *o31w, *o31b, *o32w, *o32b, *o41w, *o41b, *o42w, *o42b;  // DCN offset convs (18 channels)
  float *l1, *l2, *l3, *l4;                                // laterals 1x1 -> 32
  float *s0, *s2, *s4, *s6;                                // score head
  float *w0T, *b0, *w2, *b2;                               // SDDH offset convs (w0 transposed to [1152][32])
  __half *sfh, *sfl, *agh, *agl;                           // SDDH sf_conv [128][128] and agg as [128 d][16*128 (p,c)], fp16 hi/lo
  CUtensorMap m_sf[2], m_ag[2];
  float *off = nullptr, *dsc = nullptr;                    // per-keypoint scratch (sel_cap entries)
  __half *fsh = nullptr, *fsl = nullptr, *f2h = nullptr, *f2l = nullptr;
  CUtensorMap m_fs[2], m_f2[2];
  // workspace (max size)
  size_t maxP = 0;
  float *img, *pad, *t1a, *x1, *p2, *t2a, *x2, *sc2, *p3, *off3, *t3a, *x3, *sc3, *p4, *off4, *t4a, *x4, *sc4;
  float *l2o, *l3o, *l4o, *sh0, *sh1, *sh2, *score_pad, *feat, *score, *nms;
  int *cand_idx, *chunk_count, *chunk_off, *cand_count, *sel_idx, *sel_count;
  float *cand_score, *sel_score, *kxy, *disp, *kscore, *o_kpts, *o_desc;
  float* thr_dev = nullptr;
  int sel_cap = 0, out_cap = 0;
  TopkScratch topk;  // grid-wide top-k (keypoint limit > kMaxTopK)
};

namespace {

constexpr int kAlikedNLimit = 20000;  // ALIKED.n_limit_max (aliked.py:585): the cut when max_num_keypoints <= 0

// Keypoints the selection keeps at most: top-k mode's K, or threshold / mean mode's n_limit (aliked.py:585-592)
int aliked_limit(const dimb_aliked_conf& c) { return c.max_num_keypoints > 0 ? c.max_num_keypoints : kAlikedNLimit; }

int up_f32(dimb_ctx* ctx, float** d, const float* src, size_t n) {
  DIMB_TRY(dimb_alloc_t(ctx, d, n, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*d, src, n * sizeof(float), cudaMemcpyHostToDevice));
  return DIMB_OK;
}

// fp32 [n][k] weight -> fp16 hi/lo B operand + tensor maps (box = 128 rows)
int up_split(dimb_ctx* ctx, __half** dh, __half** dl, CUtensorMap (&maps)[2], const float* w, int n, int k) {
  const size_t cnt = static_cast<size_t>(n) * k;
  std::vector<__half> h, l;
  al_split_host(w, cnt, h, l);
  DIMB_TRY(dimb_alloc_t(ctx, dh, cnt, false));
  DIMB_TRY(dimb_alloc_t(ctx, dl, cnt, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*dh, h.data(), cnt * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*dl, l.data(), cnt * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_TRY(dimb_tmap_2d(ctx, &maps[0], *dh, n, k, k, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &maps[1], *dl, n, k, k, 128));
  return DIMB_OK;
}

// conv weight + eval BatchNorm -> w, alpha = invstd*gamma, beta = bias - mean*alpha (ATen batch_norm inference transform)
int make_bnconv(dimb_ctx* ctx, BnConv& c, const float*& p, int cout, int cin, bool dcn_offsets_first, float** offw, float** offb) {
  c.cin = cin;
  c.cout = cout;
  if (dcn_offsets_first) {  // state_dict order: offset_conv.weight, offset_conv.bias, regular_conv.weight
    DIMB_TRY(up_f32(ctx, offw, p, static_cast<size_t>(18) * cin * 9));
    p += static_cast<size_t>(18) * cin * 9;
    DIMB_TRY(up_f32(ctx, offb, p, 18));
    p += 18;
  }
  if (dcn_offsets_first) {  // deformable: regular_conv weights transposed to [Cin][9][Cout] for al_deform_conv_kernel
    const std::vector<float> wt = al_dcn_weight(p, cout, cin);
    DIMB_TRY(up_f32(ctx, &c.w, wt.data(), wt.size()));
  } else {
    DIMB_TRY(up_f32(ctx, &c.w, p, static_cast<size_t>(cout) * cin * 9));
  }
  p += static_cast<size_t>(cout) * cin * 9;
  std::vector<float> al, be;
  al_bn_fold(p, p + cout, p + 2 * cout, p + 3 * cout, cout, al, be);
  p += 4 * cout;
  DIMB_TRY(up_f32(ctx, &c.alpha, al.data(), cout));
  DIMB_TRY(up_f32(ctx, &c.beta, be.data(), cout));
  return DIMB_OK;
}


}  // namespace

extern "C" {

int dimb_aliked_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_aliked_conf* conf, dimb_aliked** out) {
  if (!ctx || !weights || !conf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t need = 678316;  // aliked-n16 / n16rot float parameters (state_dict order, without num_batches_tracked)
  if (n_floats != need) {
    dimb_set_error(ctx, "dimb_aliked_create: weight blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(need) +
                            " (aliked-n16 / aliked-n16rot)");
    return DIMB_ERR_ARG;
  }
  if (conf->nms_radius < 1 || conf->nms_radius > 5 || conf->max_height < 32 || conf->max_width < 32) {
    dimb_set_error(ctx, "dimb_aliked_create: unsupported configuration (nms_radius 1..5, max_height and max_width >= 32)");
    return DIMB_ERR_UNSUPPORTED;
  }
  dimb_aliked* al = new dimb_aliked();
  al->ctx = ctx;
  std::unique_ptr<dimb_aliked, void (*)(dimb_aliked*)> guard(al, dimb_aliked_destroy);  // a failed create releases what it built
  OwnerScope own(ctx, &al->mem);
  al->conf = *conf;
  const float* p = weights;
  DIMB_TRY(make_bnconv(ctx, al->b1c1, p, 16, 3, false, nullptr, nullptr));
  DIMB_TRY(make_bnconv(ctx, al->b1c2, p, 16, 16, false, nullptr, nullptr));
  DIMB_TRY(make_bnconv(ctx, al->b2c1, p, 32, 16, false, nullptr, nullptr));
  DIMB_TRY(make_bnconv(ctx, al->b2c2, p, 32, 32, false, nullptr, nullptr));
  DIMB_TRY(up_f32(ctx, &al->b2dw, p, 32 * 16));
  p += 32 * 16;
  DIMB_TRY(up_f32(ctx, &al->b2db, p, 32));
  p += 32;
  DIMB_TRY(make_bnconv(ctx, al->b3c1, p, 64, 32, true, &al->o31w, &al->o31b));
  DIMB_TRY(make_bnconv(ctx, al->b3c2, p, 64, 64, true, &al->o32w, &al->o32b));
  DIMB_TRY(up_f32(ctx, &al->b3dw, p, 64 * 32));
  p += 64 * 32;
  DIMB_TRY(up_f32(ctx, &al->b3db, p, 64));
  p += 64;
  DIMB_TRY(make_bnconv(ctx, al->b4c1, p, 128, 64, true, &al->o41w, &al->o41b));
  DIMB_TRY(make_bnconv(ctx, al->b4c2, p, 128, 128, true, &al->o42w, &al->o42b));
  DIMB_TRY(up_f32(ctx, &al->b4dw, p, 128 * 64));
  p += 128 * 64;
  DIMB_TRY(up_f32(ctx, &al->b4db, p, 128));
  p += 128;
  DIMB_TRY(up_f32(ctx, &al->l1, p, 32 * 16));
  p += 32 * 16;
  DIMB_TRY(up_f32(ctx, &al->l2, p, 32 * 32));
  p += 32 * 32;
  DIMB_TRY(up_f32(ctx, &al->l3, p, 32 * 64));
  p += 32 * 64;
  DIMB_TRY(up_f32(ctx, &al->l4, p, 32 * 128));
  p += 32 * 128;
  DIMB_TRY(up_f32(ctx, &al->s0, p, 8 * 128));
  p += 8 * 128;
  DIMB_TRY(up_f32(ctx, &al->s2, p, 4 * 8 * 9));
  p += 4 * 8 * 9;
  DIMB_TRY(up_f32(ctx, &al->s4, p, 4 * 4 * 9));
  p += 4 * 4 * 9;
  DIMB_TRY(up_f32(ctx, &al->s6, p, 1 * 4 * 9));
  p += 4 * 9;
  {  // desc_head.agg_weights [p][c][d] -> B operand [d][p*128 + c] (K-major), fp16 hi/lo
    const std::vector<float> t = al_sddh_agg(p);
    DIMB_TRY(up_split(ctx, &al->agh, &al->agl, al->m_ag, t.data(), 128, 2048));
    p += 16 * 128 * 128;
  }
  {  // desc_head.offset_conv.0.weight [32][1152] -> [1152][32]
    const std::vector<float> t = al_sddh_w0T(p);
    DIMB_TRY(up_f32(ctx, &al->w0T, t.data(), t.size()));
    p += 32 * 128 * 9;
  }
  DIMB_TRY(up_f32(ctx, &al->b0, p, 32));
  p += 32;
  DIMB_TRY(up_f32(ctx, &al->w2, p, 32 * 32));
  p += 32 * 32;
  DIMB_TRY(up_f32(ctx, &al->b2, p, 32));
  p += 32;
  DIMB_TRY(up_split(ctx, &al->sfh, &al->sfl, al->m_sf, p, 128, 128));  // desc_head.sf_conv.weight [d][c] is already K-major
  p += 128 * 128;
  if (static_cast<size_t>(p - weights) != need) {
    dimb_set_error(ctx, "dimb_aliked_create: internal weight-layout mismatch");
    return DIMB_ERR_ARG;
  }
  // ---- workspace for the padded maximum size
  const size_t Hp = round_up(conf->max_height, 32), Wp = round_up(conf->max_width, 32), P = Hp * Wp;
  al->maxP = P;
  auto A = [&](float** q, size_t n) -> int { return dimb_alloc_t(ctx, q, n, false); };
  DIMB_TRY(A(&al->img, P * 3));
  DIMB_TRY(A(&al->pad, P * 3));
  DIMB_TRY(A(&al->t1a, P * 16));
  DIMB_TRY(A(&al->x1, P * 16));
  DIMB_TRY(A(&al->p2, P / 4 * 16));
  DIMB_TRY(A(&al->t2a, P / 4 * 32));
  DIMB_TRY(A(&al->x2, P / 4 * 32));
  DIMB_TRY(A(&al->sc2, P / 4 * 32));
  DIMB_TRY(A(&al->p3, P / 64 * 32));
  DIMB_TRY(A(&al->off3, P / 64 * 18));
  DIMB_TRY(A(&al->t3a, P / 64 * 64));
  DIMB_TRY(A(&al->x3, P / 64 * 64));
  DIMB_TRY(A(&al->sc3, P / 64 * 64));
  DIMB_TRY(A(&al->p4, P / 1024 * 64));
  DIMB_TRY(A(&al->off4, P / 1024 * 18));
  DIMB_TRY(A(&al->t4a, P / 1024 * 128));
  DIMB_TRY(A(&al->x4, P / 1024 * 128));
  DIMB_TRY(A(&al->sc4, P / 1024 * 128));
  DIMB_TRY(A(&al->l2o, P / 4 * 32));
  DIMB_TRY(A(&al->l3o, P / 64 * 32));
  DIMB_TRY(A(&al->l4o, P / 1024 * 32));
  DIMB_TRY(A(&al->sh0, P * 8));
  DIMB_TRY(A(&al->sh1, P * 4));
  DIMB_TRY(A(&al->sh2, P * 4));
  DIMB_TRY(A(&al->score_pad, P));
  DIMB_TRY(A(&al->feat, P * 128));
  DIMB_TRY(A(&al->score, P));
  DIMB_TRY(A(&al->nms, P));
  DIMB_TRY(A(&al->cand_score, P));
  DIMB_TRY(dimb_alloc_t(ctx, &al->cand_idx, P));
  const size_t nch = ceil_div(static_cast<int>(P), kChunk);
  DIMB_TRY(dimb_alloc_t(ctx, &al->chunk_count, nch));
  DIMB_TRY(dimb_alloc_t(ctx, &al->chunk_off, nch));
  DIMB_TRY(dimb_alloc_t(ctx, &al->cand_count, 1));
  DIMB_TRY(dimb_alloc_t(ctx, &al->sel_count, 1));
  DIMB_TRY(dimb_alloc_t(ctx, &al->thr_dev, 1));
  if (aliked_limit(*conf) > kMaxTopK) DIMB_TRY(topk_reserve(ctx, al->topk, 1, static_cast<int>(P), aliked_limit(*conf)));
  *out = guard.release();
  return DIMB_OK;
}

void dimb_aliked_destroy(dimb_aliked* al) {
  if (!al) return;
  dimb_release(al->ctx, al->mem);
  delete al;
}

// Device-pointer variant: image fp32 (H,W,channels) 0..255 in device memory; outputs in device memory: kpts [cap][2]
// sub-pixel (x,y), scores [cap] (= score dispersity, reference quirk A.5), desc [128][cap], count [1].  No host
// synchronisation: the caller checks count <= cap (entries beyond cap are not written).
int dimb_aliked_extract_dev(dimb_aliked* al, const float* image, int H, int W, int channels, float* kpts, float* scores, float* desc,
                            int* count, int cap, void* stream) {
  if (!al || !image || !kpts || !scores || !desc || !count || (channels != 1 && channels != 3) || cap < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = al->ctx;
  OwnerScope own(ctx, &al->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const dimb_aliked_conf& cf = al->conf;
  int Hp, Wp, top, left;
  al_input_padder(H, W, Hp, Wp, top, left);
  if (static_cast<size_t>(Hp) * Wp > al->maxP || H < 8 || W < 8) {
    dimb_set_error(ctx, "dimb_aliked_extract: image larger than the workspace given at create time");
    return DIMB_ERR_ARG;
  }
  // top-k mode (detection_threshold <= 0 < max_num_keypoints): the K largest of the border-zeroed NMS map, as torch.topk; otherwise
  // K is the n_limit cut of threshold / mean mode
  const bool topk = cf.detection_threshold <= 0.f && cf.max_num_keypoints > 0;
  const int K = aliked_limit(cf);
  if (topk && static_cast<long long>(K) > static_cast<long long>(H) * W) {
    dimb_set_error(ctx, "dimb_aliked_extract: max_num_keypoints " + std::to_string(K) + " exceeds the " + std::to_string(H * W) +
                            " pixels of the image (top-k mode)");
    return DIMB_ERR_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t P = static_cast<size_t>(Hp) * Wp;
  const int H2 = Hp / 2, W2 = Wp / 2, H8 = Hp / 8, W8 = Wp / 8, H32 = Hp / 32, W32 = Wp / 32;
  {
    ProfScope prof(ctx, st, "al.block1");
    DIMB_TRY(launch_al_pad(ctx, st, image, H, W, channels, al->pad, Hp, Wp, top, left));
    // block1
    DIMB_TRY(conv3(ctx, st, al->pad, 3, Hp, Wp, al->b1c1.w, al->b1c1.alpha, al->b1c1.beta, nullptr, al->t1a, 16, 1));
    DIMB_TRY(conv3(ctx, st, al->t1a, 16, Hp, Wp, al->b1c2.w, al->b1c2.alpha, al->b1c2.beta, nullptr, al->x1, 16, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block2");  // ResBlock, regular convs
    DIMB_TRY(launch_al_avgpool(ctx, st, al->x1, 16, Hp, Wp, 2, al->p2));
    DIMB_TRY(conv3(ctx, st, al->p2, 16, H2, W2, al->b2c1.w, al->b2c1.alpha, al->b2c1.beta, nullptr, al->t2a, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->p2, 16, P / 4, al->b2dw, al->b2db, al->sc2, 32, 0));
    DIMB_TRY(conv3(ctx, st, al->t2a, 32, H2, W2, al->b2c2.w, al->b2c2.alpha, al->b2c2.beta, al->sc2, al->x2, 32, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block3");  // deformable
    DIMB_TRY(launch_al_avgpool(ctx, st, al->x2, 32, H2, W2, 4, al->p3));
    DIMB_TRY(dcn(ctx, st, al->p3, 32, H8, W8, al->o31w, al->o31b, al->off3, al->b3c1, nullptr, al->t3a, 1));
    DIMB_TRY(conv1(ctx, st, al->p3, 32, P / 64, al->b3dw, al->b3db, al->sc3, 64, 0));
    DIMB_TRY(dcn(ctx, st, al->t3a, 64, H8, W8, al->o32w, al->o32b, al->off3, al->b3c2, al->sc3, al->x3, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block4");  // deformable
    DIMB_TRY(launch_al_avgpool(ctx, st, al->x3, 64, H8, W8, 4, al->p4));
    DIMB_TRY(dcn(ctx, st, al->p4, 64, H32, W32, al->o41w, al->o41b, al->off4, al->b4c1, nullptr, al->t4a, 1));
    DIMB_TRY(conv1(ctx, st, al->p4, 64, P / 1024, al->b4dw, al->b4db, al->sc4, 128, 0));
    DIMB_TRY(dcn(ctx, st, al->t4a, 128, H32, W32, al->o42w, al->o42b, al->off4, al->b4c2, al->sc4, al->x4, 1));
  }
  {
    ProfScope prof(ctx, st, "al.aggregate");
    DIMB_TRY(conv1(ctx, st, al->x2, 32, P / 4, al->l2, nullptr, al->l2o, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->x3, 64, P / 64, al->l3, nullptr, al->l3o, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->x4, 128, P / 1024, al->l4, nullptr, al->l4o, 32, 1));
    DIMB_TRY(launch_al_fuse(ctx, st, al->x1, al->l1, al->l2o, al->l3o, al->l4o, al->s0, Hp, Wp, top, left, H, W, al->sh0, al->feat));
  }
  {
    ProfScope prof(ctx, st, "al.score_head");
    DIMB_TRY(conv3(ctx, st, al->sh0, 8, Hp, Wp, al->s2, nullptr, nullptr, nullptr, al->sh1, 4, 1));
    DIMB_TRY(conv3(ctx, st, al->sh1, 4, Hp, Wp, al->s4, nullptr, nullptr, nullptr, al->sh2, 4, 1));
    DIMB_TRY(conv3(ctx, st, al->sh2, 4, Hp, Wp, al->s6, nullptr, nullptr, nullptr, al->score_pad, 1, 2));
    DIMB_TRY(launch_al_crop(ctx, st, al->score_pad, Hp, Wp, top, left, al->score, H, W));
  }
  const int r = cf.nms_radius;
  {
  ProfScope prof(ctx, st, "al.detect");
  DIMB_TRY(launch_nms(ctx, st, al->score, al->nms, 1, H, W, r, kNmsProductionVer));
  const CandBufs cand{al->chunk_count, al->chunk_off, al->cand_count, al->cand_idx, al->cand_score};
  if (topk) {
    // the nonzero pixels of the border-zeroed NMS map; topk_fill_kernel appends zero pixels when there are fewer than K
    DIMB_TRY(launch_candidates(ctx, st, al->nms, cand, 1, H, W, 0.f, r, nullptr, true));
  } else {
    // threshold mode (aliked.py:152-160): nms > detection_threshold; if nothing passes, nms > mean(score_map).  Mean mode
    // (detection_threshold <= 0): nms > mean(score_map).  Decided on the device: count, then al_threshold_kernel fixes the
    // threshold, then count / scan / compact with it.
    const bool mean_mode = cf.detection_threshold <= 0.f;
    if (!mean_mode) DIMB_TRY(launch_candidates(ctx, st, al->nms, cand, 1, H, W, cf.detection_threshold, r, nullptr, false));
    DIMB_TRY(launch_al_threshold(ctx, st, al->score, H * W, mean_mode ? nullptr : al->cand_count, cf.detection_threshold, al->thr_dev));
    DIMB_TRY(launch_candidates(ctx, st, al->nms, cand, 1, H, W, 0.f, r, al->thr_dev, true));
  }
  const int scap = std::max(cap, K);  // the selection writes up to K entries whatever cap is
  if (al->sel_cap < cap) {
    if (al->sel_cap > 0)  // release the smaller per-keypoint buffers of an earlier call
      for (void* old : {static_cast<void*>(al->sel_idx), static_cast<void*>(al->sel_score), static_cast<void*>(al->kxy), static_cast<void*>(al->kscore),
                        static_cast<void*>(al->off), static_cast<void*>(al->dsc), static_cast<void*>(al->fsh), static_cast<void*>(al->fsl),
                        static_cast<void*>(al->f2h), static_cast<void*>(al->f2l)})
        dimb_free(ctx, old);
    DIMB_TRY(dimb_alloc_t(ctx, &al->sel_idx, scap));
    DIMB_TRY(dimb_alloc_t(ctx, &al->sel_score, scap));
    DIMB_TRY(dimb_alloc_t(ctx, &al->kxy, static_cast<size_t>(cap) * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &al->kscore, cap));
    const size_t rows = static_cast<size_t>(round_up(cap, kTileM)) * 16;  // SDDH operands, padded to whole GEMM tiles
    DIMB_TRY(dimb_alloc_t(ctx, &al->off, static_cast<size_t>(cap) * 32));
    DIMB_TRY(dimb_alloc_t(ctx, &al->dsc, static_cast<size_t>(round_up(cap, kTileM)) * 128));
    DIMB_TRY(dimb_alloc_t(ctx, &al->fsh, rows * 128));
    DIMB_TRY(dimb_alloc_t(ctx, &al->fsl, rows * 128));
    DIMB_TRY(dimb_alloc_t(ctx, &al->f2h, rows * 128));
    DIMB_TRY(dimb_alloc_t(ctx, &al->f2l, rows * 128));
    DIMB_TRY(dimb_tmap_2d(ctx, &al->m_fs[0], al->fsh, rows, 128, 128, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &al->m_fs[1], al->fsl, rows, 128, 128, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &al->m_f2[0], al->f2h, rows / 16, 2048, 2048, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &al->m_f2[1], al->f2l, rows / 16, 2048, 2048, kTileM));
    al->sel_cap = cap;
  }
  DIMB_TRY(launch_select(ctx, st, cand, al->sel_idx, al->sel_score, count, 1, H * W, K, scap, &al->topk, topk));
  DIMB_TRY(launch_al_dkd(ctx, st, al->score, H, W, r, al->sel_idx, count, cap, al->kxy, scores, al->kscore));
  }
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  {
  ProfScope prof(ctx, st, "al.sddh_offsets+sample");
  DIMB_TRY(launch_al_sddh_offsets(ctx, st, al->feat, H, W, al->kxy, count, cap, al->w0T, al->b0, al->w2, al->b2, kpts, al->off));
  DIMB_TRY(launch_al_sddh_sample(ctx, st, al->feat, H, W, al->kxy, count, cap, al->off, al->fsh, exact ? al->fsl : nullptr));
  }
  DIMB_TRY(launch_al_sddh_sf_gemm(ctx, st, al->m_fs, al->m_sf, al->f2h, exact ? al->f2l : nullptr, count, cap));
  DIMB_TRY(launch_al_sddh_agg_gemm(ctx, st, al->m_f2, al->m_ag, al->dsc, count, cap));
  ProfScope prof(ctx, st, "al.sddh_norm");
  return launch_al_sddh_norm(ctx, st, al->dsc, count, cap, desc);
}

// Host variant (the plugin's entry): image host fp32 (H,W,channels); outputs host, same layouts as above.
int dimb_aliked_extract(dimb_aliked* al, const float* image, int H, int W, int channels, float* kpts, float* scores, float* desc, int* count,
                        int cap) {
  if (!al || !image || !kpts || !scores || !desc || !count || (channels != 1 && channels != 3) || cap < 1 || H < 1 || W < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = al->ctx;
  OwnerScope own(ctx, &al->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t npx = static_cast<size_t>(H) * W * channels;
  if (npx > al->maxP * 3) {
    dimb_set_error(ctx, "dimb_aliked_extract: image larger than the workspace given at create time");
    return DIMB_ERR_ARG;
  }
  if (al->out_cap < cap) {
    if (al->out_cap > 0)
      for (void* old : {static_cast<void*>(al->disp), static_cast<void*>(al->o_kpts), static_cast<void*>(al->o_desc)}) dimb_free(ctx, old);
    DIMB_TRY(dimb_alloc_t(ctx, &al->disp, cap));
    DIMB_TRY(dimb_alloc_t(ctx, &al->o_kpts, static_cast<size_t>(cap) * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &al->o_desc, static_cast<size_t>(cap) * 128));
    al->out_cap = cap;
  }
  cudaStream_t st = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(al->img, image, npx * sizeof(float), cudaMemcpyHostToDevice, st));
  // descriptors are written with leading dimension cap, so the device buffer is used with exactly this cap
  DIMB_TRY(dimb_aliked_extract_dev(al, al->img, H, W, channels, al->o_kpts, al->disp, al->o_desc, al->sel_count, cap, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(count, al->sel_count, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(kpts, al->o_kpts, static_cast<size_t>(cap) * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(scores, al->disp, static_cast<size_t>(cap) * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(desc, al->o_desc, static_cast<size_t>(cap) * 128 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  if (*count > cap) {
    dimb_set_error(ctx, "dimb_aliked_extract: more keypoints than cap");
    return DIMB_ERR_CAPACITY;
  }
  return DIMB_OK;
}

// debug taps of the last call: 0 = score map [H][W], 1 = feature map [128][H][W]
int dimb_aliked_debug_read(dimb_aliked* al, int which, float* out, size_t n_floats) {
  if (!al || !out) return DIMB_ERR_ARG;
  dimb_ctx* ctx = al->ctx;
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  if (which == 0) {
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, al->score, n_floats * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  // the device map is pixel-major [H][W][128]; the tap keeps the reference's [128][H][W] layout
  if (n_floats % 128) return DIMB_ERR_ARG;
  const size_t px = n_floats / 128;
  std::vector<float> tmp(n_floats);
  DIMB_CUDA_OK(ctx, cudaMemcpy(tmp.data(), al->feat, n_floats * sizeof(float), cudaMemcpyDeviceToHost));
  for (size_t p = 0; p < px; ++p)
    for (int c = 0; c < 128; ++c) out[static_cast<size_t>(c) * px + p] = tmp[p * 128 + c];
  return DIMB_OK;
}

}  // extern "C"
