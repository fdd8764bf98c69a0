// fstore.cu - device-resident feature store (dimb_fstore_*): the features.h5 boundary of the reference kept in HBM.
//
// The reference writes every image's FeaturesDict to features.h5 - every array cast to float16, gzip level 9
// (extractors/extractor_base.py:56-99) - and re-opens and re-reads the file for each image of each pair
// (io/h5.py:45-89 via matchers/matcher_base.py:221-222).  The store keeps exactly the h5 CONTENT - float16 keypoints, scores,
// tile_idx and (D,N) descriptors plus the int image_size - one fixed-size block per image in one contiguous device allocation:
//   * extractors put features without leaving the device (dimb_fstore_put_dev: the float16 cast of the h5 writer happens here),
//   * matchers read them in place (dimb_fstore_feats_dev -> dimb_lg_match_dev / dimb_nn_match_dev, no rounding left to do),
//   * get_features' contract (float32 arrays that are float16-exact, int32 image_size) is served by dimb_fstore_get,
//   * the multi-GPU path all-gathers whole blocks over NCCL (dimb_fstore_block_dev) - SURVEY 8(e),
//   * one bulk copy of the blocks to the host is all a features.h5 writer needs afterwards.
#include <algorithm>
#include <memory>
#include <vector>

#include "fstore.cuh"

namespace {
// float32 features (layouts of dimb_sp_extract_dev / dimb_aliked_extract_dev) -> one float16 block.  grid.x covers cap in 256s,
// grid.y = D + 1: row y < D converts descriptor row y, row D converts keypoints / scores / tile_idx and writes the header.
__global__ void fs_put_kernel(const float* __restrict__ kpts, const float* __restrict__ scores, const float* __restrict__ tile_idx,
                              const float* __restrict__ desc, int ld, const int* __restrict__ count, int n_host, SlotPtrs s, int cap, int D,
                              int H, int W) {
  const int n = min(count ? *count : n_host, cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (y < D) {
    if (i < cap) s.desc[static_cast<size_t>(y) * cap + i] = i < n ? __float2half_rn(desc[static_cast<size_t>(y) * ld + i]) : __half(0.f);
    return;
  }
  if (i == 0) {
    s.hdr[0] = n;
    // image_size goes through float16 like every other array of the group (extractor_base.py:80-86, quirk A.8) and comes back as
    // int32 (io/h5.py:75-77): odd sizes above 2048 px are rounded, exactly as the reference's matcher sees them
    s.hdr[1] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(H), 65504.f))));
    s.hdr[2] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(W), 65504.f))));
    s.hdr[3] = 1;
  }
  if (i >= cap) return;
  const bool live = i < n;
  s.kpts[2 * i] = live ? __float2half_rn(kpts[2 * i]) : __half(0.f);
  s.kpts[2 * i + 1] = live ? __float2half_rn(kpts[2 * i + 1]) : __half(0.f);
  s.scores[i] = live ? __float2half_rn(scores ? scores[i] : 1.f) : __half(0.f);   // absent scores -> ones (extractor_base.py:371-373)
  s.tile[i] = live ? __float2half_rn(tile_idx ? tile_idx[i] : 0.f) : __half(0.f);  // no tiling -> zeros (extractor_base.py:226)
}
}  // namespace

static SlotPtrs slot_ptrs(const dimb_fstore* fs, int slot) { return fs_layout(fs).at(slot); }

extern "C" {

int dimb_fstore_create(dimb_ctx* ctx, int n_slots, int cap, int desc_dim, dimb_fstore** out) {
  if (!ctx || !out || n_slots < 1 || cap < 1 || desc_dim < 1) return DIMB_ERR_ARG;
  *out = nullptr;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  dimb_fstore* fs = new dimb_fstore();
  fs->ctx = ctx;
  std::unique_ptr<dimb_fstore, void (*)(dimb_fstore*)> guard(fs, dimb_fstore_destroy);
  OwnerScope own(ctx, &fs->mem);
  fs->n_slots = n_slots;
  fs->cap = round_up(cap, 8);  // 16-byte aligned rows
  fs->D = desc_dim;
  const size_t c = fs->cap;
  fs->off_kpts = kHdrInts * sizeof(int);
  fs->off_scores = fs->off_kpts + c * 2 * sizeof(__half);
  fs->off_tile = fs->off_scores + c * sizeof(__half);
  fs->off_desc = fs->off_tile + c * sizeof(__half);
  fs->slot_bytes = (fs->off_desc + static_cast<size_t>(desc_dim) * c * sizeof(__half) + 255) / 256 * 256;
  DIMB_TRY(dimb_alloc_t(ctx, &fs->base, fs->slot_bytes * n_slots));
  *out = guard.release();
  return DIMB_OK;
}

void dimb_fstore_destroy(dimb_fstore* fs) {
  if (!fs) return;
  dimb_release(fs->ctx, fs->mem);
  delete fs;
}

int dimb_fstore_put_dev(dimb_fstore* fs, int slot, const float* d_kpts, const float* d_scores, const float* d_tile_idx, const float* d_desc,
                        int desc_ld, const int* d_count, int height, int width, void* stream) {
  if (!fs || slot < 0 || slot >= fs->n_slots || !d_kpts || !d_desc || !d_count) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  fs_put_kernel<<<dim3(ceil_div(fs->cap, 256), fs->D + 1), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      d_kpts, d_scores, d_tile_idx, d_desc, desc_ld ? desc_ld : fs->cap, d_count, 0, slot_ptrs(fs, slot), fs->cap, fs->D, height, width);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_fstore_put(dimb_fstore* fs, int slot, const float* kpts, const float* scores, const float* tile_idx, const float* desc, int n,
                    int height, int width) {
  if (!fs || slot < 0 || slot >= fs->n_slots || n < 0 || (n > 0 && (!kpts || !desc))) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  if (n > fs->cap) {
    dimb_set_error(ctx, "dimb_fstore_put: " + std::to_string(n) + " keypoints exceed the store's capacity " + std::to_string(fs->cap));
    return DIMB_ERR_CAPACITY;
  }
  OwnerScope own(ctx, &fs->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t c = fs->cap;
  if (!fs->st_k) {
    DIMB_TRY(dimb_alloc_t(ctx, &fs->st_k, c * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &fs->st_s, c));
    DIMB_TRY(dimb_alloc_t(ctx, &fs->st_t, c));
    DIMB_TRY(dimb_alloc_t(ctx, &fs->st_d, c * fs->D));
  }
  cudaStream_t st = 0;
  if (n > 0) {
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(fs->st_k, kpts, static_cast<size_t>(n) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
    if (scores) DIMB_CUDA_OK(ctx, cudaMemcpyAsync(fs->st_s, scores, static_cast<size_t>(n) * sizeof(float), cudaMemcpyHostToDevice, st));
    if (tile_idx) DIMB_CUDA_OK(ctx, cudaMemcpyAsync(fs->st_t, tile_idx, static_cast<size_t>(n) * sizeof(float), cudaMemcpyHostToDevice, st));
    DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(fs->st_d, c * sizeof(float), desc, static_cast<size_t>(n) * sizeof(float), static_cast<size_t>(n) * sizeof(float),
                                        fs->D, cudaMemcpyHostToDevice, st));
  }
  fs_put_kernel<<<dim3(ceil_div(fs->cap, 256), fs->D + 1), 256, 0, st>>>(fs->st_k, scores ? fs->st_s : nullptr, tile_idx ? fs->st_t : nullptr,
                                                                         fs->st_d, fs->cap, nullptr, n, slot_ptrs(fs, slot), fs->cap, fs->D,
                                                                         height, width);
  DIMB_LAUNCH_CHECK(ctx);
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  return DIMB_OK;
}

int dimb_fstore_count(dimb_fstore* fs, int slot, int* n, int* image_size) {
  if (!fs || slot < 0 || slot >= fs->n_slots || !n) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  int hdr[kHdrInts];
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  DIMB_CUDA_OK(ctx, cudaMemcpy(hdr, slot_ptrs(fs, slot).hdr, sizeof(hdr), cudaMemcpyDeviceToHost));
  *n = hdr[3] ? hdr[0] : -1;  // -1: nothing stored in this slot
  if (image_size) image_size[0] = hdr[1], image_size[1] = hdr[2];
  return DIMB_OK;
}

int dimb_fstore_get(dimb_fstore* fs, int slot, float* kpts, float* scores, float* tile_idx, float* desc, int* n, int* image_size, int cap) {
  if (!fs || slot < 0 || slot >= fs->n_slots || !n) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  fs->host.resize(fs->slot_bytes);
  DIMB_CUDA_OK(ctx, cudaMemcpy(fs->host.data(), fs->base + static_cast<size_t>(slot) * fs->slot_bytes, fs->slot_bytes, cudaMemcpyDeviceToHost));
  const int* hdr = reinterpret_cast<const int*>(fs->host.data());
  if (!hdr[3]) {
    dimb_set_error(ctx, "dimb_fstore_get: slot " + std::to_string(slot) + " is empty");
    return DIMB_ERR_ARG;
  }
  const int cnt = hdr[0];
  *n = cnt;
  if (image_size) image_size[0] = hdr[1], image_size[1] = hdr[2];
  if (cnt > cap) return DIMB_ERR_CAPACITY;
  const __half* hk = reinterpret_cast<const __half*>(fs->host.data() + fs->off_kpts);
  const __half* hs = reinterpret_cast<const __half*>(fs->host.data() + fs->off_scores);
  const __half* ht = reinterpret_cast<const __half*>(fs->host.data() + fs->off_tile);
  const __half* hd = reinterpret_cast<const __half*>(fs->host.data() + fs->off_desc);
  for (int i = 0; i < cnt; ++i) {
    if (kpts) kpts[2 * i] = __half2float(hk[2 * i]), kpts[2 * i + 1] = __half2float(hk[2 * i + 1]);
    if (scores) scores[i] = __half2float(hs[i]);
    if (tile_idx) tile_idx[i] = __half2float(ht[i]);
  }
  if (desc)  // (D, n) dense, the FeaturesDict layout
    for (int c = 0; c < fs->D; ++c)
      for (int i = 0; i < cnt; ++i) desc[static_cast<size_t>(c) * cnt + i] = __half2float(hd[static_cast<size_t>(c) * fs->cap + i]);
  return DIMB_OK;
}

int dimb_fstore_feats_dev(dimb_fstore* fs, int slot, dimb_feats_dev* out) {
  if (!fs || slot < 0 || slot >= fs->n_slots || !out) return DIMB_ERR_ARG;
  const SlotPtrs s = slot_ptrs(fs, slot);
  *out = dimb_feats_dev{};
  out->keypoints = reinterpret_cast<const float*>(s.kpts);
  out->descriptors = reinterpret_cast<const float*>(s.desc);
  out->n = s.hdr;
  out->n_cap = fs->cap;
  out->desc_layout = 0;
  out->desc_ld = fs->cap;
  out->f16 = 1;
  out->size_dev = s.hdr + 1;  // [H, W] exactly as image_size is stored (quirk A.3)
  return DIMB_OK;
}

int dimb_fstore_sg_feats_dev(dimb_fstore* fs, int slot, dimb_sg_feats_dev* out) {
  if (!fs || slot < 0 || slot >= fs->n_slots || !out) return DIMB_ERR_ARG;
  const SlotPtrs s = slot_ptrs(fs, slot);
  *out = dimb_sg_feats_dev{};
  out->keypoints = s.kpts;
  out->descriptors = s.desc;
  out->scores = s.scores;
  out->n = s.hdr;
  out->n_cap = fs->cap;
  out->desc_ld = fs->cap;
  out->f16 = 1;
  out->size_dev = s.hdr + 1;
  return DIMB_OK;
}

int dimb_fstore_block_dev(dimb_fstore* fs, void** d_base, size_t* slot_bytes, int* n_slots, int* cap) {
  if (!fs) return DIMB_ERR_ARG;
  if (d_base) *d_base = fs->base;
  if (slot_bytes) *slot_bytes = fs->slot_bytes;
  if (n_slots) *n_slots = fs->n_slots;
  if (cap) *cap = fs->cap;
  return DIMB_OK;
}

}  // extern "C"
