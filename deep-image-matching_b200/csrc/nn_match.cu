// nn_match.cu - brute-force descriptor matcher (dimb_nn_match*), replacing KorniaMatcher._match_pairs
// (reference matchers/kornia_matcher.py:27-54 -> kornia.feature.DescriptorMatcher nn/mnn/snn/smnn).
//
// The reference materialises the full n0 x n1 distance matrix (torch.cdist, 268 MB at 8192^2) and runs
// min / topk over it.  Here the distance tile never leaves the SM: the tensor-core GEMM of gemm.cuh
// produces a 128 x 128 tile of dot products in registers and its epilogue turns it into distances
// (|a|^2 + |b|^2 - 2ab, clamped, sqrt) and a per-row running (best, second best, argbest) over each
// 32-column chunk; a small merge kernel reduces the chunk partials.  The column statistics needed by the
// mutual / symmetric modes are the same kernel with the operands swapped.
//
// One batched engine serves P pairs = 2P sides per call with the keypoint counts on the device (dimb_nn_match_batch_dev);
// dimb_nn_match_dev and dimb_nn_match are its P = 1 callers.  Side s owns rows [s * NPp, (s + 1) * NPp) of the operand buffers
// (NPp = the largest n_cap rounded up to 128), pair p is sides 2p and 2p + 1:
//   prep   : one launch over all sides: fp16 hi (/ lo) planes, squared norms (zero on padding rows) and the live count of every side
//            (0 for both sides of a pair kornia leaves empty, so that no later kernel works on it)
//   top2   : one persistent GEMM over all pairs per direction (rows of sides 2p, then of sides 2p + 1 for mnn / smnn); tiles past a
//            side's count, and pairs with an empty partner, are skipped on the device.  The host-count callers (P = 1) launch exactly
//            the tiles of their counts with the counts as kernel arguments and a B panel that may stay resident in shared memory
//   merge  : chunk partials -> (best, second, argbest) per live row, one launch per direction (the directions share the partials)
//   select : one CTA per pair, kornia's mode logic and the ordered compaction into [P][cap] tables
#include "nn_kernels.cuh"

extern "C" {

// P pairs on device features with device counts (contract in dimb200.h): validation before any CUDA call, then the engine.
int dimb_nn_match_batch_dev(dimb_ctx* ctx, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int D, int mode, float th,
                            int64_t* d_idx, float* d_dist, int* d_n, int cap, void* stream) {
  if (!ctx || !f0 || !f1 || !d_idx || !d_dist || !d_n || P < 1 || cap < 1 || D < 1 || mode < 0 || mode > 3) {
    if (ctx) dimb_set_error(ctx, "dimb_nn_match_batch_dev: invalid argument (NULL array or output, P >= 1, cap >= 1, D >= 1, mode 0..3)");
    return DIMB_ERR_ARG;
  }
  std::vector<NNSideIn> sides(2 * P);
  int max_cap = 0;
  bool any_f32 = false;
  for (int p = 0; p < P; ++p)
    for (int sd = 0; sd < 2; ++sd) {
      const dimb_feats_dev& f = sd ? f1[p] : f0[p];
      if (!f.descriptors || !f.n || f.n_cap < 0 || f.desc_layout != 0 || f.desc_ld < 0) {
        dimb_set_error(ctx, "dimb_nn_match_batch_dev: pair " + std::to_string(p) + " side " + std::to_string(sd) +
                                ": NULL descriptors / n, n_cap < 0, or desc_layout other than 0 ((D,n) rows)");
        return DIMB_ERR_ARG;
      }
      sides[2 * p + sd] = NNSideIn{f.descriptors, f.n, f.n_cap, f.desc_ld ? f.desc_ld : f.n_cap, f.f16 ? 1 : 0, f.round_fp16 ? 1 : 0};
      max_cap = std::max(max_cap, f.n_cap);
      any_f32 |= !f.f16 && !f.round_fp16;
    }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const bool split = any_f32 && ctx->precision == DIMB_PRECISION_EXACT;
  return nn_run(ctx, static_cast<cudaStream_t>(stream), sides, nn_shape(P, max_cap, nullptr), D, mode, th, split ? 1 : 0,
                reinterpret_cast<long long*>(d_idx), d_dist, d_n, cap);
}

// Device-resident entry: descriptors (D,n) with row pitch ld in HBM (fp32, or fp16 as the device feature store keeps them),
// results in device buffers, asynchronous on `stream`.  fp16 input takes the single-MMA path (the values ARE fp16: exact products).
int dimb_nn_match_dev(dimb_ctx* ctx, const void* d_desc0, int n0, int ld0, const void* d_desc1, int n1, int ld1, int D, int desc_f16,
                      int mode, float th, int64_t* d_idx, float* d_dist, int* d_n, int cap, void* stream) {
  if (!ctx || !d_idx || !d_dist || !d_n || n0 < 0 || n1 < 0 || D < 1 || mode < 0 || mode > 3 || cap < 1) {
    if (ctx) dimb_set_error(ctx, "dimb_nn_match_dev: invalid argument (descriptor dimension >= 1, mode 0..3, cap >= 1)");
    return DIMB_ERR_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (nn_trivially_empty(n0, n1, mode)) {
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(d_n, 0, sizeof(int), st));
    return DIMB_OK;
  }
  if (!d_desc0 || !d_desc1) return DIMB_ERR_ARG;
  const int f16 = desc_f16 ? 1 : 0, hn[2] = {n0, n1};
  const std::vector<NNSideIn> sides = {NNSideIn{d_desc0, nullptr, n0, ld0 ? ld0 : n0, f16, 0},
                                       NNSideIn{d_desc1, nullptr, n1, ld1 ? ld1 : n1, f16, 0}};
  const bool split = !desc_f16 && ctx->precision == DIMB_PRECISION_EXACT;  // fp32 input: no host round trip to learn whether lo == 0
  return nn_run(ctx, st, sides, nn_shape(1, std::max(n0, n1), hn), D, mode, th, split ? 1 : 0, reinterpret_cast<long long*>(d_idx), d_dist,
                d_n, cap);
}

int dimb_nn_match(dimb_ctx* ctx, const float* d0, int n0, const float* d1, int n1, int D, int mode, float th, int64_t* idx, float* dist,
                  int* n, int cap) {
  if (!ctx || !idx || !dist || !n || n0 < 0 || n1 < 0 || D < 1 || mode < 0 || mode > 3 || cap < 1) {
    if (ctx) dimb_set_error(ctx, "dimb_nn_match: invalid argument (descriptor dimension >= 1, mode nn/mnn/snn/smnn, cap >= 1)");
    return DIMB_ERR_ARG;
  }
  *n = 0;
  if (nn_trivially_empty(n0, n1, mode)) return DIMB_OK;
  if (!d0 || !d1) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = 0;
  float *raw0, *raw1, *o_dist;
  long long* o_idx;
  int* o_n;
  DIMB_TRY(dimb_scratch(ctx, 0, static_cast<size_t>(D) * n0 * sizeof(float), reinterpret_cast<void**>(&raw0)));
  DIMB_TRY(dimb_scratch(ctx, 1, static_cast<size_t>(D) * n1 * sizeof(float), reinterpret_cast<void**>(&raw1)));
  DIMB_TRY(dimb_scratch(ctx, 2, static_cast<size_t>(cap) * 2 * sizeof(long long), reinterpret_cast<void**>(&o_idx)));
  DIMB_TRY(dimb_scratch(ctx, 3, static_cast<size_t>(cap) * sizeof(float), reinterpret_cast<void**>(&o_dist)));
  DIMB_TRY(dimb_scratch(ctx, 4, sizeof(int), reinterpret_cast<void**>(&o_n)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(raw0, d0, static_cast<size_t>(D) * n0 * sizeof(float), cudaMemcpyHostToDevice, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(raw1, d1, static_cast<size_t>(D) * n1 * sizeof(float), cudaMemcpyHostToDevice, st));
  const int hn[2] = {n0, n1};
  const std::vector<NNSideIn> sides = {NNSideIn{raw0, nullptr, n0, n0, 0, 0}, NNSideIn{raw1, nullptr, n1, n1, 0, 0}};
  // descriptors read back from features.h5 are exactly fp16: then the lo planes are zero and one MMA has exact products
  const int split = ctx->precision == DIMB_PRECISION_EXACT ? -1 : 0;
  DIMB_TRY(nn_run(ctx, st, sides, nn_shape(1, std::max(n0, n1), hn), D, mode, th, split, o_idx, o_dist, o_n, cap));
  int cnt = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(&cnt, o_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  *n = cnt;
  if (cnt > cap) {
    dimb_set_error(ctx, "dimb_nn_match: more matches than cap");
    return DIMB_ERR_CAPACITY;
  }
  if (cnt > 0) {
    DIMB_CUDA_OK(ctx, cudaMemcpy(idx, o_idx, static_cast<size_t>(cnt) * 2 * sizeof(long long), cudaMemcpyDeviceToHost));
    DIMB_CUDA_OK(ctx, cudaMemcpy(dist, o_dist, static_cast<size_t>(cnt) * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return DIMB_OK;
}

}  // extern "C"
