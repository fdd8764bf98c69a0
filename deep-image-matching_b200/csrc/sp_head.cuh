// sp_head.cuh - the two SuperPoint head kernels around detection (detect.cuh): the 65-way softmax of the score head with its
// depth-to-space, and the bilinear sampling of the descriptor head at the selected keypoints.
#pragma once
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ softmax over 65 logits + depth-to-space
// one warp per cell; logits [B*h*w][65] fp32 -> scores [B][8h][8w]       (superpoint.py:175-179)
__global__ void sp_softmax_d2s_kernel(const float* __restrict__ logits, float* __restrict__ scores, int B, int h, int w) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * h * w) return;
  const float* L = logits + static_cast<size_t>(warp) * 65;
  const float a = L[lane], b2 = L[lane + 32], c = (lane == 0) ? L[64] : -INFINITY;
  float m = fmaxf(fmaxf(a, b2), c);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float ea = expf(a - m), eb = expf(b2 - m), ec = (lane == 0) ? expf(c - m) : 0.f;
  float s = ea + eb + ec;
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const int b = warp / (h * w), cell = warp - b * h * w, cy = cell / w, cx = cell - cy * w;
  float* out = scores + (static_cast<size_t>(b) * h * 8 + cy * 8) * (w * 8) + cx * 8;
  out[(lane >> 3) * (w * 8) + (lane & 7)] = ea / s;            // channel j = lane     -> (j/8, j%8)
  out[((lane >> 3) + 4) * (w * 8) + (lane & 7)] = eb / s;      // channel j = lane+32
}

// ------------------------------------------------------------------ keypoints + descriptor sampling
// warp per keypoint.  dense: [B][h*w][256] fp32 (convDb output, not yet normalised)
__global__ void sp_describe_kernel(const int* __restrict__ sel_idx, const float* __restrict__ sel_score,
                                   const int* __restrict__ sel_count, const float* __restrict__ dense, float* __restrict__ kpts,
                                   float* __restrict__ scores, float* __restrict__ desc, int W8, int h, int w, int cap,
                                   int fix_sampling) {
  const int b = blockIdx.y;
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int n = min(sel_count[b], cap);
  if (k >= n) return;
  const int p = sel_idx[static_cast<size_t>(b) * cap + k];
  const int py = p / W8, px = p - py * W8;
  const float x = static_cast<float>(px), y = static_cast<float>(py);
  if (lane == 0) {
    kpts[(static_cast<size_t>(b) * cap + k) * 2 + 0] = x;  // torch.flip(k,[1]).float(): (x, y)
    kpts[(static_cast<size_t>(b) * cap + k) * 2 + 1] = y;
    scores[static_cast<size_t>(b) * cap + k] = sel_score[static_cast<size_t>(b) * cap + k];
  }
  float ix, iy;
  if (fix_sampling) {  // extractors/superpoint.py:16-27, align_corners=False
    const float gx = (x + 0.5f) / (static_cast<float>(w) * 8.f) * 2.f - 1.f;
    const float gy = (y + 0.5f) / (static_cast<float>(h) * 8.f) * 2.f - 1.f;
    ix = ((gx + 1.f) * w - 1.f) / 2.f;
    iy = ((gy + 1.f) * h - 1.f) / 2.f;
  } else {  // thirdparty superpoint.py:81-98, align_corners=True
    const float gx = (x - 4.f + 0.5f) / (w * 8.f - 4.f - 0.5f) * 2.f - 1.f;
    const float gy = (y - 4.f + 0.5f) / (h * 8.f - 4.f - 0.5f) * 2.f - 1.f;
    ix = ((gx + 1.f) / 2.f) * (w - 1);
    iy = ((gy + 1.f) / 2.f) * (h - 1);
  }
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  const float wx1 = ix - fx, wx0 = (fx + 1.f) - ix, wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const float* D = dense + static_cast<size_t>(b) * h * w * 256;
#pragma unroll
  for (int cidx = 0; cidx < 4; ++cidx) {
    const int cx = x0 + (cidx & 1), cy = y0 + (cidx >> 1);
    const float wgt = ((cidx & 1) ? wx1 : wx0) * ((cidx >> 1) ? wy1 : wy0);
    if (cx < 0 || cx >= w || cy < 0 || cy >= h) continue;  // padding_mode="zeros"
    const float* d = D + (static_cast<size_t>(cy) * w + cx) * 256 + lane * 8;
    const float4 q0 = *reinterpret_cast<const float4*>(d), q1 = *reinterpret_cast<const float4*>(d + 4);
    const float e[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(e[j], e[j], ss);
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);  // F.normalize(descriptors, p=2, dim=1)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(wgt, e[j] * inv, acc[j]);
  }
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) ss = fmaf(acc[j], acc[j], ss);
#pragma unroll
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  float* o = desc + static_cast<size_t>(b) * 256 * cap + k;
#pragma unroll
  for (int j = 0; j < 8; ++j) o[static_cast<size_t>(lane * 8 + j) * cap] = acc[j] * inv;  // (D,N) layout
}

inline int launch_sp_softmax(dimb_ctx* ctx, cudaStream_t st, const float* logits, float* scores, int B, int h, int w) {
  sp_softmax_d2s_kernel<<<ceil_div(B * h * w * 32, 256), 256, 0, st>>>(logits, scores, B, h, w);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// keypoints (x, y) [B][cap][2], scores [B][cap] and descriptors [B][256][cap] of the first min(sel_count[b], cap) selected pixels
inline int launch_sp_describe(dimb_ctx* ctx, cudaStream_t st, const int* sel_idx, const float* sel_score, const int* sel_count,
                              const float* dense, float* kpts, float* scores, float* desc, int B, int h, int w, int cap, int fix_sampling) {
  sp_describe_kernel<<<dim3(ceil_div(cap * 32, 256), B), 256, 0, st>>>(sel_idx, sel_score, sel_count, dense, kpts, scores, desc, w * 8, h, w,
                                                                        cap, fix_sampling);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
