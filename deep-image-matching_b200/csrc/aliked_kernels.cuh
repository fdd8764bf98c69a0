// aliked_kernels.cuh - the kernels of ALIKED extraction, their launch helpers and the host transforms of the weights they read:
// dimb_aliked_extract_dev (aliked.cu) runs the network through these helpers, and the self-test library (selftest.cu,
// dimb_selftest_aliked_*) runs each stage through the same helpers on caller-given inputs.  See aliked.cu for the stages.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "gemm.cuh"

namespace {


__device__ __forceinline__ float selu_f(float x) {
  // torch.selu: x > 0 ? scale*x : scale*alpha*(exp(x)-1)   (ATen elu kernel with negcoef = alpha*scale)
  const float scale = 1.0507009873554804934193349852946f, alpha = 1.6732632423543772848170429916717f;
  return x > 0.f ? x * scale : (expf(x) - 1.f) * (alpha * scale);
}
__device__ __forceinline__ float act_f(float x, int act) { return act == 1 ? selu_f(x) : (act == 2 ? 1.f / (1.f + expf(-x)) : x); }

// image (H,W,3) or (H,W) float 0..255 -> planar [3][Hp][Wp] in [0,1], replicate padded (InputPadder, aliked.py:247-264)
__global__ void al_pad_kernel(const float* __restrict__ img, int H, int W, int channels, float* __restrict__ out, int Hp, int Wp,
                              int pad_top, int pad_left) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
  if (x >= Wp) return;
  const int sy = min(max(y - pad_top, 0), H - 1), sx = min(max(x - pad_left, 0), W - 1);
  const float v = channels == 3 ? img[(static_cast<size_t>(sy) * W + sx) * 3 + c] : img[static_cast<size_t>(sy) * W + sx];
  out[(static_cast<size_t>(c) * Hp + y) * Wp + x] = __fdiv_rn(v, 255.f);
}

// 3x3 conv, zero padding 1.  out = act(alpha[co]*conv + beta[co] (+ resid)).
// CTA = 64 x 8 output pixels x CO_T output channels (blockIdx.z); thread = 4 pixels of one row x CO_T channels in
// registers.  Input channels stream through shared memory 8 at a time; weights sit in shared memory as [ci][tap][co] so
// that one broadcast LDS.128 feeds 16 FMAs.  Per accumulator the summation order is ci ascending, tap ascending.
constexpr int kCiT = 8, kCoT = 16;
template <int CO_T, int PXT>  // PXT pixels per thread: 4 (tile 64 x 8) or 1 (tile 16 x 8, for the low-resolution maps)
__global__ void __launch_bounds__(128) al_conv3x3_kernel(const float* __restrict__ in, int Cin, int H, int W,
                                                         const float* __restrict__ wgt /*[Cout][Cin][9]*/,
                                                         const float* __restrict__ alpha, const float* __restrict__ beta,
                                                         const float* __restrict__ resid, float* __restrict__ out, int Cout, int act) {
  __shared__ __align__(16) float s_in[kCiT][10][68];
  __shared__ __align__(16) float s_w[kCiT][9][CO_T];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  constexpr int TW = 16 * PXT;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * 8, co0 = blockIdx.z * CO_T;
  float acc[PXT][CO_T];
#pragma unroll
  for (int p = 0; p < PXT; ++p)
#pragma unroll
    for (int j = 0; j < CO_T; ++j) acc[p][j] = 0.f;
  for (int ci0 = 0; ci0 < Cin; ci0 += kCiT) {
    for (int e = threadIdx.x; e < kCiT * 10 * (TW + 2); e += 128) {
      const int c = e / (10 * (TW + 2)), rem = e - c * 10 * (TW + 2), yy = rem / (TW + 2), xx = rem - yy * (TW + 2);
      const int gy = y0 + yy - 1, gx = x0 + xx - 1, ci = ci0 + c;
      s_in[c][yy][xx] = (ci < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W) ? in[(static_cast<size_t>(ci) * H + gy) * W + gx] : 0.f;
    }
    for (int e = threadIdx.x; e < kCiT * 9 * CO_T; e += 128) {
      const int c = e / (9 * CO_T), rem = e - c * 9 * CO_T, t = rem / CO_T, j = rem - t * CO_T;
      s_w[c][t][j] = (co0 + j < Cout && ci0 + c < Cin) ? wgt[(static_cast<size_t>(co0 + j) * Cin + ci0 + c) * 9 + t] : 0.f;
    }
    __syncthreads();
#pragma unroll 2
    for (int c = 0; c < kCiT; ++c) {
      float v[3][PXT + 2];
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        if (PXT == 4) {
          const float4 a = *reinterpret_cast<const float4*>(&s_in[c][ty + dy][tx * 4]);
          const float2 b = *reinterpret_cast<const float2*>(&s_in[c][ty + dy][tx * 4 + 4]);
          v[dy][0] = a.x, v[dy][1] = a.y, v[dy][2] = a.z, v[dy][3] = a.w, v[dy][PXT] = b.x, v[dy][PXT + 1] = b.y;
        } else {
#pragma unroll
          for (int i = 0; i < PXT + 2; ++i) v[dy][i] = s_in[c][ty + dy][tx * PXT + i];
        }
      }
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        float w[CO_T];
#pragma unroll
        for (int j4 = 0; j4 < CO_T / 4; ++j4) {
          const float4 q = *reinterpret_cast<const float4*>(&s_w[c][t][j4 * 4]);
          w[j4 * 4] = q.x, w[j4 * 4 + 1] = q.y, w[j4 * 4 + 2] = q.z, w[j4 * 4 + 3] = q.w;
        }
#pragma unroll
        for (int p = 0; p < PXT; ++p) {
          const float xv = v[t / 3][p + t % 3];
#pragma unroll
          for (int j = 0; j < CO_T; ++j) acc[p][j] = fmaf(xv, w[j], acc[p][j]);
        }
      }
    }
    __syncthreads();
  }
  const int x = x0 + tx * PXT, y = y0 + ty;
  if (y >= H || x >= W) return;
  const bool vec = PXT == 4 && (W & 3) == 0;  // then x + 3 < W and the row start is 16-byte aligned
#pragma unroll
  for (int j = 0; j < CO_T; ++j) {
    const int co = co0 + j;
    if (co >= Cout) break;
    const size_t o = (static_cast<size_t>(co) * H + y) * W + x;
    const float al = alpha ? alpha[co] : 1.f, be = beta ? beta[co] : 0.f;
    float r[PXT];
#pragma unroll
    for (int p = 0; p < PXT; ++p) r[p] = acc[p][j] * al + be;
    if (vec) {
      if (resid) {
        const float4 q = *reinterpret_cast<const float4*>(resid + o);
        r[0] += q.x, r[1 % PXT] += q.y, r[2 % PXT] += q.z, r[3 % PXT] += q.w;
      }
      *reinterpret_cast<float4*>(out + o) =
          make_float4(act_f(r[0], act), act_f(r[1 % PXT], act), act_f(r[2 % PXT], act), act_f(r[3 % PXT], act));
    } else {
#pragma unroll
      for (int p = 0; p < PXT; ++p)
        if (x + p < W) out[o + p] = act_f(r[p] + (resid ? resid[o + p] : 0.f), act);
    }
  }
}

// 1x1 conv: out[co][p] = act(sum_ci w[co][ci] in[ci][p] + b[co]); thread per pixel, 16 output channels per blockIdx.y
__global__ void __launch_bounds__(256) al_conv1x1_kernel(const float* __restrict__ in, int Cin, size_t P, const float* __restrict__ w,
                                                         const float* __restrict__ bias, float* __restrict__ out, int Cout, int act) {
  extern __shared__ float sw1[];  // [16][Cin]
  const int co0 = blockIdx.y * kCoT;
  for (int e = threadIdx.x; e < kCoT * Cin; e += 256) sw1[e] = (co0 + e / Cin < Cout) ? w[static_cast<size_t>(co0 + e / Cin) * Cin + e % Cin] : 0.f;
  __syncthreads();
  const size_t p = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (p >= P) return;
  float acc[kCoT];
#pragma unroll
  for (int j = 0; j < kCoT; ++j) acc[j] = 0.f;
  for (int ci = 0; ci < Cin; ++ci) {
    const float v = in[static_cast<size_t>(ci) * P + p];
#pragma unroll
    for (int j = 0; j < kCoT; ++j) acc[j] = fmaf(v, sw1[j * Cin + ci], acc[j]);
  }
#pragma unroll
  for (int j = 0; j < kCoT; ++j)
    if (co0 + j < Cout) out[static_cast<size_t>(co0 + j) * P + p] = act_f(acc[j] + (bias ? bias[co0 + j] : 0.f), act);
}

__global__ void al_avgpool_kernel(const float* __restrict__ in, int C, int H, int W, int k, float* __restrict__ out) {
  const int Ho = H / k, Wo = W / k;
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(C) * Ho * Wo) return;
  const int x = static_cast<int>(i % Wo), y = static_cast<int>((i / Wo) % Ho), c = static_cast<int>(i / (static_cast<size_t>(Wo) * Ho));
  float s = 0.f;
  for (int dy = 0; dy < k; ++dy)
    for (int dx = 0; dx < k; ++dx) s += in[(static_cast<size_t>(c) * H + y * k + dy) * W + x * k + dx];
  out[i] = s / static_cast<float>(k * k);
}

// torchvision deform_conv2d bilinear_interpolate
__device__ __forceinline__ float dcn_bilinear(const float* __restrict__ in, int H, int W, float h, float w) {
  if (h <= -1.f || static_cast<float>(H) <= h || w <= -1.f || static_cast<float>(W) <= w) return 0.f;
  const int hl = static_cast<int>(floorf(h)), wl = static_cast<int>(floorf(w)), hh_ = hl + 1, wh_ = wl + 1;
  const float lh = h - hl, lw = w - wl, hh = 1.f - lh, hw = 1.f - lw;
  const float v1 = (hl >= 0 && wl >= 0) ? in[hl * W + wl] : 0.f;
  const float v2 = (hl >= 0 && wh_ <= W - 1) ? in[hl * W + wh_] : 0.f;
  const float v3 = (hh_ <= H - 1 && wl >= 0) ? in[hh_ * W + wl] : 0.f;
  const float v4 = (hh_ <= H - 1 && wh_ <= W - 1) ? in[hh_ * W + wh_] : 0.f;
  return hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4;
}

// deformable 3x3 conv (pad 1, stride 1, one offset group): offsets [18][H][W] = (dy,dx) per tap, clamped to +-max_off.
// out = act(alpha*conv + beta (+resid)).  CTA = 16 pixels x all Cout: per chunk of 8 input channels the 8 x 9 x 16
// bilinear samples are taken once into shared memory (they are shared by every output channel) next to the matching
// weight slab [8][9][Cout]; thread = (pixel, group of Cout/8 channels).  Summation order per output: ci, tap ascending.
constexpr int kDcnPx = 16;
template <int CPT>  // output channels per thread = Cout / 8
__global__ void __launch_bounds__(128) al_deform_conv_kernel(const float* __restrict__ in, int Cin, int H, int W,
                                                             const float* __restrict__ offs, float max_off,
                                                             const float* __restrict__ wgt /*[Cin][9][Cout]*/,
                                                             const float* __restrict__ alpha, const float* __restrict__ beta,
                                                             const float* __restrict__ resid, float* __restrict__ out, int act) {
  constexpr int Cout = CPT * 8;
  extern __shared__ __align__(16) float dsm[];
  float* s_w = dsm;                               // [8][9][Cout]
  float* s_v = s_w + kCiT * 9 * Cout;             // [8][9][16]
  float* s_y = s_v + kCiT * 9 * kDcnPx;           // [9][16] sample rows
  float* s_x = s_y + 9 * kDcnPx;                  // [9][16] sample columns
  const int t = threadIdx.x, px = t & (kDcnPx - 1), cg = t >> 4;
  const int HW = H * W, p0 = blockIdx.x * kDcnPx;
  for (int e = t; e < 9 * kDcnPx; e += 128) {
    const int tap = e / kDcnPx, q = e - tap * kDcnPx, p = min(p0 + q, HW - 1);
    const int y = p / W, x = p - y * W;
    const float oy = fminf(fmaxf(offs[static_cast<size_t>(2 * tap) * HW + p], -max_off), max_off);
    const float ox = fminf(fmaxf(offs[static_cast<size_t>(2 * tap + 1) * HW + p], -max_off), max_off);
    s_y[e] = static_cast<float>(y - 1 + tap / 3) + oy;
    s_x[e] = static_cast<float>(x - 1 + tap % 3) + ox;
  }
  float acc[CPT];
#pragma unroll
  for (int j = 0; j < CPT; ++j) acc[j] = 0.f;
  __syncthreads();
  for (int ci0 = 0; ci0 < Cin; ci0 += kCiT) {
    for (int e = t; e < kCiT * 9 * kDcnPx; e += 128) {
      const int c = e / (9 * kDcnPx), rem = e - c * 9 * kDcnPx;  // rem = tap * 16 + pixel
      s_v[e] = dcn_bilinear(in + static_cast<size_t>(ci0 + c) * HW, H, W, s_y[rem], s_x[rem]);
    }
    {  // weights are stored [Cin][9][Cout] (transposed at create time): the slab of this chunk is contiguous
      const float4* src = reinterpret_cast<const float4*>(wgt + static_cast<size_t>(ci0) * 9 * Cout);
      for (int e = t; e < kCiT * 9 * Cout / 4; e += 128) reinterpret_cast<float4*>(s_w)[e] = src[e];
    }
    __syncthreads();
#pragma unroll 4
    for (int ct = 0; ct < kCiT * 9; ++ct) {
      const float v = s_v[ct * kDcnPx + px];
      const float* wr = s_w + ct * Cout + cg * CPT;
#pragma unroll
      for (int j4 = 0; j4 < CPT / 4; ++j4) {
        const float4 q = *reinterpret_cast<const float4*>(wr + j4 * 4);
        acc[j4 * 4] = fmaf(v, q.x, acc[j4 * 4]);
        acc[j4 * 4 + 1] = fmaf(v, q.y, acc[j4 * 4 + 1]);
        acc[j4 * 4 + 2] = fmaf(v, q.z, acc[j4 * 4 + 2]);
        acc[j4 * 4 + 3] = fmaf(v, q.w, acc[j4 * 4 + 3]);
      }
    }
    __syncthreads();
  }
  const int p = p0 + px;
  if (p >= HW) return;
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int co = cg * CPT + j;
    const size_t o = static_cast<size_t>(co) * HW + p;
    float r = acc[j] * alpha[co] + beta[co];
    if (resid) r += resid[o];
    out[o] = act_f(r, act);
  }
}

// upsample_bilinear2d, align_corners=True (ATen: scale = (in-1)/(out-1); idx0 = (int)src; lambda1 = src - idx0)
__device__ __forceinline__ float up_bilinear(const float* __restrict__ plane, int h, int w, float sy, float sx, int y, int x) {
  const float fy = sy * y, fx = sx * x;
  const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
  const int yp = (y0 < h - 1) ? 1 : 0, xp = (x0 < w - 1) ? 1 : 0;
  const float l1y = fy - y0, l0y = 1.f - l1y, l1x = fx - x0, l0x = 1.f - l1x;
  const float* q = plane + static_cast<size_t>(y0) * w + x0;
  return l0y * (l0x * q[0] + l1x * q[xp]) + l1y * (l0x * q[yp * w] + l1x * q[yp * w + xp]);
}

// Fused full-resolution tail of extract_dense_map (aliked.py:658-672), one thread per padded pixel:
//   x1' = selu(conv1(x1));  x1234 = cat[x1', up2(x2'), up8(x3'), up32(x4')]  (128 values in registers)
//   sh0 = selu(score_head.0(x1234))                     -> [8][Hp][Wp]
//   feature_map = x1234 / max(||x1234||_2, 1e-12)       -> cropped, pixel-major [H][W][128]: the descriptor head gathers whole
//                                                          128-channel pixels (3x3 patches, 16 deformed samples per keypoint), which
//                                                          are 512 contiguous bytes this way instead of 128 sectors of 128 planes
// The 128-channel full-resolution tensor never exists in HBM un-normalised: traffic = 16 planes in, 8 + 128 planes out.
__global__ void __launch_bounds__(128) al_fuse_kernel(const float* __restrict__ x1 /*[16][Hp][Wp]*/, const float* __restrict__ wl1 /*[32][16]*/,
                                                      const float* __restrict__ l2o, const float* __restrict__ l3o,
                                                      const float* __restrict__ l4o, const float* __restrict__ ws0 /*[8][128]*/, int Hp,
                                                      int Wp, int top, int left, int H, int W, float* __restrict__ sh0,
                                                      float* __restrict__ feat) {
  __shared__ __align__(16) float sw1[32 * 16];   // [co][ci]
  __shared__ __align__(16) float ss0[128 * 8];   // [c][j] (transposed so that one LDS.128 feeds 4 FMAs)
  for (int e = threadIdx.x; e < 32 * 16; e += 128) sw1[e] = wl1[e];
  for (int e = threadIdx.x; e < 8 * 128; e += 128) ss0[(e & 127) * 8 + (e >> 7)] = ws0[e];
  __syncthreads();
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= Wp) return;
  const size_t P = static_cast<size_t>(Hp) * Wp, p = static_cast<size_t>(y) * Wp + x;
  float v[128];
  {
    float xin[16];
#pragma unroll
    for (int ci = 0; ci < 16; ++ci) xin[ci] = x1[ci * P + p];
#pragma unroll
    for (int co = 0; co < 32; ++co) {
      float a = 0.f;
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4) {
        const float4 q = *reinterpret_cast<const float4*>(&sw1[co * 16 + c4 * 4]);
        a = fmaf(xin[c4 * 4], q.x, a);
        a = fmaf(xin[c4 * 4 + 1], q.y, a);
        a = fmaf(xin[c4 * 4 + 2], q.z, a);
        a = fmaf(xin[c4 * 4 + 3], q.w, a);
      }
      v[co] = selu_f(a);
    }
  }
#pragma unroll
  for (int lvl = 1; lvl < 4; ++lvl) {
    const int f = lvl == 1 ? 2 : (lvl == 2 ? 8 : 32);
    const int h = Hp / f, w = Wp / f;
    const float* src = lvl == 1 ? l2o : (lvl == 2 ? l3o : l4o);
    const float sy = h > 1 ? static_cast<float>(h - 1) / static_cast<float>(Hp - 1) : 0.f;
    const float sx = w > 1 ? static_cast<float>(w - 1) / static_cast<float>(Wp - 1) : 0.f;
#pragma unroll
    for (int cc = 0; cc < 32; ++cc) v[lvl * 32 + cc] = up_bilinear(src + static_cast<size_t>(cc) * h * w, h, w, sy, sx, y, x);
  }
  {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
#pragma unroll
    for (int c = 0; c < 128; ++c) {
      const float4 q0 = *reinterpret_cast<const float4*>(&ss0[c * 8]), q1 = *reinterpret_cast<const float4*>(&ss0[c * 8 + 4]);
      a[0] = fmaf(v[c], q0.x, a[0]), a[1] = fmaf(v[c], q0.y, a[1]), a[2] = fmaf(v[c], q0.z, a[2]), a[3] = fmaf(v[c], q0.w, a[3]);
      a[4] = fmaf(v[c], q1.x, a[4]), a[5] = fmaf(v[c], q1.y, a[5]), a[6] = fmaf(v[c], q1.z, a[6]), a[7] = fmaf(v[c], q1.w, a[7]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sh0[j * P + p] = selu_f(a[j]);
  }
  const int yo = y - top, xo = x - left;
  if (yo < 0 || yo >= H || xo < 0 || xo >= W) return;
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < 128; ++c) ss = fmaf(v[c], v[c], ss);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  float4* o = reinterpret_cast<float4*>(feat + (static_cast<size_t>(yo) * W + xo) * 128);
#pragma unroll
  for (int c = 0; c < 32; ++c) o[c] = make_float4(v[4 * c] * inv, v[4 * c + 1] * inv, v[4 * c + 2] * inv, v[4 * c + 3] * inv);
}

// crops [C][Hp][Wp] -> [C][H][W]
__global__ void al_crop_kernel(const float* __restrict__ in, int Hp, int Wp, int top, int left, float* __restrict__ out, int H, int W) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
  if (x >= W) return;
  out[(static_cast<size_t>(c) * H + y) * W + x] = in[(static_cast<size_t>(c) * Hp + y + top) * Wp + x + left];
}

// DKD sub-pixel refinement (aliked.py:180-222); thread per keypoint.  Outputs normalised keypoints in [-1,1].
__global__ void al_dkd_refine_kernel(const float* __restrict__ score, int H, int W, int r, const int* __restrict__ sel_idx,
                                     const int* __restrict__ count, int cap, float* __restrict__ kxy, float* __restrict__ disp,
                                     float* __restrict__ kscore) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(*count, cap);
  if (i >= n) return;
  const int idx = sel_idx[i], py = idx / W, px = idx - py * W;
  float mx = -INFINITY;
  for (int dy = -r; dy <= r; ++dy)
    for (int dx = -r; dx <= r; ++dx) {
      const int yy = py + dy, xx = px + dx;
      const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? score[static_cast<size_t>(yy) * W + xx] : 0.f;  // Unfold zero padding
      mx = fmaxf(mx, v);
    }
  float se = 0.f, sxw = 0.f, syw = 0.f;
  for (int dy = -r; dy <= r; ++dy)
    for (int dx = -r; dx <= r; ++dx) {
      const int yy = py + dy, xx = px + dx;
      const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? score[static_cast<size_t>(yy) * W + xx] : 0.f;
      const float e = expf((v - mx) / 0.1f);
      se += e;
      sxw = fmaf(e, static_cast<float>(dx), sxw);
      syw = fmaf(e, static_cast<float>(dy), syw);
    }
  const float rx = sxw / se, ry = syw / se;
  float sd = 0.f;
  for (int dy = -r; dy <= r; ++dy)
    for (int dx = -r; dx <= r; ++dx) {
      const int yy = py + dy, xx = px + dx;
      const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? score[static_cast<size_t>(yy) * W + xx] : 0.f;
      const float e = expf((v - mx) / 0.1f);
      const float ux = (static_cast<float>(dx) - rx) / static_cast<float>(r), uy = (static_cast<float>(dy) - ry) / static_cast<float>(r);
      const float nrm = sqrtf(ux * ux + uy * uy);
      sd = fmaf(e, nrm * nrm, sd);
    }
  disp[i] = sd / se;
  const float kx = (static_cast<float>(px) + rx) / static_cast<float>(W - 1) * 2.f - 1.f;
  const float ky = (static_cast<float>(py) + ry) / static_cast<float>(H - 1) * 2.f - 1.f;
  kxy[2 * i] = kx;
  kxy[2 * i + 1] = ky;
  // grid_sample(score_map, bilinear, align_corners=True, zeros padding)
  const float ix = ((kx + 1.f) / 2.f) * (W - 1), iy = ((ky + 1.f) / 2.f) * (H - 1);
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  float acc = 0.f;
  for (int c = 0; c < 4; ++c) {
    const int cx = x0 + (c & 1), cy = y0 + (c >> 1);
    const float wgt = ((c & 1) ? ix - fx : fx + 1.f - ix) * ((c >> 1) ? iy - fy : fy + 1.f - iy);
    if (cx >= 0 && cx < W && cy >= 0 && cy < H) acc = fmaf(score[static_cast<size_t>(cy) * W + cx], wgt, acc);
  }
  kscore[i] = acc;
}

// ---------------------------------------------------------------- SDDH (aliked.py:503-558)
// Four steps.  The two contractions that carry the FLOPs (sf_conv: [16N x 128] x [128 x 128]; the aggregation einsum
// 'ncp,pcd->nd': [N x 2048] x [2048 x 128]) run on the tensor cores through gemm.cuh (fp16 hi/lo split, fp32 accumulate).
//   al_sddh_offsets_kernel  3x3 patch -> offset_conv.0 + SELU -> offset_conv.2 -> 16 clamped (dx,dy); also the final
//                           pixel coordinates of the keypoints.  CTA = 8 keypoints so that w0 is read once per 8.
//   al_sddh_sample_kernel   bilinear samples of the 16 positions x 128 channels -> A operand [16N][128] (hi/lo)
//   GEMM 1 + EpiSeluSplit   selu(sf_conv) -> A operand [N][16*128]
//   GEMM 2 + EpiRowsF32     aggregation -> [N][128] fp32;  al_sddh_norm_kernel: L2 normalise, store (D,N)
constexpr int kSddhKp = 8;
__global__ void __launch_bounds__(128) al_sddh_offsets_kernel(const float* __restrict__ feat, int H, int W, const float* __restrict__ kxy,
                                                              const int* __restrict__ count, int cap,
                                                              const float* __restrict__ w0T /*[1152][32]*/, const float* __restrict__ b0,
                                                              const float* __restrict__ w2 /*[32][32]*/, const float* __restrict__ b2,
                                                              float* __restrict__ kpts_px, float* __restrict__ off /*[cap][32]*/) {
  constexpr int C = 128, E = C * 9;
  const int n = min(*count, cap), k0 = blockIdx.x * kSddhKp, t = threadIdx.x;
  if (k0 >= n) return;
  __shared__ float patch[kSddhKp][E];
  __shared__ float hid[kSddhKp][32];
  __shared__ int corner[kSddhKp][2];
  const float whx = static_cast<float>(W - 1), why = static_cast<float>(H - 1);
  if (t < kSddhKp) {
    const int k = min(k0 + t, n - 1);
    const float kwx = (kxy[2 * k] / 2.f + 0.5f) * whx, kwy = (kxy[2 * k + 1] / 2.f + 0.5f) * why;
    // get_patches: corner = (long(kwh) - K/2 + 1).long(), clamped so that the 3x3 patch stays inside (aliked.py:52-56)
    int cx = static_cast<int>(static_cast<float>(static_cast<int>(kwx)) - 1.5f + 1.f);
    int cy = static_cast<int>(static_cast<float>(static_cast<int>(kwy)) - 1.5f + 1.f);
    corner[t][0] = min(max(cx, 0), W - 1 - 3);
    corner[t][1] = min(max(cy, 0), H - 1 - 3);
    if (k0 + t < n) {  // final pixel coordinates: wh * (k + 1) / 2   (aliked.py:689)
      kpts_px[2 * k] = whx * (kxy[2 * k] + 1.f) / 2.f;
      kpts_px[2 * k + 1] = why * (kxy[2 * k + 1] + 1.f) / 2.f;
    }
  }
  __syncthreads();
  for (int e = t; e < kSddhKp * E; e += 128) {  // lanes run over the channels of one patch pixel: 512-byte coalesced reads
    const int q = e / E, r = e - q * E, pos = r >> 7, c = r & 127, j = pos / 3, i = pos - 3 * j;
    patch[q][c * 9 + pos] = feat[(static_cast<size_t>(corner[q][1] + j) * W + corner[q][0] + i) * C + c];
  }
  __syncthreads();
  {  // offset_conv.0 (3x3 valid conv = dot over 1152) + SELU: lane = output channel, warp = keypoints 2w, 2w+1
    const int o = t & 31, q0 = (t >> 5) * 2;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
    for (int e = 0; e < E; ++e) {
      const float wv = __ldg(w0T + e * 32 + o);
      a0 = fmaf(patch[q0][e], wv, a0);
      a1 = fmaf(patch[q0 + 1][e], wv, a1);
    }
    hid[q0][o] = selu_f(a0 + b0[o]);
    hid[q0 + 1][o] = selu_f(a1 + b0[o]);
  }
  __syncthreads();
  const float mo = static_cast<float>(max(H, W)) / 4.f;
  for (int e = t; e < kSddhKp * 32; e += 128) {  // offset_conv.2 (1x1) + clamp
    const int q = e >> 5, o = e & 31;
    if (k0 + q >= n) continue;
    float a = b2[o];
#pragma unroll
    for (int i = 0; i < 32; ++i) a = fmaf(hid[q][i], w2[o * 32 + i], a);
    off[static_cast<size_t>(k0 + q) * 32 + o] = fminf(fmaxf(a, -mo), mo);
  }
}

// CTA = one keypoint, thread = channel: grid_sample(bilinear, align_corners, zeros) of the 16 deformed positions
__global__ void __launch_bounds__(128) al_sddh_sample_kernel(const float* __restrict__ feat, int H, int W, const float* __restrict__ kxy,
                                                             const int* __restrict__ count, int cap, const float* __restrict__ off,
                                                             __half* __restrict__ fh, __half* __restrict__ fl /*[cap*16][128]*/) {
  constexpr int M = 16;
  const int k = blockIdx.x, t = threadIdx.x;
  if (k >= min(*count, cap)) return;
  const float whx = static_cast<float>(W - 1), why = static_cast<float>(H - 1);
  const float kwx = (kxy[2 * k] / 2.f + 0.5f) * whx, kwy = (kxy[2 * k + 1] / 2.f + 0.5f) * why;
  const float* plane = feat + t;  // pixel-major map: channel t of pixel p is plane[p * 128]
#pragma unroll 4
  for (int p = 0; p < M; ++p) {
    const float posx = kwx + off[k * 32 + p], posy = kwy + off[k * 32 + M + p];
    const float gx = 2.f * posx / whx - 1.f, gy = 2.f * posy / why - 1.f;
    const float ix = ((gx + 1.f) / 2.f) * whx, iy = ((gy + 1.f) / 2.f) * why;
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
    float acc = 0.f;
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      const int qx = x0 + (c4 & 1), qy = y0 + (c4 >> 1);
      const float wgt = ((c4 & 1) ? ix - fx : fx + 1.f - ix) * ((c4 >> 1) ? iy - fy : fy + 1.f - iy);
      if (qx >= 0 && qx < W && qy >= 0 && qy < H) acc = fmaf(plane[(static_cast<size_t>(qy) * W + qx) * 128], wgt, acc);
    }
    __half h, l;
    split_f32(acc, h, l);
    const size_t o = (static_cast<size_t>(k) * M + p) * 128 + t;
    fh[o] = h;
    if (fl) fl[o] = l;
  }
}

// GEMM 1 epilogue: selu(acc) -> fp16 hi/lo, row-major [rows][128]; tiles beyond the live keypoints are skipped
struct EpiSeluSplit : EpiBase {
  __half *hi, *lo;  // lo null in FAST mode
  const int* count;
  int rows_per_kp, cap, ldc;
  __device__ bool tile_active(const TileCoord& tc) const { return tc.m0 < min(*count, cap) * rows_per_kp; }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    float4 f[8];
    warp_transpose32(v, sc, f);
    const int lane = r & 31, col = n + (lane & 7) * 4;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = tc.m0 + (r & ~31) + it * 4 + (lane >> 3);
      if (row >= cap * rows_per_kp) continue;
      const size_t o = static_cast<size_t>(row) * ldc + col;
      store_split4(hi + o, lo ? lo + o : nullptr, make_float4(selu_f(f[it].x), selu_f(f[it].y), selu_f(f[it].z), selu_f(f[it].w)));
    }
  }
};

// GEMM 2 epilogue: plain fp32 rows [cap][128]
struct EpiRowsF32 : EpiBase {
  float* out;
  const int* count;
  int cap;
  __device__ bool tile_active(const TileCoord& tc) const { return tc.m0 < min(*count, cap); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    float4 f[8];
    warp_transpose32(v, sc, f);
    const int lane = r & 31, col = n + (lane & 7) * 4;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = tc.m0 + (r & ~31) + it * 4 + (lane >> 3);
      if (row < cap) *reinterpret_cast<float4*>(out + static_cast<size_t>(row) * 128 + col) = f[it];
    }
  }
};

// warp per keypoint: descriptors = F.normalize(d), stored in the FeaturesDict (D,N) layout
__global__ void al_sddh_norm_kernel(const float* __restrict__ d /*[cap][128]*/, const int* __restrict__ count, int cap,
                                    float* __restrict__ desc /*[128][cap]*/) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= min(*count, cap)) return;
  const float4 v = *reinterpret_cast<const float4*>(d + static_cast<size_t>(k) * 128 + lane * 4);
  float ss = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
#pragma unroll
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  desc[static_cast<size_t>(lane * 4) * cap + k] = v.x * inv;
  desc[static_cast<size_t>(lane * 4 + 1) * cap + k] = v.y * inv;
  desc[static_cast<size_t>(lane * 4 + 2) * cap + k] = v.z * inv;
  desc[static_cast<size_t>(lane * 4 + 3) * cap + k] = v.w * inv;
}

// thr_out = thr if some pixel passed it, else mean(score_map) (aliked.py:158-160); cand_count null: always the mean (mean mode)
__global__ void __launch_bounds__(1024) al_threshold_kernel(const float* __restrict__ score, int HW, const int* __restrict__ cand_count,
                                                            float thr, float* __restrict__ thr_out) {
  if (cand_count && *cand_count > 0) {
    if (threadIdx.x == 0) *thr_out = thr;
    return;
  }
  __shared__ double red[32];
  double acc = 0;
  for (int i = threadIdx.x; i < HW; i += 1024) acc += score[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 32; ++i) t += red[i];
    *thr_out = static_cast<float>(t / HW);
  }
}

struct BnConv {
  float *w = nullptr, *alpha = nullptr, *beta = nullptr;
  int cin = 0, cout = 0;
};

// ---------------------------------------------------------------- host transforms of the state_dict weights
// eval BatchNorm -> alpha = invstd*gamma, beta = bias - mean*alpha (ATen batch_norm inference transform); g, b, m, v: [cout] each
inline void al_bn_fold(const float* g, const float* b, const float* m, const float* v, int cout, std::vector<float>& al,
                       std::vector<float>& be) {
  al.resize(cout);
  be.resize(cout);
  for (int i = 0; i < cout; ++i) {
    const float invstd = 1.f / std::sqrt(v[i] + 1e-5f);
    al[i] = invstd * g[i];
    be[i] = b[i] - m[i] * al[i];
  }
}

// deformable regular_conv weights [Cout][Cin][3][3] -> [Cin][9][Cout], the layout al_deform_conv_kernel reads
inline std::vector<float> al_dcn_weight(const float* p, int cout, int cin) {
  std::vector<float> wt(static_cast<size_t>(cout) * cin * 9);
  for (int co = 0; co < cout; ++co)
    for (int ct = 0; ct < cin * 9; ++ct) wt[static_cast<size_t>(ct) * cout + co] = p[static_cast<size_t>(co) * cin * 9 + ct];
  return wt;
}

// desc_head.offset_conv.0.weight [32][1152] -> [1152][32] (w0T of al_sddh_offsets_kernel)
inline std::vector<float> al_sddh_w0T(const float* p) {
  std::vector<float> t(static_cast<size_t>(1152) * 32);
  for (int o = 0; o < 32; ++o)
    for (int e = 0; e < 1152; ++e) t[static_cast<size_t>(e) * 32 + o] = p[static_cast<size_t>(o) * 1152 + e];
  return t;
}

// desc_head.agg_weights [p][c][d] -> B operand [d][p*128 + c] (K-major) of the aggregation GEMM
inline std::vector<float> al_sddh_agg(const float* p) {
  std::vector<float> t(static_cast<size_t>(128) * 2048);
  for (int q = 0; q < 16; ++q)
    for (int c = 0; c < 128; ++c)
      for (int d = 0; d < 128; ++d) t[static_cast<size_t>(d) * 2048 + q * 128 + c] = p[(static_cast<size_t>(q) * 128 + c) * 128 + d];
  return t;
}

// fp32 GEMM operand -> fp16 hi / lo (hi = rn(w), lo = rn(w - hi))
inline void al_split_host(const float* w, size_t cnt, std::vector<__half>& h, std::vector<__half>& l) {
  h.resize(cnt);
  l.resize(cnt);
  for (size_t i = 0; i < cnt; ++i) {
    h[i] = __float2half_rn(w[i]);
    l[i] = __float2half_rn(w[i] - __half2float(h[i]));
  }
}

// ---------------------------------------------------------------- launch helpers

// The al_conv3x3_kernel instantiation conv3 runs: 1 = <8,1> (maps of at most 64 x 64 pixels: small tiles so that the grid still fills
// the SMs), 2 = <16,4> (Cout >= 16), 3 = <8,4>
inline int al_conv3_plan(int H, int W, int cout) {
  if (static_cast<size_t>(H) * W <= 64 * 64) return 1;
  return cout >= 16 ? 2 : 3;
}
// conv3 on a given instantiation (al_conv3_plan's numbering)
inline int conv3_as(dimb_ctx* ctx, cudaStream_t st, int plan, const float* in, int cin, int H, int W, const float* w, const float* alpha,
                    const float* beta, const float* resid, float* out, int cout, int act) {
  if (plan == 1) {
    dim3 grid(ceil_div(W, 16), ceil_div(H, 8), ceil_div(cout, 8));
    al_conv3x3_kernel<8, 1><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  } else if (plan == 2) {
    dim3 grid(ceil_div(W, 64), ceil_div(H, 8), ceil_div(cout, 16));
    al_conv3x3_kernel<16, 4><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  } else {
    dim3 grid(ceil_div(W, 64), ceil_div(H, 8), ceil_div(cout, 8));
    al_conv3x3_kernel<8, 4><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int conv3(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, int H, int W, const float* w, const float* alpha, const float* beta,
                 const float* resid, float* out, int cout, int act) {
  return conv3_as(ctx, st, al_conv3_plan(H, W, cout), in, cin, H, W, w, alpha, beta, resid, out, cout, act);
}
inline int conv1(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, size_t P, const float* w, const float* bias, float* out, int cout,
                 int act) {
  dim3 grid(static_cast<unsigned>((P + 255) / 256), ceil_div(cout, kCoT));
  al_conv1x1_kernel<<<grid, 256, kCoT * cin * sizeof(float), st>>>(in, cin, P, w, bias, out, cout, act);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
// deformable conv on given offsets [18][H][W] (clamped to +-max_off in the kernel); c.cout 64 or 128, cin a multiple of 8
inline int launch_al_deform(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, int H, int W, const float* offs, float max_off,
                            const BnConv& c, const float* resid, float* out, int act) {
  const size_t smem = (static_cast<size_t>(kCiT) * 9 * (c.cout + kDcnPx) + 18 * kDcnPx) * sizeof(float);
  const int grid = ceil_div(H * W, kDcnPx);
  if (c.cout == 64) {
    al_deform_conv_kernel<8><<<grid, 128, smem, st>>>(in, cin, H, W, offs, max_off, c.w, c.alpha, c.beta, resid, out, act);
  } else if (c.cout == 128) {
    al_deform_conv_kernel<16><<<grid, 128, smem, st>>>(in, cin, H, W, offs, max_off, c.w, c.alpha, c.beta, resid, out, act);
  } else {
    return DIMB_ERR_UNSUPPORTED;
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int dcn(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, int H, int W, const float* offw, const float* offb, float* offbuf,
               const BnConv& c, const float* resid, float* out, int act) {
  // offsets = offset_conv(x) (3x3, bias), clamped inside the deform kernel
  DIMB_TRY(conv3(ctx, st, in, cin, H, W, offw, nullptr, offb, nullptr, offbuf, 18, 0));
  const float mo = static_cast<float>(std::max(H, W)) / 4.f;
  return launch_al_deform(ctx, st, in, cin, H, W, offbuf, mo, c, resid, out, act);
}

// InputPadder(h, w, 32): pad = (((x // 32) + 1) * 32 - x) % 32, split floor / ceil
inline void al_input_padder(int H, int W, int& Hp, int& Wp, int& top, int& left) {
  const int ph = (((H / 32) + 1) * 32 - H) % 32, pw = (((W / 32) + 1) * 32 - W) % 32;
  top = ph / 2, left = pw / 2, Hp = H + ph, Wp = W + pw;
}

// al_pad_kernel: image (H,W,channels) -> planar [3][Hp][Wp]
inline int launch_al_pad(dimb_ctx* ctx, cudaStream_t st, const float* image, int H, int W, int channels, float* out, int Hp, int Wp,
                         int top, int left) {
  al_pad_kernel<<<dim3(ceil_div(Wp, 128), Hp, 3), 128, 0, st>>>(image, H, W, channels, out, Hp, Wp, top, left);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
// k x k average pooling, stride k, of C planes of H x W
inline int launch_al_avgpool(dimb_ctx* ctx, cudaStream_t st, const float* in, int C, int H, int W, int k, float* out) {
  const size_t n = static_cast<size_t>(C) * (H / k) * (W / k);
  al_avgpool_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(in, C, H, W, k, out);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int launch_al_fuse(dimb_ctx* ctx, cudaStream_t st, const float* x1, const float* wl1, const float* l2o, const float* l3o,
                          const float* l4o, const float* ws0, int Hp, int Wp, int top, int left, int H, int W, float* sh0, float* feat) {
  al_fuse_kernel<<<dim3(ceil_div(Wp, 128), Hp), 128, 0, st>>>(x1, wl1, l2o, l3o, l4o, ws0, Hp, Wp, top, left, H, W, sh0, feat);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
// one plane [Hp][Wp] -> [H][W]
inline int launch_al_crop(dimb_ctx* ctx, cudaStream_t st, const float* in, int Hp, int Wp, int top, int left, float* out, int H, int W) {
  al_crop_kernel<<<dim3(ceil_div(W, 128), H, 1), 128, 0, st>>>(in, Hp, Wp, top, left, out, H, W);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int launch_al_threshold(dimb_ctx* ctx, cudaStream_t st, const float* score, int HW, const int* cand_count, float thr, float* thr_out) {
  al_threshold_kernel<<<1, 1024, 0, st>>>(score, HW, cand_count, thr, thr_out);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int launch_al_dkd(dimb_ctx* ctx, cudaStream_t st, const float* score, int H, int W, int r, const int* sel_idx, const int* count,
                         int cap, float* kxy, float* disp, float* kscore) {
  al_dkd_refine_kernel<<<ceil_div(cap, 128), 128, 0, st>>>(score, H, W, r, sel_idx, count, cap, kxy, disp, kscore);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
inline int launch_al_sddh_offsets(dimb_ctx* ctx, cudaStream_t st, const float* feat, int H, int W, const float* kxy, const int* count,
                                  int cap, const float* w0T, const float* b0, const float* w2, const float* b2, float* kpts_px, float* off) {
  al_sddh_offsets_kernel<<<ceil_div(cap, kSddhKp), 128, 0, st>>>(feat, H, W, kxy, count, cap, w0T, b0, w2, b2, kpts_px, off);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
// fl null: FAST precision (hi only)
inline int launch_al_sddh_sample(dimb_ctx* ctx, cudaStream_t st, const float* feat, int H, int W, const float* kxy, const int* count,
                                 int cap, const float* off, __half* fh, __half* fl) {
  al_sddh_sample_kernel<<<cap, 128, 0, st>>>(feat, H, W, kxy, count, cap, off, fh, fl);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
// sf_conv + SELU: [16 cap][128] x [128][128]^T -> f2 hi / lo (lo null: FAST).  a: samples (rows of 16 cap, padded to whole tiles),
// b: sf_conv.weight
inline int launch_al_sddh_sf_gemm(dimb_ctx* ctx, cudaStream_t st, const CUtensorMap (&a)[2], const CUtensorMap (&b)[2], __half* f2h,
                                  __half* f2l, const int* count, int cap) {
  EpiSeluSplit e;
  e.hi = f2h, e.lo = f2l, e.count = count, e.rows_per_kp = 16, e.cap = cap, e.ldc = 128;
  TcOperands ops;
  ops.Ah = a[0], ops.Al = a[1], ops.Bh = b[0], ops.Bl = b[1];
  GemmArgs g{};
  g.num_kb = 2, g.M = cap * 16, g.N = 128;
  return launch_gemm<128, false>(ctx, st, ops, g, e, ceil_div(cap * 16, kTileM), 128, "al.sddh_sf_gemm");
}
// aggregation einsum 'ncp,pcd->nd': [cap][2048] x [128][2048]^T -> dsc [cap][128] fp32.  a: f2, b: the reordered agg_weights
inline int launch_al_sddh_agg_gemm(dimb_ctx* ctx, cudaStream_t st, const CUtensorMap (&a)[2], const CUtensorMap (&b)[2], float* dsc,
                                   const int* count, int cap) {
  EpiRowsF32 e;
  e.out = dsc, e.count = count, e.cap = cap;
  TcOperands ops;
  ops.Ah = a[0], ops.Al = a[1], ops.Bh = b[0], ops.Bl = b[1];
  GemmArgs g{};
  g.num_kb = 32, g.M = cap, g.N = 128;
  return launch_gemm<128, false>(ctx, st, ops, g, e, ceil_div(cap, kTileM), 128, "al.sddh_agg_gemm");
}
inline int launch_al_sddh_norm(dimb_ctx* ctx, cudaStream_t st, const float* dsc, const int* count, int cap, float* desc) {
  al_sddh_norm_kernel<<<ceil_div(cap * 32, 256), 256, 0, st>>>(dsc, count, cap, desc);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
