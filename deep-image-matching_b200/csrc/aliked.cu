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
#include <algorithm>
#include <memory>
#include <cmath>
#include <cstring>
#include <vector>

#include "detect.cuh"
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

}  // namespace

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
  std::vector<__half> h(cnt), l(cnt);
  for (size_t i = 0; i < cnt; ++i) {
    h[i] = __float2half_rn(w[i]);
    l[i] = __float2half_rn(w[i] - __half2float(h[i]));
  }
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
    std::vector<float> wt(static_cast<size_t>(cout) * cin * 9);
    for (int co = 0; co < cout; ++co)
      for (int ct = 0; ct < cin * 9; ++ct) wt[static_cast<size_t>(ct) * cout + co] = p[static_cast<size_t>(co) * cin * 9 + ct];
    DIMB_TRY(up_f32(ctx, &c.w, wt.data(), wt.size()));
  } else {
    DIMB_TRY(up_f32(ctx, &c.w, p, static_cast<size_t>(cout) * cin * 9));
  }
  p += static_cast<size_t>(cout) * cin * 9;
  const float *g = p, *b = p + cout, *m = p + 2 * cout, *v = p + 3 * cout;
  std::vector<float> al(cout), be(cout);
  for (int i = 0; i < cout; ++i) {
    const float invstd = 1.f / std::sqrt(v[i] + 1e-5f);
    al[i] = invstd * g[i];
    be[i] = b[i] - m[i] * al[i];
  }
  p += 4 * cout;
  DIMB_TRY(up_f32(ctx, &c.alpha, al.data(), cout));
  DIMB_TRY(up_f32(ctx, &c.beta, be.data(), cout));
  return DIMB_OK;
}

int conv3(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, int H, int W, const float* w, const float* alpha, const float* beta,
          const float* resid, float* out, int cout, int act) {
  if (static_cast<size_t>(H) * W <= 64 * 64) {  // low-resolution maps: small tiles so that the grid still fills the SMs
    dim3 grid(ceil_div(W, 16), ceil_div(H, 8), ceil_div(cout, 8));
    al_conv3x3_kernel<8, 1><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  } else if (cout >= 16) {
    dim3 grid(ceil_div(W, 64), ceil_div(H, 8), ceil_div(cout, 16));
    al_conv3x3_kernel<16, 4><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  } else {
    dim3 grid(ceil_div(W, 64), ceil_div(H, 8), ceil_div(cout, 8));
    al_conv3x3_kernel<8, 4><<<grid, 128, 0, st>>>(in, cin, H, W, w, alpha, beta, resid, out, cout, act);
  }
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
int conv1(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, size_t P, const float* w, const float* bias, float* out, int cout, int act) {
  dim3 grid(static_cast<unsigned>((P + 255) / 256), ceil_div(cout, kCoT));
  al_conv1x1_kernel<<<grid, 256, kCoT * cin * sizeof(float), st>>>(in, cin, P, w, bias, out, cout, act);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}
int dcn(dimb_ctx* ctx, cudaStream_t st, const float* in, int cin, int H, int W, const float* offw, const float* offb, float* offbuf,
        const BnConv& c, const float* resid, float* out, int act) {
  // offsets = offset_conv(x) (3x3, bias), clamped inside the deform kernel
  DIMB_TRY(conv3(ctx, st, in, cin, H, W, offw, nullptr, offb, nullptr, offbuf, 18, 0));
  const float mo = static_cast<float>(std::max(H, W)) / 4.f;
  const size_t smem = (static_cast<size_t>(kCiT) * 9 * (c.cout + kDcnPx) + 18 * kDcnPx) * sizeof(float);
  const int grid = ceil_div(H * W, kDcnPx);
  if (c.cout == 64) {
    al_deform_conv_kernel<8><<<grid, 128, smem, st>>>(in, cin, H, W, offbuf, mo, c.w, c.alpha, c.beta, resid, out, act);
  } else if (c.cout == 128) {
    al_deform_conv_kernel<16><<<grid, 128, smem, st>>>(in, cin, H, W, offbuf, mo, c.w, c.alpha, c.beta, resid, out, act);
  } else {
    return DIMB_ERR_UNSUPPORTED;
  }
  DIMB_LAUNCH_CHECK(ctx);
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
    std::vector<float> t(static_cast<size_t>(128) * 2048);
    for (int q = 0; q < 16; ++q)
      for (int c = 0; c < 128; ++c)
        for (int d = 0; d < 128; ++d) t[static_cast<size_t>(d) * 2048 + q * 128 + c] = p[(static_cast<size_t>(q) * 128 + c) * 128 + d];
    DIMB_TRY(up_split(ctx, &al->agh, &al->agl, al->m_ag, t.data(), 128, 2048));
    p += 16 * 128 * 128;
  }
  {  // desc_head.offset_conv.0.weight [32][1152] -> [1152][32]
    std::vector<float> t(static_cast<size_t>(1152) * 32);
    for (int o = 0; o < 32; ++o)
      for (int e = 0; e < 1152; ++e) t[static_cast<size_t>(e) * 32 + o] = p[static_cast<size_t>(o) * 1152 + e];
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
  // InputPadder(h, w, 32): pad = (((x // 32) + 1) * 32 - x) % 32, split floor / ceil
  const int ph = (((H / 32) + 1) * 32 - H) % 32, pw = (((W / 32) + 1) * 32 - W) % 32;
  const int top = ph / 2, left = pw / 2, Hp = H + ph, Wp = W + pw;
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
    al_pad_kernel<<<dim3(ceil_div(Wp, 128), Hp, 3), 128, 0, st>>>(image, H, W, channels, al->pad, Hp, Wp, top, left);
    DIMB_LAUNCH_CHECK(ctx);
    // block1
    DIMB_TRY(conv3(ctx, st, al->pad, 3, Hp, Wp, al->b1c1.w, al->b1c1.alpha, al->b1c1.beta, nullptr, al->t1a, 16, 1));
    DIMB_TRY(conv3(ctx, st, al->t1a, 16, Hp, Wp, al->b1c2.w, al->b1c2.alpha, al->b1c2.beta, nullptr, al->x1, 16, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block2");  // ResBlock, regular convs
    al_avgpool_kernel<<<static_cast<unsigned>((P / 4 * 16 + 255) / 256), 256, 0, st>>>(al->x1, 16, Hp, Wp, 2, al->p2);
    DIMB_LAUNCH_CHECK(ctx);
    DIMB_TRY(conv3(ctx, st, al->p2, 16, H2, W2, al->b2c1.w, al->b2c1.alpha, al->b2c1.beta, nullptr, al->t2a, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->p2, 16, P / 4, al->b2dw, al->b2db, al->sc2, 32, 0));
    DIMB_TRY(conv3(ctx, st, al->t2a, 32, H2, W2, al->b2c2.w, al->b2c2.alpha, al->b2c2.beta, al->sc2, al->x2, 32, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block3");  // deformable
    al_avgpool_kernel<<<static_cast<unsigned>((P / 64 * 32 + 255) / 256), 256, 0, st>>>(al->x2, 32, H2, W2, 4, al->p3);
    DIMB_LAUNCH_CHECK(ctx);
    DIMB_TRY(dcn(ctx, st, al->p3, 32, H8, W8, al->o31w, al->o31b, al->off3, al->b3c1, nullptr, al->t3a, 1));
    DIMB_TRY(conv1(ctx, st, al->p3, 32, P / 64, al->b3dw, al->b3db, al->sc3, 64, 0));
    DIMB_TRY(dcn(ctx, st, al->t3a, 64, H8, W8, al->o32w, al->o32b, al->off3, al->b3c2, al->sc3, al->x3, 1));
  }
  {
    ProfScope prof(ctx, st, "al.block4");  // deformable
    al_avgpool_kernel<<<static_cast<unsigned>((P / 1024 * 64 + 255) / 256), 256, 0, st>>>(al->x3, 64, H8, W8, 4, al->p4);
    DIMB_LAUNCH_CHECK(ctx);
    DIMB_TRY(dcn(ctx, st, al->p4, 64, H32, W32, al->o41w, al->o41b, al->off4, al->b4c1, nullptr, al->t4a, 1));
    DIMB_TRY(conv1(ctx, st, al->p4, 64, P / 1024, al->b4dw, al->b4db, al->sc4, 128, 0));
    DIMB_TRY(dcn(ctx, st, al->t4a, 128, H32, W32, al->o42w, al->o42b, al->off4, al->b4c2, al->sc4, al->x4, 1));
  }
  {
    ProfScope prof(ctx, st, "al.aggregate");
    DIMB_TRY(conv1(ctx, st, al->x2, 32, P / 4, al->l2, nullptr, al->l2o, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->x3, 64, P / 64, al->l3, nullptr, al->l3o, 32, 1));
    DIMB_TRY(conv1(ctx, st, al->x4, 128, P / 1024, al->l4, nullptr, al->l4o, 32, 1));
    al_fuse_kernel<<<dim3(ceil_div(Wp, 128), Hp), 128, 0, st>>>(al->x1, al->l1, al->l2o, al->l3o, al->l4o, al->s0, Hp, Wp, top, left, H, W,
                                                                  al->sh0, al->feat);
    DIMB_LAUNCH_CHECK(ctx);
  }
  {
    ProfScope prof(ctx, st, "al.score_head");
    DIMB_TRY(conv3(ctx, st, al->sh0, 8, Hp, Wp, al->s2, nullptr, nullptr, nullptr, al->sh1, 4, 1));
    DIMB_TRY(conv3(ctx, st, al->sh1, 4, Hp, Wp, al->s4, nullptr, nullptr, nullptr, al->sh2, 4, 1));
    DIMB_TRY(conv3(ctx, st, al->sh2, 4, Hp, Wp, al->s6, nullptr, nullptr, nullptr, al->score_pad, 1, 2));
    al_crop_kernel<<<dim3(ceil_div(W, 128), H, 1), 128, 0, st>>>(al->score_pad, Hp, Wp, top, left, al->score, H, W);
    DIMB_LAUNCH_CHECK(ctx);
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
    al_threshold_kernel<<<1, 1024, 0, st>>>(al->score, H * W, mean_mode ? nullptr : al->cand_count, cf.detection_threshold, al->thr_dev);
    DIMB_LAUNCH_CHECK(ctx);
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
  al_dkd_refine_kernel<<<ceil_div(cap, 128), 128, 0, st>>>(al->score, H, W, r, al->sel_idx, count, cap, al->kxy, scores, al->kscore);
  DIMB_LAUNCH_CHECK(ctx);
  }
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  {
  ProfScope prof(ctx, st, "al.sddh_offsets+sample");
  al_sddh_offsets_kernel<<<ceil_div(cap, kSddhKp), 128, 0, st>>>(al->feat, H, W, al->kxy, count, cap, al->w0T, al->b0, al->w2, al->b2, kpts,
                                                                 al->off);
  DIMB_LAUNCH_CHECK(ctx);
  al_sddh_sample_kernel<<<cap, 128, 0, st>>>(al->feat, H, W, al->kxy, count, cap, al->off, al->fsh, exact ? al->fsl : nullptr);
  DIMB_LAUNCH_CHECK(ctx);
  }
  {  // sf_conv + SELU: [16 cap][128] x [128][128]^T
    EpiSeluSplit e;
    e.hi = al->f2h, e.lo = exact ? al->f2l : nullptr, e.count = count, e.rows_per_kp = 16, e.cap = cap, e.ldc = 128;
    TcOperands ops;
    ops.Ah = al->m_fs[0], ops.Al = al->m_fs[1], ops.Bh = al->m_sf[0], ops.Bl = al->m_sf[1];
    GemmArgs g{};
    g.num_kb = 2, g.M = cap * 16, g.N = 128;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, ceil_div(cap * 16, kTileM), 128, "al.sddh_sf_gemm")));
  }
  {  // aggregation einsum 'ncp,pcd->nd': [cap][2048] x [128][2048]^T
    EpiRowsF32 e;
    e.out = al->dsc, e.count = count, e.cap = cap;
    TcOperands ops;
    ops.Ah = al->m_f2[0], ops.Al = al->m_f2[1], ops.Bh = al->m_ag[0], ops.Bl = al->m_ag[1];
    GemmArgs g{};
    g.num_kb = 32, g.M = cap, g.N = 128;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, g, e, ceil_div(cap, kTileM), 128, "al.sddh_agg_gemm")));
  }
  ProfScope prof(ctx, st, "al.sddh_norm");
  al_sddh_norm_kernel<<<ceil_div(cap * 32, 256), 256, 0, st>>>(al->dsc, count, cap, desc);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
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
