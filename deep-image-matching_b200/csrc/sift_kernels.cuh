// sift_kernels.cuh - the per-keypoint and selection kernels of SIFT extraction and their launch helpers: sift_run (sift.cu) calls
// them on its pyramid, and the self-test library (selftest.cu, dimb_selftest_sift_*) calls the same helpers on caller-given levels,
// candidates and records.  See sift.cu for the stages and the OpenCV functions each one restates.
#pragma once
#include <algorithm>
#include <climits>
#include <cmath>

#include "common.cuh"
#include "detect.cuh"

namespace {

constexpr int kBorder = 5;          // SIFT_IMG_BORDER
constexpr int kMaxInterp = 5;       // SIFT_MAX_INTERP_STEPS
constexpr int kOriBins = 36;        // SIFT_ORI_HIST_BINS
constexpr int kDescHist = 6 * 6 * 10;  // (d + 2)^2 (n + 2) for d = 4, n = 8
constexpr int kWarps = 4;           // warps per CTA of the orientation and descriptor kernels
enum { kFx = 0, kFy, kFsize, kFangle, kFresp, kFoct, kNumFields };

// cv::fastAtan2 (hal fastAtan32f, degrees): a degree-7 polynomial; the histogram bins depend on it, so atan2f is not a substitute
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
  const float p1 = 0.9997878412794807f * 57.29577951308232f, p3 = -0.3258083974640975f * 57.29577951308232f;
  const float p5 = 0.1555786518463281f * 57.29577951308232f, p7 = -0.04432655554792128f * 57.29577951308232f;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + static_cast<float>(2.220446049250313e-16));
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + static_cast<float>(2.220446049250313e-16));
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

__device__ __forceinline__ int cv_round(float v) { return __float2int_rn(v); }

// ------------------------------------------------------------------ sift.extrema, sift.ori
struct Geo {
  int B, L, n_oct;
  float contrast, edge, sigma;
  int h[16], w[16];
  size_t gauss[16], dog[16];  // element offsets of each octave's level 0 ([levels][B][h][w])
};

__host__ __device__ __forceinline__ const float* level_ptr(const float* base, const Geo& g, bool is_dog, int o, int lv, int b) {
  const size_t plane = static_cast<size_t>(g.h[o]) * g.w[o];
  return base + (is_dog ? g.dog[o] : g.gauss[o]) + (static_cast<size_t>(lv) * g.B + b) * plane;
}

// adjustLocalExtrema: false when the candidate is dropped; on success r, c, layer, xc, xr, xi and contr are the refined values
__device__ bool sift_refine(const float* pyr, const Geo& g, int b, int o, int& layer, int& r, int& c, float& xc, float& xr, float& xi,
                            float& contr) {
  const float img_scale = 1.f / 255.f, deriv_scale = img_scale * 0.5f, second_scale = img_scale, cross_scale = img_scale * 0.25f;
  const int w = g.w[o], h = g.h[o];
  float dD[3];
  int i = 0;
  xi = xr = xc = 0.f;
  for (; i < kMaxInterp; ++i) {
    const float* img = level_ptr(pyr, g, true, o, layer, b);
    const float* prv = level_ptr(pyr, g, true, o, layer - 1, b);
    const float* nxt = level_ptr(pyr, g, true, o, layer + 1, b);
    auto I = [&](const float* p, int y, int x) { return p[static_cast<size_t>(y) * w + x]; };
    dD[0] = (I(img, r, c + 1) - I(img, r, c - 1)) * deriv_scale;
    dD[1] = (I(img, r + 1, c) - I(img, r - 1, c)) * deriv_scale;
    dD[2] = (I(nxt, r, c) - I(prv, r, c)) * deriv_scale;
    const float v2 = I(img, r, c) * 2.f;
    const float dxx = (I(img, r, c + 1) + I(img, r, c - 1) - v2) * second_scale;
    const float dyy = (I(img, r + 1, c) + I(img, r - 1, c) - v2) * second_scale;
    const float dss = (I(nxt, r, c) + I(prv, r, c) - v2) * second_scale;
    const float dxy = (I(img, r + 1, c + 1) - I(img, r + 1, c - 1) - I(img, r - 1, c + 1) + I(img, r - 1, c - 1)) * cross_scale;
    const float dxs = (I(nxt, r, c + 1) - I(nxt, r, c - 1) - I(prv, r, c + 1) + I(prv, r, c - 1)) * cross_scale;
    const float dys = (I(nxt, r + 1, c) - I(nxt, r - 1, c) - I(prv, r + 1, c) + I(prv, r - 1, c)) * cross_scale;
    // Matx33f::solve(DECOMP_LU) of a 3x3 system: Cramer's rule in float, zeros when the determinant is 0
    const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
    float X0 = 0.f, X1 = 0.f, X2 = 0.f;
    float d = a00 * (a11 * a22 - a21 * a12) - a01 * (a10 * a22 - a20 * a12) + a02 * (a10 * a21 - a20 * a11);
    if (d != 0.f) {
      d = 1.f / d;
      const float b0 = dD[0], b1 = dD[1], b2 = dD[2];
      X0 = d * (b0 * (a11 * a22 - a12 * a21) - a01 * (b1 * a22 - a12 * b2) + a02 * (b1 * a21 - a11 * b2));
      X1 = d * (a00 * (b1 * a22 - a12 * b2) - b0 * (a10 * a22 - a12 * a20) + a02 * (a10 * b2 - b1 * a20));
      X2 = d * (a00 * (a11 * b2 - b1 * a21) - a01 * (a10 * b2 - b1 * a20) + b0 * (a10 * a21 - a11 * a20));
    }
    xi = -X2, xr = -X1, xc = -X0;
    if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
    const float big = static_cast<float>(INT_MAX / 3);
    if (fabsf(xi) > big || fabsf(xr) > big || fabsf(xc) > big) return false;
    c += cv_round(xc);
    r += cv_round(xr);
    layer += cv_round(xi);
    if (layer < 1 || layer > g.L || c < kBorder || c >= w - kBorder || r < kBorder || r >= h - kBorder) return false;
  }
  if (i >= kMaxInterp) return false;
  const float* img = level_ptr(pyr, g, true, o, layer, b);
  const float* prv = level_ptr(pyr, g, true, o, layer - 1, b);
  const float* nxt = level_ptr(pyr, g, true, o, layer + 1, b);
  auto I = [&](const float* p, int y, int x) { return p[static_cast<size_t>(y) * w + x]; };
  dD[0] = (I(img, r, c + 1) - I(img, r, c - 1)) * deriv_scale;
  dD[1] = (I(img, r + 1, c) - I(img, r - 1, c)) * deriv_scale;
  dD[2] = (I(nxt, r, c) - I(prv, r, c)) * deriv_scale;
  const float t = dD[0] * xc + dD[1] * xr + dD[2] * xi;
  contr = I(img, r, c) * img_scale + t * 0.5f;
  if (fabsf(contr) * g.L < g.contrast) return false;
  const float v2 = I(img, r, c) * 2.f;
  const float dxx = (I(img, r, c + 1) + I(img, r, c - 1) - v2) * second_scale;
  const float dyy = (I(img, r + 1, c) + I(img, r - 1, c) - v2) * second_scale;
  const float dxy = (I(img, r + 1, c + 1) - I(img, r + 1, c - 1) - I(img, r - 1, c + 1) + I(img, r - 1, c - 1)) * cross_scale;
  const float tr = dxx + dyy, det = dxx * dyy - dxy * dxy;
  if (det <= 0 || tr * tr * g.edge >= (g.edge + 1) * (g.edge + 1) * det) return false;
  return true;
}

// ------------------------------------------------------------------ sift.extrema
// A refined extremum (adjustLocalExtrema passed): the integer position after interpolation and its offsets and contrast
struct Cand {
  unsigned ol;  // octave << 8 | layer
  unsigned rc;  // row << 16 | column
  float xc, xr, xi, contr;
};

// DoG layers 1..L of octave o: 26-neighbour extrema (>= / <= every neighbour, above thr), each refined by the thread that found it;
// only the extrema that pass the interpolation, contrast and edge tests are appended, so flat DoG plateaus (every pixel an
// extremum, all rejected by the contrast test) take no buffer space
__global__ void sift_extrema_kernel(const float* __restrict__ pyr, Geo g, int o, float thr, Cand* __restrict__ cand,
                                    int* __restrict__ cand_count, int ccap) {
  const int B = g.B, h = g.h[o], w = g.w[o];
  const int c = blockIdx.x * blockDim.x + threadIdx.x + kBorder, r = blockIdx.y + kBorder;
  const int b = blockIdx.z % B, layer = blockIdx.z / B + 1;
  if (c >= w - kBorder) return;
  const size_t lvl = static_cast<size_t>(h) * w * B;
  const float* cur = level_ptr(pyr, g, true, o, layer, b) + static_cast<size_t>(r) * w + c;
  const float val = *cur;
  if (!(fabsf(val) > thr)) return;
  bool ext = true;
  if (val > 0) {
    for (int dl = -1; dl <= 1 && ext; ++dl)
      for (int dy = -1; dy <= 1 && ext; ++dy)
        for (int dx = -1; dx <= 1; ++dx)
          if (!(val >= cur[dl * static_cast<ptrdiff_t>(lvl) + dy * w + dx])) {
            ext = false;
            break;
          }
  } else {
    for (int dl = -1; dl <= 1 && ext; ++dl)
      for (int dy = -1; dy <= 1 && ext; ++dy)
        for (int dx = -1; dx <= 1; ++dx)
          if (!(val <= cur[dl * static_cast<ptrdiff_t>(lvl) + dy * w + dx])) {
            ext = false;
            break;
          }
  }
  if (!ext) return;
  int ly = layer, rr = r, cc = c;
  float xc, xr, xi, contr;
  if (!sift_refine(pyr, g, b, o, ly, rr, cc, xc, xr, xi, contr)) return;
  const int slot = atomicAdd(&cand_count[b], 1);
  if (slot < ccap)
    cand[static_cast<size_t>(b) * ccap + slot] = Cand{static_cast<unsigned>(o << 8 | ly), static_cast<unsigned>(rr << 16 | cc), xc, xr, xi, contr};
}

// Keypoint records: rec [B][kNumFields][kcap] (float fields; the packed octave as int bits), before the final 0.5 scaling
__global__ void __launch_bounds__(kWarps * 32) sift_ori_kernel(const float* __restrict__ pyr, Geo g, const Cand* __restrict__ cand,
                                                             const int* __restrict__ cand_count, int ccap, float* __restrict__ rec,
                                                             int* __restrict__ kp_count, int kcap) {
  const int b = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int n = min(cand_count[b], ccap);
  __shared__ float hist_s[kWarps][kOriBins + 4];
  __shared__ float stage_w[kWarps][32];
  __shared__ int stage_b[kWarps][32];
  float* temphist = hist_s[wid] + 2;
  for (int ci = blockIdx.x * kWarps + wid; ci < n; ci += gridDim.x * kWarps) {
    const Cand cd = cand[static_cast<size_t>(b) * ccap + ci];
    const int o = cd.ol >> 8, layer = cd.ol & 255, r = cd.rc >> 16, c = cd.rc & 0xffff;
    const float xc = cd.xc, xr = cd.xr, xi = cd.xi, contr = cd.contr;
    const float size = g.sigma * powf(2.f, (layer + xi) / g.L) * static_cast<float>(1 << o) * 2.f;
    const float scl_octv = size * 0.5f / static_cast<float>(1 << o);
    const int radius = cv_round(4.5f * scl_octv);
    const float sig = 1.5f * scl_octv, expf_scale = -1.f / (2.f * sig * sig);
    const float* img = level_ptr(pyr, g, false, o, layer, b);
    const int w = g.w[o], h = g.h[o];
    for (int i = lane; i < kOriBins + 4; i += 32) hist_s[wid][i] = 0.f;
    __syncwarp();
    const int side = 2 * radius + 1, len = side * side;
    for (int base = 0; base < len; base += 32) {
      const int p = base + lane;
      int bin = -1;
      float wm = 0.f;
      if (p < len) {
        const int i = p / side - radius, j = p % side - radius;
        const int y = r + i, x = c + j;
        if (y > 0 && y < h - 1 && x > 0 && x < w - 1) {
          const float dx = img[static_cast<size_t>(y) * w + x + 1] - img[static_cast<size_t>(y) * w + x - 1];
          const float dy = img[static_cast<size_t>(y - 1) * w + x] - img[static_cast<size_t>(y + 1) * w + x];
          const float wt = expf((i * i + j * j) * expf_scale);
          const float ori = fast_atan2_deg(dy, dx), mag = sqrtf(dx * dx + dy * dy);
          bin = cv_round((kOriBins / 360.f) * ori);
          if (bin >= kOriBins) bin -= kOriBins;
          if (bin < 0) bin += kOriBins;
          wm = wt * mag;
        }
      }
      stage_b[wid][lane] = bin;
      stage_w[wid][lane] = wm;
      __syncwarp();
      if (lane == 0)  // in sample order, as the sequential loop of calcOrientationHist
        for (int q = 0; q < 32; ++q)
          if (stage_b[wid][q] >= 0) temphist[stage_b[wid][q]] += stage_w[wid][q];
      __syncwarp();
    }
    if (lane == 0) {
      temphist[-1] = temphist[kOriBins - 1];
      temphist[-2] = temphist[kOriBins - 2];
      temphist[kOriBins] = temphist[0];
      temphist[kOriBins + 1] = temphist[1];
      float hist[kOriBins];
      float omax = 0.f;
      for (int i = 0; i < kOriBins; ++i) {
        hist[i] = (temphist[i - 2] + temphist[i + 2]) * (1.f / 16.f) + (temphist[i - 1] + temphist[i + 1]) * (4.f / 16.f) +
                  temphist[i] * (6.f / 16.f);
        omax = i == 0 ? hist[0] : fmaxf(omax, hist[i]);
      }
      const float mag_thr = omax * 0.8f;
      const float kx = (c + xc) * static_cast<float>(1 << o), ky = (r + xr) * static_cast<float>(1 << o);
      const int oct = o + (layer << 8) + (static_cast<int>(rint((xi + 0.5) * 255)) << 16);
      float* rb = rec + static_cast<size_t>(b) * kNumFields * kcap;
      for (int j = 0; j < kOriBins; ++j) {
        const int l = j > 0 ? j - 1 : kOriBins - 1, r2 = j < kOriBins - 1 ? j + 1 : 0;
        if (hist[j] > hist[l] && hist[j] > hist[r2] && hist[j] >= mag_thr) {
          float bin = j + 0.5f * (hist[l] - hist[r2]) / (hist[l] - 2 * hist[j] + hist[r2]);
          bin = bin < 0 ? kOriBins + bin : bin >= kOriBins ? bin - kOriBins : bin;
          float angle = 360.f - (360.f / kOriBins) * bin;
          if (fabsf(angle - 360.f) < 1.1920929e-7f) angle = 0.f;
          const int slot = atomicAdd(&kp_count[b], 1);
          if (slot < kcap) {
            rb[kFx * static_cast<size_t>(kcap) + slot] = kx;
            rb[kFy * static_cast<size_t>(kcap) + slot] = ky;
            rb[kFsize * static_cast<size_t>(kcap) + slot] = size;
            rb[kFangle * static_cast<size_t>(kcap) + slot] = angle;
            rb[kFresp * static_cast<size_t>(kcap) + slot] = fabsf(contr);
            rb[kFoct * static_cast<size_t>(kcap) + slot] = __int_as_float(oct);
          }
        }
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------ sift.select
// per image: keypoints to sort (0 when a buffer overflowed) into the sort state word detect.cuh's radix passes read
__global__ void sift_select_init_kernel(const int* __restrict__ cand_count, const int* __restrict__ kp_count, int ccap, int kcap,
                                        unsigned* __restrict__ state, int* __restrict__ n_sorted, int* __restrict__ ovf) {
  const int b = blockIdx.x;
  if (threadIdx.x) return;
  const bool over = cand_count[b] > ccap || kp_count[b] > kcap;
  ovf[b] = over;
  n_sorted[b] = over ? 0 : kp_count[b];
  state[b * kTkState + kTkSort] = over ? 0u : static_cast<unsigned>(kp_count[b]);
}

// 32-bit sort key of field f, ascending in KeyPoint_LessThan's order (every field is >= 0, so float bits order as the floats)
__device__ __forceinline__ unsigned field_key(const float* rb, int kcap, int f, int idx) {
  const unsigned u = __float_as_uint(rb[static_cast<size_t>(f) * kcap + idx]);
  return (f == kFsize || f == kFresp || f == kFoct) ? ~u : u;
}

__global__ void sift_sort_keys_kernel(const float* __restrict__ rec, const int* __restrict__ n_sorted, unsigned long long* __restrict__ keys,
                                      int kcap, int f, int first) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_sorted[b]) return;
  unsigned long long* k = keys + static_cast<size_t>(b) * kcap;
  const int idx = first ? i : static_cast<int>(k[i] & 0xffffffffull);
  k[i] = static_cast<unsigned long long>(field_key(rec + static_cast<size_t>(b) * kNumFields * kcap, kcap, f, idx)) << 32 |
         static_cast<unsigned>(idx);
}

// Ordered compaction in chunks of kChunk: mode 0 (removeDuplicatedSorted) walks the sorted keys and keeps a keypoint unless its
// (x, y, size, angle) equals its predecessor's; mode 1 (retainBest) walks the deduplicated list and keeps responses >= the
// radix-selected threshold when the image has more than n_features keypoints.
template <int MODE>
__device__ __forceinline__ bool sift_keep(const float* rb, int kcap, const unsigned long long* keys, const int* sel, const float* resp,
                                          const unsigned* st, int i) {
  if (MODE == 0) {
    if (i == 0) return true;
    const int a = static_cast<int>(keys[i] & 0xffffffffull), p = static_cast<int>(keys[i - 1] & 0xffffffffull);
    for (int f = kFx; f <= kFangle; ++f)
      if (rb[static_cast<size_t>(f) * kcap + a] != rb[static_cast<size_t>(f) * kcap + p]) return true;
    return false;
  }
  return !st[kTkSelect] || __float_as_uint(resp[i]) >= st[kTkPrefix];
}

template <int MODE>
__global__ void __launch_bounds__(256) sift_compact_count_kernel(const float* __restrict__ rec, const unsigned long long* __restrict__ keys,
                                                                 const int* __restrict__ sel, const float* __restrict__ resp,
                                                                 const unsigned* __restrict__ state, const int* __restrict__ n_in,
                                                                 int* __restrict__ chunk_cnt, int kcap, int nchunks) {
  const int b = blockIdx.y, chunk = blockIdx.x, n = n_in[b];
  if (chunk * kChunk >= n) return;
  const float* rb = rec + static_cast<size_t>(b) * kNumFields * kcap;
  const size_t off = static_cast<size_t>(b) * kcap;
  int cnt = 0;
  for (int q = 0; q < kChunk / 256; ++q) {
    const int i = chunk * kChunk + threadIdx.x * (kChunk / 256) + q;
    if (i < n) cnt += sift_keep<MODE>(rb, kcap, keys + off, sel + off, resp + off, state + b * kTkState, i);
  }
  __shared__ int red[8];
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    chunk_cnt[b * nchunks + chunk] = t;
  }
}

__global__ void sift_compact_scan_kernel(int* __restrict__ chunk_cnt, const int* __restrict__ n_in, int* __restrict__ n_out, int nchunks) {
  const int b = blockIdx.x;
  if (threadIdx.x) return;
  int run = 0;
  for (int i = 0; i < ceil_div(n_in[b], kChunk); ++i) {
    const int c = chunk_cnt[b * nchunks + i];
    chunk_cnt[b * nchunks + i] = run;
    run += c;
  }
  n_out[b] = run;
}

struct SiftOut {
  float *kpts, *desc, *frames;
  int *octave, *counts;
  int cap;
};

// MODE 0 writes sel (record index) and resp of the deduplicated list; MODE 1 writes the outputs (x, y, size scaled by 0.5, the
// octave field with octave - 1, as detectAndCompute does for firstOctave = -1) and the record index of each output row to sel_out
template <int MODE>
__global__ void __launch_bounds__(256) sift_compact_write_kernel(const float* __restrict__ rec, const unsigned long long* __restrict__ keys,
                                                                 int* __restrict__ sel, float* __restrict__ resp,
                                                                 const unsigned* __restrict__ state, const int* __restrict__ n_in,
                                                                 const int* __restrict__ chunk_off, int* __restrict__ sel_out,
                                                                 const int* __restrict__ ovf, SiftOut out, const int* __restrict__ n_out,
                                                                 int kcap, int nchunks) {
  const int b = blockIdx.y, chunk = blockIdx.x, n = n_in[b];
  if (MODE == 1 && chunk == 0 && threadIdx.x == 0) out.counts[b] = ovf[b] ? -1 : n_out[b];
  if (chunk * kChunk >= n) return;
  const float* rb = rec + static_cast<size_t>(b) * kNumFields * kcap;
  const size_t off = static_cast<size_t>(b) * kcap;
  constexpr int kPer = kChunk / 256;
  bool keep[kPer];
  int cnt = 0;
  const int i0 = chunk * kChunk + threadIdx.x * kPer;
  for (int q = 0; q < kPer; ++q) {
    const int i = i0 + q;
    keep[q] = i < n && sift_keep<MODE>(rb, kcap, keys + off, sel + off, resp + off, state + b * kTkState, i);
    cnt += keep[q];
  }
  __shared__ int wsum[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) wsum[wid] = inc;
  __syncthreads();
  int pos = chunk_off[b * nchunks + chunk] + inc - cnt;
  for (int q = 0; q < wid; ++q) pos += wsum[q];
  for (int q = 0; q < kPer; ++q) {
    if (!keep[q]) continue;
    const int i = i0 + q;
    if (MODE == 0) {
      const int idx = static_cast<int>(keys[off + i] & 0xffffffffull);
      sel_out[off + pos] = idx;
      resp[off + pos] = rb[static_cast<size_t>(kFresp) * kcap + idx];
    } else if (pos < out.cap) {
      const int idx = sel[off + i];
      auto F = [&](int f) { return rb[static_cast<size_t>(f) * kcap + idx]; };
      const size_t ob = static_cast<size_t>(b) * out.cap + pos;
      out.kpts[ob * 2] = F(kFx) * 0.5f;
      out.kpts[ob * 2 + 1] = F(kFy) * 0.5f;
      if (out.frames) {
        out.frames[ob * 3] = F(kFsize) * 0.5f;
        out.frames[ob * 3 + 1] = F(kFangle);
        out.frames[ob * 3 + 2] = F(kFresp);
      }
      const int oct = __float_as_int(F(kFoct));
      if (out.octave) out.octave[ob] = (oct & ~255) | ((oct - 1) & 255);
      sel_out[ob] = idx;
    }
    ++pos;
  }
}

// ------------------------------------------------------------------ sift.desc
// calcSIFTDescriptor(img, ptf, 360 - angle, size / 2, d = 4, n = 8) of the output rows, one warp per keypoint: the lanes compute
// samples 32 at a time and lanes 0..7 add the eight trilinear shares of each sample, in sample order, to the histogram
__global__ void __launch_bounds__(kWarps * 32) sift_desc_kernel(const float* __restrict__ pyr, Geo g, const float* __restrict__ rec,
                                                              const int* __restrict__ sel_out, const int* __restrict__ counts, int kcap,
                                                              float* __restrict__ desc, int cap) {
  const int b = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int n = min(counts[b], cap);
  __shared__ float hist_s[kWarps][kDescHist];
  __shared__ float stage_v[kWarps][32][8];
  __shared__ int stage_i[kWarps][32];
  float* hist = hist_s[wid];
  const float* rb = rec + static_cast<size_t>(b) * kNumFields * kcap;
  constexpr int d = 4, nb = 8;
  for (int row = blockIdx.x * kWarps + wid; row < n; row += gridDim.x * kWarps) {
    const int idx = sel_out[static_cast<size_t>(b) * cap + row];
    auto F = [&](int f) { return rb[static_cast<size_t>(f) * kcap + idx]; };
    const int oct = __float_as_int(F(kFoct));
    const int o = oct & 255, layer = (oct >> 8) & 255;
    // unpackOctave of the scaled keypoint: octave o - 1, scale 2 for octave -1, else 1 / 2^(o - 1)
    const float scale = o == 0 ? 2.f : 1.f / static_cast<float>(1 << (o - 1));
    const float size = F(kFsize) * 0.5f * scale;
    const float ptx = F(kFx) * 0.5f * scale, pty = F(kFy) * 0.5f * scale;
    float ori = 360.f - F(kFangle);
    if (fabsf(ori - 360.f) < 1.1920929e-7f) ori = 0.f;
    const float scl = size * 0.5f;
    const float* img = level_ptr(pyr, g, false, o, layer, b);
    const int w = g.w[o], h = g.h[o];
    const int px = cv_round(ptx), py = cv_round(pty);
    float cos_t = cosf(ori * static_cast<float>(3.141592653589793 / 180)), sin_t = sinf(ori * static_cast<float>(3.141592653589793 / 180));
    const float bins_per_rad = nb / 360.f, exp_scale = -1.f / (d * d * 0.5f), hist_width = 3.f * scl;
    int radius = cv_round(hist_width * 1.4142135623730951f * (d + 1) * 0.5f);
    radius = min(radius, static_cast<int>(sqrt(static_cast<double>(w) * w + static_cast<double>(h) * h)));
    cos_t /= hist_width;
    sin_t /= hist_width;
    for (int i = lane; i < kDescHist; i += 32) hist[i] = 0.f;
    __syncwarp();
    const int side = 2 * radius + 1, len = side * side;
    for (int base = 0; base < len; base += 32) {
      const int p = base + lane;
      int hidx = -1;
      float v[8];
      if (p < len) {
        const int i = p / side - radius, j = p % side - radius;
        const float c_rot = j * cos_t - i * sin_t, r_rot = j * sin_t + i * cos_t;
        float rbin = r_rot + d / 2 - 0.5f, cbin = c_rot + d / 2 - 0.5f;
        const int y = py + i, x = px + j;
        if (rbin > -1 && rbin < d && cbin > -1 && cbin < d && y > 0 && y < h - 1 && x > 0 && x < w - 1) {
          const float dx = img[static_cast<size_t>(y) * w + x + 1] - img[static_cast<size_t>(y) * w + x - 1];
          const float dy = img[static_cast<size_t>(y - 1) * w + x] - img[static_cast<size_t>(y + 1) * w + x];
          const float wt = expf((c_rot * c_rot + r_rot * r_rot) * exp_scale);
          float obin = (fast_atan2_deg(dy, dx) - ori) * bins_per_rad;
          const float mag = sqrtf(dx * dx + dy * dy) * wt;
          const int r0 = static_cast<int>(floorf(rbin)), c0 = static_cast<int>(floorf(cbin));
          int o0 = static_cast<int>(floorf(obin));
          rbin -= r0, cbin -= c0, obin -= o0;
          if (o0 < 0) o0 += nb;
          if (o0 >= nb) o0 -= nb;
          const float v_r1 = mag * rbin, v_r0 = mag - v_r1;
          const float v_rc11 = v_r1 * cbin, v_rc10 = v_r1 - v_rc11, v_rc01 = v_r0 * cbin, v_rc00 = v_r0 - v_rc01;
          v[7] = v_rc11 * obin, v[6] = v_rc11 - v[7];
          v[5] = v_rc10 * obin, v[4] = v_rc10 - v[5];
          v[3] = v_rc01 * obin, v[2] = v_rc01 - v[3];
          v[1] = v_rc00 * obin, v[0] = v_rc00 - v[1];
          hidx = ((r0 + 1) * (d + 2) + c0 + 1) * (nb + 2) + o0;
        }
      }
      stage_i[wid][lane] = hidx;
      if (hidx >= 0)
        for (int q = 0; q < 8; ++q) stage_v[wid][lane][q] = v[q];
      __syncwarp();
      if (lane < 8) {
        // corner q = (r, c, o) bits (4, 2, 1) of v_rco[r][c][o] -> offsets of the eight histogram updates
        const int dr = lane >> 2, dc = (lane >> 1) & 1, dq = lane & 1;
        const int add = dr * (d + 2) * (nb + 2) + dc * (nb + 2) + dq;
        for (int s = 0; s < 32; ++s) {
          const int hi = stage_i[wid][s];
          if (hi >= 0) hist[hi + add] += stage_v[wid][s][lane];
          __syncwarp(0xffu);  // a bin shared by two samples takes their shares in sample order
        }
      }
      __syncwarp();
    }
    // wrap the circular orientation bins, then 0.2 clamp, 512 / norm and saturation, four outputs per lane
    float val[4];
    float nrm = 0.f;
    for (int q = 0; q < 4; ++q) {
      const int k = lane * 4 + q, cell = k / nb, ob = k % nb, i = cell / d, j = cell % d;
      const int hb = ((i + 1) * (d + 2) + (j + 1)) * (nb + 2);
      val[q] = hist[hb + ob] + (ob < 2 ? hist[hb + nb + ob] : 0.f);
      nrm += val[q] * val[q];
    }
    for (int o2 = 16; o2; o2 >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o2);
    const float thr = sqrtf(nrm) * 0.2f;
    nrm = 0.f;
    for (int q = 0; q < 4; ++q) {
      val[q] = fminf(val[q], thr);
      nrm += val[q] * val[q];
    }
    for (int o2 = 16; o2; o2 >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o2);
    const float f = 512.f / fmaxf(sqrtf(nrm), 1.1920929e-7f);
    for (int q = 0; q < 4; ++q)
      desc[(static_cast<size_t>(b) * 128 + lane * 4 + q) * cap + row] = fminf(fmaxf(rintf(val[q] * f), 0.f), 255.f);
    __syncwarp();
  }
}

// ------------------------------------------------------------------ launch helpers
// findScaleSpaceExtrema's integer threshold of the 26-neighbour test: floor(0.5 * contrastThreshold / nOctaveLayers * 255)
inline float sift_extrema_thr(double contrast, int L) {
  return static_cast<float>(static_cast<int>(std::floor(0.5 * contrast / L * 255)));
}

// sift.extrema over every octave larger than 2 kBorder pixels each way: refined candidates of image b go to cand [b][ccap] in
// atomic order; cand_count [B] (zero on entry) counts every survivor, stored or not
inline int launch_sift_extrema(dimb_ctx* ctx, cudaStream_t st, const float* pyr, const Geo& g, float thr, Cand* cand, int* cand_count,
                               int ccap) {
  for (int o = 0; o < g.n_oct; ++o) {
    if (g.h[o] <= 2 * kBorder || g.w[o] <= 2 * kBorder) continue;
    const dim3 grid(ceil_div(g.w[o] - 2 * kBorder, 128), g.h[o] - 2 * kBorder, g.B * g.L);
    sift_extrema_kernel<<<grid, 128, 0, st>>>(pyr, g, o, thr, cand, cand_count, ccap);
    DIMB_LAUNCH_CHECK(ctx);
  }
  return DIMB_OK;
}

// sift.ori: the first min(cand_count[b], ccap) candidates of each image -> records rec [B][kNumFields][kcap] in atomic order;
// kp_count [B] (zero on entry) counts every keypoint, stored or not
inline int launch_sift_ori(dimb_ctx* ctx, cudaStream_t st, const float* pyr, const Geo& g, const Cand* cand, const int* cand_count, int ccap,
                           float* rec, int* kp_count, int kcap) {
  const int B = g.B;
  const int blocks = std::max(1, std::min(ceil_div(ccap, kWarps), 4 * ctx->num_sms * 8 / std::max(B, 1)));
  sift_ori_kernel<<<dim3(blocks, B), kWarps * 32, 0, st>>>(pyr, g, cand, cand_count, ccap, rec, kp_count, kcap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// Scratch of sift.select, per image: n_sorted, n_dedup, ovf, dummy [B]; sel, resp, keys0, keys1 [B][kcap]; chunk
// [B][ceil(kcap / kChunk)]; digit_off [B][ceil(kcap / kSortTile)][256]; state [B][kTkState]; hist [B][256].  sel_out [B][out.cap]
// receives the record index of each output row.
struct SiftSelectBufs {
  int *n_sorted, *n_dedup, *ovf, *dummy, *sel, *chunk, *digit_off, *sel_out;
  float* resp;
  unsigned *state, *hist;
  unsigned long long *keys0, *keys1;
};

// sift.select: sort the records of each image, drop duplicates, retainBest(n_features) (0: keep all), and write the output rows of
// `out` (counts -1 for an image whose candidate or keypoint count exceeded ccap or kcap)
inline int launch_sift_select(dimb_ctx* ctx, cudaStream_t st, int B, const float* rec, const int* cand_count, const int* kp_count, int ccap,
                              int kcap, int n_features, const SiftSelectBufs& s, const SiftOut& out) {
  sift_select_init_kernel<<<B, 32, 0, st>>>(cand_count, kp_count, ccap, kcap, s.state, s.n_sorted, s.ovf);
  DIMB_LAUNCH_CHECK(ctx);
  // stable LSD passes, least significant field first: the keys carry the record index in their low word
  const int nblk = ceil_div(kcap, kSortTile);
  const dim3 kg(ceil_div(kcap, 256), B), sg(nblk, B);
  const int order[kNumFields] = {kFoct, kFresp, kFangle, kFsize, kFy, kFx};
  for (int fi = 0; fi < kNumFields; ++fi) {
    sift_sort_keys_kernel<<<kg, 256, 0, st>>>(rec, s.n_sorted, s.keys0, kcap, order[fi], fi == 0);
    DIMB_LAUNCH_CHECK(ctx);
    for (int pass = 0; pass < 4; ++pass) {
      const unsigned long long* src = pass & 1 ? s.keys1 : s.keys0;
      unsigned long long* dst = pass & 1 ? s.keys0 : s.keys1;
      const int shift = 32 + 8 * pass;
      topk_sort_pass_kernel<false><<<sg, kTopkThreads, 0, st>>>(src, dst, nullptr, nullptr, s.digit_off, s.state, kcap, 0, nblk, shift);
      DIMB_LAUNCH_CHECK(ctx);
      topk_sort_scan_kernel<<<B, 256, 0, st>>>(s.digit_off, s.state, nblk);
      DIMB_LAUNCH_CHECK(ctx);
      topk_sort_pass_kernel<true><<<sg, kTopkThreads, 0, st>>>(src, dst, nullptr, nullptr, s.digit_off, s.state, kcap, 0, nblk, shift);
      DIMB_LAUNCH_CHECK(ctx);
    }
  }
  const int nch = ceil_div(kcap, kChunk);
  const dim3 cg(nch, B);
  sift_compact_count_kernel<0><<<cg, 256, 0, st>>>(rec, s.keys0, s.sel, s.resp, s.state, s.n_sorted, s.chunk, kcap, nch);
  DIMB_LAUNCH_CHECK(ctx);
  sift_compact_scan_kernel<<<B, 32, 0, st>>>(s.chunk, s.n_sorted, s.n_dedup, nch);
  DIMB_LAUNCH_CHECK(ctx);
  sift_compact_write_kernel<0><<<cg, 256, 0, st>>>(rec, s.keys0, nullptr, s.resp, s.state, s.n_sorted, s.chunk, s.sel, s.ovf, out, s.n_dedup,
                                                   kcap, nch);
  DIMB_LAUNCH_CHECK(ctx);
  // retainBest: the n_features-th largest response by detect.cuh's radix select (kTkSelect = more than n_features remain)
  const int K = n_features > 0 ? n_features : INT_MAX;
  topk_init_kernel<<<B, kTopkThreads, 0, st>>>(s.n_dedup, K, 0, s.hist, s.state, s.dummy);
  DIMB_LAUNCH_CHECK(ctx);
  if (n_features > 0) {
    const dim3 hg(std::min(kTopkSelGrid, ceil_div(kcap, kTopkThreads * 16)), B);
    for (int shift = 24; shift >= 0; shift -= 8) {
      topk_hist_kernel<<<hg, kTopkThreads, 0, st>>>(s.resp, s.n_dedup, s.state, s.hist, kcap, shift);
      DIMB_LAUNCH_CHECK(ctx);
      topk_digit_kernel<<<B, kTopkThreads, 0, st>>>(s.hist, s.state, shift);
      DIMB_LAUNCH_CHECK(ctx);
    }
  }
  sift_compact_count_kernel<1><<<cg, 256, 0, st>>>(rec, s.keys0, s.sel, s.resp, s.state, s.n_dedup, s.chunk, kcap, nch);
  DIMB_LAUNCH_CHECK(ctx);
  sift_compact_scan_kernel<<<B, 32, 0, st>>>(s.chunk, s.n_dedup, s.n_sorted, nch);  // n_sorted now holds the kept counts
  DIMB_LAUNCH_CHECK(ctx);
  sift_compact_write_kernel<1><<<cg, 256, 0, st>>>(rec, s.keys0, s.sel, s.resp, s.state, s.n_dedup, s.chunk, s.sel_out, s.ovf, out,
                                                   s.n_sorted, kcap, nch);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// sift.desc: descriptors out.desc [B][128][out.cap] of the first min(out.counts[b], out.cap) output rows, row k being record
// sel_out[b][k] of rec [B][kNumFields][kcap]
inline int launch_sift_desc(dimb_ctx* ctx, cudaStream_t st, const float* pyr, const Geo& g, const float* rec, const int* sel_out, int kcap,
                            const SiftOut& out) {
  const int B = g.B;
  const int blocks = std::max(1, std::min(ceil_div(out.cap, kWarps), 4 * ctx->num_sms * 8 / std::max(B, 1)));
  sift_desc_kernel<<<dim3(blocks, B), kWarps * 32, 0, st>>>(pyr, g, rec, sel_out, out.counts, kcap, out.desc, out.cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
