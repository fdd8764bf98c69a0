// sift.cu - SIFT extraction as cv2.SIFT_create(nfeatures, nOctaveLayers, contrastThreshold, edgeThreshold, sigma)
// .detectAndCompute(gray_uint8, None) computes it (OpenCV 4.x sift.simd.hpp, enable_precise_upscale = false), batched over B images
// of one size on one stream, with no host synchronisation inside an extraction.
//
// Stages (profile groups):
//   sift.pyr      uint8 conversion, 2x INTER_LINEAR upsampling, the separable Gaussian blurs (BORDER_REFLECT_101), the every-other-
//                 pixel octave starts and the DoG levels;
//   sift.extrema  26-neighbour extrema outside a 5-pixel border; the thread that finds one runs the interpolation (up to 5 steps,
//                 3x3 Cramer solve) and the contrast and edge tests, and appends a survivor per image with an atomic counter;
//   sift.ori      one warp per refined extremum builds the 36-bin orientation histogram in sample order, and every peak >= 0.8 of
//                 the maximum is appended as its own keypoint;
//   sift.select   the keypoints of each image are sorted under a total order (x asc, y asc, size desc, angle asc, response desc,
//                 packed octave desc: KeyPoint_LessThan of removeDuplicatedSorted) by stable 8-bit LSD radix passes over the six
//                 fields, duplicates in (x, y, size, angle) dropped, then retainBest(n_features): the n-th largest response is found
//                 by detect.cuh's radix select and every keypoint at or above it is kept (ties at the boundary included), in the
//                 sorted order.  The atomic appends above make the buffer order run-dependent; the sort makes the output not.
//   sift.desc     one warp per output keypoint: 4 x 4 x 8 histogram with trilinear weights, accumulated in sample order, the 0.2
//                 clamp, the factor 512 and saturation to 0..255.
//
// Memory (per image, sized at create time for max_height x max_width): nOctaveLayers + 3 Gaussian and nOctaveLayers + 2 DoG levels
// per octave plus one octave -1 level of blur scratch, float32; octave -1 is 2H x 2W (50 MB per level at 2048 x 1536), every later
// octave a quarter of the one before.  The refined-extremum and keypoint buffers hold one entry per 16 pixels of the nOctaveLayers
// searched DoG levels (about 72 bytes per entry); a fuller image is reported (count -1) rather than cut.  At 2048 x 1536 and 3 layers that is
// about 0.8 GB of pyramid and 0.23 GB of keypoint buffers per image.
#include <algorithm>
#include <cmath>
#include <climits>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "detect.cuh"
#include "sift_kernels.cuh"

namespace {

constexpr int kMaxTaps = 127;       // largest Gaussian kernel the blur kernels take (radius 63)
constexpr int kCandDiv = 16;        // one candidate / keypoint slot per kCandDiv searched DoG pixels

struct Taps {
  float k[kMaxTaps / 2 + 1];  // k[0] centre, k[j] = k[-j]
  int r;
};

__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while (static_cast<unsigned>(p) >= static_cast<unsigned>(len)) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// ------------------------------------------------------------------ sift.pyr
// convertTo(CV_8U) of the input (round half to even, saturate), then resize(2W, 2H, INTER_LINEAR): source coordinate
// (d + 0.5) / 2 - 0.5 clamped at the edges.  Every product and sum is exact (weights 1/4, 3/4 on integers).
template <class T>
__global__ void sift_upsample_kernel(const T* __restrict__ src, float* __restrict__ dst, int H, int W) {
  const int W2 = 2 * W, H2 = 2 * H;
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y, b = blockIdx.z;
  if (dx >= W2) return;
  const T* s = src + static_cast<size_t>(b) * H * W;
  auto px = [&](int y, int x) -> float {
    float v = static_cast<float>(s[static_cast<size_t>(y) * W + x]);
    return fminf(fmaxf(rintf(v), 0.f), 255.f);
  };
  auto coord = [](int d, int n, int& s0, float& a) {
    const float f = (d + 0.5f) * 0.5f - 0.5f;
    s0 = static_cast<int>(floorf(f));
    a = f - s0;
    if (s0 < 0) s0 = 0, a = 0.f;
    if (s0 >= n - 1) s0 = n - 1, a = 0.f;
  };
  int sx, sy;
  float ax, ay;
  coord(dx, W, sx, ax);
  coord(dy, H, sy, ay);
  const int sx1 = min(sx + 1, W - 1), sy1 = min(sy + 1, H - 1);
  const float r0 = px(sy, sx) * (1.f - ax) + px(sy, sx1) * ax;
  const float r1 = px(sy1, sx) * (1.f - ax) + px(sy1, sx1) * ax;
  dst[(static_cast<size_t>(b) * H2 + dy) * W2 + dx] = r0 * (1.f - ay) + r1 * ay;
}

// separable Gaussian, row pass then column pass (sepFilter2D's order), reflect-101 borders; B images of h x w
__global__ void sift_blur_row_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, Taps t) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const float* s = src + (static_cast<size_t>(b) * h + y) * w;
  float acc = s[x] * t.k[0];
  for (int j = 1; j <= t.r; ++j) acc += (s[reflect101(x - j, w)] + s[reflect101(x + j, w)]) * t.k[j];
  dst[(static_cast<size_t>(b) * h + y) * w + x] = acc;
}

__global__ void sift_blur_col_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, Taps t) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  const float* s = src + static_cast<size_t>(b) * h * w;
  float acc = s[static_cast<size_t>(y) * w + x] * t.k[0];
  for (int j = 1; j <= t.r; ++j)
    acc += (s[static_cast<size_t>(reflect101(y - j, h)) * w + x] + s[static_cast<size_t>(reflect101(y + j, h)) * w + x]) * t.k[j];
  dst[(static_cast<size_t>(b) * h + y) * w + x] = acc;
}

// resize(src, (w / 2, h / 2), INTER_NEAREST): every other pixel
__global__ void sift_half_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, int h2, int w2) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w2) return;
  dst[(static_cast<size_t>(b) * h2 + y) * w2 + x] = src[(static_cast<size_t>(b) * h + 2 * y) * w + 2 * x];
}

// DoG level i of an octave = Gaussian i + 1 - Gaussian i, for i = 0 .. L + 1 (L + 3 Gaussian levels of B images each)
__global__ void sift_dog_kernel(const float* __restrict__ gauss, float* __restrict__ dog, size_t level) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= level) return;
  const size_t lv = blockIdx.y;
  dog[lv * level + i] = gauss[(lv + 1) * level + i] - gauss[lv * level + i];
}


// getGaussianKernel(cvRound(sigma * 8 + 1) | 1, sigma, CV_32F): taps in double, stored as float, normalised by the float sum
int gauss_taps(double sigma, Taps& t) {
  const int n = static_cast<int>(std::lrint(sigma * 8 + 1)) | 1;
  if (n > kMaxTaps) return DIMB_ERR_UNSUPPORTED;
  std::vector<float> k(n);
  const double s2 = -0.5 / (sigma * sigma);
  double sum = 0;
  for (int i = 0; i < n; ++i) {
    const double x = i - (n - 1) * 0.5;
    k[i] = static_cast<float>(std::exp(s2 * x * x));
    sum += k[i];
  }
  sum = 1. / sum;
  t.r = n / 2;
  for (int j = 0; j <= t.r; ++j) t.k[j] = static_cast<float>(k[t.r + j] * sum);
  return DIMB_OK;
}

// Octave sizes and level offsets for B images of H x W
struct Layout {
  Geo g;
  size_t total = 0;     // floats of all levels
  size_t searched = 0;  // pixels of the L searched DoG levels of one image
};

int sift_octaves(int H, int W) {
  return static_cast<int>(std::lrint(std::log(static_cast<double>(std::min(2 * H, 2 * W))) / std::log(2.) - 2)) + 1;
}

bool make_layout(const dimb_sift_conf& cf, int B, int H, int W, Layout& out) {
  Geo& g = out.g;
  g.B = B, g.L = cf.n_octave_layers, g.contrast = static_cast<float>(cf.contrast_threshold), g.edge = static_cast<float>(cf.edge_threshold);
  g.sigma = static_cast<float>(cf.sigma);
  g.n_oct = sift_octaves(H, W);
  if (g.n_oct > 16) return false;
  if (g.n_oct < 1) g.n_oct = 0;  // an image of one row or column: no octave, so no keypoints, as cv2.SIFT finds none
  size_t off = 0;
  int h = 2 * H, w = 2 * W;
  out.searched = 0;
  for (int o = 0; o < g.n_oct; ++o) {
    if (o) h /= 2, w /= 2;
    if (h < 1 || w < 1) return false;
    g.h[o] = h, g.w[o] = w;
    const size_t plane = static_cast<size_t>(h) * w * B;
    g.gauss[o] = off;
    off += plane * (g.L + 3);
    g.dog[o] = off;
    off += plane * (g.L + 2);
    out.searched += static_cast<size_t>(h) * w * g.L;
  }
  out.total = off;
  return true;
}

}  // namespace

struct dimb_sift {
  std::vector<void*> mem;
  dimb_ctx* ctx;
  dimb_sift_conf conf;
  size_t pyr_floats = 0, tmp_floats = 0;
  int ccap = 0, kcap = 0;
  float *pyr = nullptr, *tmp = nullptr, *rec = nullptr, *resp = nullptr;
  Cand* cand = nullptr;
  int *cand_count = nullptr, *kp_count = nullptr, *n_sorted = nullptr, *n_dedup = nullptr, *ovf = nullptr, *sel = nullptr;
  int *sel_out = nullptr, *chunk = nullptr, *digit_off = nullptr, *dummy = nullptr;
  unsigned *state = nullptr, *hist = nullptr;
  unsigned long long *keys0 = nullptr, *keys1 = nullptr;
  // host entry staging
  unsigned char* img_u8 = nullptr;
  float *o_kpts = nullptr, *o_desc = nullptr, *o_frames = nullptr;
  int *o_oct = nullptr, *o_counts = nullptr;
  int o_cap = 0, sel_cap = 0;
  Layout last{};  // layout of the last call (debug taps)
  bool has_last = false;
};

namespace {

int sift_run(dimb_sift* s, const void* d_images, bool u8, int B, int H, int W, const SiftOut& out, cudaStream_t st) {
  dimb_ctx* ctx = s->ctx;
  const dimb_sift_conf& cf = s->conf;
  Layout lay;
  if (!make_layout(cf, B, H, W, lay) || lay.total > s->pyr_floats) {
    dimb_set_error(ctx, "dimb_sift_extract: image larger than the workspace given at create time");
    return DIMB_ERR_ARG;
  }
  const Geo& g = lay.g;
  const int L = cf.n_octave_layers;
  // Lowe's incremental sigmas (buildGaussianPyramid)
  std::vector<Taps> taps(L + 3);
  {
    const double k = std::pow(2., 1. / L);
    // createInitialImage, in float: sigma^2 - 4 * SIFT_INIT_SIGMA^2 for the doubled image
    const float sf = static_cast<float>(cf.sigma), sig_diff = std::sqrt(std::max(sf * sf - 1.f, 0.01f));
    if (gauss_taps(sig_diff, taps[0]) != DIMB_OK) {
      dimb_set_error(ctx, "dimb_sift_extract: Gaussian kernel wider than 127 taps");
      return DIMB_ERR_UNSUPPORTED;
    }
    for (int i = 1; i < L + 3; ++i) {
      const double prev = std::pow(k, static_cast<double>(i - 1)) * cf.sigma, total = prev * k;
      if (gauss_taps(std::sqrt(total * total - prev * prev), taps[i]) != DIMB_OK) {
        dimb_set_error(ctx, "dimb_sift_extract: Gaussian kernel wider than 127 taps");
        return DIMB_ERR_UNSUPPORTED;
      }
    }
  }
  if (g.n_oct == 0) {  // H or W = 1: no octave to search
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(out.counts, 0, sizeof(int) * B, st));
    return DIMB_OK;
  }
  float* pyr = s->pyr;
  auto blur = [&](const float* src, float* dst, int o, const Taps& t) -> int {
    const dim3 grid(ceil_div(g.w[o], 128), g.h[o], B);
    sift_blur_row_kernel<<<grid, 128, 0, st>>>(src, s->tmp, g.h[o], g.w[o], t);
    DIMB_LAUNCH_CHECK(ctx);
    sift_blur_col_kernel<<<grid, 128, 0, st>>>(s->tmp, dst, g.h[o], g.w[o], t);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  {
    ProfScope prof(ctx, st, "sift.pyr");
    float* up = pyr + g.dog[0];  // the first DoG level is free until the DoG pass
    const dim3 ug(ceil_div(2 * W, 128), 2 * H, B);
    if (u8)
      sift_upsample_kernel<unsigned char><<<ug, 128, 0, st>>>(static_cast<const unsigned char*>(d_images), up, H, W);
    else
      sift_upsample_kernel<float><<<ug, 128, 0, st>>>(static_cast<const float*>(d_images), up, H, W);
    DIMB_LAUNCH_CHECK(ctx);
    for (int o = 0; o < g.n_oct; ++o) {
      const size_t plane = static_cast<size_t>(g.h[o]) * g.w[o] * B;
      float* g0 = pyr + g.gauss[o];
      if (o == 0) {
        DIMB_TRY(blur(up, g0, 0, taps[0]));
      } else {
        // level 0 of octave o: every other pixel of level L of octave o - 1
        const size_t prev_plane = static_cast<size_t>(g.h[o - 1]) * g.w[o - 1] * B;
        sift_half_kernel<<<dim3(ceil_div(g.w[o], 128), g.h[o], B), 128, 0, st>>>(pyr + g.gauss[o - 1] + L * prev_plane, g0, g.h[o - 1],
                                                                                g.w[o - 1], g.h[o], g.w[o]);
        DIMB_LAUNCH_CHECK(ctx);
      }
      for (int i = 1; i < L + 3; ++i) DIMB_TRY(blur(g0 + (i - 1) * plane, g0 + i * plane, o, taps[i]));
      const dim3 dg(static_cast<unsigned>((plane + 255) / 256), L + 2);
      sift_dog_kernel<<<dg, 256, 0, st>>>(g0, pyr + g.dog[o], plane);
      DIMB_LAUNCH_CHECK(ctx);
    }
  }
  const int ccap = s->ccap, kcap = s->kcap;
  {
    ProfScope prof(ctx, st, "sift.extrema");
    // cand_count [max_batch] is followed by kp_count [max_batch]: one memset clears both
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(s->cand_count, 0, sizeof(int) * s->conf.max_batch * 2, st));
    DIMB_TRY(launch_sift_extrema(ctx, st, pyr, g, sift_extrema_thr(cf.contrast_threshold, L), s->cand, s->cand_count, ccap));
  }
  {
    ProfScope prof(ctx, st, "sift.ori");
    DIMB_TRY(launch_sift_ori(ctx, st, pyr, g, s->cand, s->cand_count, ccap, s->rec, s->kp_count, kcap));
  }
  {
    ProfScope prof(ctx, st, "sift.select");
    const SiftSelectBufs sb{s->n_sorted, s->n_dedup, s->ovf, s->dummy, s->sel, s->chunk, s->digit_off, s->sel_out, s->resp, s->state,
                            s->hist, s->keys0, s->keys1};
    DIMB_TRY(launch_sift_select(ctx, st, B, s->rec, s->cand_count, s->kp_count, ccap, kcap, cf.n_features, sb, out));
  }
  {
    ProfScope prof(ctx, st, "sift.desc");
    DIMB_TRY(launch_sift_desc(ctx, st, pyr, g, s->rec, s->sel_out, kcap, out));
  }
  s->last = lay;
  s->has_last = true;
  return DIMB_OK;
}

int sift_reserve_out(dimb_sift* s, int cap) {
  dimb_ctx* ctx = s->ctx;
  if (s->o_cap >= cap) return DIMB_OK;
  for (void* p : {static_cast<void*>(s->o_kpts), static_cast<void*>(s->o_desc), static_cast<void*>(s->o_frames), static_cast<void*>(s->o_oct)})
    dimb_free(ctx, p);
  const size_t n = cap;  // the host entry runs one image
  DIMB_TRY(dimb_alloc_t(ctx, &s->o_kpts, n * 2));
  DIMB_TRY(dimb_alloc_t(ctx, &s->o_desc, n * 128));
  DIMB_TRY(dimb_alloc_t(ctx, &s->o_frames, n * 3));
  DIMB_TRY(dimb_alloc_t(ctx, &s->o_oct, n));
  s->o_cap = cap;
  if (cap > s->sel_cap) {
    dimb_free(ctx, s->sel_out);
    s->sel_out = nullptr;
    DIMB_TRY(dimb_alloc_t(ctx, &s->sel_out, static_cast<size_t>(s->conf.max_batch) * cap));
    s->sel_cap = cap;
  }
  return DIMB_OK;
}

}  // namespace

extern "C" {

int dimb_sift_create(dimb_ctx* ctx, const dimb_sift_conf* conf, dimb_sift** out) {
  if (!ctx || !conf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  const dimb_sift_conf& c = *conf;
  if (c.n_features < 0 || c.n_octave_layers < 1 || c.n_octave_layers > 32 || !(c.contrast_threshold >= 0) || !(c.edge_threshold > 0) ||
      !(c.sigma > 0) || c.max_batch < 1 || c.max_batch * c.n_octave_layers > 65535 || c.max_height < 1 || c.max_width < 1 || c.max_height > 16384 ||
      c.max_width > 16384) {
    dimb_set_error(ctx, "dimb_sift_create: n_features >= 0, 1 <= n_octave_layers <= 32, contrast_threshold >= 0, edge_threshold > 0, "
                        "sigma > 0, max_batch >= 1 with max_batch * n_octave_layers <= 65535 and 1 <= max_height, max_width <= 16384 are required");
    return DIMB_ERR_ARG;
  }
  Layout lay;
  if (!make_layout(c, c.max_batch, c.max_height, c.max_width, lay)) {
    dimb_set_error(ctx, "dimb_sift_create: unsupported image size");
    return DIMB_ERR_ARG;
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  dimb_sift* s = new dimb_sift();
  s->ctx = ctx;
  s->conf = c;
  std::unique_ptr<dimb_sift, void (*)(dimb_sift*)> guard(s, dimb_sift_destroy);
  OwnerScope own(ctx, &s->mem);
  const size_t B = c.max_batch;
  s->pyr_floats = lay.total;
  s->tmp_floats = lay.g.n_oct ? static_cast<size_t>(lay.g.h[0]) * lay.g.w[0] * B : 0;
  const size_t cc = lay.searched / kCandDiv + 1024;
  if (cc > static_cast<size_t>(INT_MAX / kNumFields)) {
    dimb_set_error(ctx, "dimb_sift_create: image too large");
    return DIMB_ERR_ARG;
  }
  s->ccap = s->kcap = static_cast<int>(cc);
  const size_t kc = s->kcap, nch = ceil_div(s->kcap, kChunk), nblk = ceil_div(s->kcap, kSortTile);
  DIMB_TRY(dimb_alloc_t(ctx, &s->pyr, s->pyr_floats, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->tmp, s->tmp_floats, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->cand, B * s->ccap, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->rec, B * kNumFields * kc, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->resp, B * kc, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->sel, B * kc, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->keys0, B * kc, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->keys1, B * kc, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->cand_count, B * 2));
  s->kp_count = s->cand_count + B;
  DIMB_TRY(dimb_alloc_t(ctx, &s->n_sorted, B));
  DIMB_TRY(dimb_alloc_t(ctx, &s->n_dedup, B));
  DIMB_TRY(dimb_alloc_t(ctx, &s->ovf, B));
  DIMB_TRY(dimb_alloc_t(ctx, &s->dummy, B));
  DIMB_TRY(dimb_alloc_t(ctx, &s->chunk, B * nch));
  DIMB_TRY(dimb_alloc_t(ctx, &s->digit_off, B * nblk * 256));
  DIMB_TRY(dimb_alloc_t(ctx, &s->state, B * kTkState));
  DIMB_TRY(dimb_alloc_t(ctx, &s->hist, B * 256));
  DIMB_TRY(dimb_alloc_t(ctx, &s->img_u8, B * c.max_height * c.max_width, false));
  DIMB_TRY(dimb_alloc_t(ctx, &s->o_counts, B));
  *out = guard.release();
  return DIMB_OK;
}

void dimb_sift_destroy(dimb_sift* s) {
  if (!s) return;
  dimb_release(s->ctx, s->mem);
  delete s;
}

int dimb_sift_extract_dev(dimb_sift* s, const float* d_images, int B, int H, int W, float* d_kpts, float* d_desc, float* d_frames,
                          int* d_octave, int* d_counts, int cap, void* stream) {
  if (!s || !d_images || !d_kpts || !d_desc || !d_counts || cap < 1 || B < 1 || B > s->conf.max_batch || H < 1 || W < 1 ||
      H > s->conf.max_height || W > s->conf.max_width)
    return DIMB_ERR_ARG;
  dimb_ctx* ctx = s->ctx;
  OwnerScope own(ctx, &s->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (cap > s->sel_cap) {
    dimb_free(ctx, s->sel_out);
    s->sel_out = nullptr;
    DIMB_TRY(dimb_alloc_t(ctx, &s->sel_out, static_cast<size_t>(s->conf.max_batch) * cap));
    s->sel_cap = cap;
  }
  const SiftOut out{d_kpts, d_desc, d_frames, d_octave, d_counts, cap};
  return sift_run(s, d_images, false, B, H, W, out, static_cast<cudaStream_t>(stream));
}

int dimb_sift_extract(dimb_sift* s, const uint8_t* image, int H, int W, float* kpts, float* desc, float* frames, int* octave, int* count,
                      int cap) {
  if (!s || !image || !kpts || !desc || !count || cap < 1 || H < 1 || W < 1 || H > s->conf.max_height || W > s->conf.max_width)
    return DIMB_ERR_ARG;
  dimb_ctx* ctx = s->ctx;
  OwnerScope own(ctx, &s->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DIMB_TRY(sift_reserve_out(s, cap));
  cudaStream_t st = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(s->img_u8, image, static_cast<size_t>(H) * W, cudaMemcpyHostToDevice, st));
  const SiftOut out{s->o_kpts, s->o_desc, s->o_frames, s->o_oct, s->o_counts, cap};
  DIMB_TRY(sift_run(s, s->img_u8, true, 1, H, W, out, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(count, s->o_counts, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(kpts, s->o_kpts, static_cast<size_t>(cap) * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(desc, s->o_desc, static_cast<size_t>(cap) * 128 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (frames) DIMB_CUDA_OK(ctx, cudaMemcpyAsync(frames, s->o_frames, static_cast<size_t>(cap) * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (octave) DIMB_CUDA_OK(ctx, cudaMemcpyAsync(octave, s->o_oct, static_cast<size_t>(cap) * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  if (*count < 0) {
    dimb_set_error(ctx, "dimb_sift_extract: more extrema than the candidate buffers sized at create time hold");
    return DIMB_ERR_CAPACITY;
  }
  if (*count > cap) {
    dimb_set_error(ctx, "dimb_sift_extract: more keypoints than cap");
    return DIMB_ERR_CAPACITY;
  }
  return DIMB_OK;
}

int dimb_sift_debug_read(dimb_sift* s, int which, int image, int level, float* out, size_t n_floats) {
  if (!s || !out || (which != 0 && which != 1)) return DIMB_ERR_ARG;
  dimb_ctx* ctx = s->ctx;
  if (!s->has_last) {
    dimb_set_error(ctx, "dimb_sift_debug_read: no extraction yet");
    return DIMB_ERR_ARG;
  }
  const Geo& g = s->last.g;
  const int per = g.L + 3 - which, o = level / per, lv = level % per;
  if (level < 0 || o >= g.n_oct || image < 0 || image >= g.B) return DIMB_ERR_ARG;
  const size_t plane = static_cast<size_t>(g.h[o]) * g.w[o];
  if (n_floats != plane) {
    dimb_set_error(ctx, "dimb_sift_debug_read: expected " + std::to_string(plane) + " floats");
    return DIMB_ERR_ARG;
  }
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  const float* src = level_ptr(s->pyr, g, which == 1, o, lv, image);
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, src, plane * sizeof(float), cudaMemcpyDeviceToHost));
  return DIMB_OK;
}

}  // extern "C"
