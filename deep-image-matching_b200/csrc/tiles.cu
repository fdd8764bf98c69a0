// tiles.cu - tiled extraction and matching of image sets on the device (dimb_tile_*).
//
// The reference tiles high-resolution images on the host: ExtractorBase._extract_by_tile (extractor_base.py:279-390) extracts every
// tile, shifts the keypoints by the tile origin, drops points within 2 px of the image border, records tile_idx and applies
// np.unique; MatcherBase._match_by_tile (matcher_base.py:362-485) matches the features of each selected tile pair, maps the indices
// back to the full arrays and applies np.unique.  Here the same steps run on feature-store slots:
//   * dimb_tile_cut_dev         cuts B images into their tiles (Tiler.compute_tiles_by_size geometry, zero padding),
//   * dimb_tile_merge_dev       turns the extractor outputs of an image's tiles into its merged feature-store slot,
//   * dimb_tile_views_dev       splits merged slots into one slot per (image, tile) plus the view-row -> merged-row map,
//   * dimb_tile_match_merge_dev maps the tile-pair match tables of each image pair back to merged rows and de-duplicates them.
// np.unique is a sort followed by "keep the first of each run of equal keys".  The sort here is a segmented merge sort of
// (64-bit key, 32-bit source index) records: 1024-record chunks sorted in shared memory, then pairwise merges in global memory
// where every record finds its output slot by binary search in the partner run.  Every source index is distinct, so the order is
// total and the result does not depend on the launch configuration or on which other segments share the launch.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "fstore.cuh"

namespace {

constexpr int kMaxTiles = 2048;        // tile_idx is stored as float16: integers up to 2048 are exact
constexpr int kChunk = 1024;           // records per shared-memory sort
constexpr int kScanThreads = 1024;     // threads of the one-CTA-per-segment scans
constexpr int kSlotKeysA = 64, kSlotKeysB = 65, kSlotParams = 66, kSlotSrc = 67, kSlotCount = 68;  // context scratch slots
constexpr int kSlotResizeTab = 69, kSlotPreSides = 70, kSlotPyrA = 71, kSlotPyrB = 72, kSlotRescale = 73, kSlotRotCodes = 74;
constexpr int kSlotUnrotate = 75;
constexpr int kRotTile = 32;            // dimb_rot90_dev: source tile side (pixels), staged in shared memory
constexpr int kCvFloatLanes = 4;        // float32 lanes of OpenCV's 128-bit baseline SIMD (ResizeAreaFastVec_SIMD_32f)
constexpr unsigned long long kNoKey = ~0ull;
constexpr int kBorder = 2;             // border_thr of extractor_base.py:335

struct Grid {
  int H, W, th, tw, sy, sx, pad_top, pad_left, rows, cols;
  __host__ __device__ int tiles() const { return rows * cols; }
  __host__ __device__ int origin_x(int t) const { return -pad_left + (t % cols) * sx; }
  __host__ __device__ int origin_y(int t) const { return -pad_top + (t / cols) * sy; }
};

int py_mod(int a, int b) {
  const int r = a % b;
  return r < 0 ? r + b : r;
}

// tiling.compute_tiles_by_size: kornia.contrib.compute_padding called without the stride (quirk A.7), so the padding makes
// (size - window) % window == 0 while the tiles step by window - overlap; the odd padding pixel goes to the bottom / right.
bool make_grid(int H, int W, int th, int tw, int oy, int ox, Grid* g) {
  if (H < 1 || W < 1 || th < 1 || tw < 1 || oy < 0 || ox < 0 || oy >= th || ox >= tw) return false;
  if (H > (1 << 20) || W > (1 << 20) || th > (1 << 14) || tw > (1 << 14)) return false;
  const int ry = py_mod(H - th, th), rx = py_mod(W - tw, tw);
  const int pad_y = ry ? th - ry : 0, pad_x = rx ? tw - rx : 0;
  g->H = H, g->W = W, g->th = th, g->tw = tw, g->sy = th - oy, g->sx = tw - ox;
  g->pad_top = pad_y / 2, g->pad_left = pad_x / 2;
  g->rows = (H + pad_y - th) / g->sy + 1;
  g->cols = (W + pad_x - tw) / g->sx + 1;
  return static_cast<long long>(g->rows) * g->cols <= kMaxTiles;
}

struct alignas(16) Rec {
  unsigned long long k;
  unsigned s;
  unsigned pad;
};

__device__ __forceinline__ bool rec_less(const Rec& a, const Rec& b) { return a.k < b.k || (a.k == b.k && a.s < b.s); }

// ---------------------------------------------------------------------------------------------------------------- tile cut
__global__ void tile_cut_kernel(const float* __restrict__ img, float* __restrict__ tiles, Grid g, int C) {
  const int T = g.tiles();
  const int bt = blockIdx.y;
  const int b = bt / T, t = bt % T;
  const int per_tile = g.th * g.tw * C;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= per_tile) return;
  const int c = e % C, px = (e / C) % g.tw, py = e / (C * g.tw);
  const int x = g.origin_x(t) + px, y = g.origin_y(t) + py;
  const bool in = x >= 0 && x < g.W && y >= 0 && y < g.H;
  tiles[static_cast<size_t>(bt) * per_tile + e] = in ? img[(static_cast<size_t>(b) * g.H + y) * g.W * C + static_cast<size_t>(x) * C + c] : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------- segmented sort
__global__ void __launch_bounds__(kChunk / 2) seg_chunk_sort_kernel(Rec* __restrict__ recs, int L) {
  __shared__ Rec s[kChunk];
  Rec* seg = recs + static_cast<size_t>(blockIdx.y) * L;
  const int base = blockIdx.x * kChunk;
  for (int i = threadIdx.x; i < kChunk; i += blockDim.x) s[i] = base + i < L ? seg[base + i] : Rec{kNoKey, ~0u, 0};
  __syncthreads();
  for (int k = 2; k <= kChunk; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < kChunk; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const Rec a = s[i], c = s[ixj];
          if (rec_less(c, a) == ((i & k) == 0)) s[i] = c, s[ixj] = a;
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < kChunk && base + i < L; i += blockDim.x) seg[base + i] = s[i];
}

__device__ __forceinline__ int count_less(const Rec* seg, int lo, int hi, const Rec& e) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (rec_less(seg[mid], e)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One merge pass: sorted runs of length w pairwise into runs of 2w.  A record's output slot is its rank in its own run plus the
// number of records of the partner run that order before it.
__global__ void seg_merge_kernel(const Rec* __restrict__ in, Rec* __restrict__ out, int L, int w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const size_t off = static_cast<size_t>(blockIdx.y) * L;
  const Rec* seg = in + off;
  const Rec e = seg[i];
  const int run = i / w, base = (run & ~1) * w;
  int pos;
  if ((run & 1) == 0) {
    const int lo = base + w, hi = min(base + 2 * w, L);
    pos = lo < L ? i + count_less(seg, lo, hi, e) - lo : i;
  } else {
    pos = i - w + count_less(seg, base, base + w, e) - base;
  }
  out[off + pos] = e;
}

// Sorts n_seg segments of L records in place of a / b; returns the buffer holding the result.
int seg_sort(dimb_ctx* ctx, cudaStream_t st, Rec* a, Rec* b, int n_seg, int L, Rec** sorted) {
  seg_chunk_sort_kernel<<<dim3(ceil_div(L, kChunk), n_seg), kChunk / 2, 0, st>>>(a, L);
  DIMB_LAUNCH_CHECK(ctx);
  for (int w = kChunk; w < L; w *= 2) {
    seg_merge_kernel<<<dim3(ceil_div(L, 256), n_seg), 256, 0, st>>>(a, b, L, w);
    DIMB_LAUNCH_CHECK(ctx);
    std::swap(a, b);
  }
  *sorted = a;
  return DIMB_OK;
}

// Exclusive prefix of one flag per thread over a kScanThreads block; `total` = number of set flags.
__device__ __forceinline__ int block_scan(bool f, int* wsum, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if (lane == 0) wsum[wid] = __popc(bal);
  __syncthreads();
  int off = __popc(bal & ((1u << lane) - 1u));
  total = 0;
  for (int w = 0; w < kScanThreads / 32; ++w) {
    off += w < wid ? wsum[w] : 0;
    total += wsum[w];
  }
  __syncthreads();  // wsum is rewritten by the next call
  return off;
}

// One CTA per sorted segment: the first record of every run of equal keys, in sorted order (np.unique).  Records with kNoKey sort
// last and are dropped, so the scan stops at the first chunk that ends in one.
template <class Emit>
__global__ void __launch_bounds__(kScanThreads) seg_unique_kernel(const Rec* __restrict__ recs, int L, Emit emit) {
  __shared__ int wsum[kScanThreads / 32];
  const int b = blockIdx.x;
  const Rec* seg = recs + static_cast<size_t>(b) * L;
  int done = 0;
  for (int base = 0; base < L; base += kScanThreads) {
    const int i = base + threadIdx.x;
    bool first = false;
    Rec e{};
    if (i < L) {
      e = seg[i];
      first = e.k != kNoKey && (i == 0 || seg[i - 1].k != e.k);
    }
    int n;
    const int pos = done + block_scan(first, wsum, n);
    if (first) emit.row(b, pos, e);
    done += n;
    if (seg[min(base + kScanThreads, L) - 1].k == kNoKey) break;
  }
  if (threadIdx.x == 0) emit.count(b, done);
}

// ---------------------------------------------------------------------------------------------------------------- tile merge
struct TileOut {  // extractor outputs of B * T tiles: kpts [B*T][K][2], scores [B*T][K], desc [B*T][D][K], counts [B*T]
  const float *kpts, *scores, *desc;
  const int* counts;
  int K;
};

__global__ void tile_merge_keys_kernel(TileOut in, Grid g, Rec* __restrict__ recs, int L) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const int T = g.tiles(), t = i / in.K, r = i % in.K;
  const int bt = b * T + t;
  Rec e{kNoKey, static_cast<unsigned>(i), 0};
  if (r < min(in.counts[bt], in.K)) {
    const size_t k = (static_cast<size_t>(bt) * in.K + r) * 2;
    const float x = in.kpts[k] + static_cast<float>(g.origin_x(t)), y = in.kpts[k + 1] + static_cast<float>(g.origin_y(t));
    if (x >= kBorder && x < static_cast<float>(g.W - kBorder) && y >= kBorder && y < static_cast<float>(g.H - kBorder))  // x, y >= 2 > 0:
      // the float bit patterns order as the values do
      e.k = (static_cast<unsigned long long>(__float_as_uint(x)) << 32) | __float_as_uint(y);
  }
  recs[static_cast<size_t>(b) * L + i] = e;
}

struct MergeEmit {
  unsigned* src;  // [B][L] source record (t * K + r) of each merged row
  int* n;         // [B]
  int L;
  __device__ void row(int b, int pos, const Rec& e) const { src[static_cast<size_t>(b) * L + pos] = e.s; }
  __device__ void count(int b, int c) const { n[b] = c; }
};

// fs_put_kernel's float16 cast over the merged rows.  grid = (cap / 256, D + 1, B): row y < D converts descriptor row y, row D
// writes keypoints / scores / tile_idx and the header.
__global__ void tile_merge_write_kernel(TileOut in, Grid g, const unsigned* __restrict__ src, const int* __restrict__ n_merged,
                                        const int* __restrict__ slots, FsLayout fs, int L) {
  const int b = blockIdx.z, y = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_merged[b], T = g.tiles();
  const SlotPtrs s = fs.at(slots[b]);
  const bool live = i < n;
  const unsigned e = live ? src[static_cast<size_t>(b) * L + i] : 0u;
  const int t = e / in.K, r = e % in.K;
  const size_t bt = static_cast<size_t>(b) * T + t;
  if (y < fs.D) {
    if (i < fs.cap) s.desc[static_cast<size_t>(y) * fs.cap + i] = live ? __float2half_rn(in.desc[(bt * fs.D + y) * in.K + r]) : __half(0.f);
    return;
  }
  if (i == 0) {
    s.hdr[0] = n;
    s.hdr[1] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(g.H), 65504.f))));
    s.hdr[2] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(g.W), 65504.f))));
    s.hdr[3] = 1;
  }
  if (i >= fs.cap) return;
  const size_t k = (bt * in.K + r) * 2;
  s.kpts[2 * i] = live ? __float2half_rn(in.kpts[k] + static_cast<float>(g.origin_x(t))) : __half(0.f);
  s.kpts[2 * i + 1] = live ? __float2half_rn(in.kpts[k + 1] + static_cast<float>(g.origin_y(t))) : __half(0.f);
  s.scores[i] = live ? __float2half_rn(in.scores[bt * in.K + r]) : __half(0.f);
  s.tile[i] = live ? __float2half_rn(static_cast<float>(t)) : __half(0.f);
}

// ---------------------------------------------------------------------------------------------------------------- tile views
// One CTA per (tile, image): the merged rows of tile t in merged order -> map row of the view slot; view header.
__global__ void __launch_bounds__(kScanThreads) tile_views_scan_kernel(FsLayout src, FsLayout dst, const int* __restrict__ slots, int B,
                                                                       int* __restrict__ map) {
  __shared__ int wsum[kScanThreads / 32];
  const int t = blockIdx.x, b = blockIdx.y;
  const SlotPtrs s = src.at(slots[b]);
  const int ds = slots[B + b] + t;
  const SlotPtrs d = dst.at(ds);
  int* m = map + static_cast<size_t>(ds) * dst.cap;
  const int n = s.hdr[0];
  const __half ht = __float2half_rn(static_cast<float>(t));
  int done = 0;
  for (int base = 0; base < n; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const bool in = i < n && __heq(s.tile[i], ht);
    int c;
    const int pos = done + block_scan(in, wsum, c);
    if (in && pos < dst.cap) m[pos] = i;
    done += c;
  }
  if (threadIdx.x == 0) {
    d.hdr[0] = min(done, dst.cap);
    d.hdr[1] = s.hdr[1];  // the full image's [H, W] (matcher_base.py:1389, quirk A.3)
    d.hdr[2] = s.hdr[2];
    d.hdr[3] = 1;
  }
}

// grid = (cap / 256, D + 1, B * T): copies the mapped rows (float16 to float16) and zeroes the rest of the view slot.
__global__ void tile_views_copy_kernel(FsLayout src, FsLayout dst, const int* __restrict__ slots, int B, int T, const int* __restrict__ map) {
  const int b = blockIdx.z / T, t = blockIdx.z % T, y = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dst.cap) return;
  const SlotPtrs s = src.at(slots[b]);
  const int ds = slots[B + b] + t;
  const SlotPtrs d = dst.at(ds);
  const bool live = i < d.hdr[0];
  const int j = live ? map[static_cast<size_t>(ds) * dst.cap + i] : 0;
  const __half z(0.f);
  if (y < dst.D) {
    d.desc[static_cast<size_t>(y) * dst.cap + i] = live ? s.desc[static_cast<size_t>(y) * src.cap + j] : z;
    return;
  }
  d.kpts[2 * i] = live ? s.kpts[2 * j] : z;
  d.kpts[2 * i + 1] = live ? s.kpts[2 * j + 1] : z;
  d.scores[i] = live ? s.scores[j] : z;
  d.tile[i] = live ? s.tile[j] : z;
}

// ---------------------------------------------------------------------------------------------------------------- match merge
// params: offsets [Q + 1] of each image pair's tile pairs, then view0 [P], view1 [P] (map rows of both sides of every tile pair).
__global__ void match_merge_keys_kernel(const int* __restrict__ params, int Q, const int* __restrict__ maps, int map_ld,
                                        const int64_t* __restrict__ matches, const int* __restrict__ n_matches, int cap, Rec* __restrict__ recs,
                                        int L) {
  const int q = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const int* off = params;
  const int P = off[Q];
  const int p = off[q] + i / cap, r = i % cap;
  Rec e{kNoKey, static_cast<unsigned>(i), 0};
  if (p < off[q + 1] && r < min(n_matches[p], cap)) {
    const int64_t* m = matches + (static_cast<size_t>(p) * cap + r) * 2;
    const unsigned i0 = static_cast<unsigned>(maps[static_cast<size_t>(params[Q + 1 + p]) * map_ld + m[0]]);
    const unsigned i1 = static_cast<unsigned>(maps[static_cast<size_t>(params[Q + 1 + P + p]) * map_ld + m[1]]);
    e.k = (static_cast<unsigned long long>(i0) << 32) | i1;
  }
  recs[static_cast<size_t>(q) * L + i] = e;
}

struct MatchEmit {
  int64_t* out;  // [Q][cap2][2]
  int* n;        // [Q], the full count
  int cap2;
  __device__ void row(int q, int pos, const Rec& e) const {
    if (pos >= cap2) return;
    int64_t* o = out + (static_cast<size_t>(q) * cap2 + pos) * 2;
    o[0] = static_cast<int64_t>(e.k >> 32);
    o[1] = static_cast<int64_t>(e.k & 0xffffffffull);
  }
  __device__ void count(int q, int c) const { n[q] = c; }
};

// ---------------------------------------------------------------------------------------------------------------- preselection
// OpenCV's computeResizeAreaTab (imgproc/src/resize.cpp) for one axis, cn = 1: every weight in double, stored as float.
void area_tab(int ssize, int dsize, std::vector<int>* di, std::vector<int>* si, std::vector<float>* alpha) {
  const double scale = 1.0 / (static_cast<double>(dsize) / ssize);
  auto push = [&](int d, int s, float a) { di->push_back(d), si->push_back(s), alpha->push_back(a); };
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = std::min(scale, ssize - fsx1);
    int sx1 = static_cast<int>(std::ceil(fsx1)), sx2 = static_cast<int>(std::floor(fsx2));
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    if (sx1 - fsx1 > 1e-3) push(dx, sx1 - 1, static_cast<float>((sx1 - fsx1) / cell));
    for (int sx = sx1; sx < sx2; ++sx) push(dx, sx, static_cast<float>(1.0 / cell));
    if (fsx2 - sx2 > 1e-3) push(dx, sx2, static_cast<float>(std::min(std::min(fsx2 - sx2, 1.), cell) / cell));
  }
}

// cv::resize's is_area_fast: the factor 1 / (dsize / ssize) is an integer within DBL_EPSILON (0 otherwise).
int area_fast_factor(int ssize, int dsize) {
  const double scale = 1.0 / (static_cast<double>(dsize) / ssize);
  const int i = static_cast<int>(std::lround(scale));
  return std::abs(scale - i) < 2.220446049250313e-16 ? i : 0;
}

struct AreaTab {  // per axis: the entries of output index d are [ofs[d], ofs[d + 1]) of src / alpha, in OpenCV's order
  const int *xofs, *xsrc, *yofs, *ysrc;
  const float *xa, *ya;
};

// The source pixels of the INTER_AREA kernels, read through a pointer to a pixel's first value: a gray image [H][W] as it is, or an
// RGB image [H][W][3] made gray per pixel by the project's gray rule (pairs_generator.gray_from_rgb): each channel rounded half to
// even and clamped to 0..255 (cvRound, then saturate_cast<uchar>), then cv::cvtColor's RGB2GRAY in 15-bit fixed point,
// (9798 R + 19235 G + 3735 B + 2^14) >> 15.  The gray value is an integer in 0..255, so the arithmetic after it is the gray path's.
struct GrayPixel {
  static constexpr int kChannels = 1;
  static __device__ __forceinline__ float load(const float* px) { return *px; }
};
struct RgbGrayPixel {
  static constexpr int kChannels = 3;
  static __device__ __forceinline__ float load(const float* px) {
    const auto u8 = [](float v) { return min(max(__float2int_rn(v), 0), 255); };
    return static_cast<float>((9798 * u8(px[0]) + 19235 * u8(px[1]) + 3735 * u8(px[2]) + 16384) >> 15);
  }
};

// resizeArea_: per output pixel, the rows of the y-table in order; buf = sum of S * alpha in x-table order from 0; the first row sets
// sum = beta * buf, the others add beta * buf.  Every product and sum is rounded on its own, as OpenCV's scalar code does.
template <class Px>
__global__ void resize_area_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int H2, int W2, AreaTab t) {
  constexpr int C = Px::kChannels;
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y, b = blockIdx.z;
  if (dx >= W2) return;
  const float* img = src + static_cast<size_t>(b) * H * W * C;
  const int x0 = t.xofs[dx], x1 = t.xofs[dx + 1], j0 = t.yofs[dy], j1 = t.yofs[dy + 1];
  float sum = 0.f;
  for (int j = j0; j < j1; ++j) {
    const float* row = img + static_cast<size_t>(t.ysrc[j]) * W * C;
    float buf = 0.f;
    for (int k = x0; k < x1; ++k) buf = __fadd_rn(buf, __fmul_rn(Px::load(row + t.xsrc[k] * C), t.xa[k]));
    const float v = __fmul_rn(t.ya[j], buf);
    sum = j == j0 ? v : __fadd_rn(sum, v);
  }
  dst[(static_cast<size_t>(b) * H2 + dy) * W2 + dx] = sum;
}

// resizeAreaFast_ for integer factors (fy, fx): the block row-major, sum += ((a + b) + c) + d per four pixels, then sum * (1.f / area).
// For 2 x 2 OpenCV's vector loop (ResizeAreaFastVec_SIMD_32f) covers the columns dx < vec_end and computes ((a + b) + (c + d)) * 0.25f;
// the scalar loop above takes the rest of the row.  fy = fx = 1 with vec_end = 0 returns the source pixels exactly.
template <class Px>
__global__ void resize_area_fast_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int H2, int W2, int fy, int fx,
                                        int vec_end) {
  constexpr int C = Px::kChannels;
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y, b = blockIdx.z;
  if (dx >= W2) return;
  const float* S = src + ((static_cast<size_t>(b) * H + static_cast<size_t>(dy) * fy) * W + static_cast<size_t>(dx) * fx) * C;
  const int area = fy * fx;
  auto at = [&](int k) { return Px::load(S + (static_cast<size_t>(k / fx) * W + k % fx) * C); };
  if (dx < vec_end) {
    dst[(static_cast<size_t>(b) * H2 + dy) * W2 + dx] = __fmul_rn(__fadd_rn(__fadd_rn(at(0), at(1)), __fadd_rn(at(2), at(3))), 0.25f);
    return;
  }
  float sum = 0.f;
  int k = 0;
  for (; k <= area - 4; k += 4) sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(__fadd_rn(at(k), at(k + 1)), at(k + 2)), at(k + 3)));
  for (; k < area; ++k) sum = __fadd_rn(sum, at(k));
  dst[(static_cast<size_t>(b) * H2 + dy) * W2 + dx] = __fmul_rn(sum, __fdiv_rn(1.f, static_cast<float>(area)));
}

// cv::resize's coefficient loop for INTER_AREA when an axis is enlarged (area_mode, ksize 2), one axis: inv = dsize / ssize and
// scale = 1 / inv in double, as hal::resize computes them.  Returns xmax, the first d whose sx + 1 reaches the border (dsize if none).
int area_linear_tab(int ssize, int dsize, int* s_idx, float* alpha) {
  const double inv = static_cast<double>(dsize) / ssize, scale = 1.0 / inv;
  int xmax = dsize;
  for (int d = 0; d < dsize; ++d) {
    int sx = static_cast<int>(std::floor(d * scale));
    float fx = static_cast<float>((d + 1) - (sx + 1) * inv);
    fx = fx <= 0 ? 0.f : fx - std::floor(fx);
    if (sx + 1 >= ssize) {
      xmax = std::min(xmax, d);
      if (sx >= ssize - 1) fx = 0.f, sx = ssize - 1;
    }
    s_idx[d] = sx;
    alpha[2 * d] = 1.f - fx;
    alpha[2 * d + 1] = fx;
  }
  return xmax;
}

struct LinearTab {  // per axis: the source index [dsize] and the weight pairs [dsize][2]; columns dx >= xmax copy S[sx]
  const int *xs, *ys;
  const float2 *xa, *ya;
  int xmax;
};

// resizeGeneric_ with HResizeLinear / VResizeLinear in float: each of the two source rows sy and min(sy + 1, H - 1) is resampled
// horizontally as S[sx] * a0 + S[sx + 1] * a1 (S[sx] from xmax on), then out = row0 * b0 + row1 * b1; every product and sum is
// rounded on its own (no FMA).
template <class Px>
__global__ void resize_area_linear_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int H2, int W2,
                                          LinearTab t) {
  constexpr int C = Px::kChannels;
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y, b = blockIdx.z;
  if (dx >= W2) return;
  const int sx = t.xs[dx], sy = t.ys[dy];
  const float2 a = t.xa[dx], be = t.ya[dy];
  const float* img = src + static_cast<size_t>(b) * H * W * C;
  auto hrow = [&](int y) {
    const float* S = img + static_cast<size_t>(y) * W * C;
    return dx < t.xmax ? __fadd_rn(__fmul_rn(Px::load(S + sx * C), a.x), __fmul_rn(Px::load(S + (sx + 1) * C), a.y)) : Px::load(S + sx * C);
  };
  const float r0 = hrow(sy), r1 = hrow(min(sy + 1, H - 1));
  dst[(static_cast<size_t>(b) * H2 + dy) * W2 + dx] = __fadd_rn(__fmul_rn(r0, be.x), __fmul_rn(r1, be.y));
}

// The launches of the INTER_AREA entries for source pixels Px, arguments checked by the entry: the integer-factor kernel when both
// factors are integers (1 x 1 included), otherwise the table kernel with one upload of both axes' tables.
template <class Px>
int resize_area_launch(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                       cudaStream_t st) {
  const dim3 grid(ceil_div(width2, 128), height2, B);
  const int fy = area_fast_factor(height, height2), fx = area_fast_factor(width, width2);
  if (fy && fx) {
    // OpenCV's baseline build vectorises float rows 128 bits (4 lanes) wide; only 2 x 2 has a vector loop
    const int vec_end = fy == 2 && fx == 2 ? width2 / kCvFloatLanes * kCvFloatLanes : 0;
    ProfScope prof(ctx, st, "tile.resize");
    resize_area_fast_kernel<Px><<<grid, 128, 0, st>>>(d_src, d_dst, height, width, height2, width2, fy, fx, vec_end);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  }
  // one upload: x offsets [W2 + 1], x sources, y offsets [H2 + 1], y sources, then the x and y weights (float bits)
  std::vector<int> xd, xs, yd, ys;
  std::vector<float> xa, ya;
  area_tab(width, width2, &xd, &xs, &xa);
  area_tab(height, height2, &yd, &ys, &ya);
  auto offsets = [](const std::vector<int>& d, int n) {
    std::vector<int> o(n + 1, 0);
    for (int v : d) ++o[v + 1];
    for (int i = 0; i < n; ++i) o[i + 1] += o[i];
    return o;
  };
  std::vector<int> hp = offsets(xd, width2);
  const size_t o_xs = hp.size();
  hp.insert(hp.end(), xs.begin(), xs.end());
  const size_t o_yofs = hp.size();
  const std::vector<int> yo = offsets(yd, height2);
  hp.insert(hp.end(), yo.begin(), yo.end());
  const size_t o_ys = hp.size();
  hp.insert(hp.end(), ys.begin(), ys.end());
  const size_t o_xa = hp.size();
  hp.resize(o_xa + xa.size() + ya.size());
  std::memcpy(hp.data() + o_xa, xa.data(), xa.size() * sizeof(float));
  std::memcpy(hp.data() + o_xa + xa.size(), ya.data(), ya.size() * sizeof(float));
  int* d_tab;
  DIMB_TRY(dimb_scratch(ctx, kSlotResizeTab, hp.size() * sizeof(int), reinterpret_cast<void**>(&d_tab)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_tab, hp.data(), hp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const AreaTab t{d_tab, d_tab + o_xs, d_tab + o_yofs, d_tab + o_ys, reinterpret_cast<const float*>(d_tab + o_xa),
                  reinterpret_cast<const float*>(d_tab + o_xa + xa.size())};
  ProfScope prof(ctx, st, "tile.resize");
  resize_area_kernel<Px><<<grid, 128, 0, st>>>(d_src, d_dst, height, width, height2, width2, t);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// The bilinear emulation of INTER_AREA when an axis is enlarged, for source pixels Px, arguments checked by the entry.
template <class Px>
int resize_area_linear_launch(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                              cudaStream_t st) {
  // one upload: the x and y weight pairs (float bits, first so that the float2 reads stay aligned), then x and y sources
  std::vector<int> hp(3 * static_cast<size_t>(width2 + height2));
  float* xa = reinterpret_cast<float*>(hp.data());
  float* ya = xa + 2 * width2;
  int* xs = hp.data() + 2 * (width2 + height2);
  int* ys = xs + width2;
  const int xmax = area_linear_tab(width, width2, xs, xa);
  area_linear_tab(height, height2, ys, ya);
  int* d_tab;
  DIMB_TRY(dimb_scratch(ctx, kSlotResizeTab, hp.size() * sizeof(int), reinterpret_cast<void**>(&d_tab)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_tab, hp.data(), hp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const float2* d_w = reinterpret_cast<const float2*>(d_tab);
  const int* d_s = d_tab + 2 * (width2 + height2);
  const LinearTab t{d_s, d_s + width2, d_w, d_w + width2, xmax};
  ProfScope prof(ctx, st, "tile.resize");
  resize_area_linear_kernel<Px><<<dim3(ceil_div(width2, 128), height2, B), 128, 0, st>>>(d_src, d_dst, height, width, height2, width2, t);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// cv::borderInterpolate with BORDER_REFLECT_101 (BORDER_DEFAULT): gfedcb|abcdefgh|gfedcba.
__host__ __device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// The 1 4 6 4 1 tap sum of pyrDown_ in its two orders: OpenCV's scalar loops, s2 * 6 + (s1 + s3) * 4 + s0 + s4 left to right, and its
// baseline-SIMD horizontal loop (PyrDownVecH, v_muladd without FMA), s2 * 6 + ((s1 + s3) * 4 + (s0 + s4)).
__device__ __forceinline__ float pyr5_scalar(float s0, float s1, float s2, float s3, float s4) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s2, 6.f), __fmul_rn(__fadd_rn(s1, s3), 4.f)), s0), s4);
}
__device__ __forceinline__ float pyr5_vec(float s0, float s1, float s2, float s3, float s4) {
  return __fadd_rn(__fmul_rn(s2, 6.f), __fadd_rn(__fmul_rn(__fadd_rn(s1, s3), 4.f), __fadd_rn(s0, s4)));
}

// cv::pyrDown (pyrDown_ with FltCast<float, 8>) of B images [H][W][C] -> [H2][W2][C], H2 = (H + 1) / 2, W2 = (W + 1) / 2; one
// thread per output value.  Horizontal pass per source row: output column 0 and the columns from width0 = min((W - 3) / 2 + 1, W2)
// on (the tabR border columns) use the scalar order, and so does the scalar tail of the vector loop, which covers columns
// [1, 1 + floor((width0 - 1) / 4) * 4) for C = 1 and [1, width0 - 1) for C = 3 (one pixel per 4-lane step).  Vertical pass over the
// five rows 2y - 2 .. 2y + 2 (reflect-101): PyrDownVecV's ((r1 + r3) + r2) * 4 + ((r0 + r4) + (r2 + r2)) on the first
// floor(W2 * C / 4) * 4 values of the row, the scalar order on the rest, then * (1 / 256).  Every operation rounded on its own.
__global__ void __launch_bounds__(128) pyr_down_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int C, int H2,
                                                       int W2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  const int row_len = W2 * C;
  if (j >= row_len) return;
  const int x = j / C, c = j - x * C;
  const int width0 = min((W - 3) / 2 + 1, W2);  // C division truncates: 0 for W = 1
  const bool hvec = C == 1 ? (x >= 1 && x < 1 + (width0 - 1) / 4 * 4) : (x >= 1 && x < width0 - 1);
  int sx[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) sx[k] = reflect101(2 * x - 2 + k, W) * C + c;
  const float* img = src + static_cast<size_t>(b) * H * W * C;
  float r[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const float* S = img + static_cast<size_t>(reflect101(2 * y - 2 + k, H)) * W * C;
    r[k] = hvec ? pyr5_vec(S[sx[0]], S[sx[1]], S[sx[2]], S[sx[3]], S[sx[4]]) : pyr5_scalar(S[sx[0]], S[sx[1]], S[sx[2]], S[sx[3]], S[sx[4]]);
  }
  const float v = j < (row_len & ~(kCvFloatLanes - 1))
                      ? __fadd_rn(__fmul_rn(__fadd_rn(__fadd_rn(r[1], r[3]), r[2]), 4.f), __fadd_rn(__fadd_rn(r[0], r[4]), __fadd_rn(r[2], r[2])))
                      : pyr5_scalar(r[0], r[1], r[2], r[3], r[4]);
  dst[(static_cast<size_t>(b) * H2 + y) * row_len + j] = __fmul_rn(v, 1.f / 256.f);
}

// cv::pyrUp (pyrUp_ with FltCast<float, 6>) of B images [H][W][C] -> [2H][2W][C]; one thread per output value.  Horizontal pass per
// source row, output column X of source column x = X / 2: even X gives (S[x - 1] + S[x] * 6) + S[x + 1], odd X (S[x] + S[x + 1]) * 4,
// except at the borders: X = 0 gives S[0] * 6 + S[1] * 2, X = 2W - 2 gives S[W - 2] + S[W - 1] * 7, X = 2W - 1 gives S[W - 1] * 8, and
// a one-column image gives S[0] * 8 on both.  Vertical pass over the source rows y - 1, y, y + 1 of y = Y / 2 (row s read at
// reflect101(2s, 2H) / 2): even Y gives (r0 + r1 * 6) + r2, odd Y (r1 + r2) * 4, then * (1 / 64).  Every operation rounded on its own.
__global__ void __launch_bounds__(128) pyr_up_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int C) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y, b = blockIdx.z;
  const int row_len = 2 * W * C;
  if (j >= row_len) return;
  const int X = j / C, c = j - X * C, x = X >> 1;
  const bool odd = X & 1;
  const float* img = src + static_cast<size_t>(b) * H * W * C;
  auto hrow = [&](int sy) {
    const float* S = img + static_cast<size_t>(sy) * W * C + c;
    if (W == 1) return __fmul_rn(S[0], 8.f);
    if (odd) return x == W - 1 ? __fmul_rn(S[x * C], 8.f) : __fmul_rn(__fadd_rn(S[x * C], S[(x + 1) * C]), 4.f);
    if (x == 0) return __fadd_rn(__fmul_rn(S[0], 6.f), __fmul_rn(S[C], 2.f));
    if (x == W - 1) return __fadd_rn(S[(x - 1) * C], __fmul_rn(S[x * C], 7.f));
    return __fadd_rn(__fadd_rn(S[(x - 1) * C], __fmul_rn(S[x * C], 6.f)), S[(x + 1) * C]);
  };
  const int y = Y >> 1;
  const float r1 = hrow(y), r2 = hrow(reflect101(2 * y + 2, 2 * H) / 2);
  const float v = (Y & 1) ? __fmul_rn(__fadd_rn(r1, r2), 4.f)
                          : __fadd_rn(__fadd_rn(hrow(reflect101(2 * y - 2, 2 * H) / 2), __fmul_rn(r1, 6.f)), r2);
  dst[(static_cast<size_t>(b) * 2 * H + Y) * row_len + j] = __fmul_rn(v, 1.f / 64.f);
}

// The keypoint pass shared by the store remaps below: for a non-empty slot, thread (0, 0) writes [H, W] into the header as
// fs_put_kernel does, and keypoint i (one per thread of a (cap / 256)-wide grid row) becomes map(x, y) in float32, rounded to float16.
// Empty slots are left alone.
template <class Map>
__device__ __forceinline__ void fs_remap_slot(const FsLayout& L, int slot, int H, int W, Map map) {
  const SlotPtrs s = L.at(slot);
  if (!s.hdr[3]) return;
  const int n = min(s.hdr[0], L.cap), i = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    s.hdr[1] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(H), 65504.f))));
    s.hdr[2] = static_cast<int>(__half2float(__float2half_rn(fminf(static_cast<float>(W), 65504.f))));
  }
  if (i >= n) return;
  const float2 p = map(__half2float(s.kpts[2 * i]), __half2float(s.kpts[2 * i + 1]));
  s.kpts[2 * i] = __float2half_rn(p.x);
  s.kpts[2 * i + 1] = __float2half_rn(p.y);
}

// Multiplies the float16 keypoints of B store slots by `scale` (a power of two) and writes [H, W] into their headers.  grid (cap / 256, B).
__global__ void fs_rescale_kernel(FsLayout L, const int* __restrict__ slots, float scale, int H, int W) {
  fs_remap_slot(L, slots[blockIdx.y], H, W, [scale](float x, float y) { return make_float2(__fmul_rn(x, scale), __fmul_rn(y, scale)); });
}

struct Unrotate {  // one slot of dimb_fstore_unrotate_dev: its rotation code (0..3 quarter turns clockwise) and original size
  int slot, quarter, H, W;
};

// The inverse of cv2.rotate on pixel indices of the original H x W image, per slot: (x', y') in the rotated image ->
// 90: (y', H - 1 - x'), 180: (W - 1 - x', H - 1 - y'), 270: (W - 1 - y', x'), each difference one float32 rounding.  grid (cap / 256, B).
__global__ void fs_unrotate_kernel(FsLayout L, const Unrotate* __restrict__ items) {
  const Unrotate u = items[blockIdx.y];
  const float h1 = static_cast<float>(u.H - 1), w1 = static_cast<float>(u.W - 1);
  const int q = u.quarter;
  fs_remap_slot(L, u.slot, u.H, u.W, [=](float x, float y) {
    if (q == 1) return make_float2(y, __fsub_rn(h1, x));
    if (q == 2) return make_float2(__fsub_rn(w1, x), __fsub_rn(h1, y));
    if (q == 3) return make_float2(__fsub_rn(w1, y), x);
    return make_float2(x, y);
  });
}

// cv2.rotate of B float32 images [H][W][C] by per-image quarter turns quarter[b] (0 = copy, 1 = 90 clockwise, 2 = 180, 3 = 270); image
// b of dst starts at b * H * W * C and is [H][W][C] (0, 180) or [W][H][C] (90, 270).  One CTA per 32 x 32-pixel source tile, staged in
// shared memory (row stride 32 C + 1 floats, so that the transposed reads of 90 / 270 hit 32 distinct banks); the CTA then writes the
// tile's image under the rotation row by row, so global reads and writes both run along rows.  A permutation: bitwise cv2.rotate.
// grid (ceil(W / 32), ceil(H / 32), B), block (32, 8).
__global__ void __launch_bounds__(256) rot90_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int C,
                                                    const int* __restrict__ quarter) {
  __shared__ float tile[kRotTile][kRotTile * 3 + 1];
  const int q = quarter[blockIdx.z], x0 = blockIdx.x * kRotTile, y0 = blockIdx.y * kRotTile, lane = threadIdx.x;
  const size_t img = static_cast<size_t>(blockIdx.z) * H * W * C;
  const int row_len = min(kRotTile, W - x0) * C;
  for (int r = threadIdx.y; r < kRotTile && y0 + r < H; r += blockDim.y)
    for (int e = lane; e < row_len; e += kRotTile) tile[r][e] = src[img + (static_cast<size_t>(y0 + r) * W + x0) * C + e];
  __syncthreads();
  // destination row a of the tile's image (a = 0..31) and pixel p along it -> source pixel (sy, sx) of the tile
  const bool turn = q & 1;
  const int Wd = turn ? H : W;
  for (int a = threadIdx.y; a < kRotTile; a += blockDim.y) {
    for (int e = lane; e < kRotTile * C; e += kRotTile) {
      const int p = e / C, c = e - p * C;
      int sy, sx, dy, dx;
      if (q == 0) sy = a, sx = p, dy = y0 + a, dx = x0 + p;
      else if (q == 1) sy = kRotTile - 1 - p, sx = a, dy = x0 + a, dx = H - y0 - kRotTile + p;
      else if (q == 2) sy = kRotTile - 1 - a, sx = kRotTile - 1 - p, dy = H - y0 - kRotTile + a, dx = W - x0 - kRotTile + p;
      else sy = p, sx = kRotTile - 1 - a, dy = W - x0 - kRotTile + a, dx = y0 + p;
      if (y0 + sy >= H || x0 + sx >= W) continue;
      dst[img + (static_cast<size_t>(dy) * Wd + dx) * C + c] = tile[sy][sx * C + c];
    }
  }
}

// One CTA per image: size = (1 + max) - min per axis over its keypoints, {1, 1} without keypoints (min / max are exact in any order).
__global__ void __launch_bounds__(256) kpts_extent_kernel(const float* __restrict__ kpts, int ld, const int* __restrict__ counts,
                                                          float* __restrict__ out) {
  __shared__ float red[4][8];
  const int b = blockIdx.x, n = min(max(counts[b], 0), ld);
  const float2* k = reinterpret_cast<const float2*>(kpts) + static_cast<size_t>(b) * ld;
  float mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float2 p = k[i];
    mn0 = fminf(mn0, p.x), mx0 = fmaxf(mx0, p.x), mn1 = fminf(mn1, p.y), mx1 = fmaxf(mx1, p.y);
  }
  for (int o = 16; o; o >>= 1) {
    mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)), mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o)), mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[0][w] = mn0, red[1][w] = mx0, red[2][w] = mn1, red[3][w] = mx1;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < 8; ++i) mn0 = fminf(mn0, red[0][i]), mx0 = fmaxf(mx0, red[1][i]), mn1 = fminf(mn1, red[2][i]), mx1 = fmaxf(mx1, red[3][i]);
  out[2 * b] = n ? __fsub_rn(__fadd_rn(1.f, mx0), mn0) : 1.f;
  out[2 * b + 1] = n ? __fsub_rn(__fadd_rn(1.f, mx1), mn1) : 1.f;
}

struct PreSide {  // keypoints of one side of one pair (dimb_feats_dev's keypoints / f16 / round_fp16)
  const void* kpts;
  int f16, round_fp16;
};

__device__ __forceinline__ float pre_kpt(const PreSide& s, int64_t i) {
  if (s.f16) return __half2float(static_cast<const __half*>(s.kpts)[i]);
  const float v = static_cast<const float*>(s.kpts)[i];
  return s.round_fp16 ? __half2float(__float2half_rn(v)) : v;
}

// The tiles along one axis whose open interval (origin, origin + size) holds v: a float estimate widened by one on both sides, then
// the exact test on every candidate (origins are integers below 2^21, exact in float).
__device__ __forceinline__ void axis_cover(float v, int pad, int step, int size, int n, int& lo, int& hi) {
  const float u = v + static_cast<float>(pad);
  lo = max(0, static_cast<int>(floorf((u - static_cast<float>(size)) / static_cast<float>(step))) - 1);
  hi = min(n - 1, static_cast<int>(floorf(u / static_cast<float>(step))) + 1);
}

__device__ __forceinline__ bool in_open(float v, int o, int size) { return v > static_cast<float>(o) && v < static_cast<float>(o + size); }

struct PrePair {  // one image pair of a preselection batch: both sides' keypoints, tile grids and scales, and its count block
  PreSide s0, s1;
  Grid g0, g1;
  float sc0, sc1;
  size_t off;  // first element of the pair's [T0][T1] block of counts / flags
};

// grid (cap / 128, Q): one thread per match row; +1 for every (t0, t1) whose boxes both hold the row's full-resolution points.
__global__ void tile_preselect_count_kernel(const PrePair* __restrict__ pairs, const int64_t* __restrict__ matches,
                                            const int* __restrict__ n_matches, int cap, int* __restrict__ counts) {
  const int q = blockIdx.y, r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= min(n_matches[q], cap)) return;
  const int64_t* m = matches + (static_cast<size_t>(q) * cap + r) * 2;
  const PrePair& p = pairs[q];
  const Grid g0 = p.g0, g1 = p.g1;
  const float x0 = __fdiv_rn(pre_kpt(p.s0, 2 * m[0]), p.sc0), y0 = __fdiv_rn(pre_kpt(p.s0, 2 * m[0] + 1), p.sc0);
  const float x1 = __fdiv_rn(pre_kpt(p.s1, 2 * m[1]), p.sc1), y1 = __fdiv_rn(pre_kpt(p.s1, 2 * m[1] + 1), p.sc1);
  constexpr float kFar = 4194304.f;  // 2^22: beyond every box (image and tile sides are below 2^20 / 2^14), and keeps the estimates in int
  if (!(fabsf(x0) < kFar && fabsf(y0) < kFar && fabsf(x1) < kFar && fabsf(y1) < kFar)) return;
  const int T1 = g1.tiles();
  int* c = counts + p.off;
  int r0lo, r0hi, c0lo, c0hi, r1lo, r1hi, c1lo, c1hi;
  axis_cover(y0, g0.pad_top, g0.sy, g0.th, g0.rows, r0lo, r0hi);
  axis_cover(x0, g0.pad_left, g0.sx, g0.tw, g0.cols, c0lo, c0hi);
  axis_cover(y1, g1.pad_top, g1.sy, g1.th, g1.rows, r1lo, r1hi);
  axis_cover(x1, g1.pad_left, g1.sx, g1.tw, g1.cols, c1lo, c1hi);
  for (int ra = r0lo; ra <= r0hi; ++ra) {
    if (!in_open(y0, -g0.pad_top + ra * g0.sy, g0.th)) continue;
    for (int ca = c0lo; ca <= c0hi; ++ca) {
      if (!in_open(x0, -g0.pad_left + ca * g0.sx, g0.tw)) continue;
      const int t0 = ra * g0.cols + ca;
      for (int rb = r1lo; rb <= r1hi; ++rb) {
        if (!in_open(y1, -g1.pad_top + rb * g1.sy, g1.th)) continue;
        for (int cb = c1lo; cb <= c1hi; ++cb)
          if (in_open(x1, -g1.pad_left + cb * g1.sx, g1.tw)) atomicAdd(c + static_cast<size_t>(t0) * T1 + rb * g1.cols + cb, 1);
      }
    }
  }
}

__global__ void tile_preselect_flag_kernel(const int* __restrict__ counts, size_t n, int min_matches, unsigned char* __restrict__ flags) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    flags[i] = counts[i] > min_matches;
}

}  // namespace

extern "C" {

int dimb_tile_grid(int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w, int* out) {
  Grid g;
  if (!out || !make_grid(height, width, tile_h, tile_w, overlap_h, overlap_w, &g)) return DIMB_ERR_ARG;
  out[0] = g.rows, out[1] = g.cols, out[2] = g.pad_top, out[3] = g.pad_left, out[4] = g.sy, out[5] = g.sx;
  return DIMB_OK;
}

int dimb_tile_cut_dev(dimb_ctx* ctx, const float* d_images, int B, int height, int width, int channels, int tile_h, int tile_w, int overlap_h,
                      int overlap_w, float* d_tiles, void* stream) {
  Grid g;
  if (!ctx || !d_images || !d_tiles || B < 1 || (channels != 1 && channels != 3) ||
      !make_grid(height, width, tile_h, tile_w, overlap_h, overlap_w, &g) || static_cast<long long>(B) * g.tiles() > 65535 ||
      static_cast<long long>(tile_h) * tile_w * channels >= (1ll << 31))
    return DIMB_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope prof(ctx, st, "tile.cut");
  tile_cut_kernel<<<dim3(ceil_div(tile_h * tile_w * channels, 256), B * g.tiles()), 256, 0, st>>>(d_images, d_tiles, g, channels);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_tile_merge_dev(dimb_fstore* fs, int B, const int* slots, int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w,
                        const float* d_kpts, const float* d_scores, const float* d_desc, const int* d_counts, int K, void* stream) {
  Grid g;
  if (!fs || !slots || !d_kpts || !d_scores || !d_desc || !d_counts || B < 1 || B > 65535 || K < 1 ||
      !make_grid(height, width, tile_h, tile_w, overlap_h, overlap_w, &g))
    return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b)
    if (slots[b] < 0 || slots[b] >= fs->n_slots) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  const long long L = static_cast<long long>(g.tiles()) * K;
  if (L >= (1ll << 30)) return DIMB_ERR_ARG;
  if (L > fs->cap) {
    dimb_set_error(ctx, "dimb_tile_merge_dev: " + std::to_string(g.tiles()) + " tiles x " + std::to_string(K) +
                            " keypoints exceed the store's capacity " + std::to_string(fs->cap));
    return DIMB_ERR_CAPACITY;
  }
  const int Li = static_cast<int>(L);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  Rec *ra, *rb, *sorted;
  unsigned* src;
  int *d_slots, *d_n;
  DIMB_TRY(dimb_scratch(ctx, kSlotKeysA, static_cast<size_t>(B) * Li * sizeof(Rec), reinterpret_cast<void**>(&ra)));
  DIMB_TRY(dimb_scratch(ctx, kSlotKeysB, static_cast<size_t>(B) * Li * sizeof(Rec), reinterpret_cast<void**>(&rb)));
  DIMB_TRY(dimb_scratch(ctx, kSlotParams, static_cast<size_t>(B) * sizeof(int), reinterpret_cast<void**>(&d_slots)));
  DIMB_TRY(dimb_scratch(ctx, kSlotSrc, static_cast<size_t>(B) * Li * sizeof(unsigned), reinterpret_cast<void**>(&src)));
  DIMB_TRY(dimb_scratch(ctx, kSlotCount, static_cast<size_t>(B) * sizeof(int), reinterpret_cast<void**>(&d_n)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_slots, slots, B * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.merge");
  const TileOut in{d_kpts, d_scores, d_desc, d_counts, K};
  tile_merge_keys_kernel<<<dim3(ceil_div(Li, 256), B), 256, 0, st>>>(in, g, ra, Li);
  DIMB_LAUNCH_CHECK(ctx);
  DIMB_TRY(seg_sort(ctx, st, ra, rb, B, Li, &sorted));
  seg_unique_kernel<<<B, kScanThreads, 0, st>>>(sorted, Li, MergeEmit{src, d_n, Li});
  DIMB_LAUNCH_CHECK(ctx);
  tile_merge_write_kernel<<<dim3(ceil_div(fs->cap, 256), fs->D + 1, B), 256, 0, st>>>(in, g, src, d_n, d_slots, fs_layout(fs), Li);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_tile_views_dev(dimb_fstore* src, int B, const int* src_slots, int n_tiles, dimb_fstore* dst, const int* dst_slots, int* d_map,
                        void* stream) {
  if (!src || !dst || !src_slots || !dst_slots || !d_map || B < 1 || B > 65535 || n_tiles < 1 || n_tiles > kMaxTiles ||
      static_cast<long long>(B) * n_tiles > 65535 || src->D != dst->D || src->ctx != dst->ctx)
    return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b)
    if (src_slots[b] < 0 || src_slots[b] >= src->n_slots || dst_slots[b] < 0 || dst_slots[b] > dst->n_slots - n_tiles) return DIMB_ERR_ARG;
  dimb_ctx* ctx = src->ctx;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<int> hp(src_slots, src_slots + B);
  hp.insert(hp.end(), dst_slots, dst_slots + B);
  int* d_slots;
  DIMB_TRY(dimb_scratch(ctx, kSlotParams, hp.size() * sizeof(int), reinterpret_cast<void**>(&d_slots)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_slots, hp.data(), hp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.views");
  tile_views_scan_kernel<<<dim3(n_tiles, B), kScanThreads, 0, st>>>(fs_layout(src), fs_layout(dst), d_slots, B, d_map);
  DIMB_LAUNCH_CHECK(ctx);
  tile_views_copy_kernel<<<dim3(ceil_div(dst->cap, 256), dst->D + 1, B * n_tiles), 256, 0, st>>>(fs_layout(src), fs_layout(dst), d_slots, B,
                                                                                               n_tiles, d_map);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_tile_match_merge_dev(dimb_ctx* ctx, int Q, const int* pair_offsets, const int* view0, const int* view1, const int* d_maps, int map_ld,
                              const int64_t* d_matches, const int* d_n_matches, int cap, int64_t* d_out, int* d_n_out, int cap2, void* stream) {
  if (!ctx || !pair_offsets || !d_maps || !d_n_out || !d_out || Q < 1 || Q > 65535 || map_ld < 1 || cap < 1 || cap2 < 1 ||
      pair_offsets[0] != 0)
    return DIMB_ERR_ARG;
  int widest = 0;
  for (int q = 0; q < Q; ++q) {
    if (pair_offsets[q + 1] < pair_offsets[q]) return DIMB_ERR_ARG;
    widest = std::max(widest, pair_offsets[q + 1] - pair_offsets[q]);
  }
  const int P = pair_offsets[Q];
  if (P > 0 && (!view0 || !view1 || !d_matches || !d_n_matches)) return DIMB_ERR_ARG;
  for (int p = 0; p < P; ++p)
    if (view0[p] < 0 || view1[p] < 0) return DIMB_ERR_ARG;
  const long long L = static_cast<long long>(widest) * cap;
  if (L >= (1ll << 30)) return DIMB_ERR_ARG;
  const int Li = static_cast<int>(L);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<int> hp(pair_offsets, pair_offsets + Q + 1);
  if (P > 0) {
    hp.insert(hp.end(), view0, view0 + P);
    hp.insert(hp.end(), view1, view1 + P);
  }
  Rec *ra, *rb, *sorted = nullptr;
  int* d_params;
  DIMB_TRY(dimb_scratch(ctx, kSlotKeysA, std::max<size_t>(1, static_cast<size_t>(Q) * Li) * sizeof(Rec), reinterpret_cast<void**>(&ra)));
  DIMB_TRY(dimb_scratch(ctx, kSlotKeysB, std::max<size_t>(1, static_cast<size_t>(Q) * Li) * sizeof(Rec), reinterpret_cast<void**>(&rb)));
  DIMB_TRY(dimb_scratch(ctx, kSlotParams, hp.size() * sizeof(int), reinterpret_cast<void**>(&d_params)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_params, hp.data(), hp.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.match_merge");
  if (Li > 0) {
    match_merge_keys_kernel<<<dim3(ceil_div(Li, 256), Q), 256, 0, st>>>(d_params, Q, d_maps, map_ld, d_matches, d_n_matches, cap, ra, Li);
    DIMB_LAUNCH_CHECK(ctx);
    DIMB_TRY(seg_sort(ctx, st, ra, rb, Q, Li, &sorted));
  }
  seg_unique_kernel<<<Q, kScanThreads, 0, st>>>(Li > 0 ? sorted : ra, Li, MatchEmit{d_out, d_n_out, cap2});
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_resize_area_tab(int ssize, int dsize, int* d_idx, int* s_idx, float* alpha, int cap, int* n) {
  if (!n || ssize < 1 || dsize < 1 || dsize > ssize || cap < 0 || (cap > 0 && (!d_idx || !s_idx || !alpha))) return DIMB_ERR_ARG;
  std::vector<int> di, si;
  std::vector<float> a;
  area_tab(ssize, dsize, &di, &si, &a);
  *n = static_cast<int>(di.size());
  if (*n > cap) return DIMB_ERR_CAPACITY;
  std::copy(di.begin(), di.end(), d_idx);
  std::copy(si.begin(), si.end(), s_idx);
  std::copy(a.begin(), a.end(), alpha);
  return DIMB_OK;
}

int dimb_resize_area_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2, void* stream) {
  if (!ctx || !d_src || !d_dst || B < 1 || B > 65535 || height < 1 || width < 1 || height > (1 << 20) || width > (1 << 20) || height2 < 1 ||
      width2 < 1 || height2 > height || width2 > width || height2 > 65535)
    return DIMB_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (height2 == height && width2 == width) {
    ProfScope prof(ctx, st, "tile.resize");
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_dst, d_src, static_cast<size_t>(B) * height * width * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return DIMB_OK;
  }
  return resize_area_launch<GrayPixel>(ctx, d_src, B, height, width, d_dst, height2, width2, st);
}

int dimb_resize_area_linear_tab(int ssize, int dsize, int* s_idx, float* alpha, int* xmax) {
  if (ssize < 1 || dsize < 1 || !s_idx || !alpha || !xmax) return DIMB_ERR_ARG;
  *xmax = area_linear_tab(ssize, dsize, s_idx, alpha);
  return DIMB_OK;
}

int dimb_resize_area_linear_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                                void* stream) {
  if (!ctx || !d_src || !d_dst || B < 1 || B > 65535 || height < 1 || width < 1 || height > (1 << 20) || width > (1 << 20) || height2 < 1 ||
      width2 < 1 || height2 > 65535 || width2 > (1 << 20) || (height2 <= height && width2 <= width))
    return DIMB_ERR_ARG;
  return resize_area_linear_launch<GrayPixel>(ctx, d_src, B, height, width, d_dst, height2, width2, static_cast<cudaStream_t>(stream));
}

int dimb_resize_area_rgb_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                             void* stream) {
  if (!ctx || !d_src || !d_dst || B < 1 || B > 65535 || height < 1 || width < 1 || height > (1 << 20) || width > (1 << 20) || height2 < 1 ||
      width2 < 1 || height2 > 65535 || width2 > (1 << 20))
    return DIMB_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (height2 > height || width2 > width)
    return resize_area_linear_launch<RgbGrayPixel>(ctx, d_src, B, height, width, d_dst, height2, width2, st);
  return resize_area_launch<RgbGrayPixel>(ctx, d_src, B, height, width, d_dst, height2, width2, st);  // equal size: factors 1 x 1
}

int dimb_pyr_size(int height, int width, int level, int* height2, int* width2) {
  if (!height2 || !width2 || level < -1 || level > 3 || height < 1 || width < 1 || height > (1 << 20) || width > (1 << 20)) return DIMB_ERR_ARG;
  int h = height, w = width;
  if (level < 0) h *= 2, w *= 2;
  for (int l = 0; l < level; ++l) h = (h + 1) / 2, w = (w + 1) / 2;
  *height2 = h, *width2 = w;
  return DIMB_OK;
}

int dimb_pyr_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, int channels, int level, float* d_dst, void* stream) {
  int h2, w2;
  if (!ctx || !d_src || !d_dst || B < 1 || B > 65535 || (channels != 1 && channels != 3) || dimb_pyr_size(height, width, level, &h2, &w2) != DIMB_OK)
    return DIMB_ERR_ARG;
  // every launch has one CTA row per output row; the widest row is the source's (down) or the output's (up)
  const long long rows = level < 0 ? 2ll * height : (height + 1) / 2, row_len = (level < 0 ? 2ll * width : width) * channels;
  if (rows > 65535 || row_len >= (1ll << 30)) return DIMB_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (level == 0) {
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_dst, d_src, static_cast<size_t>(B) * height * width * channels * sizeof(float),
                                      cudaMemcpyDeviceToDevice, st));
    return DIMB_OK;
  }
  float* mid[2] = {nullptr, nullptr};
  for (int l = 1; l < level; ++l) {  // intermediates of a chain: level l's output in mid[(l - 1) % 2]
    int hl, wl;
    dimb_pyr_size(height, width, l, &hl, &wl);
    DIMB_TRY(dimb_scratch(ctx, (l - 1) % 2 ? kSlotPyrB : kSlotPyrA, static_cast<size_t>(B) * hl * wl * channels * sizeof(float),
                          reinterpret_cast<void**>(&mid[(l - 1) % 2])));
  }
  ProfScope prof(ctx, st, "tile.pyr");
  if (level < 0) {
    pyr_up_kernel<<<dim3(ceil_div(2 * width * channels, 128), 2 * height, B), 128, 0, st>>>(d_src, d_dst, height, width, channels);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  }
  const float* in = d_src;
  int h = height, w = width;
  for (int l = 1; l <= level; ++l) {
    const int hn = (h + 1) / 2, wn = (w + 1) / 2;
    float* out = l == level ? d_dst : mid[(l - 1) % 2];
    pyr_down_kernel<<<dim3(ceil_div(wn * channels, 128), hn, B), 128, 0, st>>>(in, out, h, w, channels, hn, wn);
    DIMB_LAUNCH_CHECK(ctx);
    in = out, h = hn, w = wn;
  }
  return DIMB_OK;
}

int dimb_fstore_rescale_dev(dimb_fstore* fs, int B, const int* slots, int level, int height, int width, void* stream) {
  if (!fs || !slots || B < 1 || B > 65535 || level < -1 || level > 3 || height < 1 || width < 1) return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b)
    if (slots[b] < 0 || slots[b] >= fs->n_slots) return DIMB_ERR_ARG;
  dimb_ctx* ctx = fs->ctx;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* d_slots;
  DIMB_TRY(dimb_scratch(ctx, kSlotRescale, static_cast<size_t>(B) * sizeof(int), reinterpret_cast<void**>(&d_slots)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_slots, slots, B * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.pyr");
  fs_rescale_kernel<<<dim3(ceil_div(fs->cap, 256), B), 256, 0, st>>>(fs_layout(fs), d_slots, std::ldexp(1.f, level), height, width);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// upright (image_matching.py:496 rotates the images, :703 rotates the keypoints back)
int dimb_rot90_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, int channels, const int* rotations, float* d_dst,
                   void* stream) {
  if (!ctx || !d_src || !d_dst || !rotations || B < 1 || B > 65535 || (channels != 1 && channels != 3) || height < 1 || width < 1 ||
      height > (1 << 20) || width > (1 << 20) || ceil_div(height, kRotTile) > 65535)
    return DIMB_ERR_ARG;
  std::vector<int> quarter(B);
  for (int b = 0; b < B; ++b) {
    if (rotations[b] != 0 && rotations[b] != 90 && rotations[b] != 180 && rotations[b] != 270) return DIMB_ERR_ARG;
    quarter[b] = rotations[b] / 90;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* d_quarter;
  DIMB_TRY(dimb_scratch(ctx, kSlotRotCodes, static_cast<size_t>(B) * sizeof(int), reinterpret_cast<void**>(&d_quarter)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_quarter, quarter.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.rot");
  rot90_kernel<<<dim3(ceil_div(width, kRotTile), ceil_div(height, kRotTile), B), dim3(kRotTile, 8), 0, st>>>(d_src, d_dst, height, width,
                                                                                                              channels, d_quarter);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_fstore_unrotate_dev(dimb_fstore* fs, int B, const int* slots, const int* rotations, const int* heights, const int* widths,
                             void* stream) {
  if (!fs || !slots || !rotations || !heights || !widths || B < 1 || B > 65535) return DIMB_ERR_ARG;
  std::vector<Unrotate> items(B);
  for (int b = 0; b < B; ++b) {
    const int r = rotations[b];
    if (slots[b] < 0 || slots[b] >= fs->n_slots || (r != 0 && r != 90 && r != 180 && r != 270) || heights[b] < 1 || widths[b] < 1)
      return DIMB_ERR_ARG;
    items[b] = {slots[b], r / 90, heights[b], widths[b]};
  }
  dimb_ctx* ctx = fs->ctx;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  Unrotate* d_items;
  DIMB_TRY(dimb_scratch(ctx, kSlotUnrotate, static_cast<size_t>(B) * sizeof(Unrotate), reinterpret_cast<void**>(&d_items)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_items, items.data(), B * sizeof(Unrotate), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.rot");
  fs_unrotate_kernel<<<dim3(ceil_div(fs->cap, 256), B), 256, 0, st>>>(fs_layout(fs), d_items);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_kpts_extent_dev(dimb_ctx* ctx, int B, const float* d_kpts, int kpt_ld, const int* d_counts, float* d_size_out, void* stream) {
  if (!ctx || !d_kpts || !d_counts || !d_size_out || B < 1 || kpt_ld < 1) return DIMB_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope prof(ctx, st, "tile.extent");
  kpts_extent_kernel<<<B, 256, 0, st>>>(d_kpts, kpt_ld, d_counts, d_size_out);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_tile_preselect_pairs_dev(dimb_ctx* ctx, int Q, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                                  const int* d_n_matches, int cap, const int* sizes, int tile_h, int tile_w, int overlap_h, int overlap_w,
                                  const double* scales, int min_matches_per_tile, int* d_counts, unsigned char* d_flags, void* stream) {
  if (!ctx || !f0 || !f1 || !d_matches || !d_n_matches || !sizes || !scales || !d_counts || !d_flags || Q < 1 || Q > 65535 || cap < 1 ||
      min_matches_per_tile < 0)
    return DIMB_ERR_ARG;
  std::vector<PrePair> hp(Q);
  size_t n = 0;
  for (int q = 0; q < Q; ++q) {
    PrePair& p = hp[q];
    const int* s = sizes + 4 * q;
    if (!f0[q].keypoints || !f1[q].keypoints || !make_grid(s[0], s[1], tile_h, tile_w, overlap_h, overlap_w, &p.g0) ||
        !make_grid(s[2], s[3], tile_h, tile_w, overlap_h, overlap_w, &p.g1))
      return DIMB_ERR_ARG;
    p.sc0 = static_cast<float>(scales[2 * q]), p.sc1 = static_cast<float>(scales[2 * q + 1]);  // numpy: float32 array / Python float in float32
    if (!(std::isfinite(p.sc0) && p.sc0 > 0.f && std::isfinite(p.sc1) && p.sc1 > 0.f)) return DIMB_ERR_ARG;
    p.s0 = PreSide{f0[q].keypoints, f0[q].f16, f0[q].round_fp16};
    p.s1 = PreSide{f1[q].keypoints, f1[q].f16, f1[q].round_fp16};
    p.off = n;
    n += static_cast<size_t>(p.g0.tiles()) * p.g1.tiles();
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  PrePair* d_pairs;
  DIMB_TRY(dimb_scratch(ctx, kSlotPreSides, hp.size() * sizeof(PrePair), reinterpret_cast<void**>(&d_pairs)));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(d_pairs, hp.data(), hp.size() * sizeof(PrePair), cudaMemcpyHostToDevice, st));
  ProfScope prof(ctx, st, "tile.preselect");
  DIMB_CUDA_OK(ctx, cudaMemsetAsync(d_counts, 0, n * sizeof(int), st));
  tile_preselect_count_kernel<<<dim3(ceil_div(cap, 128), Q), 128, 0, st>>>(d_pairs, d_matches, d_n_matches, cap, d_counts);
  DIMB_LAUNCH_CHECK(ctx);
  tile_preselect_flag_kernel<<<static_cast<int>(std::min<size_t>((n + 255) / 256, 4096)), 256, 0, st>>>(d_counts, n, min_matches_per_tile,
                                                                                                    d_flags);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

int dimb_tile_preselect_dev(dimb_ctx* ctx, int Q, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                            const int* d_n_matches, int cap, int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w,
                            double scale0, double scale1, int min_matches_per_tile, int* d_counts, unsigned char* d_flags, void* stream) {
  if (Q < 1 || Q > 65535) return DIMB_ERR_ARG;
  std::vector<int> sizes(4 * static_cast<size_t>(Q));
  std::vector<double> scales(2 * static_cast<size_t>(Q));
  for (int q = 0; q < Q; ++q) {
    sizes[4 * q] = sizes[4 * q + 2] = height, sizes[4 * q + 1] = sizes[4 * q + 3] = width;
    scales[2 * q] = scale0, scales[2 * q + 1] = scale1;
  }
  return dimb_tile_preselect_pairs_dev(ctx, Q, f0, f1, d_matches, d_n_matches, cap, sizes.data(), tile_h, tile_w, overlap_h, overlap_w,
                                       scales.data(), min_matches_per_tile, d_counts, d_flags, stream);
}

}  // extern "C"
