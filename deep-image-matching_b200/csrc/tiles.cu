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
#include <vector>

#include "fstore.cuh"

namespace {

constexpr int kMaxTiles = 2048;        // tile_idx is stored as float16: integers up to 2048 are exact
constexpr int kChunk = 1024;           // records per shared-memory sort
constexpr int kScanThreads = 1024;     // threads of the one-CTA-per-segment scans
constexpr int kSlotKeysA = 64, kSlotKeysB = 65, kSlotParams = 66, kSlotSrc = 67, kSlotCount = 68;  // context scratch slots
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

}  // extern "C"
