/* dimb200.h - C ABI of libdimb200.so: the H100-native (sm_90a) hot path of
 * 3DOM-FBK/deep-image-matching behind plain pointers and sizes.
 *
 * Each entry point replaces the body of one reference plugin method (paths are
 * relative to src/deep_image_matching/ of the reference at 74d7bd5):
 *
 *   dimb_sp_extract      <- SuperPointExtractor._extract      extractors/superpoint.py:107-132
 *                           (+ model thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:160-227)
 *   dimb_lg_match        <- LightGlueMatcher._match_pairs     matchers/lightglue.py:102-125
 *                           (+ featuresDict2Lightglue :8-66, model thirdparty/LightGlue/lightglue/lightglue.py:424-579)
 *   dimb_nn_match        <- KorniaMatcher._match_pairs        matchers/kornia_matcher.py:27-54
 *                           (kornia.feature.DescriptorMatcher modes nn/mnn/snn/smnn)
 *   *_dev variants       :  same computation on device pointers and a caller stream, so that
 *                           features never leave HBM between extraction and matching
 *                           (the reference round-trips them through features.h5, extractor_base.py:56-99).
 *
 * Conventions: every function returns DIMB_OK (0) or a negative error code; the message is
 * available from dimb_last_error(ctx) and contains "CUDA out of memory" for allocation failures
 * (matchers/matcher_base.py:251-254 keys its tile fallback on that text).  Caller owns all host
 * buffers; the library owns device memory inside its handles.  One ctx per device, not thread-safe.
 * There is NO CPU fallback: without a CUDA device every create call fails.
 */
#ifndef DIMB200_H
#define DIMB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dimb_ctx dimb_ctx;
typedef struct dimb_sp dimb_sp;
typedef struct dimb_lg dimb_lg;

enum {
  DIMB_OK = 0,
  DIMB_ERR_CUDA = -1,
  DIMB_ERR_OOM = -2,
  DIMB_ERR_ARG = -3,
  DIMB_ERR_UNSUPPORTED = -4,
  DIMB_ERR_CAPACITY = -5
};

/* Arithmetic mode of the tensor-core contractions (SURVEY Appendix C):
 *   EXACT: fp16 hi+lo split operands, 3 MMAs per product, fp32 accumulate -> fp32-class results
 *          (parity mode, graded against the fp32 oracle at 1e-4).
 *   FAST : plain fp16 operands (statistically equivalent to the reference's TF32/fp16 GPU path). */
enum { DIMB_PRECISION_EXACT = 0, DIMB_PRECISION_FAST = 1 };

/* ------------------------------------------------------------------ context */
int dimb_ctx_create(int device, dimb_ctx** out);
void dimb_ctx_destroy(dimb_ctx* ctx);
const char* dimb_last_error(dimb_ctx* ctx);
int dimb_ctx_set_precision(dimb_ctx* ctx, int precision);
/* Number of kernels this library has launched on ctx (bench.py "gpu_launches"). */
unsigned long long dimb_ctx_launch_count(dimb_ctx* ctx);
const char* dimb_version(void);
/* Synchronising device -> host copy of a buffer the library exposed through a *_dev accessor (tests, debug taps). */
int dimb_read_dev(dimb_ctx* ctx, void* dst, const void* d_src, size_t bytes);
/* Per-kernel-group device timing with CUDA events on the launching stream (bench.py roofline):
 * dimb_ctx_profile(ctx, 1) starts recording, dimb_ctx_profile_read returns the JSON text
 * {"<group>": [total_ms, launches], ...}; dimb_ctx_profile(ctx, 0) stops and clears. */
int dimb_ctx_profile(dimb_ctx* ctx, int enable);
int dimb_ctx_profile_read(dimb_ctx* ctx, char* buf, size_t n);

/* ------------------------------------------------------------------ SuperPoint */
typedef struct {
  int nms_radius;            /* config.py:96  (3)      */
  float keypoint_threshold;  /* config.py:97  (0.0005) */
  int max_keypoints;         /* config.py:98  (2048); -1 = unlimited; any positive limit (above 16384 a grid-wide top-k runs) */
  int remove_borders;        /* superpoint.py default (4) */
  int fix_sampling;          /* 0: thirdparty superpoint.py:81-98, 1: extractors/superpoint.py:16-27 */
  int max_batch;             /* workspace sizing: images per call */
  int max_height, max_width; /* workspace sizing */
} dimb_sp_conf;

/* weights: packed fp32, PyTorch OIHW tensors in this order, each weight followed by its bias:
 * conv1a conv1b conv2a conv2b conv3a conv3b conv4a conv4b convPa convPb convDa convDb
 * (1,300,865 floats for superpoint_v1). */
int dimb_sp_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_sp_conf* conf, dimb_sp** out);
void dimb_sp_destroy(dimb_sp* sp);

/* images: host float32 [B][H][W], gray 0..255 (what ExtractorBase.extract hands to _extract).
 * Outputs (host, caller allocated): kpts [B][cap][2] (x,y) float32, scores [B][cap],
 * desc [B][256][cap] i.e. (D,N) with row pitch cap, counts [B].  Order: reference order
 * (row-major if <= max_keypoints candidates, else score-descending).  Returns
 * DIMB_ERR_CAPACITY (counts filled) if an image yields more than cap keypoints. */
int dimb_sp_extract(dimb_sp* sp, const float* images, int B, int H, int W, float* kpts, float* scores, float* desc,
                    int* counts, int cap);
/* Same on device pointers, asynchronous on `stream` (a cudaStream_t); counts stay on device. */
int dimb_sp_extract_dev(dimb_sp* sp, const float* d_images, int B, int H, int W, float* d_kpts, float* d_scores,
                        float* d_desc, int* d_counts, int cap, void* stream);
/* Debug taps (device->host copies of intermediates of the LAST extract call, image 0):
 * which: 0 = dense score map [H8*8][W8*8], 1 = nms map, 2 = encoder output [h][w][128] (fp32, NHWC),
 * 3 = dense descriptors (un-normalised convDb output) [h][w][256]. */
int dimb_sp_debug_read(dimb_sp* sp, int which, float* out, size_t n_floats);

/* ------------------------------------------------------------------ LightGlue */
typedef struct {
  int input_dim;           /* 256 superpoint, 128 aliked/disk (lightglue.py:330-359) */
  int descriptor_dim;      /* 256 (tensor-core kernels); any other shape, e.g. LighterGlue's 96, runs the generic fp32 path */
  int n_layers;            /* 9 (LighterGlue: 6) */
  int num_heads;           /* 4 (LighterGlue: 1); head dim = descriptor_dim / num_heads must be even and <= 128 */
  double depth_confidence; /* 0.95, -1 disables early exit (double: compared as float(x), like torch) */
  double width_confidence; /* 0.99, -1 disables point pruning; the keep test uses float(1 - width_confidence) */
  double filter_threshold; /* 0.1 */
  int prune_min_kpts;      /* 1536 = reference CUDA+flash semantics (lightglue.py:318-323,606-610) */
  int max_pairs;           /* workspace sizing: pairs per call */
  int max_kpts;            /* workspace sizing: keypoints per image */
} dimb_lg_conf;

/* weights: packed fp32 in this order (names as in the reference state_dict, SURVEY Appendix D):
 *   posenc.Wr.weight (hd/2,2); [input_proj.weight (d,din), input_proj.bias] iff din != d;
 *   for i in layers: self_attn.{Wqkv,out_proj,ffn.0}.{weight,bias}, ffn.1.{weight,bias}, ffn.3.{weight,bias},
 *                    cross_attn.{to_qk,to_v,to_out,ffn.0}.{weight,bias}, ffn.1.{weight,bias}, ffn.3.{weight,bias};
 *   for i in layers: log_assignment.i.matchability.{weight,bias}, log_assignment.i.final_proj.{weight,bias};
 *   for i in layers-1: token_confidence.i.token.0.{weight,bias}.
 * Replaces LightGlue.__init__ + load_state_dict (lightglue.py:325-398) and, for descriptor_dim 96 / one head / 6 layers /
 * input_dim 64, LighterGlue.__init__ (thirdparty/accelerated_features/modules/lighterglue.py:29-48). */
int dimb_lg_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* conf, dimb_lg** out);
void dimb_lg_destroy(dimb_lg* lg);

typedef struct {
  const float* keypoints;   /* (n,2) x,y float32 */
  const float* descriptors; /* float32; layout below */
  int n;                    /* number of keypoints */
  int desc_layout;          /* 0: (D,n) rows of pitch desc_ld (FeaturesDict layout), 1: (n,D) rows of pitch desc_ld */
  int desc_ld;              /* row pitch in floats (0 = dense) */
  int has_size;             /* 0: size := 1 + max(kpts) - min(kpts) (lightglue.py:26-27) */
  float size0, size1;       /* image_size exactly as the caller stores it ([H,W] in DIM; quirk A.3) */
} dimb_feats;

/* P pairs.  Outputs (host): matches [P][cap][2] int64 (ascending in column 0), mscores [P][cap],
 * n_matches [P], stop_layer [P] (1-based layer count executed, the reference's "stop").  The pairs are staged into
 * dimb_lg_match_dev; all P are checked before any launch, and a count above cap returns DIMB_ERR_CAPACITY after every pair's
 * outputs (its first cap matches, its full count) are written.
 * Replaces LightGlueMatcher._match_pairs (matchers/lightglue.py:102-125) and LighterGlueMatcher._match_pairs
 * (matchers/lighterglue.py:105-262). */
int dimb_lg_match(dimb_lg* lg, int P, const dimb_feats* f0, const dimb_feats* f1, int64_t* matches, float* mscores,
                  int* n_matches, int* stop_layer, int cap);

typedef struct {
  const float* keypoints;   /* device (n_cap,2) */
  const float* descriptors; /* device; layout below */
  const int* n;             /* device scalar: number of valid keypoints (<= n_cap) */
  int n_cap;
  int desc_layout;          /* 0: (D,n) rows of pitch desc_ld, 1: (n,D) rows of pitch desc_ld */
  int desc_ld;
  float size0, size1;
  int round_fp16;           /* 1: round keypoints/descriptors to fp16 first, as the features.h5 round trip does */
  int f16;                  /* 1: keypoints and descriptors ARE float16 arrays (device feature store blocks); round_fp16 is moot */
  const int* size_dev;      /* non-NULL: device int[2] holding image_size ([H,W]); overrides size0 / size1 */
  const float* size_f32_dev; /* non-NULL: device float[2] used as the normalisation size as is (e.g. dimb_kpts_extent_dev's
                                own-extent size); overrides size0 / size1 / size_dev */
} dimb_feats_dev;

/* Device-resident variant, asynchronous on `stream` (no host synchronisation once its scratch, sized for max_pairs by the first
 * call, exists); d_matches [P][cap][2] int64 ascending in column 0, d_mscores [P][cap], d_n_matches [P] (the full count, also above
 * cap; only cap rows are written), d_stop_layer [P] are device buffers.  A pair with an empty side gets stop 1 and 0 matches.
 * DIMB_ERR_ARG, before any CUDA call, for P outside [1, max_pairs], cap < 1, n_cap above max_kpts or a NULL pointer.  Every shape:
 * descriptor_dim 256 / 4 heads runs the tensor-core kernels; other shapes (LighterGlue: 96 / 1 head) run the shape-generic
 * engine.  dimb_lg_match stages host pairs into this entry for both.  For the shape-generic engine, size0 = size1 = 0 with no
 * size_dev / size_f32_dev normalises by the keypoints' own extent (1 + max) - min, as dimb_lg_match does without has_size. */
int dimb_lg_match_dev(dimb_lg* lg, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches,
                      float* d_mscores, int* d_n_matches, int* d_stop_layer, int cap, void* stream);
/* Debug tap: fp32 descriptors x[side][row][d] after the last executed layer of the LAST call (host copy). */
int dimb_lg_debug_read(dimb_lg* lg, int which, int side, float* out, size_t n_floats);

/* ------------------------------------------------------------------ brute-force descriptor NN */
enum { DIMB_NN_NN = 0, DIMB_NN_MNN = 1, DIMB_NN_SNN = 2, DIMB_NN_SMNN = 3 };

/* d0: (D,n0) float32 host (FeaturesDict layout), d1: (D,n1); any descriptor size D >= 1 (zero-padded to a multiple of 64 on
 * device, which changes no distance).  Outputs: idx [cap][2] int64 sorted by column 0, dist [cap] (distance for nn/mnn, ratio
 * for snn/smnn), n = number of matches.  Descriptors that are exactly fp16-representable (everything read back from
 * features.h5 is, extractor_base.py:56-99) are detected on device and take the single-MMA path: its products are then exact and
 * only the fp32 accumulation rounds, so integer descriptors whose squared norms add up to less than 2^24 (ORB's and SIFT's) get
 * correctly rounded distances and tables that follow kornia's rules exactly, ties included. */
int dimb_nn_match(dimb_ctx* ctx, const float* d0, int n0, const float* d1, int n1, int D, int mode, float th,
                  int64_t* idx, float* dist, int* n, int cap);
/* Same on device pointers, asynchronous on `stream`: d_desc0 / d_desc1 are (D,n) arrays of row pitch ld0 / ld1 elements
 * (0 = dense), float32 (desc_f16 = 0) or float16 (desc_f16 = 1: the layout the device feature store keeps, single-MMA
 * path); d_idx [cap][2] int64, d_dist [cap], d_n [1] are device buffers.  The sequential-pair workload of
 * pairs_generator.py:22-34 keeps every image's descriptors in HBM and calls this once per pair. */
int dimb_nn_match_dev(dimb_ctx* ctx, const void* d_desc0, int n0, int ld0, const void* d_desc1, int n1, int ld1, int D, int desc_f16,
                      int mode, float th, int64_t* d_idx, float* d_dist, int* d_n, int cap, void* stream);
/* P pairs, asynchronous on `stream`, never synchronises once its scratch has grown to the call's size.  f0[p] / f1[p] (host arrays
 * of P): only descriptors, n (device), n_cap, desc_layout (0 only), desc_ld, f16 and round_fp16 are read; rows = min(*n, n_cap).
 * d_idx [P][cap][2] int64, d_dist [P][cap] (distance for nn / mnn, ratio for snn / smnn), d_n [P] = the full count (only the first
 * cap rows are written), in the order and with the empty-input rules of dimb_nn_match (kornia's).  round_fp16 = 1 rounds float32
 * descriptors to fp16 first (round to nearest even, the features.h5 cast).  Three MMAs per product (EXACT) only when some side is
 * float32 without round_fp16; fp16 inputs need one (exact products).  Results per pair do not depend on the other pairs of the call.
 * dimb_nn_match_dev and dimb_nn_match run this engine with P = 1.  DIMB_ERR_ARG, before any CUDA call, for a NULL ctx / array /
 * output / descriptors / n, P < 1, cap < 1, D < 1, mode outside 0..3, n_cap < 0 or desc_layout != 0.
 * Scratch (context slots, grow-only), NPp = the largest n_cap rounded up to 128, Dp = D rounded up to 64: the fp16 operands
 * 2P x NPp x Dp x 2 B (twice with the three-MMA split), and the chunk partials of the top-2 GEMM, P x NPp x NPp / 32 x 12 B, shared
 * by the two directions of mnn / smnn: about 25 MB per pair at 8192 keypoints, 1.6 MB at 2048.
 * Profile groups: nn.prep, nn.top2_gemm, nn.merge, nn.select. */
int dimb_nn_match_batch_dev(dimb_ctx* ctx, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int D, int mode, float th,
                            int64_t* d_idx, float* d_dist, int* d_n, int cap, void* stream);

/* ------------------------------------------------------------------ device feature store (the features.h5 boundary kept in HBM)
 * Replaces, for the hot path, save_features_h5 (extractors/extractor_base.py:56-99: every array cast to float16, gzip-9, one
 * group per image) and get_features (io/h5.py:45-89: re-read per image per pair, matchers/matcher_base.py:221-222).  One
 * fixed-size block per image: int32 header {n, H, W, valid}, then float16 keypoints [cap][2], scores [cap], tile_idx [cap],
 * descriptors [D][cap] - the exact values features.h5 would hold.  Blocks are contiguous so that the multi-GPU path can
 * all-gather them over NCCL (SURVEY 8e) and an h5 writer needs one bulk copy. */
typedef struct dimb_fstore dimb_fstore;
int dimb_fstore_create(dimb_ctx* ctx, int n_slots, int cap, int desc_dim, dimb_fstore** out);
void dimb_fstore_destroy(dimb_fstore* fs);
/* Device put (asynchronous on `stream`): float32 features in the layouts of dimb_sp_extract_dev / dimb_aliked_extract_dev
 * (d_desc (D,n) rows of pitch desc_ld, d_count device scalar); d_scores / d_tile_idx may be NULL (ones / zeros, as
 * ExtractorBase.extract fills them, extractor_base.py:226,371-373).  The float16 cast of the h5 writer happens here. */
int dimb_fstore_put_dev(dimb_fstore* fs, int slot, const float* d_kpts, const float* d_scores, const float* d_tile_idx, const float* d_desc,
                        int desc_ld, const int* d_count, int height, int width, void* stream);
/* Host put: kpts (n,2), scores (n,) or NULL, tile_idx (n,) or NULL, desc (D,n) dense. */
int dimb_fstore_put(dimb_fstore* fs, int slot, const float* kpts, const float* scores, const float* tile_idx, const float* desc, int n,
                    int height, int width);
/* n = keypoints stored in the slot (-1: empty); image_size[2] = [H,W].  Synchronises. */
int dimb_fstore_count(dimb_fstore* fs, int slot, int* n, int* image_size);
/* get_features' contract: float32 host arrays whose values are float16-exact, desc (D,n) dense; any output may be NULL. */
int dimb_fstore_get(dimb_fstore* fs, int slot, float* kpts, float* scores, float* tile_idx, float* desc, int* n, int* image_size, int cap);
/* The slot as a dimb_feats_dev with f16 = 1, for dimb_lg_match_dev; its descriptors also feed dimb_nn_match_dev (desc_f16 = 1, ld = cap). */
int dimb_fstore_feats_dev(dimb_fstore* fs, int slot, dimb_feats_dev* out);
/* Raw blocks: base pointer, bytes per slot, slot count, keypoint capacity (slot s starts at base + s * slot_bytes). */
int dimb_fstore_block_dev(dimb_fstore* fs, void** d_base, size_t* slot_bytes, int* n_slots, int* cap);

/* ------------------------------------------------------------------ geometric verification (fundamental-matrix RANSAC)
 * Replaces the estimator inside geometric_verification (utils/geometric_verification.py:45-179: pydegensac.findFundamentalMatrix /
 * cv2.findFundamentalMat), the step after _match_pairs (matchers/matcher_base.py:298-340).  Three estimators (dimb_gv_conf.estimator),
 * both with Sampson inliers (threshold in pixels) and two least-squares refits of the final model:
 *   ransac8: max(64, min(max_iters, 8192)) 8-point hypotheses per pair in parallel, no adaptive stopping;
 *   lo-ransac: 7-point hypotheses in waves of 1024, local optimisation of each wave's new best model (inner RANSAC on 16-inlier
 *     least-squares fits, each iterated 4 times) and confidence stopping, up to min(max_iters, 65536) hypotheses;
 *   degensac: lo-ransac plus DEGENSAC's dominant-plane test of each 7-point model (H from F and three points over five triplets,
 *     5 of 7 sample points within 2 x threshold transfer error) and plane-and-parallax recovery of F = [e']_x H from up to 1024
 *     pairs of off-plane matches when a wave finds a better plane; n_hypotheses counts the 7-point hypotheses.
 * Stochastic like the reference's estimators (seeded, reproducible here): parity is statistical.  F row-major, x1^T F x0 = 0; zeros
 * and an all-ones mask when fewer than 8 matches exist or no model is found (the reference returns F = None, mask all True).
 * dimb_gv_fundamental is dimb_gv_estimate with ransac8. */
int dimb_gv_fundamental(dimb_ctx* ctx, const float* kpts0, const float* kpts1, int n, float threshold, int max_iters, unsigned seed, float* F,
                        unsigned char* mask, int* n_inliers);
/* P pairs on device buffers, asynchronous on `stream`: matches in the output layout of dimb_lg_match_dev / dimb_pipe_* ([P][cap][2]
 * int64 + [P] counts) indexing the per-pair keypoint arrays d_kpts0[p] / d_kpts1[p] ((N,2) float32; the pointer ARRAYS are host). */
int dimb_gv_fundamental_batch_dev(dimb_ctx* ctx, int P, const float* const* d_kpts0, const float* const* d_kpts1, const int64_t* d_matches,
                                  const int* d_n_matches, int cap, float threshold, int max_iters, unsigned seed, float* d_F,
                                  unsigned char* d_mask, int* d_n_inliers, void* stream);
/* Verification of an image set's match tables (the step between _match_pairs and the COLMAP database).  Every GV entry is bitwise
 * reproducible: a pair's mask, F and count depend on its matches, its seed and the configuration only. */
typedef struct {
  float threshold;          /* Sampson distance threshold in pixels, > 0 */
  int max_iters;            /* ransac8: hypotheses per pair = max(64, min(max_iters, 8192)); lo-ransac, degensac: at most
                               min(max_iters, 65536) */
  int min_inliers;          /* gate: a pair keeps its verified table iff n_inliers >= min_inliers ... */
  float min_inlier_ratio;   /* ... and float(n_inliers) >= min_inlier_ratio * float(n_raw), in [0, 1] (0 / 0: every pair kept) */
  int estimator;            /* 0: ransac8, 1: lo-ransac, 3: degensac; 2 and every other value are refused (a zero-filled trailing part of the struct means
                               ransac8) */
  float confidence;         /* lo-ransac and degensac only: stop once the best model leaves a chance below 1 - confidence of having missed a
                               better all-inlier 7-point sample, in (0, 1) */
} dimb_gv_conf;
/* One pair on host buffers (n,2) float32 with the estimator of `conf` (its gate fields are not read): F [9], mask [n], n_inliers as
 * dimb_gv_fundamental; n_hypotheses (may be NULL): the hypotheses that ran (ransac8: its fixed count; 0 when n < 8).  Equal to
 * dimb_gv_verify_dev on the same points and seed.  DIMB_ERR_ARG, before any CUDA call, for the argument errors of
 * dimb_gv_fundamental, an unknown estimator, and with lo-ransac or degensac confidence outside (0, 1) or max_iters < 1. */
int dimb_gv_estimate(dimb_ctx* ctx, const float* kpts0, const float* kpts1, int n, const dimb_gv_conf* conf, unsigned seed, float* F,
                     unsigned char* mask, int* n_inliers, int* n_hypotheses);
/* P pairs, asynchronous on `stream`, never synchronises (once its scratch has grown to the call's size).  Keypoints come from
 * f0[p] / f1[p], of which only keypoints, f16 and round_fp16 are read: feature-store slots or float32 extractor outputs.
 * d_matches [P][cap][2] int64 + d_n_matches [P] in the layout of dimb_lg_match_dev / dimb_sg_match_dev (n_raw = min(d_n_matches[p],
 * cap)).  seeds: HOST array [P], the RNG seed of each pair (independent of the pair's position in the call).  Outputs (device):
 * d_verified [P][cap][2] int64 = the rows of d_matches whose mask is 1, in their original order; d_n_verified [P] = n_inliers, or 0
 * when the gate rejects the pair; d_F [P][9] (x1^T F x0 = 0, zeros when no model); d_mask [P][cap]; d_n_inliers [P].  Pairs with
 * fewer than 8 raw matches (or no model): mask all ones, F zeros, n_inliers = n_raw, then the gate.  DIMB_ERR_ARG, before any CUDA
 * call, for a NULL ctx / f0 / f1 / seeds / conf / buffer / keypoint pointer, P < 1, cap < 1, threshold <= 0, min_inliers < 0,
 * min_inlier_ratio outside [0, 1], an unknown estimator, and with lo-ransac or degensac confidence outside (0, 1) or max_iters < 1. */
int dimb_gv_verify_dev(dimb_ctx* ctx, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                       const int* d_n_matches, int cap, const unsigned* seeds, const dimb_gv_conf* conf, int64_t* d_verified,
                       int* d_n_verified, float* d_F, unsigned char* d_mask, int* d_n_inliers, void* stream);

/* ------------------------------------------------------------------ tiled image sets
 * Device counterparts of ExtractorBase._extract_by_tile (extractors/extractor_base.py:279-390) and MatcherBase._match_by_tile
 * (matchers/matcher_base.py:362-485).  Every entry is asynchronous on `stream` and never synchronises (once its context scratch has
 * grown to the call's size), is bitwise reproducible and independent of how images or pairs are batched, and returns DIMB_ERR_ARG
 * before any CUDA call for a NULL pointer or an out-of-range size.
 * Profile groups: tile.cut, tile.merge, tile.views, tile.match_merge.
 *
 * Tile geometry (utils/tiling.py Tiler.compute_tiles_by_size): tile_h x tile_w windows stepped by (tile - overlap), on the image
 * zero-padded by kornia's compute_padding called WITHOUT the stride (quirk A.7: the padding makes (size - tile) % tile == 0, the
 * odd pixel at the bottom / right; with an overlap the last `overlap` padded pixels are never covered).  Tiles are numbered
 * row-major; tile t = row * n_cols + col has its origin at (x, y) = (-pad_left + col * stride_w, -pad_top + row * stride_h) in the
 * un-padded image.  At most 2048 tiles (tile_idx is stored as float16).
 * Host only (no CUDA call): out[6] = {n_rows, n_cols, pad_top, pad_left, stride_h, stride_w}. */
int dimb_tile_grid(int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w, int* out);
/* d_images: B float32 images [B][H][W][channels], channels 1 (gray) or 3 (RGB).  d_tiles: [B * T][tile_h][tile_w][channels], the
 * T tiles of image 0 first; pixels in the padding are 0.  B * T <= 65535. */
int dimb_tile_cut_dev(dimb_ctx* ctx, const float* d_images, int B, int height, int width, int channels, int tile_h, int tile_w, int overlap_h,
                      int overlap_w, float* d_tiles, void* stream);
/* Tile-feature merge of B images into the store slots slots[b] (host array).  Input: the float32 extractor outputs of the T tiles
 * of every image in the layouts of dimb_sp_extract_dev / dimb_aliked_extract_dev with capacity K per tile: d_kpts [B*T][K][2],
 * d_scores [B*T][K], d_desc [B*T][D][K], d_counts [B*T] (device; rows = min(count, K)).  Per tile t in order: keypoints shifted by
 * the tile origin (float32 add), kept iff 2 <= x < W - 2 and 2 <= y < H - 2, concatenated; then np.unique(kpts, axis=0,
 * return_index=True): sorted by (x, y), the first of exact duplicates in concatenation order kept.  Descriptors, scores and
 * tile_idx = t follow; the slot gets the float16 cast of dimb_fstore_put_dev and the header n = merged count, [H, W] of the full
 * image.  DIMB_ERR_CAPACITY when the store's capacity is below T * K. */
int dimb_tile_merge_dev(dimb_fstore* fs, int B, const int* slots, int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w,
                        const float* d_kpts, const float* d_scores, const float* d_desc, const int* d_counts, int K, void* stream);
/* Tile views (matcher_base.py:1380-1391 get_features_by_tile) of B merged slots src_slots[b]: view slot dst_slots[b] + t of `dst`
 * receives the merged rows with tile_idx == t in merged order, and row dst_slot of d_map ([dst n_slots][dst cap] int32) maps each view
 * row to its merged row.  The view header carries the FULL image's [H, W] (quirk A.3), so dimb_fstore_feats_dev /
 * dimb_fstore_sg_feats_dev of a view slot feed dimb_lg_match_dev / dimb_sg_match_dev unchanged.  A tile left without rows gives
 * n = 0.  Views hold at most dst's capacity rows (a tile never contributes more than the extractor's K).  Both stores share the
 * context and the descriptor size; B * n_tiles <= 65535. */
int dimb_tile_views_dev(dimb_fstore* src, int B, const int* src_slots, int n_tiles, dimb_fstore* dst, const int* dst_slots, int* d_map,
                        void* stream);
/* Tile-pair match merge of Q image pairs.  Host CSR: image pair q owns the tile pairs p in [pair_offsets[q], pair_offsets[q+1]);
 * tile pair p matched view rows view0[p] (side 0) and view1[p] (side 1) of d_maps (rows of map_ld ints, as dimb_tile_views_dev writes
 * them).  d_matches [P][cap][2] int64 + d_n_matches [P] in the layout of dimb_lg_match_dev / dimb_sg_match_dev (rows = min(n, cap)).
 * Per image pair: both columns remapped to merged rows, concatenated, np.unique(axis=0) (sorted by (idx0, idx1), duplicates
 * dropped).  Out (device): d_out [Q][cap2][2] int64 and d_n_out [Q], the full count also when it exceeds cap2 (only the first cap2
 * rows are written).  An image pair without tile pairs gets 0. */
int dimb_tile_match_merge_dev(dimb_ctx* ctx, int Q, const int* pair_offsets, const int* view0, const int* view1, const int* d_maps, int map_ld,
                              const int64_t* d_matches, const int* d_n_matches, int cap, int64_t* d_out, int* d_n_out, int cap2, void* stream);

/* Tile preselection (matcher_base.py:1055-1148): the low-resolution SuperPoint + LightGlue pass that picks the tile pairs worth
 * matching.  Same conventions as the entries above; profile groups tile.resize, tile.extent, tile.preselect.
 *
 * cv2.resize(img, (W2, H2), interpolation=INTER_AREA) for downscaling, OpenCV's resizeArea_ / computeResizeAreaTab: per axis
 * scale = 1 / (dsize / ssize) in double; destination index d covers [d * scale, d * scale + scale) with a leading partial weight, full
 * weights 1 / cellWidth and a trailing partial weight, all computed in double and stored as float.  Host only (no CUDA call): the
 * table of one axis, entries in OpenCV's order, d_idx / s_idx / alpha of at most cap entries; *n = the entry count (<= 2 * ssize).
 * DIMB_ERR_CAPACITY (n filled) when cap is too small; DIMB_ERR_ARG unless 1 <= dsize <= ssize. */
int dimb_resize_area_tab(int ssize, int dsize, int* d_idx, int* s_idx, float* alpha, int cap, int* n);
/* B float32 gray images d_src [B][H][W] -> d_dst [B][H2][W2], bitwise the value cv2.resize(INTER_AREA) gives: per output pixel,
 * over the contributing source rows in table order, buf = sum of S[sx] * alpha in x-table order from 0, then sum = beta * buf for
 * the first row and sum += beta * buf for the others, every product and sum rounded separately (no FMA).  H2 == H and W2 == W is a
 * copy.  When both factors H / H2 and W / W2 are integers (within DBL_EPSILON, OpenCV's is_area_fast) OpenCV sums the
 * sy x sx block row-major, four pixels at a time (sum += ((a + b) + c) + d), and scales by float(1 / area); that order is used too.
 * The 2 x 2 block also has OpenCV's vector loop, ((a + b) + (c + d)) * 0.25f, over the first floor(W2 / 4) * 4 columns of each row,
 * with the scalar order for the rest: parity is with OpenCV's 128-bit baseline SIMD width (4 float lanes).  Upscaling (OpenCV
 * switches to a bilinear variant there) is refused: DIMB_ERR_ARG for H2 > H or W2 > W.  B, H2 <= 65535. */
int dimb_resize_area_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                         void* stream);
/* INTER_AREA when an axis is enlarged (pairs_generator.py's read_lowres enlarges small photos to resize_max): OpenCV then runs
 * cv::resize's area_mode, a bilinear emulation on BOTH axes, as soon as one factor dsize / ssize exceeds 1.  Host only (no CUDA
 * call): the coefficients of one axis for any 1 <= ssize, dsize, per destination index d (OpenCV's coefficient loop in double with
 * inv = dsize / ssize, scale = 1 / inv): sx = floor(d * scale), fx = float((d + 1) - (sx + 1) * inv), fx = fx <= 0 ? 0 : fx - floor(fx);
 * where sx + 1 >= ssize the first such d is *xmax (dsize if none), and for sx >= ssize - 1, sx = ssize - 1 and fx = 0.
 * Out: s_idx [dsize], alpha [dsize][2] = {1 - fx, fx}.  DIMB_ERR_ARG for a size below 1 or a NULL pointer. */
int dimb_resize_area_linear_tab(int ssize, int dsize, int* s_idx, float* alpha, int* xmax);
/* B float32 gray images d_src [B][H][W] -> d_dst [B][H2][W2], bitwise cv2.resize(INTER_AREA) when H2 > H or W2 > W (resizeGeneric_
 * with HResizeLinear / VResizeLinear in float over the tables above): each of the source rows sy and min(sy + 1, H - 1) is resampled
 * as S[sx] * a0 + S[sx + 1] * a1 (S[sx] alone for columns from xmax on), then out = row0 * b0 + row1 * b1, the weights unchanged when
 * the second row is clamped; every product and sum rounded separately (no FMA).  DIMB_ERR_ARG when no axis is enlarged (use
 * dimb_resize_area_dev), otherwise the argument limits of dimb_resize_area_dev; profile group tile.resize.  CUDA cores. */
int dimb_resize_area_linear_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                                void* stream);
/* The low-resolution gray image of an RGB image in one pass (the low-resolution passes of ALIKED sets): B float32 RGB images
 * d_src [B][H][W][3] -> gray d_dst [B][H2][W2], bitwise cv2.resize(gray_from_rgb(img), (W2, H2), interpolation=INTER_AREA) for any
 * size relation.  The gray rule (pairs_generator.gray_from_rgb) is applied to every source pixel as it is read, so no full-size gray
 * image is staged: each channel rounded half to even and clamped to 0..255, then (9798 R + 19235 G + 3735 B + 2^14) >> 15, the
 * RGB2GRAY of cv::cvtColor on uint8 (R first: not the BGR2GRAY order of the SuperPoint input).  The resize is then that of
 * dimb_resize_area_dev (integer factors, 1 x 1 for H2 == H and W2 == W, or the area tables) or, when H2 > H or W2 > W, that of
 * dimb_resize_area_linear_dev, with the same arithmetic.  DIMB_ERR_ARG (before any CUDA call) for B outside [1, 65535], H or W
 * outside [1, 2^20], H2 outside [1, 65535], W2 outside [1, 2^20] or a NULL pointer; profile group tile.resize; asynchronous on
 * `stream`.  CUDA cores. */
int dimb_resize_area_rgb_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, float* d_dst, int height2, int width2,
                             void* stream);
/* Extraction quality (ExtractorBase._resize_image / _resize_features, extractor_base.py:205,224): the reference resizes every image
 * by its `quality` before extracting and scales the keypoints back to the original image.  level: -1 = one cv2.pyrUp ("highest"),
 * 0 = none ("high"), 1..3 = that many cv2.pyrDown ("medium", "low", "lowest").  Host only (no CUDA call): the size after `level`
 * steps, pyrDown giving ((H + 1) / 2, (W + 1) / 2) and pyrUp (2H, 2W).  DIMB_ERR_ARG for a level outside [-1, 3], a size outside
 * [1, 2^20] or a NULL pointer. */
int dimb_pyr_size(int height, int width, int level, int* height2, int* width2);
/* B float32 images d_src [B][H][W][channels] (channels 1 gray or 3 interleaved RGB) -> d_dst [B][H2][W2][channels] (dimb_pyr_size),
 * bitwise cv2.pyrDown applied `level` times or cv2.pyrUp once (BORDER_DEFAULT = reflect-101), level 0 a copy.  pyrDown: horizontal
 * 1 4 6 4 1 sums per source row, then the vertical sum over rows 2y - 2 .. 2y + 2 and * (1 / 256); pyrUp: 1 6 1 / 4 4 sums on the
 * doubled grid and * (1 / 64); the order of every sum is OpenCV's, including the columns its 4-lane baseline SIMD loops cover, and
 * every product and sum is rounded on its own (no FMA).  The intermediates of a chain live in the context's grow-only scratch, so
 * the caller allocates only d_dst (which must not overlap d_src).  DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, B
 * outside [1, 65535], other channel counts, a bad size or level, or more than 65535 output rows in one step.  Profile group tile.pyr.
 * CUDA cores. */
int dimb_pyr_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, int channels, int level, float* d_dst, void* stream);
/* _resize_features on B store slots slots[b] (host array) filled from features of the resized image (dimb_fstore_put_dev, or
 * dimb_tile_merge_dev on the resized grid): their float16 keypoints are multiplied by 2^level and the header's [H, W] becomes the
 * original height x width (float16-rounded as dimb_fstore_put_dev stores it).  Scaling by a power of two commutes with rounding to
 * float16 while the values stay normal (>= 2^-14), so this equals the reference's float32 scale followed by the h5 cast.  Empty slots
 * are left alone.  DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, B outside [1, 65535], a slot out of range, a level outside
 * [-1, 3] or a size below 1.  Asynchronous on `stream`; profile group tile.pyr. */
int dimb_fstore_rescale_dev(dimb_fstore* fs, int B, const int* slots, int level, int height, int width, void* stream);
/* upright (image_matching.py:496): cv2.rotate of B float32 images d_src [B][H][W][channels] (channels 1 gray or 3 interleaved RGB) by
 * rotations[b] (host array, each 0, 90 = ROTATE_90_CLOCKWISE, 180 = ROTATE_180 or 270 = ROTATE_90_COUNTERCLOCKWISE; mixed values in
 * one call) into d_dst, image b starting at element b * H * W * channels and being [H][W][channels] (0, 180) or [W][H][channels]
 * (90, 270).  A permutation, so bitwise cv2.rotate.  One host->device copy of the codes (context scratch) and one launch; d_dst must
 * not overlap d_src.  DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, B outside [1, 65535], other channel counts, a size
 * outside [1, 2^20] or another rotation value.  Asynchronous on `stream`; profile group tile.rot.  CUDA cores, memory-bound
 * (2 * B * H * W * channels * 4 bytes). */
int dimb_rot90_dev(dimb_ctx* ctx, const float* d_src, int B, int height, int width, int channels, const int* rotations, float* d_dst,
                   void* stream);
/* upright (image_matching.py:703): the keypoints of B store slots slots[b] (host arrays throughout), extracted from their image turned
 * by rotations[b] with cv2.rotate, back on pixel indices of the original heights[b] x widths[b] image: in float32, (x', y') ->
 * 90: (y', H - 1 - x'), 180: (W - 1 - x', H - 1 - y'), 270: (W - 1 - y', x'), 0: unchanged, then rounded to float16; the header's [H, W]
 * becomes the original size (float16-rounded as dimb_fstore_put_dev stores it).  Scores, descriptors and tile_idx are untouched, and
 * empty slots are left alone.  DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, B outside [1, 65535], a slot out of range,
 * another rotation value or a size below 1.  Asynchronous on `stream`; profile group tile.rot. */
int dimb_fstore_unrotate_dev(dimb_fstore* fs, int B, const int* slots, const int* rotations, const int* heights, const int* widths,
                             void* stream);
/* normalize_keypoints' own-extent size for LightGlue without image_size (lightglue.py:26-27): per image b, over its
 * min(d_counts[b], kpt_ld) keypoints of d_kpts [B][kpt_ld][2] float32, d_size_out[b] = {(1 + max x) - min x, (1 + max y) - min y}
 * in float32, as dimb_lg_match computes it on the host; {1, 1} for an image without keypoints.  Feed it to dimb_lg_match_dev
 * through dimb_feats_dev.size_f32_dev. */
int dimb_kpts_extent_dev(dimb_ctx* ctx, int B, const float* d_kpts, int kpt_ld, const int* d_counts, float* d_size_out, void* stream);
/* The box-count loop of tile_selection's PRESELECTION for Q image pairs, each side on its own tile grid.  Pair q: the low-resolution
 * match table d_matches[q] ([Q][cap][2] int64, rows = min(d_n_matches[q], cap), as dimb_lg_match_dev writes it) indexes the keypoints
 * of f0[q] / f1[q] (host arrays of Q; keypoints, f16 and round_fp16 are read).  sizes: host [Q][4] int {H0, W0, H1, W1}, the
 * full-resolution sizes of both images, each tiled as dimb_tile_grid with the shared tile and overlap (T0[q] and T1[q] tiles);
 * scales: host [Q][2] double {scale0, scale1}, cast to float32.  Each matched keypoint maps back to full resolution as
 * kpt / float(scale) (float32 division) and counts for tile pair (t0, t1) iff it lies strictly inside both boxes:
 * ox < x < ox + tile_w and oy < y < oy + tile_h.  Out (device), pair q's block starting at element sum_{p<q} T0[p] * T1[p]:
 * d_counts int32, the count of tile pair (t0, t1) at t0 * T1[q] + t1 (row-major), and d_flags uint8 in the same layout,
 * count > min_matches_per_tile.  Integer counts: exact in any order.  DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, Q outside
 * [1, 65535], cap < 1, a bad size or grid on either side, scales that are not finite and positive, or min_matches_per_tile < 0. */
int dimb_tile_preselect_pairs_dev(dimb_ctx* ctx, int Q, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                                  const int* d_n_matches, int cap, const int* sizes, int tile_h, int tile_w, int overlap_h, int overlap_w,
                                  const double* scales, int min_matches_per_tile, int* d_counts, unsigned char* d_flags, void* stream);
/* dimb_tile_preselect_pairs_dev for Q pairs of equally sized images (height x width) and one pair of scales: d_counts / d_flags
 * [Q][T*T], the count of tile pair (t0, t1) at t0 * T + t1. */
int dimb_tile_preselect_dev(dimb_ctx* ctx, int Q, const dimb_feats_dev* f0, const dimb_feats_dev* f1, const int64_t* d_matches,
                            const int* d_n_matches, int cap, int height, int width, int tile_h, int tile_w, int overlap_h, int overlap_w,
                            double scale0, double scale1, int min_matches_per_tile, int* d_counts, unsigned char* d_flags, void* stream);

/* ------------------------------------------------------------------ fused per-pair path
 * SuperPoint on both images of every pair followed by LightGlue, features kept in HBM in between (the
 * reference's features.h5 round trip, ImageMatcher.extract_features -> match_pairs, image_matching.py:413-494,
 * is reduced to its value-level effect: fp16 rounding of keypoints and descriptors). */
typedef struct dimb_pipe dimb_pipe;
int dimb_pipe_create(dimb_sp* sp, dimb_lg* lg, int max_pairs, int H, int W, int cap, dimb_pipe** out);
void dimb_pipe_destroy(dimb_pipe* pipe);
/* images: HOST float32 [2P][H][W] gray 0..255, pair p = images 2p and 2p+1.  Outputs (HOST): matches [P][cap][2]
 * int64, mscores [P][cap], n_matches [P], stop_layer [P], n_kpts [2P], kpts [2P][cap][2] (may be NULL). */
int dimb_pipe_match_image_pairs(dimb_pipe* pipe, const float* images, int P, int64_t* matches, float* mscores,
                                int* n_matches, int* stop_layer, int* n_kpts, float* kpts);
/* Same with 8-bit gray images (the reference casts them with astype(float32), extractor_base.py:201-202): a quarter of
 * the host->device traffic, exact conversion on device. */
int dimb_pipe_match_image_pairs_u8(dimb_pipe* pipe, const uint8_t* images, int P, int64_t* matches, float* mscores,
                                   int* n_matches, int* stop_layer, int* n_kpts, float* kpts);
/* Same with the images already in device memory, asynchronous on `stream`; results stay in device buffers owned
 * by the pipe, exposed by dimb_pipe_outputs_dev (layouts as above). */
int dimb_pipe_match_image_pairs_dev(dimb_pipe* pipe, const float* d_images, int P, void* stream);
int dimb_pipe_outputs_dev(dimb_pipe* pipe, int64_t** d_matches, float** d_mscores, int** d_n_matches, int** d_stop,
                          int** d_nkpts, float** d_kpts);
/* Device buffers holding the SuperPoint features of the last call: kpts [2P][cap][2], scores [2P][cap], desc [2P][256][cap]
 * ((D,N) rows of pitch cap), counts [2P] - the arrays ExtractorBase.extract would hand to save_features_h5
 * (extractor_base.py:223-229) before the float16 cast. */
int dimb_pipe_features_dev(dimb_pipe* pipe, float** d_kpts, float** d_scores, float** d_desc, int** d_counts);
dimb_ctx* dimb_sp_ctx(dimb_sp* sp);

/* ---------------------------------------------------------------------------------------------------------
 * ALIKED extraction.  Replaces AlikedExtractor._extract (reference src/deep_image_matching/extractors/aliked.py:45-64)
 * and the model it drives (thirdparty/LightGlue/lightglue/aliked.py:560-693: encoder with deformable blocks :367-449,
 * DKD detector :92-244, SDDH descriptor head :452-558).  Supported: aliked-n16 / aliked-n16rot (dim 128, K 3, M 16), and
 * the three detection modes of DKD (top_k = -1 if detection_threshold > 0 else max_num_keypoints):
 *   threshold mode  detection_threshold > 0: NMS pixels above it (above mean(score_map) if none is), the n_limit best of them;
 *   top-k mode      detection_threshold <= 0 < max_num_keypoints: exactly max_num_keypoints keypoints, the largest of the
 *                   border-zeroed NMS map, score-descending (torch.topk).  Fewer nonzero NMS pixels than that: the rest are the
 *                   first zero pixels in row-major order.  max_num_keypoints > H * W is refused (DIMB_ERR_ARG);
 *   mean mode       detection_threshold <= 0 and max_num_keypoints <= 0: NMS pixels above mean(score_map), the 20000 best.
 * Kept keypoints are row-major when no cut fires, else score-descending (ties: smaller pixel index first).
 *
 * weights: fp32 blob, the model's state_dict tensors in state_dict order without num_batches_tracked
 * (block1.conv1.weight ... desc_head.sf_conv.weight; 678316 floats).
 * Reproduced quirk: `scores` are the DKD score *dispersities* (aliked.py:682 swaps the names; SURVEY A.5). */
typedef struct dimb_aliked dimb_aliked;
typedef struct dimb_aliked_conf {
  int max_num_keypoints;      /* threshold / mean mode: n_limit, <= 0 -> 20000 (aliked.py:585); top-k mode: K.  Any value */
  float detection_threshold;  /* 0.2; <= 0: top-k or mean mode */
  int nms_radius;             /* 2 */
  int max_height, max_width;  /* workspace size */
} dimb_aliked_conf;
int dimb_aliked_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_aliked_conf* conf, dimb_aliked** out);
void dimb_aliked_destroy(dimb_aliked* al);
/* image: host fp32 (H,W,channels) 0..255, channels 3 (RGB, ExtractorBase with grayscale=False) or 1 (replicated).
 * Out (host): kpts [cap][2] sub-pixel (x,y); scores [cap]; desc [128][cap] ((D,N) FeaturesDict layout, ld = cap); count. */
int dimb_aliked_extract(dimb_aliked* al, const float* image, int H, int W, int channels, float* kpts, float* scores, float* desc,
                        int* count, int cap);
/* Device-pointer variant (same layouts, all pointers in device memory, count [1]); no host synchronisation - the caller
 * checks count <= cap.  Feeds dimb_lg_match_dev (desc_layout 0, desc_ld = cap) without leaving HBM. */
int dimb_aliked_extract_dev(dimb_aliked* al, const float* d_image, int H, int W, int channels, float* d_kpts, float* d_scores,
                            float* d_desc, int* d_count, int cap, void* stream);
/* debug taps of the last call: 0 = score map [H][W], 1 = L2-normalised feature map [128][H][W] */
int dimb_aliked_debug_read(dimb_aliked* al, int which, float* out, size_t n_floats);

/* ---------------------------------------------------------------------------------------------------------
 * SuperGlue matching.  Replaces SuperGlueMatcher._match_pairs (reference src/deep_image_matching/matchers/superglue.py:75-106,
 * adapter features_2_sg :8-41) and the model it drives (thirdparty/SuperGluePretrainedNetwork/models/superglue.py:51-305).
 * descriptor_dim 256, 4 heads, keypoint encoder [32,64,128,256].  The GNN and the score matrix run on the wgmma kernels shared with
 * LightGlue; the keypoint encoder, Sinkhorn and the mutual-max filter are batched CUDA-core kernels (csrc/superglue.cu).
 *
 * weights: fp32 blob in THIS order (names of the reference state_dict; BatchNorm = weight, bias, running_mean, running_var):
 *   kenc.encoder.{0,3,6,9}.{weight,bias} each followed by its BatchNorm kenc.encoder.{1,4,7,10}; kenc.encoder.12.{weight,bias};
 *   for i in layers: gnn.layers.i.attn.merge.{weight,bias}, attn.proj.{0,1,2}.{weight,bias}, mlp.0.{weight,bias}, mlp.1 (BatchNorm),
 *                    mlp.3.{weight,bias};
 *   final_proj.{weight,bias}; bin_score. */
typedef struct dimb_sg dimb_sg;
typedef struct {
  int n_layers;                   /* 18 */
  unsigned long long cross_mask;  /* bit i set: GNN layer i is a cross layer (["self","cross"] * 9 -> 0x2AAAA) */
  int sinkhorn_iterations;        /* 100 (superglue.py:218; the plugin's own 20 never reaches the model, see matchers/superglue.py) */
  float match_threshold;          /* 0.2 */
  int max_kpts;                   /* workspace sizing */
  int max_pairs;                  /* workspace sizing: pairs per dimb_sg_match_dev call (0 = 1) */
} dimb_sg_conf;
typedef struct {
  const float* keypoints;   /* (n,2) x,y */
  const float* descriptors; /* (256,n) rows of pitch desc_ld (0 = n): the FeaturesDict layout */
  const float* scores;      /* (n,) */
  int n, desc_ld;
  int height, width;        /* image_size = [H,W] */
} dimb_sg_feats;
size_t dimb_sg_weight_count(int n_layers);
int dimb_sg_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_sg_conf* conf, dimb_sg** out);
void dimb_sg_destroy(dimb_sg* sg);
/* One pair.  Out (host): matches [cap][2] int64 ascending in column 0, mscores [cap] (matching_scores0 of the matched rows). */
int dimb_sg_match(dimb_sg* sg, const dimb_sg_feats* f0, const dimb_sg_feats* f1, int64_t* matches, float* mscores, int* n_matches,
                  int cap);
/* Device counterpart of dimb_sg_feats: SuperGlue needs the scores, which dimb_feats_dev does not carry. */
typedef struct {
  const void* keypoints;    /* device (n_cap,2) x,y */
  const void* descriptors;  /* device (256,n) rows of pitch desc_ld (0 = n_cap): the FeaturesDict / store layout */
  const void* scores;       /* device (n_cap,); required (features_2_sg needs scores) */
  const int* n;             /* device scalar, <= n_cap */
  int n_cap, desc_ld;
  int f16;                  /* 1: the three arrays are float16 (feature-store blocks) */
  int round_fp16;           /* 1: round float32 inputs to fp16 first (the features.h5 round trip) */
  int height, width;        /* image_size [H,W] */
  const int* size_dev;      /* non-NULL: device int[2] [H,W], overrides height / width */
} dimb_sg_feats_dev;
/* P <= max_pairs pairs on device pointers, asynchronous on `stream` (never synchronises).  Outputs as dimb_lg_match_dev:
 * d_matches [P][cap][2] int64 ascending in column 0, d_mscores [P][cap], d_n_matches [P] (the full count, also when it exceeds
 * cap; only the first cap rows are written). */
int dimb_sg_match_dev(dimb_sg* sg, int P, const dimb_sg_feats_dev* f0, const dimb_sg_feats_dev* f1, int64_t* d_matches, float* d_mscores,
                      int* d_n_matches, int cap, void* stream);
/* The slot as SuperGlue device input: f16 = 1, scores from the slot's score block, size_dev = the slot header's [H,W]. */
int dimb_fstore_sg_feats_dev(dimb_fstore* fs, int slot, dimb_sg_feats_dev* out);

/* ---------------------------------------------------------------------------------------------------------
 * SIFT extraction.  Replaces SIFTExtractor._extract (reference extractors/sift.py): cv2.SIFT_create(nfeatures, nOctaveLayers,
 * contrastThreshold, edgeThreshold, sigma).detectAndCompute(gray_uint8, None) of OpenCV 4.x with enable_precise_upscale = false
 * (csrc/sift.cu lists the stages).  Results are deterministic: an image gives bitwise the same output on every run and at every
 * position of a batch.  Output order: removeDuplicatedSorted's (x asc, y asc, size desc, angle asc, response desc, octave desc),
 * which is cv2's own order unless retainBest cuts; when it cuts, cv2's order is an artefact of std::nth_element and this order
 * replaces it.  retainBest keeps every keypoint whose response equals the n_features-th largest, so a count may exceed n_features.
 * Memory: sized at create time for max_batch images of max_height x max_width, about 0.8 GB of float32 pyramid and 0.23 GB of
 * refined-extremum and keypoint buffers per 2048 x 1536 image at 3 layers.  Profile groups sift.pyr, sift.extrema, sift.ori, sift.select,
 * sift.desc. */
typedef struct dimb_sift dimb_sift;
typedef struct {
  int n_features;             /* retainBest(n_features); 0 keeps every keypoint */
  int n_octave_layers;        /* 3 */
  double contrast_threshold;  /* 0.04 in OpenCV, 0.0004 in the sift+kornia_matcher pipeline */
  double edge_threshold;      /* 10 */
  double sigma;               /* 1.6 */
  int max_batch;              /* workspace sizing: images per call (max_batch * n_octave_layers <= 65535) */
  int max_height, max_width;  /* workspace sizing, at most 16384 */
} dimb_sift_conf;
/* DIMB_ERR_ARG, before any CUDA call, for a NULL pointer or a value outside the ranges above. */
int dimb_sift_create(dimb_ctx* ctx, const dimb_sift_conf* conf, dimb_sift** out);
void dimb_sift_destroy(dimb_sift* sift);
/* One host image, uint8 [H][W].  Out (host): kpts [cap][2] (x, y), desc [128][cap] (integral 0..255 values as float; (D,N) rows of
 * pitch cap), frames [cap][3] (size, angle, response) and octave [cap] (cv2's packed KeyPoint.octave), both optional (NULL), count.
 * DIMB_ERR_CAPACITY (count filled) when the image has more than cap keypoints, or (count -1) more extrema than the candidate
 * buffers hold. */
int dimb_sift_extract(dimb_sift* sift, const uint8_t* image, int H, int W, float* kpts, float* desc, float* frames, int* octave,
                      int* count, int cap);
/* B device float32 images [B][H][W]; each pixel is first converted as convertTo(CV_8U) does (round half to even, saturate to 0..255),
 * so integral 0..255 images are taken exactly.  Outputs (device) in the layouts of dimb_sp_extract_dev: d_kpts [B][cap][2],
 * d_desc [B][128][cap], d_counts [B]; d_frames [B][cap][3] and d_octave [B][cap] may be NULL.  d_counts holds the true count (-1 when
 * the candidate buffers overflowed); only the first cap rows are written and the caller checks the count.  Asynchronous on `stream`.
 * DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, cap < 1, B outside [1, max_batch] or a size above the workspace. */
int dimb_sift_extract_dev(dimb_sift* sift, const float* d_images, int B, int H, int W, float* d_kpts, float* d_desc, float* d_frames,
                          int* d_octave, int* d_counts, int cap, void* stream);
/* Debug taps of the last call, image `image`: which 0 = Gaussian level, level = octave * (n_octave_layers + 3) + i; which 1 = DoG
 * level, level = octave * (n_octave_layers + 2) + i.  Octave 0 is OpenCV's octave -1 (2H x 2W), each later octave halves (floor) both
 * sides; out holds exactly that octave's h * w floats (0..255 scale). */
int dimb_sift_debug_read(dimb_sift* sift, int which, int image, int level, float* out, size_t n_floats);

/* ------------------------------------------------------------------------------------------------------------------------------
 * ORB extraction.  Replaces the host cv2.ORB of the reference's ORB extractor (extractors/orb.py): cv2.ORB_create(nfeatures,
 * scaleFactor, nlevels, edgeThreshold, firstLevel, WTA_K, scoreType, patchSize, fastThreshold).detect(gray_uint8) followed by
 * .compute of OpenCV 4.x, for firstLevel 0, WTA_K 2 and patchSize 31 (cv2's defaults; other values need the random pattern or
 * upscaled levels and are refused).  csrc/orb.cu lists the stages.  Pyramid, FAST, Harris and the descriptor tests follow cv2
 * bit for bit, the blur in the fused multiply-add order of OpenCV's vector build (its SSE2 baseline rounds a few float ties the
 * other way); results are deterministic, alone or at any position of a batch.  Output order: level ascending, then y, then x on
 * the level (cv2's order within a level is an artefact of std::nth_element).  retainBest keeps every keypoint tied with the
 * boundary response, so a count may exceed nfeatures.  Memory: sized at create time for max_batch images of max_height x
 * max_width, about 3.3 bytes of levels and 7 bytes of candidate lists per input pixel at scaleFactor 1.2.  Profile groups orb.pyr,
 * orb.fast, orb.select, orb.desc. */
typedef struct dimb_orb dimb_orb;
enum { DIMB_ORB_HARRIS_SCORE = 0, DIMB_ORB_FAST_SCORE = 1 };
typedef struct {
  int n_features;             /* nfeatures, split over the levels as ORB does; 500 in OpenCV */
  double scale_factor;        /* scaleFactor, rounded to float as cv2.ORB_create takes it; 1 < scale_factor <= 16; 1.2 */
  int nlevels;                /* 1 .. 32; 8 */
  int edge_threshold;         /* 0 .. 4096; 31 */
  int first_level;            /* 0 only */
  int wta_k;                  /* 2 only */
  int score_type;             /* DIMB_ORB_HARRIS_SCORE or DIMB_ORB_FAST_SCORE */
  int patch_size;             /* 31 only */
  int fast_threshold;         /* clamped to 0 .. 255 as FAST does; 20 */
  int max_batch;              /* workspace sizing: images per call, at most 65535 */
  int max_height, max_width;  /* workspace sizing, at most 16384 */
} dimb_orb_conf;
/* DIMB_ERR_ARG, before any CUDA call, for a NULL pointer or a value outside the ranges above. */
int dimb_orb_create(dimb_ctx* ctx, const dimb_orb_conf* conf, dimb_orb** out);
void dimb_orb_destroy(dimb_orb* orb);
/* One host image, uint8 [H][W].  Out (host): kpts [cap][2] (x, y at level 0), desc [32][cap] (descriptor bytes 0..255 as float;
 * (D,N) rows of pitch cap), frames [cap][3] (size, angle, response) and octave [cap] (the level), both optional (NULL), count.
 * DIMB_ERR_CAPACITY (count filled) when the image has more than cap keypoints.  DIMB_ERR_ARG for an image larger than the
 * workspace or so small that a level would be empty. */
int dimb_orb_extract(dimb_orb* orb, const uint8_t* image, int H, int W, float* kpts, float* desc, float* frames, int* octave, int* count,
                     int cap);
/* B device float32 images [B][H][W], converted as convertTo(CV_8U) does (round half to even, saturate), in the layouts of
 * dimb_sift_extract_dev: d_kpts [B][cap][2], d_desc [B][32][cap], d_counts [B]; d_frames [B][cap][3] and d_octave [B][cap] may be
 * NULL.  d_counts holds the true count; only the first cap rows are written and the caller checks the count.  The candidate lists
 * are sized for the most corners non-maximum suppression can leave, so no image overflows them.  Asynchronous on `stream`.
 * DIMB_ERR_ARG, before any CUDA call, for a NULL pointer, cap < 1, B outside [1, max_batch] or a size above the workspace. */
int dimb_orb_extract_dev(dimb_orb* orb, const float* d_images, int B, int H, int W, float* d_kpts, float* d_desc, float* d_frames,
                         int* d_octave, int* d_counts, int cap, void* stream);
/* Debug taps of the last call, image `image`: which 0 = pyramid level `level`, which 1 = its 7 x 7 Gaussian blur (what the
 * descriptors read); out holds that level's h * w pixel values as float. */
int dimb_orb_debug_read(dimb_orb* orb, int which, int image, int level, float* out, size_t n_floats);

#ifdef __cplusplus
}
#endif
#endif /* DIMB200_H */
