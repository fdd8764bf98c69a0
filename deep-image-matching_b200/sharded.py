"""Multi-GPU driver of the hot path (SURVEY 8e): one process per GPU (torch.distributed; nccl on GPUs, gloo in the CPU tests).

Independent-pair workloads (bench.py default): pairs are dealt to ranks, no data-path collective, one gather of the match
tables to rank 0.  Image-set workloads (exhaustive / sequential pair lists over n images - ImageMatcher.extract_features +
match_pairs, image_matching.py:413-494, is the serial loop this replaces) run in two phases:
  1. image i is extracted on rank ``i % G`` into that rank's region of the device feature store (``shard_images``,
     ``store_slot``);
  2. ONE ``all_gather`` of the float16 feature blocks (NCCL over NVLink; ~1.07 MB per SuperPoint image) gives every rank all
     features (``all_gather_blocks``), then the pair list is dealt by longest-processing-time (``shard_pairs``) and each rank
     matches its pairs (LightGlue, SuperGlue or kornia's brute-force nearest neighbours) out of its own HBM; the variable-length
     match tables are gathered to rank 0 (``gather_match_tables``).
With ``verification`` the matcher's tables of each pair batch go straight into the device geometric verification (fundamental-matrix
RANSAC, ordered inlier compaction and the per-pair gate, one launch group per batch); raw tables, verified tables and F are gathered
to rank 0 (``gather_verified``), and ``export_verified_to_colmap`` writes the COLMAP database from the store and those results.
With ``tiling`` (the reference's tile_size / tile_overlap / tile_selection) high-resolution images are cut into tiles on the device,
the extractor runs over tiles and every image's tile features are merged into its slot (ExtractorBase._extract_by_tile); after the
exchange each rank splits the merged slots into per-tile views, matches the selected tile pairs out of the views and merges their
tables into one table per image pair (MatcherBase._match_by_tile).
With ``pair_generation`` ("matching_lowres") the pair list itself comes from the device: low-resolution SuperPoint in phase 1, the
exchange of those features, LightGlue over every brute-force pair dealt to the ranks, and an all_gather of the match counts that
leaves the same kept pairs on every rank (``lowres_pairs``, ``run_lowres``).
With ``quality`` other than "high" each image is resized on the device by cv2.pyrUp / cv2.pyrDown steps before extraction (plain or
tiled) and the stored keypoints are scaled back to the original image (ExtractorBase._resize_image / _resize_features).
Images of a set may differ in size (per-image ``height`` / ``width``): each rank runs its images in groups of one size, and every slot,
tile grid and low-resolution image keeps its own image's size."""
from __future__ import annotations

import numpy as np


def shard_pairs(n_pairs: int, world: int, rank: int, costs=None) -> list:
    """Indices of the pairs rank `rank` processes.  Round-robin by default (pairs_from_bruteforce order,
    pairs_generator.py:37-38); with per-pair costs (e.g. N0*N1) a longest-processing-time deal balances the
    early-exit variance.  Deterministic on every rank."""
    if costs is None:
        return list(range(rank, n_pairs, world))
    order = sorted(range(n_pairs), key=lambda i: (-float(costs[i]), i))
    load = [0.0] * world
    mine = []
    for i in order:
        r = min(range(world), key=lambda k: (load[k], k))
        load[r] += float(costs[i])
        if r == rank:
            mine.append(i)
    return sorted(mine)


def shard_images(n_images: int, world: int, rank: int) -> list:
    """Images rank `rank` extracts: i % world == rank (tiles of one image stay on one rank)."""
    return list(range(rank, n_images, world))


def images_per_rank(n_images: int, world: int) -> int:
    return (n_images + world - 1) // world


def store_slot(image: int, n_images: int, world: int) -> int:
    """Slot of image `image` in the device feature store: rank-major, so that each rank's extractions are one contiguous run of
    blocks and the exchange is a single all_gather of equal-sized regions."""
    return (image % world) * images_per_rank(n_images, world) + image // world


def all_gather_blocks(store_tensor, n_images: int, dist=None):
    """store_tensor: uint8 tensor viewing the whole store, shape (world * images_per_rank, slot_bytes); rank r has filled rows
    [r * ipr, (r + 1) * ipr).  After the call every rank holds every block.  Returns the bytes this rank received."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return 0
    world, rank = dist.get_world_size(), dist.get_rank()
    ipr = images_per_rank(n_images, world)
    assert store_tensor.shape[0] == world * ipr, (store_tensor.shape, world, ipr)
    mine = store_tensor[rank * ipr:(rank + 1) * ipr].clone()  # send buffer (the receive buffer is the store itself)
    dist.all_gather_into_tensor(store_tensor.view(-1), mine.view(-1))
    return (world - 1) * mine.numel()


def _gather_arrays(local_ids, arrays, n_pairs: int, width: int, dtype, dist, device, everywhere: bool = False):
    """Gather {pair id -> `dtype` array of `width` columns and any number of rows} from all ranks to rank 0: one all_gather of every
    rank's (pair count, most rows), one of the padded arrays, each row of the padded buffer being (pair id, rows, values...).
    Returns the list by pair id on rank 0, pairs nobody sent left None (None elsewhere, unless `everywhere`: then on every rank)."""
    import torch

    arrays = [np.asarray(a, dtype).reshape(-1, width) for a in arrays]
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        out = [None] * n_pairs
        for i, a in zip(local_ids, arrays):
            out[i] = a
        return out
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = device if device is not None else torch.device("cpu")
    cnt = torch.tensor([len(arrays), max([len(a) for a in arrays], default=0)], dtype=torch.int64, device=dev)
    cnts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(cnts, cnt)
    cnts = torch.stack(cnts).cpu().numpy()
    kmax, smax = cnts.max(axis=0)
    buf = np.zeros((max(kmax, 1), 2 + width * max(smax, 1)), dtype)
    for j, (i, a) in enumerate(zip(local_ids, arrays)):
        buf[j, :2] = i, len(a)
        buf[j, 2:2 + a.size] = a.ravel()
    buf = torch.as_tensor(buf, device=dev)
    bufs = [torch.zeros_like(buf) for _ in range(world)]
    dist.all_gather(bufs, buf)
    if rank != 0 and not everywhere:
        return None
    out = [None] * n_pairs
    for r in range(world):
        b = bufs[r].cpu().numpy()
        for j in range(cnts[r, 0]):
            i, s = int(b[j, 0]), int(b[j, 1])
            out[i] = b[j, 2:2 + width * s].reshape(-1, width).copy()
    return out


def gather_match_tables(local_ids, local_matches, n_pairs: int, dist=None, device=None):
    """Gather {pair id -> int64 (S,2)} from all ranks to rank 0 (counts all_gather + padded all_gather).
    Returns the full list on rank 0 (None elsewhere)."""
    return _gather_arrays(local_ids, local_matches, n_pairs, 2, np.int64, dist, device)


def gather_pair_counts(local_ids, local_counts, n_pairs: int, dist=None, device=None) -> list:
    """Gather {pair id -> int count} from all ranks to EVERY rank (the same all_gathers as ``gather_match_tables``).  Returns the
    list of n_pairs ints by pair id on every rank."""
    full = _gather_arrays(local_ids, [[int(c)] for c in local_counts], n_pairs, 1, np.int64, dist, device, everywhere=True)
    return [int(a[0, 0]) for a in full]


def upright_waves(pairs, n_images: int, count, dist=None, device=None):
    """The upright search over the ranks, wave by wave (``upright.upright_schedule``): each wave's decisions are dealt round-robin
    (``shard_pairs``), ``count(my decisions, rotations so far)`` gives the four counts (rotations 0, 90, 180, 270) of each of this rank's
    decisions in order, and one ``gather_pair_counts`` (four ids per decision) gives every rank the wave's counts and so its
    rotations.  Returns (rotations, {(target, reference): [c_0, c_90, c_180, c_270]}), the same on every rank."""
    from .upright import choose, upright_schedule
    world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    rotations, counts = [0] * n_images, {}
    for wave in upright_schedule(pairs, n_images):
        mine = shard_pairs(len(wave), world, rank)
        local = np.asarray(count([wave[q] for q in mine], list(rotations)), np.int64).reshape(-1)
        full = gather_pair_counts([4 * q + r for q in mine for r in range(4)], local, 4 * len(wave), dist if world > 1 else None, device)
        for q, (t, a) in enumerate(wave):
            counts[(t, a)] = full[4 * q:4 * q + 4]
            rotations[t] = choose(counts[(t, a)])
    return rotations, counts


def gather_verified(local_ids, local_results, n_pairs: int, dist=None, device=None):
    """Gather {pair id -> (raw (S,2), verified (V,2), F (3,3) float32 or None, n_inliers)} from all ranks to rank 0: the two int64
    tables, and F and the count as one fixed-width float64 row per pair (exact for float32 and int32).
    Returns the full list of 4-tuples on rank 0 (None elsewhere)."""
    raw = _gather_arrays(local_ids, [r[0] for r in local_results], n_pairs, 2, np.int64, dist, device)
    ver = _gather_arrays(local_ids, [r[1] for r in local_results], n_pairs, 2, np.int64, dist, device)
    rows = np.zeros((len(local_ids), 11), np.float64)  # has_F, n_inliers, F row-major
    for k, r in enumerate(local_results):
        rows[k, 1] = r[3]
        if r[2] is not None:
            rows[k, 0] = 1.0
            rows[k, 2:] = np.asarray(r[2], np.float32).ravel()
    full = _gather_arrays(local_ids, rows, n_pairs, 11, np.float64, dist, device)
    if full is None:
        return None
    out = [None] * n_pairs
    for i, row in enumerate(full):
        if row is not None:
            row = row[0]
            out[i] = (raw[i], ver[i], row[2:].astype(np.float32).reshape(3, 3) if row[0] else None, int(row[1]))
    return out


def export_verified_to_colmap(store, n_images: int, world: int, pairs, results, database_path, image_names=None, **kwargs) -> dict:
    """Write the COLMAP database of a verified image set through ``io_colmap.export_to_colmap`` (call on rank 0).

    store: the device feature store (``FeatureStoreDev``; features read with ``get`` from slot ``store_slot(i, n_images, world)``,
    in image order); pairs: [(i, j), ...]; results: per pair ``(raw, verified, F, n_inliers)`` as ``run_verified`` returns them.
    Raw tables go to ``matches``; non-empty verified tables go to ``two_view_geometries`` with their F; pairs the gate rejected
    (empty verified table) are left out of it.  Image i gets database id i + 1, and each pair is handed over oriented from the lower
    to the higher id (columns swapped and F transposed for a pair (i, j) with i > j), so the stored F satisfies x_high^T F x_low = 0.
    image_names: database names of the images (default ``image_{i}``); kwargs go to ``export_to_colmap``.  Returns {name: image_id}."""
    from .io_colmap import export_to_colmap

    names = list(image_names) if image_names is not None else [f"image_{i}" for i in range(n_images)]
    if len(names) != n_images or len(set(names)) != n_images:
        raise ValueError(f"image_names must hold {n_images} distinct names")
    features = {names[i]: store.get(store_slot(i, n_images, world)) for i in range(n_images)}
    raw_tables, verified, fundamental = {}, {}, {}
    for (i, j), (raw, ver, F, _) in zip(pairs, results):
        raw = np.asarray(raw, np.int64).reshape(-1, 2)
        ver = np.asarray(ver, np.int64).reshape(-1, 2)
        if i > j:  # orient low id -> high id: export_to_colmap would swap the columns but not transpose F
            i, j, raw, ver = j, i, raw[:, ::-1], ver[:, ::-1]
            F = None if F is None else np.asarray(F).T
        key = (names[i], names[j])
        raw_tables[key] = raw
        if len(ver):
            verified[key] = ver
            if F is not None:
                fundamental[key] = np.asarray(F, np.float64)
    return export_to_colmap(features, verified, database_path, raw_matches=raw_tables, fundamental=fundamental, **kwargs)


def verification_conf(verification) -> dict | None:
    """The ``verification`` argument of ImageSetMatcher with its defaults filled in (None stays None).  Defaults: method
    "pydegensac", threshold 1.0, max_iters 10000, seed 0 (those of geometric_verification), min_inliers_per_pair 15 and
    min_inlier_ratio_per_pair 0.2 (MatcherBase's general defaults), estimator "ransac8" and confidence 0.9999 (read by
    estimators "lo-ransac" and "degensac" only, as in geometric_verification)."""
    if verification is None:
        return None
    from ._native import gv_estimator
    from .geometric_verification import method_name
    conf = {"method": "pydegensac", "threshold": 1.0, "max_iters": 10000, "seed": 0, "min_inliers_per_pair": 15,
            "min_inlier_ratio_per_pair": 0.2, "confidence": 0.9999, "estimator": "ransac8"}
    unknown = set(verification) - set(conf)
    if unknown:
        raise ValueError(f"unknown verification option(s) {sorted(unknown)}; expected some of {sorted(conf)}")
    conf.update(verification)
    conf["method"] = method_name(conf["method"])
    if not float(conf["threshold"]) > 0 or int(conf["min_inliers_per_pair"]) < 0 or not 0 <= float(conf["min_inlier_ratio_per_pair"]) <= 1:
        raise ValueError("verification needs threshold > 0, min_inliers_per_pair >= 0 and 0 <= min_inlier_ratio_per_pair <= 1")
    if gv_estimator(conf["estimator"]) != 0 and not (0 < float(conf["confidence"]) < 1 and int(conf["max_iters"]) >= 1):
        raise ValueError(f"verification with estimator {conf['estimator']} needs 0 < confidence < 1 and max_iters >= 1")
    return conf


def kornia_conf(conf) -> dict:
    """The ``lg_conf`` of ImageSetMatcher(matcher="kornia_matcher"), validated: KorniaMatcher's keys ``match_mode`` (nn, mnn, snn or
    smnn; default smnn) and ``th`` (default 0.8).  A bad mode raises the plugin's NotImplementedError."""
    from ._native import NN_MODES
    out = {"match_mode": "smnn", "th": 0.8}
    unknown = set(conf or {}) - set(out)
    if unknown:
        raise ValueError(f"unknown kornia_matcher option(s) {sorted(unknown)}; expected some of {sorted(out)}")
    out.update(conf or {})
    if out["match_mode"] not in NN_MODES:
        raise NotImplementedError(f"{out['match_mode']} is not supported. Try one of {list(NN_MODES)}")
    out["th"] = float(out["th"])
    return out


SIFT_TIE_ROOM = 64  # store rows above n_features for the keypoints retainBest keeps at the boundary response


def sift_set_conf(sp_conf) -> dict:
    """SiftNet keyword arguments of a SIFT set's ``sp_conf``: the SIFTExtractor keys (n_features, nOctaveLayers, contrastThreshold,
    edgeThreshold, sigma; missing ones take SIFTExtractor's defaults), n_features >= 1.  Raises ValueError otherwise."""
    from .extractors.sift import SIFT_KEYS, SIFTExtractor, sift_conf
    unknown = set(sp_conf or {}) - set(SIFT_KEYS) - {"name"}
    if unknown:
        raise ValueError(f"unknown SIFT option(s) {sorted(unknown)}; expected some of {list(SIFT_KEYS)}")
    conf = {**{k: SIFTExtractor._default_conf[k] for k in SIFT_KEYS}, **{k: v for k, v in (sp_conf or {}).items() if k != "name"}}
    out = sift_conf(conf)
    if out["n_features"] < 1:
        raise ValueError(f"a SIFT image set needs n_features >= 1 (it sizes the feature store), got {out['n_features']}")
    return out


def orb_tie_room(n_features: int) -> int:
    """Store rows above n_features of an ORB set.  retainBest keeps every keypoint tied with the boundary response of each level;
    FAST scores are small integers, so with scoreType FAST_SCORE such ties can add a large share of n_features."""
    return max(64, n_features // 2)


def orb_set_conf(sp_conf) -> dict:
    """OrbNet keyword arguments of an ORB set's ``sp_conf``: the ORBExtractor keys (n_features, scaleFactor, nlevels, edgeThreshold,
    firstLevel, WTA_K, scoreType, patchSize, fastThreshold; missing ones take ORBExtractor's defaults), n_features >= 1 and the
    values ORBExtractor supports.  Raises ValueError otherwise."""
    from .extractors.orb import ORB_KEYS, ORBExtractor, orb_conf
    unknown = set(sp_conf or {}) - set(ORB_KEYS) - {"name"}
    if unknown:
        raise ValueError(f"unknown ORB option(s) {sorted(unknown)}; expected some of {list(ORB_KEYS)}")
    conf = {**{k: ORBExtractor._default_conf[k] for k in ORB_KEYS}, **{k: v for k, v in (sp_conf or {}).items() if k != "name"}}
    out = orb_conf(conf)
    if out["n_features"] < 1:
        raise ValueError(f"an ORB image set needs n_features >= 1 (it sizes the feature store), got {out['n_features']}")
    return out


def lighterglue_conf(conf) -> dict:
    """The ``lg_conf`` of ImageSetMatcher(matcher="lighterglue"), validated like ``kornia_conf``: only ``filter_threshold`` (default 0.1)
    of LighterGlueMatcher's configuration reaches the network (the plugin's ``min_conf``); the network itself is ``LIGHTERGLUE_CONF``
    (depth confidence -1, width confidence 0.95)."""
    out = {"filter_threshold": 0.1}
    unknown = set(conf or {}) - set(out)
    if unknown:
        raise ValueError(f"unknown lighterglue option(s) {sorted(unknown)}; expected some of {sorted(out)}")
    out.update(conf or {})
    out["filter_threshold"] = float(out["filter_threshold"])
    return out


def given_features_conf(sp_conf) -> tuple:
    """(K, D) of an ImageSetMatcher(extractor=None): ``sp_conf`` = {"max_keypoints": K, "descriptor_dim": D}, both ints >= 1."""
    unknown = set(sp_conf or {}) - {"max_keypoints", "descriptor_dim"}
    if unknown:
        raise ValueError(f"with extractor=None sp_conf holds max_keypoints and descriptor_dim only, got {sorted(unknown)}")
    K, D = (sp_conf or {}).get("max_keypoints"), (sp_conf or {}).get("descriptor_dim")
    if not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) and v >= 1 for v in (K, D)):
        raise ValueError(f"with extractor=None sp_conf needs max_keypoints and descriptor_dim, ints >= 1, got {K!r} and {D!r}")
    return int(K), int(D)


TILE_SELECTIONS = ("grid", "exhaustive", "preselection")
TILING_KEYS = ("min_matches_per_tile", "tile_overlap", "tile_preselection_size", "tile_selection", "tile_size")


def tiling_conf(tiling) -> dict | None:
    """The ``tiling`` argument of ImageSetMatcher, validated (None stays None).  Keys as in the reference's configuration:
    ``tile_size`` (x, y) or one int (required), ``tile_overlap`` int (default 0) and ``tile_selection`` "grid" (default),
    "exhaustive" or "preselection".  Preselection also needs ``tile_preselection_size`` (positive int: the longest side of the
    down-sampled images, no default) and takes ``min_matches_per_tile`` (int >= 0, default 5, tiling.tile_selection's); grid and
    exhaustive accept and ignore both.  The returned dict adds ``tile_hw`` / ``overlap_hw``, the (H, W) order ``tiling._hw`` gives
    them."""
    if tiling is None:
        return None
    from .tiling import _hw
    unknown = set(tiling) - set(TILING_KEYS)
    if unknown:
        raise ValueError(f"unknown tiling option(s) {sorted(unknown)}; expected some of {list(TILING_KEYS)}")
    if "tile_size" not in tiling:
        raise ValueError("tiling needs tile_size")
    size, overlap = tiling["tile_size"], tiling.get("tile_overlap", 0)
    sel = str(tiling.get("tile_selection", "grid")).lower()
    ok_size = isinstance(size, int) or (isinstance(size, (tuple, list)) and len(size) == 2 and all(isinstance(v, int) for v in size))
    if not ok_size or min(_hw(size)) < 1:
        raise ValueError(f"tile_size must be a positive int or (x, y) of positive ints, got {size!r}")
    if not isinstance(overlap, int) or not 0 <= overlap < min(_hw(size)):
        raise ValueError(f"tile_overlap must be an int in [0, min(tile_size)), got {overlap!r}")
    if sel not in TILE_SELECTIONS:
        raise ValueError(f"tile_selection must be one of {TILE_SELECTIONS}, got {tiling.get('tile_selection')!r}")
    out = {"tile_size": size if isinstance(size, int) else tuple(size), "tile_overlap": overlap, "tile_selection": sel,
           "tile_hw": _hw(size), "overlap_hw": _hw(overlap)}
    if sel == "preselection":
        pre, mm = tiling.get("tile_preselection_size"), tiling.get("min_matches_per_tile", 5)
        if isinstance(pre, bool) or not isinstance(pre, int) or pre < 1:
            raise ValueError(f"tile_selection \"preselection\" needs tile_preselection_size, a positive int, got {pre!r}")
        if isinstance(mm, bool) or not isinstance(mm, int) or mm < 0:
            raise ValueError(f"min_matches_per_tile must be an int >= 0, got {mm!r}")
        out.update(tile_preselection_size=pre, min_matches_per_tile=mm)
    return out


PAIR_GENERATION_KEYS = ("min_matches", "resize_max", "strategy")


def pair_generation_conf(pair_generation) -> dict | None:
    """The ``pair_generation`` argument of ImageSetMatcher, validated (None stays None).  ``strategy`` is required and must be
    "matching_lowres" (the reference's default, pairs_generator.py:40-235); ``resize_max`` (int >= 1, default 1000) is the longest
    side of the low-resolution images and ``min_matches`` (int >= 0, default 20) the count a pair must exceed to be kept."""
    if pair_generation is None:
        return None
    unknown = set(pair_generation) - set(PAIR_GENERATION_KEYS)
    if unknown:
        raise ValueError(f"unknown pair_generation option(s) {sorted(unknown)}; expected some of {list(PAIR_GENERATION_KEYS)}")
    if "strategy" not in pair_generation:
        raise ValueError("pair_generation needs strategy")
    if pair_generation["strategy"] != "matching_lowres":
        raise ValueError(f"pair_generation strategy {pair_generation['strategy']!r} does not run on the device (only \"matching_lowres\" "
                         "does); pass `pairs` built with pairs_from_bruteforce or pairs_from_sequential instead")
    out = {"strategy": "matching_lowres", "resize_max": pair_generation.get("resize_max", 1000),
           "min_matches": pair_generation.get("min_matches", 20)}
    for key, low in (("resize_max", 1), ("min_matches", 0)):
        if isinstance(out[key], bool) or not isinstance(out[key], int) or out[key] < low:
            raise ValueError(f"{key} must be an int >= {low}, got {out[key]!r}")
    return out


UPRIGHT_KEYS = ("max_keypoints", "resize_max")


def upright_conf(upright) -> dict | None:
    """The ``upright`` argument of ImageSetMatcher, validated (None stays None): ``resize_max`` (required int >= 1, the longest side of
    the search images; no default, as none is pinned) and ``max_keypoints`` (int >= 1, default 2048, the search SuperPoint's cap:
    the plugin default -1, no cap, has no device buffer)."""
    if upright is None:
        return None
    unknown = set(upright) - set(UPRIGHT_KEYS)
    if unknown:
        raise ValueError(f"unknown upright option(s) {sorted(unknown)}; expected some of {list(UPRIGHT_KEYS)}")
    if "resize_max" not in upright:
        raise ValueError("upright needs resize_max")
    out = {"resize_max": upright["resize_max"], "max_keypoints": upright.get("max_keypoints", 2048)}
    for key in UPRIGHT_KEYS:
        if isinstance(out[key], bool) or not isinstance(out[key], int) or out[key] < 1:
            raise ValueError(f"upright {key} must be an int >= 1, got {out[key]!r}")
    return out


QUALITIES = {"highest": -1, "high": 0, "medium": 1, "low": 2, "lowest": 3}


def quality_conf(quality="high") -> int:
    """The pyramid level of the reference's extraction ``quality`` (ExtractorBase._resize_image / _resize_features): "highest" -1 (one
    cv2.pyrUp, keypoints / 2), "high" 0 (unchanged, the default), "medium" 1, "low" 2 and "lowest" 3 (that many cv2.pyrDown, keypoints
    * 2^level).  Case-insensitive; anything else raises ValueError."""
    level = QUALITIES.get(quality.lower()) if isinstance(quality, str) else None
    if level is None:
        raise ValueError(f"quality must be one of {list(QUALITIES)}, got {quality!r}")
    return level


def tile_pairs_for(selection: str, n_tiles: int, n_tiles1: int | None = None) -> list:
    """The tile pairs of one image pair under a configured selection (tiling.tile_selection), image 0 cut into `n_tiles` tiles and
    image 1 into `n_tiles1` (default: as many): "grid" pairs tile t with tile t for t < min(n_tiles, n_tiles1) (the reference zips
    the two tile lists), "exhaustive" every (t0, t1), sorted."""
    n_tiles1 = n_tiles if n_tiles1 is None else n_tiles1
    if selection == "grid":
        return [(t, t) for t in range(min(n_tiles, n_tiles1))]
    if selection == "exhaustive":
        return [(t0, t1) for t0 in range(n_tiles) for t1 in range(n_tiles1)]
    raise ValueError(f"tile_selection must be one of {TILE_SELECTIONS}, got {selection!r}")


def image_sizes(n_images: int, height, width) -> list:
    """The (H, W) of every image of a set: `height` and `width` both ints (every image has that size) or both sequences of `n_images`
    ints (image i is height[i] x width[i]).  Raises ValueError for any other form and for sizes below 1."""
    seq = [isinstance(v, (list, tuple, range, np.ndarray)) for v in (height, width)]
    if seq[0] != seq[1]:
        raise ValueError(f"height and width must both be ints or both be sequences of n_images ints, got {height!r} and {width!r}")
    if isinstance(n_images, bool) or not isinstance(n_images, (int, np.integer)) or n_images < 1:
        raise ValueError(f"an image set needs n_images >= 1, got {n_images!r}")
    hs, ws = (list(height), list(width)) if seq[0] else ([height] * n_images, [width] * n_images)
    if len(hs) != n_images or len(ws) != n_images:
        raise ValueError(f"height and width must hold one size per image: {len(hs)} and {len(ws)} for {n_images} images")
    for v in hs + ws:
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise ValueError(f"image sizes must be ints >= 1, got {v!r}")
    return [(int(h), int(w)) for h, w in zip(hs, ws)]


def _by_size(sizes, items) -> list:
    """`items` grouped by sizes[item]: [((H, W), [items...])] in order of first appearance, item order kept inside a group."""
    groups = {}
    for k in items:
        groups.setdefault(sizes[k], []).append(k)
    return list(groups.items())


def pack_tile_batches(n_tile_pairs, batch_pairs: int) -> list:
    """Consecutive image pairs packed into matcher batches of at most ``batch_pairs`` tile pairs, image pairs kept whole: a list of
    (start, end) ranges of image pairs.  Raises ValueError when one image pair alone selects more than ``batch_pairs`` tile pairs."""
    out, start, load = [], 0, 0
    for k, n in enumerate(n_tile_pairs):
        if n > batch_pairs:
            raise ValueError(f"image pair {k} selects {n} tile pairs, more than batch_pairs={batch_pairs}")
        if load + n > batch_pairs:
            out.append((start, k))
            start, load = k, 0
        load += n
    if start < len(n_tile_pairs):
        out.append((start, len(n_tile_pairs)))
    return out


def _lowres_size(height: int, width: int, size: int):
    """(scale, h, w) of an image down- or up-sampled so that its longest side is `size`, as pairs_generator.read_lowres and
    tiling.preselection_matches compute it."""
    scale = size / max(height, width)
    w, h = (int(round(x * scale)) for x in (width, height))
    return scale, h, w


class _LowResSet:
    """The low-resolution SuperPoint + LightGlue pass shared by tile preselection, pair generation and the upright search.  ``extract``
    resizes each image once with INTER_AREA to longest side `size` (gray images: dimb_resize_area_dev, or dimb_resize_area_linear_dev
    when that enlarges an axis; RGB images of an ALIKED set: dimb_resize_area_rgb_dev, gray_from_rgb's rule fused into the resize) and
    runs SuperPoint (`sp_conf`) into float32 buffers per store slot (no float16 cast: these features never pass through features.h5
    in the reference), with their own extent for LightGlue without image_size; ``buffers`` are what the exchange all-gathers (about
    (256 + 2) * 4 * K bytes per slot); ``match`` runs LightGlue (`lg_conf`) on a batch of slot pairs into m / ms / nm / sl.

    `sizes` holds every image's (H, W): ``scales`` / ``low_sizes`` are each image's scale and (h, w), and for a set of one size
    ``scale`` / ``h`` / ``w`` are those values (None otherwise).  SuperPoint is built for the largest low-resolution height and width,
    and ``low`` is one flat buffer that each batch views as (k, h, w).

    With `rotations` (the upright search) every slot holds four entries, 4 * slot + ROTATIONS.index(r): the features of its
    low-resolution image turned by r (dimb_rot90_dev).  Per batch SuperPoint runs twice, on the 0 / 180 images (h x w) and on the
    90 / 270 images (w x h), into staging rows that are then copied to their entries; ``low`` holds the four turns of one batch."""

    def __init__(self, ctx, sp_weights, lg_weights, n_slots, sizes, size, sp_conf, lg_conf, batch_images, batch_pairs, device,
                 rotations=False):
        import torch

        from . import _native
        self.ctx = ctx
        geom = {s: _lowres_size(*s, size) for s in dict.fromkeys(sizes)}
        self.scales = [geom[s][0] for s in sizes]
        self.low_sizes = [geom[s][1:] for s in sizes]
        self.scale, self.h, self.w = geom[sizes[0]] if len(geom) == 1 else (None, None, None)
        K = self.K = sp_conf["max_keypoints"]
        self.E = 4 if rotations else 1
        mh, mw = max(h for _, h, _ in geom.values()), max(w for _, _, w in geom.values())
        if rotations:
            mh = mw = max(mh, mw)
        self.sp = _native.SuperPointNet(ctx, sp_weights, max_batch=batch_images * (2 if rotations else 1), max_height=mh, max_width=mw,
                                        **sp_conf)
        self.lg = _native.LightGlueNet(ctx, lg_weights, max_pairs=batch_pairs, max_kpts=K, **lg_conf)
        self.low = torch.zeros(self.E * batch_images * max(h * w for _, h, w in geom.values()), device=device)
        self.sc = torch.zeros(self.E * batch_images, K, device=device)  # written by the extractor, not read
        n_slots *= self.E
        self.kp = torch.zeros(n_slots, K, 2, device=device)
        self.de = torch.zeros(n_slots, 256, K, device=device)
        self.n = torch.zeros(n_slots, dtype=torch.int32, device=device)
        self.size = torch.zeros(n_slots, 2, device=device)
        if rotations:  # staging rows of one batch's four turns
            self.st_kp = torch.zeros(4 * batch_images, K, 2, device=device)
            self.st_de = torch.zeros(4 * batch_images, 256, K, device=device)
            self.st_n = torch.zeros(4 * batch_images, dtype=torch.int32, device=device)
            self.st_size = torch.zeros(4 * batch_images, 2, device=device)
        self.m = torch.zeros(batch_pairs, K, 2, dtype=torch.int64, device=device)
        self.ms = torch.zeros(batch_pairs, K, device=device)
        self.nm = torch.zeros(batch_pairs, dtype=torch.int32, device=device)
        self.sl = torch.zeros(batch_pairs, dtype=torch.int32, device=device)

    @property
    def buffers(self):
        return self.kp, self.de, self.n, self.size

    def extract(self, images, image_ids, slots, st):
        """One resize batch: the equally sized images `images` (gray (k, H, W) or RGB (k, H, W, 3), at most batch_images) of images
        `image_ids`, stored in `slots`.  RGB images are made gray by ``pairs_generator.gray_from_rgb``'s rule inside the resize."""
        H, W = images.shape[1:3]
        h, w = self.low_sizes[image_ids[0]]
        if images.dim() == 4:
            resize = self.ctx.resize_area_rgb_dev
        else:
            resize = self.ctx.resize_area_linear_dev if h > H or w > W else self.ctx.resize_area_dev
        K, ss = self.K, slots
        low = self.low[:len(ss) * h * w].view(len(ss), h, w)
        resize(images.data_ptr(), len(ss), H, W, low.data_ptr(), h, w, st)
        if self.E == 4:
            return self._extract_turns(low, ss, st)
        k = 0
        while k < len(ss):  # the extractor writes consecutive rows: one call per run of consecutive slots
            e = k + 1
            while e < len(ss) and ss[e] == ss[k] + (e - k):
                e += 1
            s = ss[k]
            self.sp.extract_dev(low[k].data_ptr(), e - k, h, w, self.kp[s].data_ptr(), self.sc[k].data_ptr(), self.de[s].data_ptr(),
                                self.n[s:].data_ptr(), K, st)
            self.ctx.kpts_extent_dev(e - k, self.kp[s].data_ptr(), K, self.n[s:].data_ptr(), self.size[s].data_ptr(), st)
            k = e

    def _extract_turns(self, low, slots, st):
        """The four turns of the k resized images `low` (k, h, w): low[0:k] as it is, then 180, 90 and 270 turns in ``self.low`` (the
        0 / 180 block and the 90 / 270 block each contiguous), SuperPoint once per block into the staging rows, one copy per buffer to
        the entries 4 * slot + ROTATIONS.index(r)."""
        from .upright import ROTATIONS
        K = self.K
        k, h, w = low.shape
        turns = (0, 180, 90, 270)  # staging order: rows [j * k, (j + 1) * k) hold turn turns[j]
        for j, r in enumerate(turns[1:], 1):
            self.ctx.rot90_dev(low.data_ptr(), k, h, w, 1, [r] * k, self.low[j * k * h * w:].data_ptr(), st)
        for j0, (bh, bw) in ((0, (h, w)), (2, (w, h))):
            rows = slice(j0 * k, (j0 + 2) * k)
            self.sp.extract_dev(self.low[j0 * k * h * w:].data_ptr(), 2 * k, bh, bw, self.st_kp[rows].data_ptr(), self.sc.data_ptr(),
                                self.st_de[rows].data_ptr(), self.st_n[rows].data_ptr(), K, st)
            self.ctx.kpts_extent_dev(2 * k, self.st_kp[rows].data_ptr(), K, self.st_n[rows].data_ptr(), self.st_size[rows].data_ptr(), st)
        idx = self.n.new_tensor([4 * s + ROTATIONS.index(r) for r in turns for s in slots]).long()
        for dst, src in ((self.kp, self.st_kp), (self.de, self.st_de), (self.n, self.st_n), (self.size, self.st_size)):
            dst.index_copy_(0, idx, src[:4 * k])

    def feats(self, slot):
        """The float32 features of a slot as LightGlue input, normalised by their own extent."""
        from . import _native
        K = self.K
        return _native.FeatsDev(self.kp[slot].data_ptr(), self.de[slot].data_ptr(), self.n[slot:].data_ptr(), K, 0, K, 0.0, 0.0, 0, 0, None,
                                self.size[slot].data_ptr())

    def match(self, s0, s1, st):
        """Enqueue LightGlue on the slot pairs (s0[k], s1[k]); returns both sides' FeatsDev lists."""
        f0, f1 = [self.feats(s) for s in s0], [self.feats(s) for s in s1]
        self.lg.match_dev(f0, f1, self.m.data_ptr(), self.ms.data_ptr(), self.nm.data_ptr(), self.sl.data_ptr(), self.K, st)
        return f0, f1


class ImageSetMatcher:
    """Two-phase multi-GPU matching of an image set (module docstring): the extractor on this rank's images into the device feature
    store, one all_gather of the float16 feature blocks, the configured matcher on this rank's share of the pair list, gather of the
    match tables.  ``dist`` is ``torch.distributed`` (initialised, nccl) or None for a single process.  ``matcher``: "lightglue"
    (default), "superglue" or "kornia_matcher".

    Phase 2 is one loop over pair batches for every mode (``match`` / ``match_verified``, tiled or not): the matcher, the
    verification when asked, then the batch's results reach the host in two synchronising steps, the counts (with F and n_inliers
    when verifying) and then only the table rows in use.

    ``matcher="superglue"``: ``lg_weights`` is the SuperGlue state dict and ``lg_conf`` its configuration (``sinkhorn_iterations``,
    ``match_threshold``, ``gnn_layers``), and phase 2 runs the batched device SuperGlue on the store's slots.

    ``matcher="kornia_matcher"``: KorniaMatcher's brute-force descriptor matching (kornia DescriptorMatcher).  ``lg_conf`` holds its
    keys ``match_mode`` (nn / mnn / snn / smnn, default smnn) and ``th`` (default 0.8), checked by ``kornia_conf``; ``lg_weights`` is
    not used (None is accepted) and no network is built.  Phase 2 runs dimb_nn_match_batch_dev on each pair batch of store slots or tile
    views, counts read on the device; the tables are KorniaMatcher._match_pairs' on the store's features, and the distance (nn / mnn)
    or ratio (snn / smnn) of every match is left in the device buffer ``ms``.  SuperPoint (256-d) and ALIKED (128-d) features.

    ``extractor=None``: given features.  No extraction network is built; ``sp_conf`` is ``{"max_keypoints": K, "descriptor_dim": D}``
    (``given_features_conf``), which sizes the store, and ``put_features`` replaces ``extract`` (``run_features`` /
    ``run_features_verified`` chain the steps).  Tiling, pair generation, upright and a quality other than "high" need the images and
    are refused.  ``matcher="lighterglue"`` (given 64-d XFeat features only): the LighterGlue network (``LIGHTERGLUE_CONF``;
    ``lg_weights`` None loads the vendored checkpoint), ``lg_conf`` checked by ``lighterglue_conf`` (``filter_threshold`` only), each
    side normalised by [W, H] as LighterGlueMatcher does; pair batches run dimb_lg_match_dev on the shape-generic batched engine, and
    the tables are LighterGlueMatcher._match_pairs' on the store's features.  With given features "lightglue" takes input_dim = D (256
    or 128), "superglue" D = 256 and "kornia_matcher" any D.

    ``verification``: None (default) matches only (``run`` / ``match``).  A dict (keys and defaults in ``verification_conf``) enables
    ``run_verified`` / ``match_verified``: every pair batch is verified on the device right after matching (dimb_gv_verify_dev on the
    store's float16 keypoints, seed ``gv_seed(seed, pair id)``).  The gate: a pair keeps its verified table iff
    ``n_inliers >= min_inliers_per_pair`` and ``float32(n_inliers) >= float32(min_inlier_ratio_per_pair) * float32(n_raw)``; a
    rejected pair gets an empty verified table (its F and count are still reported).  Pairs with fewer than 8 raw matches keep
    every match and have no F (as the reference's geometric_verification returns), then face the same gate.  Method "NONE":
    verified = raw, F = None, nothing is launched.

    ``extractor``: "superpoint" (default; gray images (k, H, W)) or "aliked" (RGB images (k, H, W, 3); ``sp_weights`` / ``sp_conf``
    are the ALIKED weights and the ``AlikedNet`` configuration, one image or tile per extraction call, 128-d descriptors, LightGlue
    built with input_dim 128).  ALIKED with SuperGlue is refused.  The low-resolution passes below (tile preselection, pair generation,
    upright) run SuperPoint + SuperPoint-LightGlue for either extractor, as the reference does.  An ALIKED set feeds them the gray image
    of each RGB image by ``pairs_generator.gray_from_rgb``'s rule (R first, not the BGR2GRAY order of a SuperPoint set's input), applied
    per source pixel inside the resize (dimb_resize_area_rgb_dev); ``superpoint_weights`` is their SuperPoint (default
    ``weights.superpoint_v1()``, the checkpoint the reference's hloc SuperPoint loads; refused with SuperPoint sets, where ``sp_weights``
    is that network), and since ``lg_weights`` is then an input_dim-128 LightGlue, ``preselection_weights`` / ``lowres_weights`` /
    ``upright_weights`` are required for the passes configured, whatever the matcher.

    ``extractor="orb"``: the reference's orb+kornia_matcher pipeline, as a SIFT set: the same gray images, ``OrbNet`` (cv2.ORB's
    detect + compute), ``sp_conf`` with the ORBExtractor keys (``orb_set_conf``), D = 32, scores of ones, n_features +
    ``orb_tie_room(n_features)`` store rows (``exchange`` raises RuntimeError for an image with more), and the same refusals.

    ``extractor="sift"``: the reference's sift+kornia_matcher pipeline.  Gray images (k, H, W) as for SuperPoint, extracted by
    ``SiftNet`` (cv2.SIFT's detectAndCompute, ``batch_images`` per call); ``sp_conf`` holds the SIFTExtractor keys (``sift_set_conf``,
    n_features >= 1), ``sp_weights`` / ``lg_weights`` are not used, D = 128 and the stored scores are ones.  The store holds
    n_features + ``SIFT_TIE_ROOM`` rows per image, since retainBest keeps every keypoint tied with the n_features-th response;
    ``exchange`` raises RuntimeError for an image with more (``_check_sift_counts``).  Only ``matcher="kornia_matcher"`` with quality
    "high" is supported: other matchers, tiling (and tile preselection), pair generation, upright and other qualities raise ValueError.

    ``tiling``: None (default) or a dict checked by ``tiling_conf``.  With tiling, ``extract`` takes full-size images, cuts their tiles
    on the device, runs the extractor over tiles (SuperPoint ``batch_images`` tiles per call, network sized for one tile, with
    ``fix_sampling=True`` as the reference's tiling requires) and merges each image's tile features into its slot (store capacity
    T * K).  ``exchange`` also builds the per-tile views of every image.  ``match`` / ``match_verified`` pack whole image pairs into
    matcher batches of at most ``batch_pairs`` tile pairs, match the selected tile pairs out of the views and return one merged,
    de-duplicated table per image pair in merged-slot rows; verification and ``export_colmap`` run on the merged slots.  ``tile_pairs``
    (per image pair, a list of (t0, t1)) overrides the configured selection.

    ``tile_selection: "preselection"`` computes every pair's list on the device, equal to ``tiling.preselection_matches`` +
    ``tiling.tile_selection``: ``extract`` also down-samples each image once (INTER_AREA, longest side ``tile_preselection_size``)
    and runs SuperPoint (``tiling.SP_PRESELECTION_CONF``) into float32 per-slot buffers (about 4.2 MB per image, all-gathered by
    ``exchange``); ``match`` runs LightGlue (``tiling.LG_PRESELECTION_CONF``, keypoints normalised by their own extent) on the
    low-resolution features of each pair batch and keeps the tile pairs with more than ``min_matches_per_tile`` matches inside both
    boxes.  ``preselection_weights``: the weights of that LightGlue (default ``lg_weights``; required with SuperGlue and
    kornia_matcher, and with ALIKED).  The per-pair flags of one ``match`` call take T^2 bytes per pair on the device and
    on the host (``_preselect``), which matters only at hundreds of tiles per image.

    ``pair_generation``: None (default; the pair list is an input) or a dict checked by ``pair_generation_conf``, the reference's
    default strategy "matching_lowres" (pairs_generator.pairs_from_lowres) on the device.  ``extract`` also resizes each image once
    with INTER_AREA to longest side ``resize_max`` (enlarging too, as the reference does for small photos) and runs SuperPoint
    (``pairs_generator.SP_LOWRES_CONF``) into float32 per-slot buffers (about 2.1 MB per image, all-gathered by ``exchange``);
    ``lowres_pairs`` runs LightGlue (``pairs_generator.LG_LOWRES_CONF``, own-extent normalisation) over every brute-force pair, dealt to
    the ranks, and keeps the pairs with more than ``min_matches`` matches; ``run_lowres`` then matches the kept pairs.
    ``lowres_weights``: the weights of that LightGlue (default ``lg_weights``; required with SuperGlue, kornia_matcher and ALIKED).
    do_geometric_verification is refused (an unknown key).

    ``quality``: the reference's extraction quality, checked by ``quality_conf`` ("high", the default, changes nothing).  ``height`` /
    ``width`` stay the original image size and ``extract`` still takes full-size images: per extraction batch dimb_pyr_dev resizes them
    (bitwise cv2.pyrUp for "highest", one to three cv2.pyrDown for "medium" / "low" / "lowest") into a buffer of the resized size, the
    extractor (sized for the resized image, or tiles cut from it with the tile grid, border test and de-duplication in resized
    pixels) runs on it, and one dimb_fstore_rescale_dev multiplies the stored float16 keypoints by 2^level and records the original
    [H, W], as _resize_features and the h5 writer leave them.  Matching, verification and export then see original-pixel features.
    Pair generation reads the original images.  Tile preselection with a quality other than "high" is refused, and so is a quality
    that leaves an untiled image smaller than the extractor accepts (16 px per side for SuperPoint, 32 for ALIKED).

    Image sizes: ``height`` / ``width`` are ints (every image has that size) or sequences of ``n_images`` ints, image i being
    height[i] x width[i] (checked by ``image_sizes``; every per-size rule above is checked for each image).  All ranks pass the same
    sizes.  ``extract`` then takes a list of per-image tensors (or one stacked tensor when its images share a size), groups this rank's
    images by size and runs each group as a set of that size: its own pyramid steps, batches, tile grid (T_i tiles, store capacity
    max(T_i) * K, tile views at ``view_offsets[i]``), low-resolution size and scale, and its own [H, W] in every slot, so LightGlue,
    SuperGlue, verification and the COLMAP cameras see each image's own size.  Grid selection pairs tile t with tile t for
    t < min(T_i, T_j), as the reference's zip does.  The extractor is built for the largest extraction height and the largest width
    of the set.  Per-image values: ``sizes``, ``ext_sizes`` (after quality), ``tile_counts`` and ``view_offsets``, and ``scales`` /
    ``low_sizes`` of the low-resolution sets; for a set of one size ``H`` / ``W`` / ``h2`` / ``w2`` / ``T`` / ``G`` / ``pre_h`` /
    ``pre_w`` hold that size's values, for a mixed set they are None.  A set given as lists of equal sizes is a set of one size: the
    same launches and outputs as the int form.

    ``upright``: None (default) or a dict checked by ``upright_conf`` (``resize_max`` required, ``max_keypoints`` default 2048), the
    reference's upright option with the rules of ``upright.py``.  ``upright`` searches each image's rotation over the pair list
    (``rotations``, the same on every rank), ``extract`` then extracts the rotated images, ``match`` / ``match_verified`` match in the
    rotated frames (F mapped back to original pixels by ``upright.rotate_back_F``), and ``rotate_back`` puts the stored keypoints and
    ``image_size`` back on the original images, after which matching is refused until the next ``extract``; ``run`` /
    ``run_verified`` / ``run_lowres`` chain the steps (``run_lowres`` searches over the kept pairs), and ``export_colmap`` writes
    original-frame keypoints and camera sizes.  ``tile_idx`` keeps the rotated image's tile indices.  ``upright_weights``: the
    search's SuperPoint-LightGlue weights (default ``lg_weights``; required with SuperGlue, kornia_matcher and ALIKED).  With ALIKED
    the search runs on the gray images of the RGB originals and ALIKED extracts from the turned RGB images; ``rotate_back`` turns the
    stored float16 keypoints back and rounds them to float16 again, which ALIKED's sub-pixel keypoints can feel.  Refused: tile
    preselection, and explicit ``tile_pairs``.  Every per-size rule is checked for both orientations of every image, and the extractor
    workspace, the store and the tile views are sized for both, since the rotations are unknown at construction (a set of 1536 x 2048
    images gets a 2048 x 2048 workspace); the search holds four float32 feature entries per image (about 8.5 MB at 2048 keypoints)
    on every rank, and ``extract`` one rotated batch of batch_images full-size images at a time."""

    def __init__(self, ctx, sp_weights: dict, lg_weights: dict, n_images: int, height, width, sp_conf: dict, lg_conf: dict,
                 batch_images: int = 16, batch_pairs: int = 32, dist=None, matcher: str = "lightglue", verification: dict | None = None,
                 tiling: dict | None = None, extractor: str = "superpoint", preselection_weights: dict | None = None,
                 pair_generation: dict | None = None, lowres_weights: dict | None = None, quality: str = "high", upright: dict | None = None,
                 upright_weights: dict | None = None, superpoint_weights: dict | None = None):
        import torch

        from . import _native
        if matcher not in ("lightglue", "superglue", "kornia_matcher", "lighterglue"):
            raise ValueError(f'matcher must be "lightglue", "superglue", "kornia_matcher" or "lighterglue", got {matcher!r}')
        if extractor not in ("superpoint", "aliked", "sift", "orb", None):
            raise ValueError(f'extractor must be "superpoint", "aliked", "sift", "orb" or None (given features), got {extractor!r}')
        if extractor in ("sift", "orb"):
            name_u = extractor.upper()
            if matcher != "kornia_matcher":
                raise ValueError(f'matcher {matcher!r} with extractor="{extractor}" is not supported; {name_u} sets match with '
                                 '"kornia_matcher"')
            for name, val, off in (("tiling (and tile preselection)", tiling, None), ("pair_generation", pair_generation, None),
                                   ("upright", upright, None)):
                if val != off:
                    raise ValueError(f'{name} with extractor="{extractor}" is not supported')
            if quality_conf(quality) != 0:
                raise ValueError(f'quality {quality!r} with extractor="{extractor}" is not supported (the reference resizes uint8 '
                                 'images there); use quality="high"')
            sp_conf = sift_set_conf(sp_conf) if extractor == "sift" else orb_set_conf(sp_conf)
        if matcher == "lighterglue" and extractor is not None:
            raise ValueError(f"LighterGlue matches XFeat features only, which are given (extractor=None), not extracted by {extractor}")
        given = None
        if extractor is None:
            given = given_features_conf(sp_conf)
            for name, val, off in (("tiling", tiling, None), ("pair_generation", pair_generation, None), ("upright", upright, None),
                                   ("quality", quality, "high")):
                if val != off:
                    raise ValueError(f"{name} needs the images; with extractor=None (given features) it is not supported")
            D = given[1]
            if matcher == "lighterglue" and D != 64:
                raise ValueError(f"LighterGlue matches 64-d XFeat descriptors, got descriptor_dim {D}")
            if matcher == "lightglue":
                lg_conf = {"input_dim": D, **(lg_conf or {})}
                if D not in (256, 128) or lg_conf["input_dim"] != D:
                    raise ValueError(f"LightGlue on given features needs input_dim = descriptor_dim, 256 or 128, got {lg_conf['input_dim']} "
                                     f"and {D}")
            if matcher == "superglue" and D != 256:
                raise ValueError(f"SuperGlue matches 256-d descriptors (with scores), got descriptor_dim {D}")
        self.ltg_conf = lighterglue_conf(lg_conf) if matcher == "lighterglue" else None
        if extractor == "aliked" and matcher == "superglue":
            raise ValueError("SuperGlue matches SuperPoint features only; use matcher=\"lightglue\" with ALIKED")
        if extractor == "superpoint" and superpoint_weights is not None:
            raise ValueError("superpoint_weights is the low-resolution SuperPoint of an ALIKED set; with extractor=\"superpoint\" sp_weights "
                             "is that network")
        self.nn_conf = kornia_conf(lg_conf) if matcher == "kornia_matcher" else None
        self.tiling = tiling_conf(tiling)
        self.sizes = image_sizes(n_images, height, width)
        self.up = upright_conf(upright)
        # the distinct sizes: every per-size rule is checked once per size; with upright for both orientations of every image
        shapes = list(dict.fromkeys(self.sizes + ([(w, h) for h, w in self.sizes] if self.up else [])))
        self.presel = self.tiling is not None and self.tiling["tile_selection"] == "preselection"
        # an ALIKED set's lg_weights is an input_dim-128 LightGlue: its low-resolution passes need their SuperPoint-LightGlue weights
        aliked_lg = "the superpoint_lightglue state dict (lg_weights of an ALIKED set is an input_dim-128 LightGlue)"
        if self.up is not None:
            if extractor == "aliked" and upright_weights is None:
                raise ValueError(f"upright with extractor=\"aliked\" needs upright_weights, {aliked_lg}")
            if self.presel:
                raise ValueError("upright with tile_selection \"preselection\" is not supported; use grid or exhaustive tile selection")
            if matcher != "lightglue" and upright_weights is None:
                raise ValueError(f"upright with matcher=\"{matcher}\" needs upright_weights (SuperPoint-LightGlue weights)")
            for H, W in shapes:
                if min(_lowres_size(H, W, self.up["resize_max"])[1:]) < 1:
                    raise ValueError(f"upright resize_max {self.up['resize_max']} down-samples a {H}x{W} image to nothing")
        if self.presel:
            if extractor == "aliked" and preselection_weights is None:
                raise ValueError(f"tile preselection with extractor=\"aliked\" needs preselection_weights, {aliked_lg}")
            for H, W in shapes:
                if self.tiling["tile_preselection_size"] > max(H, W):
                    raise ValueError(f"tile_preselection_size {self.tiling['tile_preselection_size']} exceeds the image's longest side "
                                     f"{max(H, W)}: preselection only downscales")
            if matcher != "lightglue" and preselection_weights is None:
                raise ValueError(f"tile preselection with matcher=\"{matcher}\" needs preselection_weights (SuperPoint-LightGlue weights)")
            for H, W in shapes:
                if min(_lowres_size(H, W, self.tiling["tile_preselection_size"])[1:]) < 1:
                    raise ValueError(f"tile_preselection_size {self.tiling['tile_preselection_size']} down-samples a {H}x{W} image to nothing")
        self.level = quality_conf(quality)
        if self.level and self.presel:
            raise ValueError(f"tile preselection runs at the original resolution here; quality {quality!r} with tile_selection "
                             "\"preselection\" is not supported (use quality=\"high\", or grid / exhaustive tile selection)")
        # the size the extractor sees (the sizes stay the original images')
        ext = {s: s if self.level == 0 else _native.pyr_size(*s, self.level) for s in shapes}
        least = 16 if extractor == "superpoint" else 32
        for (H, W), (h2, w2) in ext.items():
            if self.level and tiling is None and min(h2, w2) < least:
                raise ValueError(f"quality {quality!r} resizes a {H}x{W} image to {h2}x{w2}, below the {least} px per side "
                                 f"the {extractor} extractor needs")
        self.pairgen = pair_generation_conf(pair_generation)
        if self.pairgen is not None:
            if extractor == "aliked" and lowres_weights is None:
                raise ValueError(f"pair generation with extractor=\"aliked\" needs lowres_weights, {aliked_lg}")
            if matcher != "lightglue" and lowres_weights is None:
                raise ValueError(f"pair generation with matcher=\"{matcher}\" needs lowres_weights (SuperPoint-LightGlue weights)")
            for H, W in shapes:
                if min(_lowres_size(H, W, self.pairgen["resize_max"])[1:]) < 1:
                    raise ValueError(f"resize_max {self.pairgen['resize_max']} down-samples a {H}x{W} image to nothing")
        uniform = len(shapes) == 1
        self._ext = ext
        # one size: the int attributes of that size; a mixed set has None there, and the per-image lists above and below
        self.H, self.W = shapes[0] if uniform else (None, None)
        self.h2, self.w2 = ext[shapes[0]] if uniform else (None, None)
        self.grid = self.T = self.G = None
        self._grids = grids = None
        if self.tiling is not None:
            self._grids = grids = {s: _native.tile_grid(*ext[s], *self.tiling["tile_hw"], *self.tiling["overlap_hw"]) for s in shapes}
        self._set_frames(self.sizes)
        if self.tiling is not None:
            if uniform:
                self.grid, self.T = grids[shapes[0]], self.tile_counts[0]
                self.G = max(1, batch_images // self.T)
        if self.tiling is not None and extractor == "superpoint":
            if "fix_sampling" in sp_conf and not sp_conf["fix_sampling"]:
                raise ValueError("tiled SuperPoint extraction runs with fix_sampling=True (the reference's rule); fix_sampling=False was given")
            sp_conf = {**sp_conf, "fix_sampling": True}
        if extractor == "aliked" and matcher == "lightglue":
            lg_conf = {"input_dim": 128, **lg_conf}
            if lg_conf["input_dim"] != 128:
                raise ValueError(f"LightGlue on ALIKED features needs input_dim=128, got {lg_conf['input_dim']}")
        self.torch, self.dist, self.ctx = torch, dist, ctx
        self.world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        self.n = n_images
        self.slots = [store_slot(i, n_images, self.world) for i in range(n_images)]
        self.extractor = extractor
        if given is not None:
            self.cap, self.D = given
        elif extractor == "sift":
            self.cap, self.D = sp_conf["n_features"] + SIFT_TIE_ROOM, 128
        elif extractor == "orb":
            self.cap, self.D = sp_conf["n_features"] + orb_tie_room(sp_conf["n_features"]), 32
        else:
            self.cap = int(sp_conf["max_keypoints"]) if extractor == "superpoint" else int(sp_conf.get("max_num_keypoints", 4000))
            self.D = 256 if extractor == "superpoint" else 128
        if self.cap < 1:
            raise ValueError(f"the image-set matcher needs a positive keypoint limit per extraction, got {self.cap}")
        self.B, self.P = batch_images, batch_pairs
        # the network takes the largest extraction height and width of the set (a set of portrait and landscape images over-sizes its
        # workspace: 2048 x 2048 for 1536 x 2048 plus 2048 x 1536), or one tile
        eh, ew = max(h for h, _ in ext.values()), max(w for _, w in ext.values())
        if self.tiling is not None:
            eh, ew = self.tiling["tile_hw"]
        if extractor == "superpoint":
            self.sp = _native.SuperPointNet(ctx, sp_weights, max_batch=batch_images, max_height=eh, max_width=ew, **sp_conf)
        elif extractor == "aliked":
            self.al = _native.AlikedNet(ctx, sp_weights, max_height=eh, max_width=ew, **sp_conf)
        elif extractor == "sift":
            self.sift = _native.SiftNet(ctx, max_batch=batch_images, max_height=eh, max_width=ew, **sp_conf)
        elif extractor == "orb":
            self.orb = _native.OrbNet(ctx, max_batch=batch_images, max_height=eh, max_width=ew, **sp_conf)
        self.matcher = matcher
        if matcher == "superglue":
            self.sg = _native.SuperGlueNet(ctx, lg_weights, max_pairs=batch_pairs, max_kpts=self.cap, **lg_conf)
        elif matcher == "lightglue":
            self.lg = _native.LightGlueNet(ctx, lg_weights, max_pairs=batch_pairs, max_kpts=self.cap, **lg_conf)
        elif matcher == "lighterglue":
            from .matchers.lighterglue import LIGHTERGLUE_CONF, lighterglue_weights
            self.lg = _native.LightGlueNet(ctx, lighterglue_weights() if lg_weights is None else lg_weights, max_pairs=batch_pairs,
                                           max_kpts=self.cap, filter_threshold=self.ltg_conf["filter_threshold"], **LIGHTERGLUE_CONF)
        self.ipr = images_per_rank(n_images, self.world)
        t_max = 1 if self.tiling is None else max(len(g["origins"]) for g in grids.values())
        self.store = _native.FeatureStoreDev(ctx, self.world * self.ipr, t_max * self.cap, self.D)
        dev = torch.device("cuda", ctx.device)
        # extraction outputs of one batch (float32, library layouts) and match outputs of one pair batch; tiled: the tiles of the
        # max(1, batch_images // T) images of one cut, T the tile count of their size
        self.C = 3 if extractor == "aliked" else 1
        n_img = {s: batch_images if self.tiling is None else max(1, batch_images // len(grids[s]["origins"])) for s in shapes}
        n_ext = batch_images
        if self.tiling is not None:
            n_ext = max(n_img[s] * len(grids[s]["origins"]) for s in shapes)
            self.tiles = torch.zeros(n_ext, eh, ew, self.C, device=dev)
        if self.level:  # the resized images of one extraction batch (tiled: of one cut), one flat buffer viewed per size
            self.resized = torch.zeros(max(n_img[s] * ext[s][0] * ext[s][1] for s in shapes) * self.C, device=dev)
        if extractor is not None:
            self.kp = torch.zeros(n_ext, self.cap, 2, device=dev)
            self.sc = torch.zeros(n_ext, self.cap, device=dev)
            self.de = torch.zeros(n_ext, self.D, self.cap, device=dev)
            self.cnt = torch.zeros(n_ext, dtype=torch.int32, device=dev)
        if extractor == "sift":  # every image's true keypoint count, checked against the store's capacity by exchange
            self.sift_counts = torch.zeros(n_images, dtype=torch.int32, device=dev)
        if extractor == "orb":
            self.orb_counts = torch.zeros(n_images, dtype=torch.int32, device=dev)
        self.m = torch.zeros(batch_pairs, self.cap, 2, dtype=torch.int64, device=dev)
        self.ms = torch.zeros(batch_pairs, self.cap, device=dev)
        self.nm = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)
        self.sl = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)
        gv_cap = self.cap
        if self.tiling is not None:
            # per-tile views of every image (slot view_offsets[i] + t) with their row maps, and the merged tables of one batch: an image
            # pair has at most min(batch_pairs, T0 * T1) distinct tile pairs of at most K rows each, so cap2 holds every merged table whole
            # (upright: room for each image's larger grid of its two orientations)
            n_views = sum(max(len(grids[s]["origins"]), len(grids[s[::-1]]["origins"]) if self.up else 0) for s in self.sizes)
            self.views = _native.FeatureStoreDev(ctx, n_views, self.cap, self.D)
            self.vmap = torch.zeros(n_views, self.views.cap, dtype=torch.int32, device=dev)
            self.cap2 = gv_cap = min(batch_pairs, t_max * t_max) * self.cap
            self.mm = torch.zeros(batch_pairs, self.cap2, 2, dtype=torch.int64, device=dev)
            self.nmm = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)
        self.pre = self.lowres = None
        low_sp = sp_weights  # the low-resolution SuperPoint: the set's own, or for an ALIKED set superpoint_weights
        if extractor == "aliked" and (self.presel or self.pairgen is not None or self.up is not None):
            from .weights import superpoint_v1
            low_sp = superpoint_v1() if superpoint_weights is None else superpoint_weights
        if self.presel:
            # PRESELECTION (matcher_base.py:1055-1089) on the device with the networks of matcher_base.py:143-159, and the box counts
            # of one pair batch
            from .tiling import LG_PRESELECTION_CONF, SP_PRESELECTION_CONF
            self.pre = _LowResSet(ctx, low_sp, lg_weights if preselection_weights is None else preselection_weights, self.world * self.ipr,
                                  self.sizes, self.tiling["tile_preselection_size"], SP_PRESELECTION_CONF, LG_PRESELECTION_CONF,
                                  batch_images, batch_pairs, dev)
            self.pre_h, self.pre_w = self.pre.h, self.pre.w
            self.pre_cnt = torch.zeros(batch_pairs, t_max * t_max, dtype=torch.int32, device=dev)
        if self.pairgen is not None:
            # matching_lowres (pairs_generator.py:40-235) with the networks of pairs_generator.py:104-126
            from .pairs_generator import LG_LOWRES_CONF, SP_LOWRES_CONF
            self.lowres = _LowResSet(ctx, low_sp, lg_weights if lowres_weights is None else lowres_weights, self.world * self.ipr,
                                     self.sizes, self.pairgen["resize_max"], SP_LOWRES_CONF, LG_LOWRES_CONF, batch_images, batch_pairs, dev)
        self.search = self.rotations = None
        self._turned_back = False
        if self.up is not None:
            # find_matches_per_rotation (image_matching.py:69-118) with the plugins' default networks; fixed descriptor sampling when
            # tiling or pair generation is configured (quirk A.6), otherwise sp_conf's
            from .upright import LG_UPRIGHT_CONF, SP_UPRIGHT_CONF
            fix = self.tiling is not None or self.pairgen is not None or bool(sp_conf.get("fix_sampling", False))
            self.search = _LowResSet(ctx, low_sp, lg_weights if upright_weights is None else upright_weights, self.world * self.ipr,
                                     self.sizes, self.up["resize_max"], {**SP_UPRIGHT_CONF, "max_keypoints": self.up["max_keypoints"],
                                                                         "fix_sampling": fix},
                                     LG_UPRIGHT_CONF, batch_images, batch_pairs, dev, rotations=True)
        self.gv = verification_conf(verification)
        if self.gv is not None and self.gv["method"] != "NONE":  # verification outputs of one pair batch
            self.v = torch.zeros(batch_pairs, gv_cap, 2, dtype=torch.int64, device=dev)
            self.nv = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)
            self.F = torch.zeros(batch_pairs, 9, device=dev)
            self.mask = torch.zeros(batch_pairs, gv_cap, dtype=torch.uint8, device=dev)
            self.ninl = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)

        class _DevArr:  # zero-copy torch view of the store's device allocation (for the NCCL all_gather)
            def __init__(self, ptr, shape):
                self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "|u1", "version": 2}

        self.store_t = torch.as_tensor(_DevArr(self.store.base, (self.world * self.ipr, self.store.slot_bytes)), device=dev)
        self.exchanged_bytes = 0

    def extract(self, d_images, image_ids):
        """Phase 1: this rank's images `image_ids` as float32 CUDA data, 0..255, gray for SuperPoint and RGB for ALIKED: one tensor
        (k, H, W) / (k, H, W, 3) when they all have the same size, or a list of k tensors (H_i, W_i) / (H_i, W_i, 3) in `image_ids`
        order.  Images are processed in groups of one size (image order kept inside a group), each group batched as a set of that
        size; a shape that is not its image's declared size raises ValueError before any launch.  With tiling the images are full
        size and are cut into tiles on the device.  A list is copied into one staging tensor per batch of batch_images, which feeds
        the low-resolution sets and (untiled) the extractor; tiled extraction stages again per cut, whose size differs.

        With upright the images are the unrotated ones, ``upright`` must have run (RuntimeError otherwise), and each staged batch is
        first turned by its images' rotations at full size (dimb_rot90_dev, one launch per batch into one buffer of the batch,
        ``_extract_turned``); everything else (quality, tile cut, extractor, by rotated size) runs on the rotated images.  The
        low-resolution sets were filled by ``upright`` from the unrotated images."""
        if self.extractor is None:
            raise RuntimeError("ImageSetMatcher was built with extractor=None: its features are given with put_features()")
        st = self.torch.cuda.current_stream().cuda_stream
        if self.up is not None:
            if self.rotations is None:
                raise RuntimeError("ImageSetMatcher was built with upright: run upright() before extract()")
            self._turned_back = False
            return self._extract_turned(d_images, image_ids, st)
        groups = self._groups(d_images, image_ids)
        lows = [low for low in (self.pre, self.lowres) if low is not None]
        if self.tiling is not None:
            if lows:
                for _, ids, src in self._batches(d_images, image_ids, groups, self.B):
                    for low in lows:
                        low.extract(src, ids, [self.slots[i] for i in ids], st)
            return self._extract_tiled(d_images, image_ids, groups, st)
        for (H, W), ids, src in self._batches(d_images, image_ids, groups, self.B):
            for low in lows:
                low.extract(src, ids, [self.slots[i] for i in ids], st)
            self._extract_batch(src, ids, H, W, st)

    def put_features(self, feats, image_ids):
        """Phase 1 with given features (extractor=None), in place of ``extract``: this rank's images `image_ids` as FeaturesDicts in
        get_features' contract (keypoints (N,2), descriptors (D,N), scores (N,), image_size [H,W]), put into their store slots with the
        float16 cast of the h5 writer (FeatureStoreDev.put).  Every entry is checked before the first put: image_size must be the
        image's declared size, D the set's descriptor_dim and N at most max_keypoints (ValueError otherwise)."""
        if self.extractor is not None:
            raise RuntimeError(f"put_features needs an ImageSetMatcher built with extractor=None, not {self.extractor!r}")
        if len(feats) != len(image_ids):
            raise ValueError(f"put_features needs one FeaturesDict per image id: {len(feats)} for {len(image_ids)} ids")
        for f, i in zip(feats, image_ids):
            k, d = np.asarray(f["keypoints"]), np.asarray(f["descriptors"])
            n = k.shape[0] if k.ndim == 2 and k.shape[1] == 2 else -1
            if n < 0:
                raise ValueError(f"image {i}: keypoints must be (N,2), got {k.shape}")
            if d.shape != (self.D, n):
                raise ValueError(f"image {i}: descriptors must be ({self.D},{n}) for descriptor_dim {self.D}, got {d.shape}")
            if n > self.cap:
                raise ValueError(f"image {i}: {n} keypoints, above max_keypoints={self.cap}")
            if f.get("scores") is not None and np.asarray(f["scores"]).shape != (n,):
                raise ValueError(f"image {i}: scores must be ({n},), got {np.asarray(f['scores']).shape}")
            size = np.asarray(f.get("image_size", ())).ravel()
            if size.shape != (2,) or tuple(int(v) for v in size) != tuple(self.sizes[i]) or np.any(size != np.round(size)):
                raise ValueError(f"image {i}: image_size must be its declared size {list(self.sizes[i])} ([H,W]), got {size.tolist()}")
        for f, i in zip(feats, image_ids):
            self.store.put(self.slots[i], f)

    def _extract_batch(self, src, ids, H, W, st):
        """Untiled extraction of the H x W images `src` (at most batch_images) of images `ids` into their slots: quality's resize, the
        extractor, put_dev, quality's rescale."""
        slots = [self.slots[i] for i in ids]
        h2, w2 = self.ext_sizes[ids[0]]
        src = self._resize(src, h2, w2, st)
        self._extract_rows(src, h2, w2, st)
        for k, s in enumerate(slots):
            scores = None if self.extractor in ("sift", "orb") else self.sc[k].data_ptr()  # no scores: the store writes ones
            self.store.put_dev(s, self.kp[k].data_ptr(), scores, self.de[k].data_ptr(), self.cap, self.cnt[k:k + 1].data_ptr(),
                               h2, w2, None, st)
        if self.extractor in ("sift", "orb"):
            counts = self.sift_counts if self.extractor == "sift" else self.orb_counts
            counts[self.torch.tensor(ids, device=self.cnt.device)] = self.cnt[:len(ids)]
        self._rescale(slots, H, W, st)

    def _extract_turned(self, d_images, image_ids, st):
        """Upright extraction: per original size, the images whose frame keeps that size (0, 180) come before those it swaps (90, 270),
        then batches of batch_images are staged (a view for consecutive rows of one tensor) and turned by one dimb_rot90_dev launch
        into one buffer of the batch, which therefore holds at most two runs of one frame size; each run goes to the extraction of a
        batch (untiled) or of cuts of its tile grid (tiled) as it is, without another copy.  Rotation 0 is copied too: one memory-bound
        pass is cheaper than the extra extractor call a third run would cost."""
        torch, C = self.torch, self.C
        px = (3,) if C == 3 else ()
        for (H, W), ks in self._groups(d_images, image_ids, self.sizes):
            ks = sorted(ks, key=lambda k: self.rotations[image_ids[k]] in (90, 270))  # stable: image order kept in each run
            for b0 in range(0, len(ks), self.B):
                part = ks[b0:b0 + self.B]
                ids = [image_ids[k] for k in part]
                buf = torch.empty(len(part) * H * W * C, device=self.kp.device)
                self.ctx.rot90_dev(self._stage(d_images, part).data_ptr(), len(part), H, W, C, [self.rotations[i] for i in ids],
                                   buf.data_ptr(), st)
                n0 = sum(self.rotations[i] in (0, 180) for i in ids)
                for a, b, (h, w) in ((0, n0, (H, W)), (n0, len(ids), (W, H))):
                    if a == b:
                        continue
                    run = buf[a * H * W * C:b * H * W * C].view((b - a, h, w) + px)
                    if self.tiling is None:
                        self._extract_batch(run, ids[a:b], h, w, st)
                        continue
                    G = max(1, self.B // self.tile_counts[ids[a]])
                    for g0 in range(0, b - a, G):
                        self._extract_cut(run[g0:g0 + G], ids[a + g0:a + g0 + G], h, w, st)

    def _batches(self, d_images, image_ids, groups, per):
        """Per size group, its batches of at most `per` images in order: ((H, W), their image ids, the images staged as one tensor)."""
        for size, ks in groups:
            for b0 in range(0, len(ks), per):
                yield size, [image_ids[k] for k in ks[b0:b0 + per]], self._stage(d_images, ks[b0:b0 + per])

    def _set_frames(self, frames):
        """The per-image sizes extraction sees, `frames` (the declared sizes, or with upright the rotated ones), and what follows from
        them: ``ext_sizes`` after quality, and with tiling ``tile_counts`` and ``view_offsets``."""
        self.frames = list(frames)
        self.ext_sizes = [self._ext[s] for s in self.frames]
        if self.tiling is not None:
            self.tile_counts = [len(self._grids[s]["origins"]) for s in self.frames]
            self.view_offsets = [int(v) for v in np.cumsum([0] + self.tile_counts[:-1])]

    def _groups(self, d_images, image_ids, sizes=None):
        """This rank's images grouped by size: [((H, W), positions in image_ids)] (``_by_size``), after checking every image's shape
        against its size in `sizes` (default: ``frames``, the declared sizes unless upright has rotated them)."""
        sizes = self.frames if sizes is None else sizes
        listed = isinstance(d_images, (list, tuple))
        if (len(d_images) != len(image_ids)) if listed else (d_images.dim() < 3 or len(d_images) < len(image_ids)):
            raise ValueError(f"extract needs one image per image id: {len(d_images)} images for {len(image_ids)} ids")
        for k, i in enumerate(image_ids):
            want = sizes[i] + ((3,) if self.C == 3 else ())
            got = tuple(d_images[k].shape) if listed else tuple(d_images.shape[1:1 + len(want)])
            if got != want or (listed and (d_images[k].dtype != self.torch.float32 or not d_images[k].is_cuda)):
                raise ValueError(f"image {i} must be a float32 CUDA tensor of shape {want} (its declared size), got {tuple(d_images[k].shape)}")
        return _by_size([sizes[i] for i in image_ids], range(len(image_ids)))

    def _stage(self, d_images, ks):
        """The images at positions `ks` of `d_images` as one contiguous (len(ks), H, W[, 3]) tensor: a view when they are consecutive
        rows of one tensor, a copy otherwise."""
        if isinstance(d_images, (list, tuple)):
            return self.torch.stack([d_images[k] for k in ks])
        if ks[-1] - ks[0] == len(ks) - 1:
            return d_images[ks[0]:ks[0] + len(ks)]
        return d_images[ks]

    def _resize(self, images, h2, w2, st):
        """The images to extract from: `images` itself at quality "high", otherwise their pyramid steps (h2 x w2) in self.resized."""
        if not self.level:
            return images
        k, H, W = images.shape[:3]
        out = self.resized[:k * h2 * w2 * self.C].view((k, h2, w2) + ((3,) if self.C == 3 else ()))
        self.ctx.pyr_dev(images.data_ptr(), k, H, W, self.C, self.level, out.data_ptr(), st)
        return out

    def _rescale(self, slots, H, W, st):
        """_resize_features on the slots just filled from resized H x W images (nothing at quality "high")."""
        if self.level:
            self.store.rescale_dev(slots, self.level, H, W, st)

    def _extract_rows(self, src, h, w, st):
        """The configured extractor on the len(src) h x w images or tiles of `src` into rows [0, len(src)) of kp / sc / de / cnt:
        SuperPoint, SIFT and ORB in calls of at most batch_images, ALIKED one per call."""
        step = 1 if self.extractor == "aliked" else self.B
        for r in range(0, len(src), step):
            if self.extractor in ("sift", "orb"):
                net = self.sift if self.extractor == "sift" else self.orb
                net.extract_dev(src[r].data_ptr(), min(step, len(src) - r), h, w, self.kp[r].data_ptr(), self.de[r].data_ptr(),
                                self.cnt[r:].data_ptr(), self.cap, stream=st)
                continue
            ptrs = (self.kp[r].data_ptr(), self.sc[r].data_ptr(), self.de[r].data_ptr(), self.cnt[r:].data_ptr(), self.cap, st)
            if self.extractor == "superpoint":
                self.sp.extract_dev(src[r].data_ptr(), min(step, len(src) - r), h, w, *ptrs)
            else:
                self.al.extract_dev(src[r].data_ptr(), h, w, 3, *ptrs)

    def _extract_tiled(self, d_images, image_ids, groups, st):
        """Per size group (its own grid of T tiles), cuts of G = max(1, batch_images // T) images: tile cut, the extractor over their
        G * T tiles, one tile merge into their slots."""
        for (H, W), ks in groups:
            G = max(1, self.B // self.tile_counts[image_ids[ks[0]]])
            for g0 in range(0, len(ks), G):
                self._extract_cut(self._stage(d_images, ks[g0:g0 + G]), [image_ids[k] for k in ks[g0:g0 + G]], H, W, st)

    def _extract_cut(self, src, ids, H, W, st):
        """One cut of the H x W images `src` (at most G of them) of images `ids`: quality's resize, tile cut, the extractor over their
        tiles, one tile merge into their slots, quality's rescale."""
        (th, tw), (oh, ow) = self.tiling["tile_hw"], self.tiling["overlap_hw"]
        (h2, w2), T = self.ext_sizes[ids[0]], self.tile_counts[ids[0]]
        src = self._resize(src, h2, w2, st)
        self.ctx.tile_cut_dev(src.data_ptr(), len(ids), h2, w2, self.C, th, tw, oh, ow, self.tiles.data_ptr(), st)
        self._extract_rows(self.tiles[:len(ids) * T], th, tw, st)
        slots = [self.slots[i] for i in ids]
        self.store.tile_merge_dev(slots, h2, w2, th, tw, oh, ow, self.kp.data_ptr(), self.sc.data_ptr(), self.de.data_ptr(),
                                  self.cnt.data_ptr(), self.cap, st)
        self._rescale(slots, H, W, st)

    def exchange(self):
        """The collective of the path: every rank's float16 feature blocks to every rank (NCCL all_gather over NVLink).  With tiling,
        every rank then builds the per-tile views of all images from the merged slots.  With upright the low-resolution sets were
        exchanged by ``upright``."""
        if self.extractor == "sift":
            self._check_sift_counts()
        if self.extractor == "orb":
            self._check_counts(self.orb_counts, "ORB", f"n_features + orb_tie_room(n_features) = {self.cap}")
        self.exchanged_bytes = all_gather_blocks(self.store_t, self.n, self.dist)
        if self.up is None:
            self.exchanged_bytes += self._exchange_lows((self.pre, self.lowres))
        if self.tiling is not None:
            st = self.torch.cuda.current_stream().cuda_stream
            for _, images in _by_size(self.frames, range(self.n)):
                T = self.tile_counts[images[0]]
                step = max(1, 65535 // T)
                for b0 in range(0, len(images), step):
                    ids = images[b0:b0 + step]
                    self.store.tile_views_dev([self.slots[i] for i in ids], T, self.views, [self.view_offsets[i] for i in ids],
                                              self.vmap.data_ptr(), st)

    def _check_sift_counts(self):
        """A SIFT store holds n_features + SIFT_TIE_ROOM rows per image; retainBest's boundary ties rarely add more than a few.  An
        image with more keypoints than that (or with more extrema than the extractor's candidate buffers hold, count -1) is an error,
        raised here before the exchange, never a silent cut."""
        self._check_counts(self.sift_counts, "SIFT", f"n_features + {SIFT_TIE_ROOM} = {self.cap}",
                           "more extrema than the SIFT candidate buffers hold")

    def _check_counts(self, counts, name, rows, negative="a failed extraction (count -1)"):
        """Raises RuntimeError for the first image whose true keypoint count is negative or above the store's rows."""
        counts = counts.cpu().tolist()
        bad = [(i, c) for i, c in enumerate(counts) if c < 0 or c > self.cap]
        if bad:
            i, c = bad[0]
            what = negative if c < 0 else f"{c} {name} keypoints, above the store's {rows} rows"
            raise RuntimeError(f"image {i}: {what}")

    def _exchange_lows(self, lows) -> int:
        """The low-resolution features of every image, for any pair: one all_gather per buffer of each set in `lows` (None skipped; a
        slot's four search entries travel together).  Returns the bytes received."""
        received = 0
        for low in lows:
            if low is not None:
                for t in low.buffers:
                    received += all_gather_blocks(t.view(self.torch.uint8).view(t.shape[0] // low.E, -1), self.n, self.dist)
        return received

    def _match_slots(self, store, s0, s1, st):
        """Enqueue the matcher on slot pairs (s0[k], s1[k]) of `store` (outputs in self.m / self.ms / self.nm)."""
        if self.matcher == "superglue":
            self.sg.match_dev([store.sg_feats_dev(s) for s in s0], [store.sg_feats_dev(s) for s in s1], self.m.data_ptr(), self.ms.data_ptr(),
                              self.nm.data_ptr(), self.cap, st)
        elif self.matcher == "kornia_matcher":  # distances / ratios go to ms
            self.ctx.nn_match_batch_dev([store.feats_dev(s) for s in s0], [store.feats_dev(s) for s in s1], self.D, self.nn_conf["match_mode"],
                                        self.nn_conf["th"], self.m.data_ptr(), self.ms.data_ptr(), self.nm.data_ptr(), self.cap, st)
        elif self.matcher == "lighterglue":  # LighterGlueMatcher's [H,W] -> [W,H] swap of image_size, as explicit sizes
            by_slot = {self.slots[i]: i for i in range(self.n)}
            f0 = [store.feats_dev(s, size=self.sizes[by_slot[s]][::-1]) for s in s0]
            f1 = [store.feats_dev(s, size=self.sizes[by_slot[s]][::-1]) for s in s1]
            self.lg.match_dev(f0, f1, self.m.data_ptr(), self.ms.data_ptr(), self.nm.data_ptr(), self.sl.data_ptr(), self.cap, st)
        else:
            self.lg.match_dev([store.feats_dev(s) for s in s0], [store.feats_dev(s) for s in s1], self.m.data_ptr(), self.ms.data_ptr(),
                              self.nm.data_ptr(), self.sl.data_ptr(), self.cap, st)

    def _preselect(self, pairs):
        """PRESELECTION tile-pair lists of `pairs` (tiling.preselection_matches + tiling.tile_selection): per batch of batch_pairs,
        LightGlue on the low-resolution slots and the tile box count (dimb_tile_preselect_pairs_dev, each pair with both images' sizes
        and scales), then ONE device->host copy of every pair's flags.  Pair (i, j) has a row-major T_i x T_j block of flags, which
        gives its list sorted.  Memory: the flags take sum(T_i * T_j) bytes over the pairs on the device and again on the host, and the
        counts of one batch (allocated with the matcher) batch_pairs * max(T)^2 int32; at T in the tens that is kilobytes per pair, but
        at hundreds of tiles per image it reaches megabytes per pair, so a very large pair list is better matched in several calls."""
        st = self.torch.cuda.current_stream().cuda_stream
        T, pre = self.tile_counts, self.pre
        (th, tw), (oh, ow) = self.tiling["tile_hw"], self.tiling["overlap_hw"]
        offsets = np.cumsum([0] + [T[i] * T[j] for i, j in pairs])
        flags = self.torch.zeros(max(int(offsets[-1]), 1), dtype=self.torch.uint8, device=self.pre_cnt.device)
        for b0 in range(0, len(pairs), self.P):
            chunk = pairs[b0:b0 + self.P]
            f0, f1 = pre.match([self.slots[i] for i, _ in chunk], [self.slots[j] for _, j in chunk], st)
            self.ctx.tile_preselect_pairs_dev(f0, f1, pre.m.data_ptr(), pre.nm.data_ptr(), pre.K, [self.sizes[i] + self.sizes[j] for i, j in chunk],
                                              th, tw, oh, ow, [(pre.scales[i], pre.scales[j]) for i, j in chunk],
                                              self.tiling["min_matches_per_tile"], self.pre_cnt.data_ptr(), flags[int(offsets[b0]):].data_ptr(), st)
        fl = flags.cpu().numpy()
        return [[(int(a), int(b)) for a, b in zip(*np.nonzero(fl[offsets[q]:offsets[q + 1]].reshape(T[i], T[j])))]
                for q, (i, j) in enumerate(pairs)]

    def _tile_pair_lists(self, pairs, tile_pairs):
        T = self.tile_counts
        if tile_pairs is None:
            if self.presel:
                return self._preselect(pairs)
            lists = {}  # one list per pair of tile counts
            return [lists.setdefault((T[i], T[j]), tile_pairs_for(self.tiling["tile_selection"], T[i], T[j])) for i, j in pairs]
        if len(tile_pairs) != len(pairs):
            raise ValueError(f"tile_pairs must hold one list per image pair: {len(tile_pairs)} lists for {len(pairs)} pairs")
        lists = []
        for (i, j), lst in zip(pairs, tile_pairs):
            lst = [(int(a), int(b)) for a, b in lst]
            if any(not (0 <= a < T[i] and 0 <= b < T[j]) for a, b in lst):
                raise ValueError(f"tile indices of image pair ({i}, {j}) must lie in [0, {T[i]}) x [0, {T[j]})")
            lists.append(lst)
        return lists

    def _enqueue_match(self, chunk, lists, st):
        """Enqueue the matcher on the image pairs `chunk` and return where it leaves their tables: (tables, counts, capacity).
        Untiled: the store slots, (m, nm, cap).  Tiled: the tile pairs `lists` out of the views (view_offsets[i] + t), then the
        tile-pair match merge, (mm, nmm, cap2)."""
        if lists is None:
            self._match_slots(self.store, [self.slots[i] for i, _ in chunk], [self.slots[j] for _, j in chunk], st)
            return self.m, self.nm, self.cap
        off = self.view_offsets
        v0 = [off[i] + a for (i, _), lst in zip(chunk, lists) for a, _ in lst]
        v1 = [off[j] + b for (_, j), lst in zip(chunk, lists) for _, b in lst]
        if v0:
            self._match_slots(self.views, v0, v1, st)
        offsets = np.concatenate([[0], np.cumsum([len(lst) for lst in lists])])
        self.ctx.tile_match_merge_dev(offsets, v0, v1, self.vmap.data_ptr(), self.views.cap, self.m.data_ptr(), self.nm.data_ptr(), self.cap,
                                      self.mm.data_ptr(), self.nmm.data_ptr(), self.cap2, st)
        return self.mm, self.nmm, self.cap2

    def _read_back(self, tables, extras, Q, stream):
        """Host copies of the first Q entries of a batch in two synchronising steps: the counts of every (tables, counts, capacity) in
        `tables` together with the `extras` tensors, then only the rows in use of each table, [:Q, :max(min(count, capacity))].
        The copies of a step are non-blocking (into pinned memory from torch's host allocator), so each step ends in one synchronise.
        Returns (per table, its Q arrays; the extras as numpy)."""
        first = [t[:Q].to("cpu", non_blocking=True) for t in [nm for _, nm, _ in tables] + list(extras)]
        stream.synchronize()
        counts = [np.minimum(h.numpy(), cap) for h, (_, _, cap) in zip(first, tables)]
        rows = [m[:Q, :int(n.max(initial=0))].to("cpu", non_blocking=True) for (m, _, _), n in zip(tables, counts)]
        stream.synchronize()
        return ([[h[k, :n[k]].copy() for k in range(Q)] for h, n in zip((r.numpy() for r in rows), counts)],
                [h.numpy() for h in first[len(tables):]])

    def _match_batches(self, pairs, pair_ids, tile_pairs, verify):
        """Phase 2 of ``match`` and, with `verify`, of ``match_verified``: per batch of image pairs the matcher, then with `verify`
        dimb_gv_verify_dev on its tables (same stream, keypoints from the store's slots), then ``_read_back``.  Untiled, every image
        pair is one unit of a batch; tiled, its tile pairs are."""
        from .geometric_verification import gv_seed
        if self.tiling is None and tile_pairs is not None:
            raise ValueError("tile_pairs needs an ImageSetMatcher built with tiling")
        if self.up is not None:
            if tile_pairs is not None:
                raise ValueError("explicit tile_pairs cannot be used with upright: the tile grids depend on the rotations the search picks")
            if self._turned_back:
                raise RuntimeError("the keypoints were rotated back (rotate_back); matching runs in the rotated frames, before it")
        stream = self.torch.cuda.current_stream()
        lists = None if self.tiling is None else self._tile_pair_lists(pairs, tile_pairs)
        g, out = self.gv, {}
        for s, e in pack_tile_batches([1] * len(pairs) if lists is None else [len(lst) for lst in lists], self.P):
            chunk, ids = pairs[s:e], pair_ids[s:e]
            m, nm, cap = self._enqueue_match(chunk, None if lists is None else lists[s:e], stream.cuda_stream)
            if not verify:
                (raw,), _ = self._read_back([(m, nm, cap)], (), e - s, stream)
                out.update(zip(ids, raw))
            else:
                f0 = [self.store.feats_dev(self.slots[i]) for i, _ in chunk]
                f1 = [self.store.feats_dev(self.slots[j]) for _, j in chunk]
                self.ctx.gv_verify_dev(f0, f1, m.data_ptr(), nm.data_ptr(), cap, [gv_seed(g["seed"], k) for k in ids], g["threshold"],
                                       g["max_iters"], g["min_inliers_per_pair"], g["min_inlier_ratio_per_pair"], self.v.data_ptr(),
                                       self.nv.data_ptr(), self.F.data_ptr(), self.mask.data_ptr(), self.ninl.data_ptr(), stream.cuda_stream,
                                       g["estimator"], g["confidence"])
                (raw, ver), (F, ninl) = self._read_back([(m, nm, cap), (self.v, self.nv, cap)], (self.F, self.ninl), e - s, stream)
                for k, (i, (a, b)) in enumerate(zip(ids, chunk)):
                    Fk = F[k].reshape(3, 3).copy() if np.any(F[k]) else None
                    if self.up is not None:  # F of the rotated frames -> original pixels
                        from .upright import rotate_back_F
                        Fk = rotate_back_F(Fk, self.rotations[a], self.sizes[a], self.rotations[b], self.sizes[b])
                    out[i] = (raw[k], ver[k], Fk, int(ninl[k]))
        return out

    def match(self, pairs, pair_ids, tile_pairs=None):
        """Phase 2: the configured matcher on `pairs` = [(i, j), ...] (this rank's share); returns {pair id: int64 (S,2)}.  Each pair
        batch comes back in two synchronising steps: the counts, then only the table rows in use.  Features are read in place from the
        store (float16, no rounding left to do).  Tiled: the tables are the merged image-pair tables; `tile_pairs` optionally gives
        each pair's list of (t0, t1)."""
        return self._match_batches(pairs, pair_ids, tile_pairs, verify=False)

    def match_verified(self, pairs, pair_ids, tile_pairs=None):
        """Phase 2 with geometric verification: returns {pair id: (raw int64 (S,2), verified int64 (V,2), F (3,3) float32 or None,
        n_inliers)}.  Per batch the matcher and dimb_gv_verify_dev are enqueued on the same stream, and the results come back in two
        synchronising steps: the raw and verified counts with F and n_inliers, then only the rows in use of both tables.  Tiled: the
        merged tables are verified against the merged slots."""
        if self.gv is None:
            raise RuntimeError("ImageSetMatcher was built without verification")
        if self.gv["method"] == "NONE":  # the reference skips the estimator: verified = raw, no F
            return {k: (m, m.copy(), None, len(m)) for k, m in self.match(pairs, pair_ids, tile_pairs).items()}
        return self._match_batches(pairs, pair_ids, tile_pairs, verify=True)

    def lowres_pairs(self):
        """Pair generation "matching_lowres" (pairs_generator.pairs_from_lowres) on the low-resolution features, after ``exchange``.
        The brute-force pairs (i < j, pairs_from_bruteforce order) are dealt by their keypoint products (one small device->host copy of
        the counts), LightGlue runs on this rank's share per batch of batch_pairs, each batch's match counts are copied into one device
        array without a host synchronise, and one device->host copy and an all_gather give every rank all counts.  Returns
        (pairs, counts), the same on every rank: the pairs with more than ``min_matches`` matches, and the count of every brute-force
        pair.  Memory: the low-resolution set holds (256 + 2) * 4 * 2048 bytes, about 2.1 MB, per image on every rank (2 GB at 1000
        images)."""
        from .pairs_generator import pairs_from_bruteforce
        if self.lowres is None:
            raise RuntimeError("ImageSetMatcher was built without pair_generation")
        torch, low = self.torch, self.lowres
        st = torch.cuda.current_stream().cuda_stream
        brute = pairs_from_bruteforce(range(self.n))
        n = low.n.cpu().numpy()[self.slots].astype(np.int64)
        mine = shard_pairs(len(brute), self.world, self.rank, [n[i] * n[j] for i, j in brute])
        counts = torch.zeros(max(len(mine), 1), dtype=torch.int32, device=low.nm.device)
        for b0 in range(0, len(mine), self.P):
            chunk = [brute[k] for k in mine[b0:b0 + self.P]]
            low.match([self.slots[i] for i, _ in chunk], [self.slots[j] for _, j in chunk], st)
            counts[b0:b0 + len(chunk)].copy_(low.nm[:len(chunk)])
        counts = gather_pair_counts(mine, counts[:len(mine)].cpu().numpy(), len(brute), self.dist if self.world > 1 else None,
                                    torch.device("cuda", self.ctx.device) if self.world > 1 else None)
        return [p for p, c in zip(brute, counts) if c > self.pairgen["min_matches"]], counts

    def run_lowres(self, d_images, my_image_ids, verified: bool = False):
        """extract -> exchange -> ``lowres_pairs`` -> ``match`` (``match_verified`` with `verified`) on this rank's share of the kept
        pairs -> gather to rank 0.  Returns (pairs, counts, results): the kept pairs and every brute-force pair's count on every rank,
        and on rank 0 the results per kept pair as ``run`` / ``run_verified`` return them (None elsewhere).  With tiling, the configured
        tile selection applies to the kept pairs."""
        match, gather = (self.match_verified, gather_verified) if verified else (self.match, gather_match_tables)
        if self.up is not None:  # pair generation reads the unrotated images, and the search runs over the kept pairs
            self._search_extract(d_images, my_image_ids)
            pairs, counts = self.lowres_pairs()
            self._search(pairs)
            self.extract(d_images, my_image_ids)
            self.exchange()
            return pairs, counts, self._match_share(match, gather, pairs, None, None)
        self.extract(d_images, my_image_ids)
        self.exchange()
        pairs, counts = self.lowres_pairs()
        return pairs, counts, self._match_share(match, gather, pairs, None, None)

    def upright(self, d_images, my_image_ids, pairs):
        """The upright search (find_matches_per_rotation, image_matching.py:69-118) over `pairs`, the schedule and rules of
        ``upright.upright_schedule`` / ``upright.upright_rotations``.  `d_images`: this rank's unrotated images, as ``extract`` takes them.

        Each rank resizes its images once (INTER_AREA, longest side ``resize_max``), turns each low-resolution image three ways
        (dimb_rot90_dev) and runs SuperPoint on all four turns (two calls per batch, one per shape) into four float32 entries per slot;
        the entries of every image then go to every rank (all_gather of about (256 + 2) * 4 * K * 4 bytes, 8.5 MB at K = 2048, per
        image).  Then wave by wave: the wave's decisions are dealt to the ranks (``shard_pairs``), LightGlue runs on the four entry
        pairs (reference at its rotation, target at each turn) of every decision in batches of batch_pairs, and one device->host copy
        of the counts and one ``gather_pair_counts`` give every rank the wave's counts, hence its rotations, which the next wave needs
        on the host.  So the search costs one host synchronise per wave: one for a brute-force list (everything hangs off image 0), up
        to n - 1 for a sequential chain.  This path runs SuperPoint 4 times per image, the reference 1 + 4 times per visited pair.

        Returns (rotations, counts), the same on every rank: the rotation of every image in degrees clockwise, and
        {(target, reference): [c_0, c_90, c_180, c_270]}; sets ``rotations``.  Afterwards ``extract`` takes the same unrotated images."""
        self._search_extract(d_images, my_image_ids)
        return self._search(pairs)

    def _search_extract(self, d_images, my_image_ids):
        """One staging pass over the unrotated images for the low-resolution work (the search entries, and the pair-generation set when
        configured), then their exchange."""
        if self.up is None:
            raise RuntimeError("ImageSetMatcher was built without upright")
        st = self.torch.cuda.current_stream().cuda_stream
        lows = [low for low in (self.lowres, self.search) if low is not None]
        for _, ids, src in self._batches(d_images, my_image_ids, self._groups(d_images, my_image_ids, self.sizes), self.B):
            for low in lows:
                low.extract(src, ids, [self.slots[i] for i in ids], st)
        self.exchanged_bytes = self._exchange_lows(lows)

    def _search(self, pairs):
        """The waves of ``upright_schedule(pairs)`` on the exchanged search entries (``upright``)."""
        from .upright import ROTATIONS, rotated_size
        torch, low = self.torch, self.search
        st = torch.cuda.current_stream().cuda_stream

        def count(decisions, rotations):  # LightGlue on the four entry pairs of each decision, counts copied on the device
            e0 = [4 * self.slots[a] + ROTATIONS.index(rotations[a]) for _, a in decisions for _ in ROTATIONS]
            e1 = [4 * self.slots[t] + r for t, _ in decisions for r in range(4)]
            got = torch.zeros(max(len(e0), 1), dtype=torch.int32, device=low.nm.device)
            for b0 in range(0, len(e0), self.P):
                q = len(e0[b0:b0 + self.P])
                low.match(e0[b0:b0 + q], e1[b0:b0 + q], st)
                got[b0:b0 + q].copy_(low.nm[:q])
            return got[:len(e0)].cpu().numpy()
        rotations, counts = upright_waves(pairs, self.n, count, self.dist if self.world > 1 else None,
                                          torch.device("cuda", self.ctx.device) if self.world > 1 else None)
        self.rotations = rotations
        self._set_frames([rotated_size(h, w, r) for (h, w), r in zip(self.sizes, rotations)])
        return rotations, counts

    def rotate_back(self):
        """Upright, after matching: the keypoints of every slot with a non-zero rotation back on its original image, and the original
        size in its header (one dimb_fstore_unrotate_dev launch; quality's rescale has already put them in the rotated full-size
        frame).  ``tile_idx`` keeps the indices of the rotated image's tile grid.  ``match`` / ``match_verified`` refuse to run after it."""
        if self.up is None or self.rotations is None:
            raise RuntimeError("rotate_back needs an ImageSetMatcher built with upright, after upright()")
        if self._turned_back:
            return
        turned = [i for i in range(self.n) if self.rotations[i]]
        if turned:
            self.store.unrotate_dev([self.slots[i] for i in turned], [self.rotations[i] for i in turned], [self.sizes[i][0] for i in turned],
                                    [self.sizes[i][1] for i in turned], self.torch.cuda.current_stream().cuda_stream)
        self._turned_back = True

    def _run(self, match, gather, d_images, my_image_ids, pairs, costs, tile_pairs):
        """extract -> exchange -> `match` on this rank's share of `pairs` -> `gather` to rank 0 (upright: the search first, and the
        keypoints rotated back before the gather)."""
        if self.up is not None:
            if tile_pairs is not None:
                raise ValueError("explicit tile_pairs cannot be used with upright: the tile grids depend on the rotations the search picks")
            self.upright(d_images, my_image_ids, pairs)
        self.extract(d_images, my_image_ids)
        self.exchange()
        return self._match_share(match, gather, pairs, costs, tile_pairs)

    def _match_share(self, match, gather, pairs, costs, tile_pairs):
        mine = shard_pairs(len(pairs), self.world, self.rank, costs)
        res = match([pairs[k] for k in mine], mine, None if tile_pairs is None else [tile_pairs[k] for k in mine])
        if self.up is not None:
            self.rotate_back()
        return gather(mine, [res[k] for k in mine], len(pairs), self.dist if self.world > 1 else None,
                      self.torch.device("cuda", self.ctx.device) if self.world > 1 else None)

    def run(self, d_images, my_image_ids, pairs, costs=None, tile_pairs=None):
        """extract -> exchange -> match my share -> gather to rank 0.  Returns the list of match tables on rank 0 (None elsewhere).
        tile_pairs (tiled only): per pair of `pairs`, its list of (t0, t1)."""
        return self._run(self.match, gather_match_tables, d_images, my_image_ids, pairs, costs, tile_pairs)

    def run_verified(self, d_images, my_image_ids, pairs, costs=None, tile_pairs=None):
        """extract -> exchange -> match and verify my share -> gather to rank 0.  Returns, on rank 0, the list of
        (raw, verified, F, n_inliers) per pair (None elsewhere); ``export_colmap`` turns it into a COLMAP database."""
        return self._run(self.match_verified, gather_verified, d_images, my_image_ids, pairs, costs, tile_pairs)

    def run_features(self, feats, my_image_ids, pairs, costs=None):
        """``run`` with given features: put_features -> exchange -> match my share -> gather to rank 0."""
        self.put_features(feats, my_image_ids)
        self.exchange()
        return self._match_share(self.match, gather_match_tables, pairs, costs, None)

    def run_features_verified(self, feats, my_image_ids, pairs, costs=None):
        """``run_verified`` with given features: put_features -> exchange -> match and verify my share -> gather to rank 0."""
        self.put_features(feats, my_image_ids)
        self.exchange()
        return self._match_share(self.match_verified, gather_verified, pairs, costs, None)

    def export_colmap(self, pairs, results, database_path, image_names=None, **kwargs) -> dict:
        """Rank 0: the COLMAP database of this image set (``export_verified_to_colmap`` on this matcher's feature store)."""
        return export_verified_to_colmap(self.store, self.n, self.world, pairs, results, database_path, image_names, **kwargs)
