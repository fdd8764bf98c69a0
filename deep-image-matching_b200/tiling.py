"""Tiling geometry and tile-pair selection around the hot path (the callers of ``_extract`` / ``_match_pairs`` when
``tile_selection != NONE``): mirror of the reference's ``utils/tiling.py:63-192`` (``Tiler.compute_tiles_by_size``) and
``matchers/matcher_base.py:989-1342`` (``tile_selection``), ``:1380-1413`` (helpers).

Only the geometry is restated (it is pure numpy in the reference too, apart from one kornia call); the two networks the
PRESELECTION mode runs on the down-sampled images - SuperPoint (hloc wrapper: ``fix_sampling=True``, ``nms_radius 5``,
``max_keypoints 4000``, ``keypoint_threshold 0.005``) and LightGlue (``depth 0.9 / width 0.95 / filter 0.3``, keypoints
normalised by their own extent because ``sp2lg`` passes no ``image_size``) ``matcher_base.py:143-159`` - run on libdimb200.
This host flow is the reference restated; ``ImageSetMatcher(tiling={..., "tile_selection": "preselection"})`` computes the same
lists on the device (``dimb_resize_area_dev``, ``dimb_kpts_extent_dev``, ``dimb_tile_preselect_dev``).

Reproduced quirk (SURVEY A.7): ``kornia.contrib.compute_padding`` is called without the stride (tiling.py:124), so the
padding assumes stride == window while the tiles are cut with stride ``window - overlap``: with an overlap the last
``overlap`` pixels of each padded axis are never visited (reference tests/test_tiling.py:91-122 pin exactly this).
"""
from __future__ import annotations

from itertools import product

import numpy as np

SP_PRESELECTION_CONF = {"nms_radius": 5, "max_keypoints": 4000, "keypoint_threshold": 0.005, "remove_borders": 4,
                        "fix_sampling": True}  # matcher_base.py:144-148 through the hloc-style wrapper (extractors/superpoint.py:31-37)
LG_PRESELECTION_CONF = {"n_layers": 9, "depth_confidence": 0.9, "width_confidence": 0.95, "filter_threshold": 0.3}  # :149-156


def compute_padding(original_size, window_size):
    """kornia.contrib.compute_padding (0.8.1, pinned by the reference's uv.lock) with stride = window: (top, bottom, left, right)
    making ``(size - window) % window == 0``, split evenly with the odd pixel at the bottom / right."""
    out = []
    for size, win in zip(original_size, window_size):
        rem = (size - win) % win
        pad = (win - rem) if rem else 0
        out += [pad // 2, pad - pad // 2]
    return tuple(out)


def _hw(v):
    """window_size / overlap as given by DIM's config are (x, y); the Tiler transposes them to (H, W) (tiling.py:96-111)."""
    if isinstance(v, int):
        return (v, v)
    return (int(v[1]), int(v[0]))


def compute_tiles_by_size(image: np.ndarray, window_size, overlap=0):
    """Tiler.compute_tiles_by_size: returns ({idx: tile (h,w[,C])}, {idx: (x, y) origin in the un-padded image}, padding)."""
    win, ov = _hw(window_size), _hw(overlap)
    arr = image if image.ndim == 3 else image[:, :, None]
    H, W = arr.shape[:2]
    pad = compute_padding((H, W), win)
    stride = [w - o for w, o in zip(win, ov)]
    padded = np.pad(arr, ((pad[0], pad[1]), (pad[2], pad[3]), (0, 0)), mode="constant", constant_values=0)
    ph, pw = padded.shape[:2]
    tiles, k = {}, 0
    for y in range(0, ph - win[0] + 1, stride[0]):
        for x in range(0, pw - win[1] + 1, stride[1]):
            t = padded[y:y + win[0], x:x + win[1]]
            # the reference hands (H,W,C) patches to _extract; single-channel images come back as (H,W,1) (tiling.py:166-173)
            tiles[k] = t
            k += 1
    n_rows = (H + pad[0] + pad[1] - win[0]) // stride[0] + 1
    n_cols = (W + pad[2] + pad[3] - win[1]) // stride[1] + 1
    origins = {}
    for row in range(n_rows):
        for col in range(n_cols):
            origins[row * n_cols + col] = (-pad[2] + col * stride[1], -pad[0] + row * stride[0])
    return tiles, origins, pad


def get_tile_bounding_box(bottom_left, tile_size):
    return [bottom_left[0], bottom_left[1], bottom_left[0] + tile_size[0], bottom_left[1] + tile_size[1]]


def points_in_rect(points: np.ndarray, rect) -> np.ndarray:
    rect = np.asarray(rect)
    return np.all(points > rect[:2], axis=1) & np.all(points < rect[2:], axis=1)


def get_features_by_tile(features: dict, tile_idx: int):
    """matcher_base.py:1380-1391: the tile's features keep the FULL-image ``image_size`` (quirk A.3)."""
    if "tile_idx" not in features:
        raise KeyError("tile_idx not found in features")
    sel = features["tile_idx"] == tile_idx
    idx = np.where(sel)[0]
    return {"keypoints": features["keypoints"][sel], "descriptors": features["descriptors"][:, sel],
            "scores": features["scores"][sel], "image_size": features["image_size"]}, idx


def preselection_matches(i0: np.ndarray, i1: np.ndarray, tile_preselection_size: int, sp_net_factory, lg_net):
    """The network part of PRESELECTION (matcher_base.py:1054-1089): both gray images down-sampled so that the longest side is
    ``tile_preselection_size`` (INTER_AREA), SuperPoint on each, LightGlue without image_size, matched keypoints scaled back
    to full resolution.  ``sp_net_factory(H, W)`` returns a SuperPointNet able to take an (H,W) image."""
    import cv2
    kps, scales = [], []
    feats = []
    for im in (i0, i1):
        size = im.shape[:2][::-1]
        scale = tile_preselection_size / max(size)
        new = tuple(int(round(x * scale)) for x in size)
        low = cv2.resize(im, new, interpolation=cv2.INTER_AREA)
        f = sp_net_factory(low.shape[0], low.shape[1]).extract(np.ascontiguousarray(low, np.float32)[None])[0]
        feats.append({"keypoints": f["keypoints"], "descriptors": f["descriptors"], "_layout": 0})
        scales.append(scale)
    res = lg_net.match([(feats[0], feats[1])])[0]
    kp0 = feats[0]["keypoints"][res["matches"][:, 0]] / scales[0]
    kp1 = feats[1]["keypoints"][res["matches"][:, 1]] / scales[1]
    return kp0, kp1


def tile_selection(i0: np.ndarray, i1: np.ndarray, method: str, tile_size, tile_overlap: int, *, kp0=None, kp1=None,
                   min_matches_per_tile: int = 5):
    """``tile_selection`` (matcher_base.py:989-1342) on already loaded gray images.  ``method``: "exhaustive" (:1047-1050),
    "grid" (:1051-1054) or "preselection" (:1055-1148; ``kp0`` / ``kp1`` = :func:`preselection_matches`).  Returns the sorted
    list of (tile index in image 0, tile index in image 1)."""
    tiles0, orig0, _ = compute_tiles_by_size(i0, tile_size, tile_overlap)
    tiles1, orig1, _ = compute_tiles_by_size(i1, tile_size, tile_overlap)
    method = str(method).lower()
    if method == "exhaustive":
        return sorted(product(tiles0.keys(), tiles1.keys()))
    if method == "grid":
        return sorted(zip(tiles0.keys(), tiles1.keys()))
    if method != "preselection":
        raise NotImplementedError(f"tile selection method {method!r} (supported: exhaustive, grid, preselection)")
    if kp0 is None or kp1 is None:
        raise ValueError("preselection needs the matched low-resolution keypoints (preselection_matches)")
    pairs = set()
    for t0, t1 in sorted(product(tiles0.keys(), tiles1.keys())):
        in0 = points_in_rect(kp0, get_tile_bounding_box(orig0[t0], tile_size))
        in1 = points_in_rect(kp1, get_tile_bounding_box(orig1[t1], tile_size))
        if int(np.sum(in0 & in1)) > min_matches_per_tile:
            pairs.add((t0, t1))
    return sorted(pairs)
