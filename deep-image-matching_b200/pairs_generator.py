"""Pair generation on libdimb200 - the part of the reference's ``pairs_generator.py`` that runs the hot path
(src/deep_image_matching/pairs_generator.py:22-235): ``pairs_from_sequential`` (:22-34), ``pairs_from_bruteforce``
(:36-37) and ``pairs_from_lowres`` (:40-235), which extracts SuperPoint features from down-sampled images and runs
LightGlue over *all* n(n-1)/2 pairs to keep those with more than ``min_matches`` matches.

Here the n images are extracted once (batched when equally sized) and the pairs go through LightGlue in batches;
the reference does one image / one pair per call with a host synchronisation after each.

Reproduced details: SuperPoint through the hloc wrapper, i.e. ``fix_sampling=True`` (thirdparty/hloc/extractors/
superpoint.py:25-31) with ``nms_radius 3, max_keypoints 2048, keypoint_threshold 0.0005`` (:108-116); LightGlue with
``n_layers 7, depth 0.9, width 0.95, filter 0.3`` (:117-126) called hloc-style *without* ``image_size`` so that keypoints
are normalised by their own extent (lightglue.py:26-27); ``use_superpoint`` is forced to True (:100); the KeyNet/AdaLAM
branch is therefore dead code in the reference and absent here; the pair is kept if ``len(matches) > min_matches``.

This host function serves images on disk; for an image set already on the device, of one size or of mixed sizes (per-image
``height`` / ``width``), ``ImageSetMatcher(pair_generation={"strategy": "matching_lowres", ...})`` gives the same pairs and counts
without leaving the device and across GPUs (``sharded.ImageSetMatcher.lowres_pairs``).
"""
from __future__ import annotations

from itertools import combinations
from pathlib import Path

import numpy as np

SP_LOWRES_CONF = {"nms_radius": 3, "max_keypoints": 2048, "keypoint_threshold": 0.0005, "remove_borders": 4, "fix_sampling": True}
LG_LOWRES_CONF = {"n_layers": 7, "depth_confidence": 0.9, "width_confidence": 0.95, "filter_threshold": 0.3}


def pairs_from_sequential(img_list, overlap: int) -> list:
    pairs = []
    for i in range(len(img_list)):
        for k in range(overlap):
            j = i + k + 1
            if j >= len(img_list):
                break
            pairs.append((img_list[i], img_list[j]))
    return pairs


def pairs_from_bruteforce(img_list) -> list:
    return list(combinations(img_list, 2))


def read_lowres(path, resize_max: int) -> np.ndarray:
    """pairs_generator.py:140-145: gray float32, longest side resized to ``resize_max`` with INTER_AREA."""
    import cv2
    i0 = cv2.imread(str(path), cv2.IMREAD_GRAYSCALE).astype(np.float32)
    size = i0.shape[:2][::-1]
    scale = resize_max / max(size)
    size_new = tuple(int(round(x * scale)) for x in size)
    return cv2.resize(i0, size_new, interpolation=cv2.INTER_AREA)


def gray_from_rgb(rgb) -> np.ndarray:
    """The gray image of an RGB image (H, W, 3), float32 0..255 as ALIKED sets hold them: the gray image the low-resolution passes of
    an ALIKED set (pair generation, tile preselection, the upright search) resize and run SuperPoint on.

    The reference reads those passes' images with ``cv2.IMREAD_GRAYSCALE``, which for JPEG returns the codec's own luma plane; that
    cannot be derived from the decoded RGB, so this project fixes the rule instead: each channel rounded half to even and clamped to
    0..255, then cv2.cvtColor RGB2GRAY, in integers ``(9798 R + 19235 G + 3735 B + 16384) >> 15``.  It is the luma with R first,
    unlike the gray images SuperPoint sets take, which carry the reference's BGR2GRAY-on-RGB order (SURVEY A.1).
    ``ImageSetMatcher`` applies the same rule on the device (dimb_resize_area_rgb_dev)."""
    import cv2
    return cv2.cvtColor(np.clip(np.rint(rgb), 0, 255).astype(np.uint8), cv2.COLOR_RGB2GRAY).astype(np.float32)


def pairs_from_lowres(img_list, resize_max: int = 1000, min_matches: int = 20, max_keypoints: int = 1024,
                      use_superpoint: bool = True, do_geometric_verification: bool = False, *, lightglue_weights: dict | None = None,
                      superpoint_weights: dict | None = None, device: int = 0, pair_batch: int = 16,
                      images: dict | None = None, return_counts: bool = False):
    """``lightglue_weights``: state dict of ``superpoint_lightglue`` (the reference downloads it; offline it has to be
    given).  ``images``: optional ``{name: gray float32 array}`` already down-sampled (tests / callers that hold the
    pixels).  Returns the kept pairs (and, with ``return_counts``, the match count of every brute-force pair)."""
    import os

    from . import _native
    from .weights import from_torch_checkpoint, load_npz, superpoint_v1
    if lightglue_weights is None:  # same lookup as LightGlueMatcher (the reference downloads superpoint_lightglue.pth)
        path = os.environ.get("DIMB_LIGHTGLUE_WEIGHTS")
        if path is None:
            raise FileNotFoundError("superpoint_lightglue weights: pass lightglue_weights=<state dict> or set DIMB_LIGHTGLUE_WEIGHTS")
        lightglue_weights = load_npz(path) if str(path).endswith(".npz") else from_torch_checkpoint(path)
    if do_geometric_verification:
        raise NotImplementedError("geometric verification (pydegensac / OpenCV RANSAC) is outside the hot path")
    img_list = [Path(p) for p in img_list]
    brute_pairs = pairs_from_bruteforce(img_list)
    ctx = _native.Context.get(device)
    low = {p.name: (images[p.name] if images is not None else read_lowres(p, resize_max)) for p in img_list}
    # ---- extraction: equally sized images go through SuperPoint as one batch
    by_shape: dict = {}
    for name, im in low.items():
        by_shape.setdefault(im.shape, []).append(name)
    feats = {}
    for (H, W), names in by_shape.items():
        net = _native.SuperPointNet(ctx, superpoint_weights or superpoint_v1(), max_batch=len(names), max_height=H, max_width=W,
                                    **SP_LOWRES_CONF)
        for name, f in zip(names, net.extract(np.stack([low[n] for n in names]))):
            feats[name] = {"keypoints": f["keypoints"], "descriptors": f["descriptors"], "_layout": 0}  # (256,N), no image_size
        del net
    # ---- matching: every brute-force pair, ``pair_batch`` pairs per LightGlue call
    kmax = max([len(f["keypoints"]) for f in feats.values()] + [1])
    lg = _native.LightGlueNet(ctx, lightglue_weights, input_dim=256, max_pairs=min(pair_batch, max(len(brute_pairs), 1)), max_kpts=kmax,
                              **LG_LOWRES_CONF)
    counts = []
    for i in range(0, len(brute_pairs), pair_batch):
        chunk = brute_pairs[i:i + pair_batch]
        res = lg.match([(feats[a.name], feats[b.name]) for a, b in chunk])
        counts += [len(r["matches"]) for r in res]
    pairs = [pr for pr, c in zip(brute_pairs, counts) if c > min_matches]
    return (pairs, counts) if return_counts else pairs
