"""Geometric verification on libdimb200 - the estimator of the reference's ``utils/geometric_verification.py:45-179`` on the GPU.

``geometric_verification(kpts0, kpts1, method, threshold, confidence, max_iters)`` keeps the reference's signature and return
contract ``(F, inlMask)``: ``F`` a (3,3) fundamental matrix or ``None``, ``inlMask`` a boolean array over the correspondences;
method NONE returns ``(None, all True)`` (:100-101) and fewer than 8 matches return ``(None, all True)`` (:107-111).  Every other
method name of the reference (PYDEGENSAC, MAGSAC, RANSAC, the OpenCV USAC family) runs the estimator chosen by ``estimator``
(csrc/gv.cu), both seeded, with Sampson inliers and two least-squares refits of the final model:

- ``"ransac8"`` (the default): max(64, min(max_iters, 8192)) 8-point hypotheses, all evaluated in parallel; ``confidence`` is
  accepted and unused (no adaptive stopping).
- ``"lo-ransac"``: 7-point hypotheses in waves of 1024, local optimisation of each wave's new best model and confidence stopping
  (``confidence`` in (0, 1)), up to min(max_iters, 65536) hypotheses - the structure of pydegensac and OpenCV's USAC, which keeps
  the true inliers at outlier ratios where ransac8 loses them.
- ``"degensac"``: lo-ransac's waves plus DEGENSAC's handling of a dominant plane (Chum, Werner, Matas, CVPR 2005), the core of
  pydegensac: a 7-point sample with 5 or more points on one plane is detected by five H-from-F-and-3-points tests, its plane's H is
  scored (transfer error below 2 x threshold), and plane and parallax recovers F = [e']_x H from pairs of off-plane matches (up to
  1024 per step, with confidence stopping).  It keeps the off-plane inliers (the parallax SfM needs) that the other two lose on
  façades, floors and aerial views of flat ground, at a higher cost per pair on such scenes.

Like the reference's estimators the result is stochastic in the sense that it depends on the seed; parity is statistical
(tests/test_geometry.py, tests/test_gv_lo.py, tests/test_gv_degensac.py).
For image sets, ``gv_seed(seed, pair_id)`` is the seed of each pair, so that a pair's result does not depend on how the pair list is
batched or sharded (``sharded.ImageSetMatcher(verification=...)``).
"""
from __future__ import annotations

import numpy as np

METHODS = ("NONE", "PYDEGENSAC", "MAGSAC", "RANSAC", "LMEDS", "RHO", "USAC_DEFAULT", "USAC_PARALLEL", "USAC_FM_8PTS", "USAC_FAST",
           "USAC_ACCURATE", "USAC_PROSAC", "USAC_MAGSAC")


def method_name(method) -> str:
    """Upper-case name in METHODS of a method given as name, enum member or index; ValueError otherwise."""
    name = getattr(method, "name", method)
    if isinstance(name, int):
        name = METHODS[name] if 0 <= name < len(METHODS) else None
    if not isinstance(name, str) or name.upper() not in METHODS:
        raise ValueError(f"Invalid Geometry Verification method. It must be one of {list(METHODS)}")
    return name.upper()


def gv_seed(seed: int, pair_id: int) -> int:
    """RNG seed (uint32) of pair `pair_id` of a pair list verified with base seed `seed`.

    A pure function of the two integers (both taken modulo 2**32): a pair's verification result depends on its global id in the
    pair list, never on the batch it was verified in or the rank that verified it.  The mix is the 32-bit "lowbias32" finaliser of
    ``seed * 0x9E3779B1 + (pair_id + 1) * 0x85EBCA77`` (mod 2**32)."""
    m = 0xFFFFFFFF
    h = ((int(seed) & m) * 0x9E3779B1 + (((int(pair_id) & m) + 1) & m) * 0x85EBCA77) & m
    h ^= h >> 16
    h = (h * 0x7FEB352D) & m
    h ^= h >> 15
    h = (h * 0x846CA68B) & m
    h ^= h >> 16
    return h


def geometric_verification(kpts0: np.ndarray = None, kpts1: np.ndarray = None, method="pydegensac", threshold: float = 1, confidence: float = 0.9999,
                           max_iters: int = 10000, quiet: bool = False, device: int = 0, seed: int = 0, estimator: str = "ransac8", **kwargs):
    from . import _native
    name = method_name(method)
    _native.gv_estimator(estimator)
    n = len(kpts0)
    if name == "NONE" or n < 8:
        return None, np.ones(n, dtype=bool)
    F, mask, _ = _native.Context.get(device).gv_estimate(kpts0, kpts1, threshold, max_iters, seed, estimator, confidence)
    return F, mask
