"""SIFTExtractor on libdimb200 - drop-in for the reference plugin (src/deep_image_matching/extractors/sift.py): same class name,
class attributes, config keys and ``_extract`` contract (uint8 (H,W) gray in - ``grayscale = True``, ``as_float = False``, since
cv2's SIFT refuses other depths - dict of numpy arrays out: keypoints (N,2) float32 as cv2.KeyPoint_convert gives them, descriptors
(128,N) float64 as ``des.astype(float).T`` gives them, no scores).  detectAndCompute runs in hand-written CUDA kernels (csrc/sift.cu)
instead of OpenCV on the host.

Differences from the reference:
- an image without keypoints returns empty arrays ((0,2) and (128,0)); the reference fails on cv2's ``None`` descriptors there;
- when ``n_features`` cuts, keypoints come in removeDuplicatedSorted's order (x, y ascending, then size descending, angle ascending,
  response descending, octave descending) instead of the order std::nth_element leaves in cv2's output.  The set of keypoints is
  cv2's, ties at the boundary response included.
``_default_conf`` holds the values of the sift+kornia_matcher pipeline in config.py; the reference plugin's own defaults are not
restated here.
"""
from __future__ import annotations

import numpy as np

from .. import _native
from ..config import confs
from .extractor_base import ExtractorBase

SIFT_KEYS = ("n_features", "nOctaveLayers", "contrastThreshold", "edgeThreshold", "sigma")


def sift_conf(cfg: dict) -> dict:
    """The SIFTExtractor keys of an extractor config as SiftNet keyword arguments."""
    return {"n_features": int(cfg["n_features"]), "n_octave_layers": int(cfg["nOctaveLayers"]),
            "contrast_threshold": float(cfg["contrastThreshold"]), "edge_threshold": float(cfg["edgeThreshold"]),
            "sigma": float(cfg["sigma"])}


class SIFTExtractor(ExtractorBase):
    _default_conf = {"name": "sift", **{k: confs["sift+kornia_matcher"]["extractor"][k] for k in SIFT_KEYS}}
    required_inputs = []
    grayscale = True
    as_float = False
    descriptor_size = 128

    def __init__(self, config: dict):
        super().__init__(config)
        self._conf = sift_conf(self.config["extractor"])
        self._ctx = _native.Context.get(int(self.config["general"].get("device", 0)))
        self._net = None
        self._net_shape = (0, 0)

    def _ensure(self, H, W):
        h, w = self._net_shape
        if self._net is None or H > h or W > w:
            self._net_shape = (max(H, h), max(W, w))
            self._net = _native.SiftNet(self._ctx, **self._conf, max_height=self._net_shape[0], max_width=self._net_shape[1])
        return self._net

    def _extract(self, image: np.ndarray) -> dict:
        image = np.asarray(image)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("SIFTExtractor takes a uint8 (H, W) gray image, as cv2.SIFT does")
        f = self._ensure(*image.shape).extract(image)
        return {"keypoints": f["keypoints"], "descriptors": f["descriptors"].astype(np.float64)}

    def _frame2tensor(self, image: np.ndarray, device: str = "cuda"):
        return image
