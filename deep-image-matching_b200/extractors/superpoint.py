"""SuperPointExtractor on libdimb200 - drop-in for the reference plugin
(src/deep_image_matching/extractors/superpoint.py:64-146): same class name, class attributes, config keys
and ``_extract`` contract (float32 (H,W) gray 0..255 in; dict of writable numpy arrays out: keypoints (N,2)
x,y, scores (N,), descriptors (256,N)).  The model arithmetic runs in hand-written sm_90a kernels
(csrc/superpoint.cu) instead of the MagicLeap torch graph.
"""
from __future__ import annotations

import numpy as np

from .. import _native
from ..config import Config
from ..weights import superpoint_v1
from .extractor_base import ExtractorBase


class SuperPointExtractor(ExtractorBase):
    _default_conf = {
        "name": "superpoint",
        "nms_radius": 4,
        "keypoint_threshold": 0.005,
        "max_keypoints": -1,
        "remove_borders": 4,
        "fix_sampling": False,
    }
    required_inputs = ["image"]
    grayscale = True
    descriptor_size = 256
    detection_noise = 2.0

    def __init__(self, config: Config):
        super().__init__(config)
        cfg = self.config["extractor"]
        self._ctx = _native.Context.get(int(self.config["general"].get("device", 0)))
        self._weights = cfg.get("weights_dict") or superpoint_v1()
        self._net = None
        self._net_shape = (0, 0, 0)

    def _ensure(self, B, H, W):
        b, h, w = self._net_shape
        if self._net is None or B > b or H > h or W > w:
            cfg = self.config["extractor"]
            self._net_shape = (max(B, b), max(H, h), max(W, w))
            self._net = _native.SuperPointNet(
                self._ctx, self._weights, nms_radius=cfg["nms_radius"], keypoint_threshold=cfg["keypoint_threshold"],
                max_keypoints=cfg["max_keypoints"], remove_borders=cfg["remove_borders"],
                fix_sampling=cfg["fix_sampling"], max_batch=self._net_shape[0], max_height=self._net_shape[1],
                max_width=self._net_shape[2])
        return self._net

    def _extract(self, image: np.ndarray) -> dict:
        image_ = self._frame2tensor(image)
        _, H, W = image_.shape
        return self._ensure(1, H, W).extract(image_)[0]

    def extract_many(self, images) -> list:
        """Batched entry (not in the reference, which is batch-1): equally sized gray images -> list of dicts."""
        arr = np.stack([self._frame2tensor(i)[0] for i in images])
        B, H, W = arr.shape
        return self._ensure(B, H, W).extract(arr)

    def _frame2tensor(self, image: np.ndarray, device: str = "cuda"):
        """(H,W) or (H,W,1) float 0..255 -> (1,H,W) float32; the /255 of the reference (:146) happens on device."""
        if image.ndim == 3:
            if image.shape[2] != 1:
                raise ValueError("SuperPoint expects a single-channel image")
            image = image[:, :, 0]
        return np.ascontiguousarray(image, dtype=np.float32)[None]
