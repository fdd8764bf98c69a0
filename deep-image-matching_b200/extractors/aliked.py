"""AlikedExtractor on libdimb200 - drop-in for the reference plugin
(src/deep_image_matching/extractors/aliked.py:10-85): same class name, class attributes, config keys and
``_extract`` contract (float32 (H,W,3) RGB 0..255 in - ``grayscale = False`` - dict of numpy arrays out:
keypoints (N,2) sub-pixel x,y; descriptors (128,N); scores (N,)).  The model runs in hand-written CUDA kernels
(csrc/aliked.cu) instead of the torch / torchvision.ops.deform_conv2d graph of the LightGlue ALIKED port.

Reproduced quirks: the config key the model reads is ``model_name`` (the plugin's own default spells it ``model``,
which the model ignores: a config without ``model_name`` gets the model default "aliked-n16", aliked.py:563);
``scores`` are the detector's score dispersities (aliked.py:682, SURVEY A.5).
"""
from __future__ import annotations

import numpy as np

from .. import _native
from ..weights import aliked as aliked_weights
from .extractor_base import ExtractorBase

_SUPPORTED = ("aliked-n16", "aliked-n16rot")  # same architecture, different checkpoints (aliked.py:574-579)


class AlikedExtractor(ExtractorBase):
    _default_conf = {
        "name:": "aliked",  # sic (reference :23)
        "model": "aliked-n16rot",
        "device": "cuda",
        "max_num_keypoints": 4000,
        "detection_threshold": 0.2,
        "nms_radius": 2,
    }
    required_inputs = []
    grayscale = False
    descriptor_size = 128

    def __init__(self, config: dict):
        super().__init__(config)
        cfg = self.config["extractor"]
        model_name = cfg.get("model_name", "aliked-n16")
        if model_name not in _SUPPORTED:
            raise NotImplementedError(f"libdimb200 implements {_SUPPORTED}; got model_name={model_name!r}")
        self._ctx = _native.Context.get(int(self.config["general"].get("device", 0)))
        self._weights = cfg.get("weights_dict") or aliked_weights(model_name)  # checkpoint follows model_name (aliked.py:581-587)
        self._net = None
        self._net_shape = (0, 0)

    def _ensure(self, H, W):
        h, w = self._net_shape
        if self._net is None or H > h or W > w:
            cfg = self.config["extractor"]
            self._net_shape = (max(H, h), max(W, w))
            self._net = _native.AlikedNet(self._ctx, self._weights, max_num_keypoints=cfg["max_num_keypoints"],
                                          detection_threshold=cfg["detection_threshold"], nms_radius=cfg["nms_radius"],
                                          max_height=self._net_shape[0], max_width=self._net_shape[1])
        return self._net

    def _extract(self, image: np.ndarray) -> dict:
        image_ = self._frame2tensor(image)
        return self._ensure(*image_.shape[:2]).extract(image_)

    def _frame2tensor(self, image: np.ndarray, device: str = "cuda"):
        """(H,W) or (H,W,3) float 0..255 -> contiguous float32; the /255 of the reference (:78) happens on device."""
        if image.ndim == 3 and image.shape[2] not in (1, 3):
            raise ValueError("ALIKED expects a 1- or 3-channel image")
        if image.ndim == 3 and image.shape[2] == 1:
            image = image[:, :, 0]
        return np.ascontiguousarray(image, dtype=np.float32)
