"""Minimal stand-in for the reference's ``Config`` object (src/deep_image_matching/config.py:339-787).

The plugin constructors only read ``.general``, ``.extractor`` and ``.matcher`` dictionaries
(extractor_base.py:134-143, matcher_base.py:110-121); the pipeline zoo below restates the entries of
``confs`` (config.py:92-296) that belong to the hot path.
"""
from __future__ import annotations

from pathlib import Path

confs = {
    "superpoint+lightglue": {  # config.py:93-110
        "extractor": {"name": "superpoint", "nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048},
        "matcher": {"name": "lightglue", "n_layers": 9, "mp": False, "flash": True, "depth_confidence": 0.95,
                    "width_confidence": 0.99, "filter_threshold": 0.1},
    },
    "superpoint+kornia_matcher": {
        "extractor": {"name": "superpoint", "nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048},
        "matcher": {"name": "kornia_matcher", "match_mode": "smnn", "th": 0.99},
    },
    "sift+kornia_matcher": {  # config.py:232-244 (SIFTExtractor: cv2.SIFT's detectAndCompute on the device, csrc/sift.cu)
        "extractor": {"name": "sift", "n_features": 2048, "nOctaveLayers": 3, "contrastThreshold": 0.0004, "edgeThreshold": 10,
                      "sigma": 1.6},
        "matcher": {"name": "kornia_matcher", "match_mode": "smnn", "th": 0.85},
    },
    "aliked+lightglue": {  # config.py:197-212
        "extractor": {"name": "aliked", "model_name": "aliked-n16rot", "max_num_keypoints": 4000, "detection_threshold": 0.2,
                      "nms_radius": 3},
        "matcher": {"name": "lightglue", "n_layers": 9, "depth_confidence": 0.95, "width_confidence": 0.99,
                    "filter_threshold": 0.1},
    },
}


class Config:
    def __init__(self, general: dict | None = None, extractor: dict | None = None, matcher: dict | None = None,
                 pipeline: str | None = None):
        base = confs.get(pipeline, {"extractor": {}, "matcher": {}}) if pipeline else {"extractor": {}, "matcher": {}}
        self.general = {"output_dir": Path("."), "verbose": False, "device": 0, "quality": "high", "tile_size": (2400, 2000),
                        "tile_overlap": 10, **(general or {})}  # tile defaults: config.py:61-63; quality: "high", the reference's default
        self.extractor = {**base["extractor"], **(extractor or {})}
        self.matcher = {**base["matcher"], **(matcher or {})}
