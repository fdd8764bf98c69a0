"""Mirror of the reference's extractor plugin surface (src/deep_image_matching/extractors/extractor_base.py).

Only what the hot path touches is restated: the constructor contract (:119-160), ``extract`` (:162-251: load,
gray conversion quirk, ``_resize_image`` by quality, ``_extract``, tile_idx, ``_resize_features``, image_size of the original
image, features.h5) and the abstract ``_extract`` / ``_frame2tensor`` (:253-277).  ``_extract_by_tile`` is restated for the tests
of the device tiling; ``extract`` itself does not tile.  The class drops in unchanged when it is replaced by the reference's own
base class (INTEGRATION.md).
"""
from __future__ import annotations

import inspect
from abc import ABCMeta, abstractmethod
from pathlib import Path
from typing import Optional, TypedDict

import numpy as np

from ..config import Config
from ..io_h5 import save_features_h5


class FeaturesDict(TypedDict):
    keypoints: np.ndarray
    descriptors: np.ndarray
    scores: Optional[np.ndarray]
    tile_idx: Optional[np.ndarray]


def extractor_loader(root, model):
    """extractor_base.py:29-53: exactly one ExtractorBase subclass per module."""
    module_path = f"{root.__name__}.{model}"
    module = __import__(module_path, fromlist=[""])
    classes = inspect.getmembers(module, inspect.isclass)
    classes = [c for c in classes if c[1].__module__ == module_path]
    classes = [c for c in classes if issubclass(c[1], ExtractorBase)]
    assert len(classes) == 1, classes
    return classes[0][1]


class ExtractorBase(metaclass=ABCMeta):
    _default_general_conf = {"force_cpu": False, "do_viz": False, "quality": "high"}
    _default_conf = {}
    required_inputs = []
    grayscale = True
    as_float = True
    descriptor_size = 128
    features_as_half = True

    def __init__(self, custom_config: Config) -> None:
        if not isinstance(custom_config, Config):
            raise TypeError("Invalid config object. 'custom_config' must be a Config object")
        self.config = {
            "general": {**self._default_general_conf, **custom_config.general},
            "extractor": {**self._default_conf, **custom_config.extractor},
        }
        if self.config["general"].get("force_cpu"):
            raise RuntimeError("dim_b200 has no CPU path (force_cpu=True is not supported)")
        self._device = "cuda"

    def extract(self, img) -> Path:
        import cv2

        im_path = Path(getattr(img, "path", img))
        if not im_path.exists():
            raise ValueError(f"Image {im_path} does not exist")
        feature_path = Path(self.config["general"]["output_dir"]) / "features.h5"
        # rasterio returns bands in file order (RGB); cv2 reads BGR -> swap so the array equals rasterio's
        image = cv2.imread(str(im_path), cv2.IMREAD_UNCHANGED)
        if image is None:
            raise ValueError(f"Cannot read {im_path}")
        if image.ndim == 3:
            image = cv2.cvtColor(image, cv2.COLOR_BGR2RGB)
        if self.grayscale and image.ndim == 3 and image.shape[2] > 1:
            image = cv2.cvtColor(image, cv2.COLOR_BGR2GRAY)  # sic: applied to an RGB array (SURVEY A.1)
        if self.as_float:
            image = image.astype(np.float32)
        quality = self.config["general"]["quality"]
        features = self._extract(self._resize_image(quality, image))
        features["tile_idx"] = np.zeros(features["keypoints"].shape[0], dtype=np.float32)
        features = self._resize_features(quality, features)
        features["image_size"] = np.array(image.shape[:2])  # the original image's size, whatever the quality
        save_features_h5(feature_path, features, im_path.name, as_half=self.features_as_half)
        return feature_path

    @staticmethod
    def _resize_image(quality, image: np.ndarray) -> np.ndarray:
        """extractor_base.py _resize_image: "highest" cv2.pyrUp, "high" unchanged, "medium" / "low" / "lowest" one, two or three
        cv2.pyrDown (``sharded.quality_conf`` gives the level)."""
        import cv2

        from ..sharded import quality_conf
        level = quality_conf(quality)
        if level < 0:
            return cv2.pyrUp(image)
        for _ in range(level):
            image = cv2.pyrDown(image)
        return image

    @staticmethod
    def _resize_features(quality, features: dict) -> dict:
        """extractor_base.py _resize_features: the keypoints (float32, in place) back to the original image, / 2 for "highest" and
        * 2, * 4, * 8 for "medium", "low", "lowest"."""
        from ..sharded import quality_conf
        level = quality_conf(quality)
        if level < 0:
            features["keypoints"] /= 2
        elif level > 0:
            features["keypoints"] *= 2 ** level
        return features

    def _extract_by_tile(self, image: np.ndarray, select_unique: bool = True) -> dict:
        """extractor_base.py:279-390: one ``_extract`` per tile of ``general.tile_size`` / ``tile_overlap``, keypoints moved to
        full-image coordinates, points closer than 2 px to the image border (or in the padding) dropped, ``tile_idx`` recorded,
        then ``np.unique`` over the coordinates (which also re-sorts the keypoints lexicographically by (x, y), quirk A.9)."""
        from ..tiling import compute_tiles_by_size

        tiles, origins, _ = compute_tiles_by_size(image, self.config["general"]["tile_size"], self.config["general"]["tile_overlap"])
        kpts, descs, scores, tidx = [], [], [], []
        for idx, tile in tiles.items():
            feat = self._extract(tile)
            kp = feat["keypoints"]
            kp += np.array(origins[idx])  # in place, like the reference (:332)
            border_thr = 2
            mask = ((kp[:, 0] >= border_thr) & (kp[:, 0] < image.shape[1] - border_thr) & (kp[:, 1] >= border_thr)
                    & (kp[:, 1] < image.shape[0] - border_thr))
            if mask.sum() > 0:
                kpts.append(kp[mask])
                descs.append(feat["descriptors"][:, mask])
                tidx.append(np.full(int(mask.sum()), idx, dtype=np.float32))
                if feat.get("scores") is not None:
                    scores.append(feat["scores"][mask])
        if kpts:
            kpts_full, desc_full, tidx_full = np.vstack(kpts), np.hstack(descs), np.concatenate(tidx)
            scores_full = np.concatenate(scores) if scores else None
        else:
            kpts_full = np.zeros((0, 2), np.float32)
            desc_full = np.zeros((self.descriptor_size, 0), np.float32)
            tidx_full, scores_full = np.zeros(0, np.float32), None
        if scores_full is None:
            scores_full = np.ones(kpts_full.shape[0], dtype=np.float32)
        if select_unique:
            kpts_full, unique_idx = np.unique(kpts_full, axis=0, return_index=True)
            desc_full, tidx_full, scores_full = desc_full[:, unique_idx], tidx_full[unique_idx], scores_full[unique_idx]
        return FeaturesDict(keypoints=kpts_full, descriptors=desc_full, scores=scores_full, tile_idx=tidx_full)

    @abstractmethod
    def _extract(self, image: np.ndarray) -> dict:
        raise NotImplementedError("Subclasses should implement _extract method!")

    @abstractmethod
    def _frame2tensor(self, image: np.ndarray, device: str = "cuda"):
        raise NotImplementedError("Subclasses should implement _frame2tensor method!")
