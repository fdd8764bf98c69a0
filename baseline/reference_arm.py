"""The reference's own SuperPoint + LightGlue path for ``bench.py --impl reference`` (CPU) and the ``gpu_reference`` leg
(eager PyTorch on the same GPU, batch 1 - the bar BASELINE.md section 3 names).

Nothing of this repository's kernels, oracle or engine is on this path: the two model files are the reference's vendored
``thirdparty/SuperGluePretrainedNetwork/models/superpoint.py`` and ``thirdparty/LightGlue/lightglue/lightglue.py``, copied
byte for byte into the git-ignored ``baseline/_ref/`` by :func:`stage` from a checkout of the reference (they are the
reference's files, not this project's, so they are not committed).  Without them ``bench.py --impl reference`` times the
oracle port instead and says so in its JSON line.  The reference
package itself cannot be imported or pip-installed here (h5py, kornia, rasterio, pydegensac, pycolmap are absent from the
image and the wheelhouse), so the thin plugin adapters around the models are restated below, each citing the lines it
follows; the models run unmodified with DIM's defaults (fp32 weights, ``flash=True``, ``mp=False``, cuDNN defaults).

LightGlue weights: the reference downloads ``superpoint_lightglue.pth`` at run time (lightglue.py:381-384); offline the
seeded LightGlue-architecture weights of the benchmark are loaded into the reference class instead (same tensors as our arm).
"""
from __future__ import annotations

import importlib.util
import os
import shutil
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
SRC = "src/deep_image_matching/thirdparty/"  # inside a checkout of the reference
FILES = {
    "superpoint.py": SRC + "SuperGluePretrainedNetwork/models/superpoint.py",
    "superpoint_v1.pth": SRC + "SuperGluePretrainedNetwork/models/weights/superpoint_v1.pth",
    "lightglue.py": SRC + "LightGlue/lightglue/lightglue.py",
}
SP_CONF = {"name": "superpoint", "nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048, "remove_borders": 4,
           "fix_sampling": False}  # config.py:93-99 over SuperPointExtractor._default_conf (extractors/superpoint.py:84-91)


def stage(reference_root: str) -> bool:
    """Copy the reference's model files from the checkout at `reference_root` into baseline/_ref/. True if the arm is available."""
    if os.path.isdir(reference_root):
        os.makedirs(REF_DIR, exist_ok=True)
        for name, rel in FILES.items():
            src, dst = os.path.join(reference_root, rel), os.path.join(REF_DIR, name)
            if not os.path.exists(dst) or os.path.getsize(dst) != os.path.getsize(src):
                shutil.copyfile(src, dst)
    return available()


def available() -> bool:
    return all(os.path.exists(os.path.join(REF_DIR, n)) for n in FILES)


def _load(name):
    spec = importlib.util.spec_from_file_location("dim_ref_" + name, os.path.join(REF_DIR, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


class ReferenceSPLG:
    """SuperPointExtractor._extract + features.h5 round trip + LightGlueMatcher._match_pairs with the reference's models."""

    def __init__(self, device: str = "cpu", fixed_work: bool = True, lg_weights: dict | None = None):
        import warnings

        import torch
        if not available():
            raise FileNotFoundError("baseline/_ref/ is not staged (baseline.reference_arm.stage(<checkout of the reference>))")
        self.torch, self.device = torch, torch.device(device)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            spmod, lgmod = _load("superpoint"), _load("lightglue")
        sd = torch.load(os.path.join(REF_DIR, "superpoint_v1.pth"), map_location="cpu")
        hub, torch.hub.load_state_dict_from_url = torch.hub.load_state_dict_from_url, (lambda *a, **k: sd)  # superpoint.py:148-150
        try:
            import contextlib
            import io
            with contextlib.redirect_stdout(io.StringIO()):  # the model prints "Loaded SuperPoint model" (bench prints ONE json line)
                self.sp = spmod.SuperPoint(dict(SP_CONF)).eval().to(self.device)  # extractors/superpoint.py:100-105
        finally:
            torch.hub.load_state_dict_from_url = hub
        cfg = {"flash": True, "mp": False, "depth_confidence": -1 if fixed_work else 0.95, "width_confidence": -1 if fixed_work else 0.99,
               "filter_threshold": 0.1}  # matchers/lightglue.py:70-77, config.py:100-109
        # features=None: no checkpoint download (lightglue.py:381-384); architecture of "superpoint" (input_dim 256, :331-334)
        self.lg = lgmod.LightGlue(features=None, input_dim=256, **cfg).eval()
        if lg_weights is not None:
            missing = self.lg.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in lg_weights.items()}, strict=False)
            assert not missing.unexpected_keys and set(missing.missing_keys) <= {"confidence_thresholds"}, missing
        self.lg = self.lg.to(self.device)

    def extract(self, image: np.ndarray) -> dict:
        """SuperPointExtractor._extract (extractors/superpoint.py:107-146): (H,W) float32 gray 0..255 -> numpy FeaturesDict."""
        torch = self.torch
        with torch.no_grad():
            image_ = torch.tensor(image[None][None] / 255.0, dtype=torch.float).to(self.device)
            feats = self.sp({"image": image_})
            feats = {k: v[0] if isinstance(v, (list, tuple)) else v for k, v in feats.items()}
            return {k: v.cpu().numpy() for k, v in feats.items()}

    @staticmethod
    def h5_roundtrip(feats: dict, image_shape) -> dict:
        """ExtractorBase.extract + save_features_h5 + get_features (extractor_base.py:56-99,223-229; io/h5.py:45-89): every array
        passes through float16; image_size = image.shape[:2] comes back as int32."""
        out = {k: v.astype(np.float16).astype(np.float32) for k, v in feats.items()}
        out["tile_idx"] = np.zeros(out["keypoints"].shape[0], np.float32)
        out["image_size"] = np.array(image_shape[:2]).astype(np.float16).astype(np.int32)
        return out

    def match(self, feats0: dict, feats1: dict) -> np.ndarray:
        """LightGlueMatcher._match_pairs (matchers/lightglue.py:102-125) incl. featuresDict2Lightglue (:8-66)."""
        torch = self.torch

        def conv(feats):
            feats = dict(feats)
            n = feats["keypoints"].shape[0]
            d = feats["descriptors"]
            if d.shape[1] == n and d.shape[0] != n:
                feats["descriptors"] = d.T
            return {k: torch.as_tensor(v[None], dtype=torch.float32, device=self.device) for k, v in feats.items()}

        with torch.no_grad():
            res = self.lg({"image0": conv(feats0), "image1": conv(feats1)})
            return res["matches"][0].cpu().numpy()

    def pair(self, g0: np.ndarray, g1: np.ndarray) -> np.ndarray:
        f = [self.h5_roundtrip(self.extract(g), g.shape) for g in (g0, g1)]
        return self.match(f[0], f[1])


_WORKER_NET = None


def _pool_worker(args):
    """One process of the CPU process pool: `n` pairs, `threads` torch threads; returns (seconds, pairs, matches)."""
    import time

    import torch
    global _WORKER_NET
    seeds, threads, size, fixed = args
    torch.set_num_threads(threads)
    if os.path.dirname(HERE) not in sys.path:
        sys.path.insert(0, os.path.dirname(HERE))
    from dim_b200 import synthetic, weights
    if _WORKER_NET is None or _WORKER_NET[0] != fixed:  # one model per worker process, built on its first task
        _WORKER_NET = (fixed, ReferenceSPLG("cpu", fixed, weights.lightglue_seeded(seed=0)))
    net = _WORKER_NET[1]
    t0 = time.perf_counter()
    nm = 0
    for s in seeds:
        g0, g1 = synthetic.synthetic_pair(s, size)
        nm += len(net.pair(g0, g1))
    return time.perf_counter() - t0, len(seeds), nm
