import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def sp_weights():
    from dim_b200 import weights
    return weights.superpoint_v1()


@pytest.fixture(scope="session")
def sp_golden():
    return np.load(os.path.join(GOLD, "superpoint_golden.npz"))


@pytest.fixture(scope="session")
def lg_golden():
    return np.load(os.path.join(GOLD, "lightglue_golden.npz"))


@pytest.fixture(scope="session")
def nn_golden():
    return np.load(os.path.join(GOLD, "nn_golden.npz"))


@pytest.fixture(scope="session")
def al_golden():
    return np.load(os.path.join(GOLD, "aliked_golden.npz"))


@pytest.fixture(scope="session")
def al_weights():
    from dim_b200 import weights
    return weights.aliked_n16rot()


@pytest.fixture(scope="session")
def ctx():
    from dim_b200 import _native
    return _native.Context.get(0)


SP_CASES = ["real240x320", "real240x320_fix_top256", "blocks384x512_top512", "real_odd237x315"]
LG_CASES = ["sp_small_fixed", "sp_small_adaptive", "sp_prune", "din128_fixed", "tiny", "cfg2_2048_adaptive", "prune_only"]


LTG_CASES = ["fixed", "lighterglue_default", "dim_plugin_default"]


def ltg_case(g, name):
    """Trained LighterGlue checkpoint on XFeat features of the reference's test photos (oracle/gen_golden.py:gen_lighterglue)."""
    from oracle import lightglue as o_lg
    dc, wc = g[name + ".conf"]
    conf = {**o_lg.DEFAULT_CONF, "input_dim": 64, "descriptor_dim": 96, "num_heads": 1, "n_layers": 6, "depth_confidence": float(dc),
            "width_confidence": float(wc)}
    f = [{"keypoints": g[f"kpts{i}"].astype(np.float32), "descriptors": g[f"desc{i}"].astype(np.float32), "image_size": g[f"size{i}"]}
         for i in (0, 1)]
    ref = {"matches": g[name + ".matches"].astype(np.int64), "scores": g[name + ".scores"], "stop": int(g[name + ".stop"]),
           "prune0": g[name + ".prune0"], "prune1": g[name + ".prune1"]}
    return f[0], f[1], conf, ref


@pytest.fixture(scope="session")
def ltg_golden():
    return np.load(os.path.join(GOLD, "lighterglue_golden.npz"))


@pytest.fixture(scope="session")
def ltg_weights():
    from dim_b200 import weights
    return weights.load_npz(os.path.join(weights.DATA, "lighterglue_weights.npz"))


AL_CASES = ["real224x288", "real_odd203x260_r3_top100", "blocks256"]


def al_case(g, name):
    mk, thr, r = g[name + ".conf"]
    conf = {"model_name": "aliked-n16rot", "max_num_keypoints": int(mk), "detection_threshold": float(thr), "nms_radius": int(r)}
    ref = {"keypoints": g[name + ".keypoints"], "scores": g[name + ".scores"], "descriptors": g[name + ".descriptors"]}
    return g[name + ".image"].astype(np.float32), conf, ref


def sp_case(g, name):
    nms, thr, mk, fix = g[name + ".conf"]
    conf = {"nms_radius": int(nms), "keypoint_threshold": float(thr), "max_keypoints": int(mk), "fix_sampling": bool(fix)}
    ref = {"keypoints": g[name + ".keypoints"].astype(np.float32), "scores": g[name + ".scores"],
           "descriptors": g[name + ".descriptors"]}
    return g[name + ".image"].astype(np.float32), conf, ref


def lg_case(g, name):
    from oracle import lightglue as o_lg
    from oracle.gen_golden import lg_pair
    seed, m, n, h, w = [int(x) for x in g[name + ".args"]]
    din, dc, wc, pm = g[name + ".conf"]
    conf = {**o_lg.DEFAULT_CONF, "input_dim": int(din), "depth_confidence": float(dc), "width_confidence": float(wc),
            "prune_min_kpts": int(pm)}
    f0, f1 = lg_pair(seed, m, n, int(din), (h, w))
    weights = o_lg.seeded_weights(conf, seed=seed)
    ref = {"matches": g[name + ".matches"].astype(np.int64), "scores": g[name + ".scores"], "stop": int(g[name + ".stop"])}
    return f0, f1, conf, weights, ref
