"""Host-side logic that needs no GPU: the C-ABI library loads and exports every declared symbol, the plugin
surface mirrors the reference's, weight packing, the features.h5 boundary, loud failure without CUDA."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT


def test_library_exports_every_declared_symbol():
    from dim_b200 import _native
    lib = _native.load_library()
    header = open(os.path.join(ROOT, "include", "dimb200.h")).read()
    declared = set(re.findall(r"\b(dimb_[a-z0-9_]+)\s*\(", header))
    assert declared >= set(_native.EXPORTS)
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert b"sm_90a" in lib.dimb_version()


def test_no_cpu_fallback():
    import torch
    from dim_b200 import _native
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_native.DimbError, match="no CPU fallback"):
        _native.Context(0)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "deep-image-matching_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_plugin_surface():
    import dim_b200.extractors as E
    import dim_b200.matchers as M
    from dim_b200.config import Config
    from dim_b200.extractors.extractor_base import ExtractorBase, extractor_loader
    from dim_b200.matchers.matcher_base import MatcherBase, matcher_loader
    sp = extractor_loader(E, "superpoint")
    lg = matcher_loader(M, "lightglue")
    km = matcher_loader(M, "kornia_matcher")
    ltg = matcher_loader(M, "lighterglue")
    assert ltg.__name__ == "LighterGlueMatcher" and issubclass(ltg, MatcherBase) and ltg.min_matches == 20
    sg = matcher_loader(M, "superglue")
    assert sg.__name__ == "SuperGlueMatcher" and sg.max_feat_no_tiling == 50000 and sg.default_config["sinkhorn_iterations"] == 20
    al = extractor_loader(E, "aliked")
    assert al.__name__ == "AlikedExtractor" and issubclass(al, ExtractorBase)
    assert al.grayscale is False and al.descriptor_size == 128 and al._default_conf["nms_radius"] == 2
    assert sp.__name__ == "SuperPointExtractor" and issubclass(sp, ExtractorBase)
    assert lg.__name__ == "LightGlueMatcher" and issubclass(lg, MatcherBase)
    assert km.__name__ == "KorniaMatcher"
    assert sp.grayscale and sp.descriptor_size == 256 and sp.features_as_half
    assert lg.max_feat_no_tiling == 200000 and lg.min_matches == 20
    assert sp._default_conf["fix_sampling"] is False and sp._default_conf["nms_radius"] == 4
    with pytest.raises(TypeError, match="Config object"):
        sp({"extractor": {}})
    with pytest.raises(TypeError, match="Config object"):
        lg({"matcher": {}})
    cfg = Config(pipeline="superpoint+lightglue")
    assert cfg.extractor["max_keypoints"] == 2048 and cfg.matcher["depth_confidence"] == 0.95


def test_featuresdict_layout_decision():
    from dim_b200.matchers.lightglue import featuresDict2Lightglue
    k = np.zeros((10, 2), np.float32)
    assert featuresDict2Lightglue({"keypoints": k, "descriptors": np.zeros((256, 10), np.float32)})["_layout"] == 0
    assert featuresDict2Lightglue({"keypoints": k, "descriptors": np.zeros((10, 256), np.float32)})["_layout"] == 1
    with pytest.raises(ValueError, match="mismatch"):
        featuresDict2Lightglue({"keypoints": k, "descriptors": np.zeros((7, 256), np.float32)})
    with pytest.raises(KeyError):
        featuresDict2Lightglue({"keypoints": k})
    # N == D is ambiguous in the reference too: treated as (N,D)   (SURVEY A.2)
    k2 = np.zeros((256, 2), np.float32)
    assert featuresDict2Lightglue({"keypoints": k2, "descriptors": np.zeros((256, 256), np.float32)})["_layout"] == 1


def test_weight_packing_sizes(sp_weights):
    from dim_b200 import _native, weights
    assert _native.pack_superpoint_weights(sp_weights).size == 1300865
    w = weights.lightglue_seeded()
    assert _native.pack_lightglue_weights(w, 256, 256, 9).size == 11851601
    w128 = weights.lightglue_seeded(input_dim=128)
    assert _native.pack_lightglue_weights(w128, 128, 256, 9).size == 11851601 + 256 * 128 + 256
    # old-style checkpoint prefixes are renamed (lightglue.py:391-396)
    old = {k.replace("transformers.3.self_attn", "self_attn.3").replace("transformers.3.cross_attn", "cross_attn.3"): v for k, v in w.items()}
    assert np.array_equal(_native.pack_lightglue_weights(old, 256, 256, 9), _native.pack_lightglue_weights(w, 256, 256, 9))


def test_aliked_and_lighterglue_weight_packing(al_weights, ltg_weights):
    """Blob sizes the C ABI checks: ALIKED-n16 state_dict order (678316 floats), LighterGlue shape (64 / 96 / 1 head / 6 layers)."""
    from dim_b200 import _native
    assert _native.pack_aliked_weights(al_weights).size == 678316
    assert len(_native.aliked_weight_names()) == 68 and set(_native.aliked_weight_names()) == set(al_weights)
    d, din, L = 96, 64, 6
    per_layer = (3 * d * d + 3 * d) + (d * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d) + 3 * (d * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d)
    need = (d // 2) * 2 + d * din + d + per_layer * L + L * (d + 1 + d * d + d) + (L - 1) * (d + 1)
    assert _native.pack_lightglue_weights(ltg_weights, din, d, L).size == need


def test_seeded_weights_are_deterministic():
    from dim_b200 import weights
    a, b = weights.lightglue_seeded(seed=3), weights.lightglue_seeded(seed=3)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert abs(float(a["transformers.0.self_attn.Wqkv.weight"][0, 0]) - float(weights.lightglue_seeded(seed=4)["transformers.0.self_attn.Wqkv.weight"][0, 0])) > 0


def test_h5_boundary_roundtrip(tmp_path):
    from dim_b200.io_h5 import as_half_roundtrip, get_features, save_features_h5
    rng = np.random.default_rng(0)
    feats = {"keypoints": rng.uniform(0, 3000, (50, 2)).astype(np.float32), "descriptors": rng.standard_normal((256, 50)).astype(np.float32),
             "scores": rng.uniform(0, 1, 50).astype(np.float32), "tile_idx": np.zeros(50, np.float32), "image_size": np.array([1536, 2048])}
    save_features_h5(tmp_path / "features.h5", dict(feats), "a.jpg")
    back = get_features(tmp_path / "features.h5", "a.jpg")
    exp = as_half_roundtrip(feats)
    for k in feats:
        assert np.array_equal(back[k], exp[k]), k
    assert back["image_size"].dtype == np.int32 and back["keypoints"].dtype == np.float32
    assert np.abs(back["keypoints"] - feats["keypoints"]).max() <= 1.0  # fp16 quantisation above 2048 px (SURVEY A.8)
    with pytest.raises(ValueError):
        get_features(tmp_path / "features.h5", "missing.jpg")


def test_synthetic_generator_is_deterministic():
    from dim_b200 import synthetic
    a0, a1 = synthetic.synthetic_pair(5, 256)
    b0, b1 = synthetic.synthetic_pair(5, 256)
    assert np.array_equal(a0, b0) and np.array_equal(a1, b1) and a0.dtype == np.float32 and a0.shape == (256, 256)


def test_pair_generators():
    """pairs_from_sequential / pairs_from_bruteforce restate pairs_generator.py:22-38."""
    from dim_b200.pairs_generator import pairs_from_bruteforce, pairs_from_sequential
    imgs = [f"im{i}.jpg" for i in range(5)]
    assert pairs_from_sequential(imgs, 1) == [(imgs[i], imgs[i + 1]) for i in range(4)]
    assert pairs_from_sequential(imgs, 2) == [("im0.jpg", "im1.jpg"), ("im0.jpg", "im2.jpg"), ("im1.jpg", "im2.jpg"), ("im1.jpg", "im3.jpg"),
                                              ("im2.jpg", "im3.jpg"), ("im2.jpg", "im4.jpg"), ("im3.jpg", "im4.jpg")]
    assert len(pairs_from_bruteforce(imgs)) == 10 and pairs_from_bruteforce(imgs)[0] == ("im0.jpg", "im1.jpg")
    assert len(pairs_from_sequential([f"d{i}" for i in range(200)], 1)) == 199  # cfg5


def test_c_abi_rejects_null_handles_without_touching_the_gpu():
    """Argument validation comes before any CUDA call: NULL handles / buffers return DIMB_ERR_ARG (-3) on a machine without a GPU."""
    import ctypes as C
    from dim_b200 import _native
    lib = _native.load_library()
    null, n = C.c_void_p(), C.c_int(0)
    buf = np.zeros(16, np.float32)
    assert lib.dimb_sp_create(null, null, 0, None, C.byref(C.c_void_p())) == -3
    assert lib.dimb_lg_create(null, null, 0, None, C.byref(C.c_void_p())) == -3
    assert lib.dimb_aliked_create(null, null, 0, None, C.byref(C.c_void_p())) == -3
    assert lib.dimb_sg_create(null, null, 0, None, C.byref(C.c_void_p())) == -3
    assert lib.dimb_sp_extract(null, _native._ptr(buf), 1, 16, 16, null, null, null, null, 1) == -3
    assert lib.dimb_aliked_extract(null, _native._ptr(buf), 16, 16, 3, null, null, null, null, 1) == -3
    assert lib.dimb_lg_match(null, 1, None, None, null, null, null, null, 1) == -3
    assert lib.dimb_nn_match(null, null, 0, null, 0, 256, 0, C.c_float(0.0), null, null, C.byref(n), 1) == -3
    assert lib.dimb_last_error(null) == b"null context"
    lib.dimb_sp_destroy(null), lib.dimb_lg_destroy(null), lib.dimb_aliked_destroy(null), lib.dimb_sg_destroy(null), lib.dimb_pipe_destroy(null)


def test_colmap_database_writer(tmp_path):
    """io_colmap.export_to_colmap writes the reference's database layout (utils/database.py / io/h5_to_db.py:44-113): read back with
    plain sqlite3 exactly as COLMAP's own database.py would."""
    import sqlite3
    from dim_b200.io_colmap import MAX_IMAGE_ID, export_to_colmap, image_ids_to_pair_id
    rng = np.random.default_rng(0)
    feats = {n: {"keypoints": rng.uniform(0, 600, (k, 2)).astype(np.float32), "image_size": np.array(hw)} for n, k, hw in
             (("a.jpg", 50, (480, 640)), ("b.jpg", 40, (640, 618)), ("c.jpg", 0, (100, 100)))}
    m_ab = np.stack([rng.permutation(50)[:30], rng.permutation(40)[:30]], 1).astype(np.int64)
    m_ba = m_ab[:10, ::-1].copy()
    F = rng.standard_normal((3, 3))
    ids = export_to_colmap(feats, {("a.jpg", "b.jpg"): m_ab[:20], ("c.jpg", "a.jpg"): np.zeros((0, 2), np.int64)}, tmp_path / "database.db",
                           raw_matches={("a.jpg", "b.jpg"): m_ab, ("b.jpg", "a.jpg"): m_ba}, fundamental={("a.jpg", "b.jpg"): F})
    assert ids == {"a.jpg": 1, "b.jpg": 2, "c.jpg": 3}
    db = sqlite3.connect(str(tmp_path / "database.db"))
    cams = db.execute("SELECT model, width, height, params, prior_focal_length FROM cameras").fetchall()
    assert len(cams) == 3 and cams[1][:3] == (2, 618, 640)
    assert np.allclose(np.frombuffer(cams[0][3], np.float64), [1.2 * 640, 320, 240, 0.1])  # simple-radial, focal prior 1.2 * max(w, h)
    rows, cols, blob = db.execute("SELECT rows, cols, data FROM keypoints WHERE image_id = 2").fetchone()
    assert (rows, cols) == (40, 2) and np.array_equal(np.frombuffer(blob, np.float32).reshape(rows, cols), feats["b.jpg"]["keypoints"])
    raw = db.execute("SELECT pair_id, rows, data FROM matches").fetchall()
    assert len(raw) == 1 and raw[0][0] == 1 * MAX_IMAGE_ID + 2 == image_ids_to_pair_id(2, 1)  # the (b, a) duplicate is skipped like the reference
    assert np.array_equal(np.frombuffer(raw[0][2], np.uint32).reshape(-1, 2), m_ab.astype(np.uint32))
    tv = dict((r[0], r[1:]) for r in db.execute("SELECT pair_id, rows, data, config, F FROM two_view_geometries").fetchall())
    assert set(tv) == {image_ids_to_pair_id(1, 2), image_ids_to_pair_id(1, 3)}
    r, data, config, Fb = tv[image_ids_to_pair_id(1, 2)]
    assert r == 20 and config == 2 and np.allclose(np.frombuffer(Fb, np.float64).reshape(3, 3), F)
    assert np.array_equal(np.frombuffer(data, np.uint32).reshape(-1, 2), m_ab[:20].astype(np.uint32))
    assert tv[image_ids_to_pair_id(1, 3)][0] == 0  # (c, a) stored under (a, c) with swapped, empty columns
    one = export_to_colmap(feats, {}, tmp_path / "database.db", single_camera=True)  # overwrites the file
    assert len(sqlite3.connect(str(tmp_path / "database.db")).execute("SELECT * FROM cameras").fetchall()) == 1 and len(one) == 3
