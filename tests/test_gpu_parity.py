"""Parity tests proper (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs and against the golden vectors.  Tolerances (BASELINE north_star): indices bit-exact, float
scores / descriptors within 1e-4 (EXACT precision mode)."""
import os

import numpy as np
import pytest

from conftest import AL_CASES, LG_CASES, LTG_CASES, SP_CASES, al_case, lg_case, ltg_case, sp_case

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _sp_net(ctx, w, conf, B, H, W):
    from dim_b200 import _native
    return _native.SuperPointNet(ctx, w, nms_radius=conf["nms_radius"], keypoint_threshold=conf["keypoint_threshold"],
                                 max_keypoints=conf["max_keypoints"], fix_sampling=conf.get("fix_sampling", False),
                                 max_batch=B, max_height=H, max_width=W)


def _check_sp(out, ref, img=None, conf=None, w=None):
    """Keypoint sets identical (differences tolerated only at the top-k cut, oracle/compare.py), floats within TOL."""
    from oracle import superpoint as o_sp
    from oracle.compare import compare_superpoint
    nms = None
    ko = {tuple(k) for k in out["keypoints"].astype(int)}
    kr = {tuple(k) for k in ref["keypoints"].astype(int)}
    if ko != kr and img is not None:
        nms = o_sp.extract(img, w, conf, return_debug=True)["_nms"]
    rep = compare_superpoint(out, ref, nms, TOL)
    if rep["boundary_diffs"]:
        print("top-k boundary differences:", rep)
    assert out["keypoints"].flags.writeable and out["keypoints"].flags.owndata  # callers mutate in place
    return rep


def _check_lg(out, ref, th=0.1):
    from oracle.compare import compare_matches
    rep = compare_matches(out, ref, th, TOL)
    if rep["boundary_diffs"]:
        print("filter-threshold boundary differences:", rep)
    assert out["matches"].dtype == np.int64
    return rep


@pytest.mark.parametrize("name", SP_CASES)
def test_superpoint_golden(ctx, sp_golden, sp_weights, name):
    img, conf, ref = sp_case(sp_golden, name)
    H, W = img.shape
    out = _sp_net(ctx, sp_weights, conf, 1, H, W).extract(img[None])[0]
    _check_sp(out, ref, img, conf, sp_weights)


def test_superpoint_cfg2_full_size_batch(ctx, sp_golden, sp_weights):
    from dim_b200 import synthetic
    from oracle import superpoint as o_sp
    conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048}
    g0, g1 = synthetic.synthetic_pair(0, 1024)
    outs = _sp_net(ctx, sp_weights, conf, 2, 1024, 1024).extract(np.stack([g0, g1]))
    ref0 = o_sp.extract(g0, sp_weights, conf)
    b = o_sp.canonical_order(ref0)  # the live oracle equals the golden vector of the reference ...
    assert np.array_equal(ref0["keypoints"][b].astype(np.int16), sp_golden["cfg2.keypoints"])
    _check_sp(outs[0], ref0, g0, conf, sp_weights)  # ... and the CUDA path equals the oracle
    _check_sp(outs[1], o_sp.extract(g1, sp_weights, conf), g1, conf, sp_weights)


def test_superpoint_plugin_matches_oracle(ctx, sp_weights):
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from oracle import superpoint as o_sp
    cfg = Config(pipeline="superpoint+lightglue", extractor={"max_keypoints": 300})
    ext = SuperPointExtractor(cfg)
    g, _ = synthetic.synthetic_pair(4, 320)
    g = g[:240]
    out = ext._extract(g)
    _check_sp(out, o_sp.extract(g, sp_weights, {**cfg.extractor}), g, {**cfg.extractor}, sp_weights)
    # properties at any size: inside the border, scores above threshold, unit descriptors, topk respected
    assert out["keypoints"].min() >= 4 and out["keypoints"][:, 0].max() < 320 - 4 and out["keypoints"][:, 1].max() < 240 - 4
    assert out["scores"].min() > 0.0005 and len(out["scores"]) <= 300
    assert np.abs(np.linalg.norm(out["descriptors"], axis=0) - 1).max() < 1e-5


@pytest.mark.parametrize("r,thr,mk", [(5, 0.005, 4000), (4, 0.005, -1), (0, 0.05, 300)])
def test_superpoint_other_nms_radii(ctx, sp_weights, r, thr, mk):
    """nms_radius 5 / 4000 kpts is the reference's tile-preselection extractor (matcher_base.py:143-148)."""
    from dim_b200 import synthetic
    from oracle import superpoint as o_sp
    conf = {"nms_radius": r, "keypoint_threshold": thr, "max_keypoints": mk}
    g, _ = synthetic.synthetic_pair(6, 384)
    g = g[:320]
    out = _sp_net(ctx, sp_weights, conf, 1, 320, 384).extract(g[None])[0]
    _check_sp(out, o_sp.extract(g, sp_weights, conf), g, conf, sp_weights)


def test_superpoint_nms_is_exact_on_its_own_score_map(ctx, sp_weights):
    """simple_nms compares floats with == (superpoint.py:47-63): given the SAME score map the result must be bit-identical.  A
    checkerboard of 8x8 blocks gives a score map full of near-equal local maxima (183 keypoints on 64 x 96); the GPU's NMS output
    and keypoint list must equal the oracle's simple_nms + threshold + border removal applied to the GPU's own score map.  (A
    constant image, the obvious tie case, yields no score above the threshold at all.)"""
    from oracle import superpoint as o_sp
    conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": -1}
    img = (np.kron((np.indices((8, 12)).sum(0) % 2).astype(np.float32), np.ones((8, 8), np.float32)) * 180 + 30).astype(np.float32)
    net = _sp_net(ctx, sp_weights, conf, 1, 64, 96)
    out = net.extract(img[None])[0]
    ref = o_sp.extract(img, sp_weights, conf)
    assert len(out["keypoints"]) == len(ref["keypoints"]) > 100
    import torch
    dense = net.debug_read(0, (64, 96))
    k = out["keypoints"].astype(int)
    nms = o_sp.simple_nms(torch.from_numpy(dense), 3).numpy()
    gnms = net.debug_read(1, (64, 96))  # the GPU's own NMS output
    bad = np.argwhere(gnms != nms)
    assert len(bad) == 0, (len(bad), bad[:8].tolist(), [(float(gnms[y, x]), float(nms[y, x]), float(dense[y, x])) for y, x in bad[:8]])
    keep = nms > conf["keypoint_threshold"]
    keep[:4], keep[-4:], keep[:, :4], keep[:, -4:] = False, False, False, False
    ys, xs = np.nonzero(keep)
    assert np.array_equal(k, np.stack([xs, ys], 1)), (len(k), len(xs))
    assert np.array_equal(out["scores"], dense[ys, xs])
    assert k[:, 0].min() >= 4 and k[:, 0].max() < 96 - 4 and k[:, 1].min() >= 4 and k[:, 1].max() < 64 - 4
    assert out["scores"].min() > conf["keypoint_threshold"]
    assert np.abs(np.linalg.norm(out["descriptors"], axis=0) - 1).max() < 1e-5
    assert np.all(np.diff(k[:, 1] * 96 + k[:, 0]) > 0)
    assert np.abs(dense - np.asarray(o_sp.extract(img, sp_weights, conf, return_debug=True)["_dense_scores"]).reshape(64, 96)).max() < TOL


def _check_al(out, ref, img, conf, w):
    from oracle import aliked as o_al
    from oracle.compare import compare_aliked
    dbg = o_al.extract(img, w, conf, return_debug=True)
    rep = compare_aliked(out, ref, dbg["_score_map"], conf["detection_threshold"], conf["nms_radius"], tol=TOL, tol_kpt=1e-3)
    if rep["boundary_diffs"]:
        print("threshold / n_limit boundary differences:", rep)
    else:
        assert rep["order_same"], "keypoint order differs from the reference"
    return rep, dbg


@pytest.mark.parametrize("name", AL_CASES)
def test_aliked_golden(ctx, al_golden, al_weights, name):
    from dim_b200 import _native
    img, conf, ref = al_case(al_golden, name)
    H, W = img.shape[:2]
    net = _native.AlikedNet(ctx, al_weights, conf["max_num_keypoints"], conf["detection_threshold"], conf["nms_radius"], H, W)
    out = net.extract(img)
    rep, dbg = _check_al(out, ref, img, conf, al_weights)
    print(name, rep["n"], rep["max_dkpt"], rep["max_dscore"], rep["max_ddesc"])
    # dense taps: score map and L2-normalised feature map against the oracle's
    assert np.abs(net.debug_read(0, (H, W)) - dbg["_score_map"]).max() < 2e-5
    assert np.abs(net.debug_read(1, (128, H, W)) - dbg["_feature_map"]).max() < 2e-5


def test_aliked_plugin_gray_and_workspace_reuse(ctx, al_weights):
    """AlikedExtractor plugin: pipeline config (nms_radius 3), a gray image (replicated to RGB like
    kornia.color.grayscale_to_rgb, aliked.py:650-651), then a smaller RGB image on the same workspace."""
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from oracle import aliked as o_al
    cfg = Config(pipeline="aliked+lightglue")
    ext = AlikedExtractor(cfg)
    assert ext.grayscale is False and ext.descriptor_size == 128
    g, _ = synthetic.synthetic_pair(2, 320)
    g = g[:250].astype(np.float32)
    out = ext._extract(g)
    _check_al(out, o_al.extract(g, al_weights, cfg.extractor), g, cfg.extractor, al_weights)
    assert out["descriptors"].shape[0] == 128 and np.abs(np.linalg.norm(out["descriptors"], axis=0) - 1).max() < 1e-5
    rgb = np.stack([g[:200, :230], g[:200, 40:270], g[30:230, :230]], axis=2)
    out = ext._extract(rgb)
    _check_al(out, o_al.extract(rgb, al_weights, cfg.extractor), rgb, cfg.extractor, al_weights)
    with pytest.raises(NotImplementedError):
        AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n32"}))


def test_aliked_degenerate_inputs(ctx, al_weights):
    """Flat image -> no keypoint at all (empty arrays of the right shapes); images barely larger than the padding unit."""
    from dim_b200 import _native, synthetic
    from oracle import aliked as o_al
    conf = {"model_name": "aliked-n16rot", "max_num_keypoints": 4000, "detection_threshold": 0.2, "nms_radius": 2}
    net = _native.AlikedNet(ctx, al_weights, 4000, 0.2, 2, 64, 80)
    flat = np.full((64, 80, 3), 128, np.float32)
    out = net.extract(flat)
    assert out["keypoints"].shape == (0, 2) and out["descriptors"].shape == (128, 0) and out["scores"].shape == (0,)
    assert len(o_al.extract(flat, al_weights, conf)["keypoints"]) == 0
    for seed, (h, w) in ((7, (40, 56)), (8, (33, 35))):
        img = synthetic.blocks_image(seed, 64)[:h, :w].astype(np.float32)
        _check_al(net.extract(img), o_al.extract(img, al_weights, conf), img, conf, al_weights)


def test_aliked_mean_threshold_fallback(ctx, al_golden, al_weights):
    """No pixel above detection_threshold -> the detector thresholds at mean(score_map) instead (aliked.py:158-160);
    decided on the device (al_threshold_kernel)."""
    from dim_b200 import _native
    from oracle import aliked as o_al
    img, conf, _ = al_case(al_golden, "blocks256")
    img = img[:160, :192]
    conf = {**conf, "detection_threshold": 0.99999, "max_num_keypoints": 4000}
    ref = o_al.extract(img, al_weights, conf)
    assert len(ref["keypoints"]) > 20
    out = _native.AlikedNet(ctx, al_weights, 4000, 0.99999, conf["nms_radius"], 160, 192).extract(img)
    dbg = o_al.extract(img, al_weights, conf, return_debug=True)
    from oracle.compare import compare_aliked
    rep = compare_aliked(out, ref, dbg["_score_map"], float(dbg["_score_map"].mean()), conf["nms_radius"], tol=TOL, tol_kpt=1e-3)
    print(rep["n"], rep["boundary_diffs"])
    # compare_aliked asserts pairing, score and descriptor errors; on top: the fallback really fired (no pixel above 0.99999)
    # and produced the oracle's keypoint count up to mean-threshold boundary cases
    assert float(dbg["_score_map"].max()) < 0.99999 and rep["n"] == len(ref["keypoints"]) > 20
    assert abs(len(out["keypoints"]) - len(ref["keypoints"])) <= len(rep["boundary_diffs"]) <= 4


@pytest.mark.parametrize("name", LG_CASES)
def test_lightglue_golden(ctx, lg_golden, name):
    from dim_b200 import _native
    f0, f1, conf, w, ref = lg_case(lg_golden, name)
    lg = _native.LightGlueNet(ctx, w, input_dim=conf["input_dim"], depth_confidence=conf["depth_confidence"],
                              width_confidence=conf["width_confidence"], prune_min_kpts=conf["prune_min_kpts"], max_pairs=1,
                              max_kpts=max(len(f0["keypoints"]), len(f1["keypoints"])))
    out = lg.match([({**f0, "_layout": 0}, {**f1, "_layout": 0})])[0]
    _check_lg(out, ref)


@pytest.mark.parametrize("env", [{"DIMB_BN256": "1"}, {"DIMB_BN256": "1", "DIMB_K32": "1"}])
def test_lightglue_kernel_variants(lg_golden, env):
    """The selectable kernel variants (128 x 256 tiles, with 32-wide K stages) against the same goldens as the
    defaults: the switches are read when a context is created, so each case runs on a context of its own."""
    from dim_b200 import _native
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        vctx = _native.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    for name in ("sp_small_adaptive", "cfg2_2048_adaptive"):
        f0, f1, conf, w, ref = lg_case(lg_golden, name)
        lg = _native.LightGlueNet(vctx, w, input_dim=conf["input_dim"], depth_confidence=conf["depth_confidence"],
                                  width_confidence=conf["width_confidence"], prune_min_kpts=conf["prune_min_kpts"], max_pairs=1,
                                  max_kpts=max(len(f0["keypoints"]), len(f1["keypoints"])))
        _check_lg(lg.match([({**f0, "_layout": 0}, {**f1, "_layout": 0})])[0], ref)


def test_lightglue_batched_pairs_and_layouts(ctx, lg_golden):
    """Several pairs of different sizes in one call, (N,D) and (D,N) layouts, non-square image_size (quirk A.3)."""
    from dim_b200 import _native
    from oracle import lightglue as o_lg
    from oracle.gen_golden import lg_pair
    conf = {**o_lg.DEFAULT_CONF}
    w = o_lg.seeded_weights(conf, seed=11)
    pairs = [lg_pair(21, 400, 333, 256, (480, 640)), lg_pair(22, 129, 700, 256, (1536, 2048)), lg_pair(23, 640, 640, 256, (1024, 1024))]
    lg = _native.LightGlueNet(ctx, w, max_pairs=3, max_kpts=700)
    feed = []
    for i, (a, b) in enumerate(pairs):
        if i == 1:  # (N,D) layout
            a, b = {**a, "descriptors": a["descriptors"].T.copy()}, {**b, "descriptors": b["descriptors"].T.copy()}
            feed.append(({**a, "_layout": 1}, {**b, "_layout": 1}))
        else:
            feed.append(({**a, "_layout": 0}, {**b, "_layout": 0}))
    outs = lg.match(feed)
    for (a, b), out in zip(pairs, outs):
        _check_lg(out, o_lg.match(a, b, w, conf))


def test_lightglue_plugin_and_empty_inputs(ctx):
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from oracle import lightglue as o_lg
    from oracle.gen_golden import lg_pair
    w = o_lg.seeded_weights({}, seed=5)
    m = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    f0, f1 = lg_pair(31, 350, 300, 256, (600, 800))
    got = m._match_pairs(f0, f1)
    exp = o_lg.match(f0, f1, w)
    assert got.dtype == np.int64 and got.shape[1] == 2 and np.array_equal(got, exp["matches"])
    empty = {"keypoints": np.zeros((0, 2), np.float32), "descriptors": np.zeros((256, 0), np.float32), "image_size": np.array([600, 800])}
    r = m.match_many([(empty, f1)], return_scores=True)[0]
    assert r["matches"].shape == (0, 2) and r["stop"] == 1  # "no keypoints" return of the reference
    # ragged batch with a single-keypoint side and a 3-keypoint side next to a regular pair
    one = {k: (v[:, :1] if k == "descriptors" else v[:1] if k in ("keypoints", "scores", "tile_idx") else v) for k, v in f0.items()}
    three = {k: (v[:, :3] if k == "descriptors" else v[:3] if k in ("keypoints", "scores", "tile_idx") else v) for k, v in f1.items()}
    from oracle.compare import compare_matches
    res = m.match_many([(one, f1), (f0, three), (f0, f1)], return_scores=True)
    for got_i, (a, b) in zip(res, [(one, f1), (f0, three), (f0, f1)]):
        compare_matches(got_i, o_lg.match(a, b, w), 0.1, TOL)


def test_aliked_lightglue_pipeline_matches_oracle(ctx, al_golden, al_weights):
    """cfg3-shaped chain through both plugins: two overlapping crops of the reference's test photo -> AlikedExtractor ->
    fp16 h5 round trip -> LightGlueMatcher(local_features="aliked", input_dim 128), against the oracle chain."""
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from oracle import aliked as o_al
    from oracle import lightglue as o_lg
    from oracle.compare import compare_matches
    imgs = [al_case(al_golden, n)[0] for n in ("real224x288", "real_odd203x260_r3_top100")]
    cfg = Config(pipeline="aliked+lightglue", extractor={"max_num_keypoints": 400})
    ext = AlikedExtractor(cfg)
    conf_lg = {**o_lg.DEFAULT_CONF, "input_dim": 128}
    w = o_lg.seeded_weights(conf_lg, seed=3)
    m = LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w}), local_features="aliked")
    feats, ofeats = [], []
    for img in imgs:
        f = ext._extract(img)
        f["image_size"] = np.array(img.shape[:2])
        feats.append(as_half_roundtrip(f))
        o = o_al.extract(img, al_weights, cfg.extractor)
        o["image_size"] = np.array(img.shape[:2])
        ofeats.append(as_half_roundtrip(o))
        assert len(f["keypoints"]) == len(o["keypoints"]) > 100
    got = m.match_many([(feats[0], feats[1])], return_scores=True)[0]
    # (1) the matcher on exactly the features it was given: tight tolerance
    rep = compare_matches(got, o_lg.match(feats[0], feats[1], w, conf_lg), 0.1, TOL)
    print("aliked+lightglue, same features:", rep["n"], "matches, max score delta", rep["max_dscore"], rep["boundary_diffs"])
    # (2) whole chain against the oracle chain: the extractor's ~1e-6 descriptor differences flip a few fp16 roundings at
    # the h5 boundary (1 fp16 ulp = 5e-4 relative), which LightGlue amplifies: same matches, scores within 2e-3
    rep = compare_matches(got, o_lg.match(ofeats[0], ofeats[1], w, conf_lg), 0.1, 2e-3)
    flips = sum(int((a["descriptors"] != b["descriptors"]).sum()) for a, b in zip(feats, ofeats))
    print("aliked+lightglue, oracle chain:", rep["n"], "matches, max score delta", rep["max_dscore"], "fp16 flips", flips)


@pytest.mark.parametrize("name", LTG_CASES)
def test_lighterglue_trained_weights_golden(ctx, ltg_golden, ltg_weights, name):
    """Trained-weights known-answer test on the GPU: the LighterGlue checkpoint the reference ships (LightGlue architecture,
    descriptor_dim 96, one head, 6 layers, input_dim 64) on XFeat features of the reference's own test photos; the expected
    matches / scores / stop layer are the outputs of the reference's LightGlue class (tests/golden/lighterglue_golden.npz).
    Score tolerance 2e-4: with trained weights the fp32 evaluation-order noise of the reference itself is 1.5e-4."""
    from dim_b200 import _native
    from oracle.compare import compare_matches
    f0, f1, conf, ref = ltg_case(ltg_golden, name)
    net = _native.LightGlueNet(ctx, ltg_weights, input_dim=64, descriptor_dim=96, n_layers=6, num_heads=1,
                               depth_confidence=conf["depth_confidence"], width_confidence=conf["width_confidence"], max_pairs=1, max_kpts=2048)
    out = net.match([({**f0, "_layout": 0}, {**f1, "_layout": 0})])[0]
    rep = compare_matches(out, ref, 0.1, 2e-4)
    print(name, rep["n"], "matches, stop", out["stop"], "max score delta", rep["max_dscore"], rep["boundary_diffs"])
    assert rep["n"] > 390


def test_lighterglue_plugin(ctx, ltg_golden, ltg_weights):
    """LighterGlueMatcher plugin: [H,W] -> [W,H] image_size swap, LighterGlue's own depth / width defaults, xfeat only."""
    from dim_b200.config import Config
    from dim_b200.matchers.lighterglue import LIGHTERGLUE_CONF, LighterGlueMatcher
    from oracle import lightglue as o_lg
    from oracle.compare import compare_matches
    f0, f1, _, _ = ltg_case(ltg_golden, "fixed")
    f0 = {k: (v[:, :700] if k == "descriptors" else v[:700] if k == "keypoints" else v) for k, v in f0.items()}
    f1 = {k: (v[:, :650] if k == "descriptors" else v[:650] if k == "keypoints" else v) for k, v in f1.items()}
    m = LighterGlueMatcher(Config(matcher={"name": "lighterglue", "weights_dict": ltg_weights}), local_features="xfeat")
    got = m.match_scored(f0, f1)
    swap = lambda f: {**f, "image_size": np.asarray(f["image_size"])[::-1].copy()}
    exp = o_lg.match(swap(f0), swap(f1), ltg_weights, {**o_lg.DEFAULT_CONF, **LIGHTERGLUE_CONF})
    rep = compare_matches(got, exp, 0.1, 2e-4)
    assert rep["n"] > 50 and m._match_pairs(f0, f1).dtype == np.int64
    with pytest.raises(ValueError, match="Unsupported local feature"):
        LighterGlueMatcher(Config(matcher={"weights_dict": ltg_weights}), local_features="superpoint")
    with pytest.raises(ValueError, match="image_size"):
        m._match_pairs({k: v for k, v in f0.items() if k != "image_size"}, f1)


@pytest.mark.parametrize("name", ["small", "tiny"])
def test_superglue_matches_oracle(ctx, name):
    """SuperGlue (csrc/superglue.cu) against the oracle (pinned to the reference class, tests/golden/superglue_golden.npz):
    seeded weights, seeded features; matches identical, matching scores within 2e-4 (100 log-space Sinkhorn sweeps)."""
    import os
    from conftest import GOLD
    from dim_b200 import _native
    from oracle import superglue as o_sg
    from oracle.compare import compare_matches
    from oracle.gen_golden import lg_pair
    g = np.load(os.path.join(GOLD, "superglue_golden.npz"))
    seed, m, n, h, w = [int(x) for x in g[name + ".args"]]
    f0, f1 = lg_pair(seed, m, n, 256, (h, w))
    wts = o_sg.seeded_weights(seed)
    out = _native.SuperGlueNet(ctx, wts, max_kpts=max(m, n)).match(f0, f1)
    ref = o_sg.match(f0, f1, wts)
    assert np.array_equal(ref["matches0"], g[name + ".matches0"])  # the live oracle equals the golden vector of the reference ...
    exp = {"matches": ref["matches"], "scores": ref["matching_scores0"][ref["matches"][:, 0]], "stop": 0}
    rep = compare_matches({**out, "stop": 0}, exp, 0.2, 2e-4)   # ... and the CUDA path equals the oracle
    print(name, rep["n"], "matches, max score delta", rep["max_dscore"], rep["boundary_diffs"])
    assert rep["n"] > 5


def test_superglue_plugin(ctx):
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from oracle import superglue as o_sg
    from oracle.gen_golden import lg_pair
    wts = o_sg.seeded_weights(4)
    f0, f1 = lg_pair(4, 200, 180, 256, (480, 640))
    m = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": wts}))
    got = m._match_pairs(f0, f1)
    exp = o_sg.match(f0, f1, wts)["matches"]
    assert got.dtype == np.int64 and len(got) > 20
    assert len({tuple(r) for r in got} ^ {tuple(r) for r in exp}) <= 1  # a match at the 0.2 threshold may flip
    with pytest.raises(KeyError, match="scores"):
        m._match_pairs({k: v for k, v in f0.items() if k != "scores"}, f1)


def test_pairs_from_lowres_matches_oracle(ctx, sp_weights):
    """pairs_from_lowres (pairs_generator.py:40-235): SuperPoint (hloc wrapper: fix_sampling) on 4 images, LightGlue
    (7 layers, 0.9 / 0.95 / 0.3, no image_size) on all 6 pairs, kept if > min_matches - against the oracle chain."""
    from pathlib import Path
    from dim_b200 import synthetic
    from dim_b200.pairs_generator import LG_LOWRES_CONF, SP_LOWRES_CONF, pairs_from_lowres
    from oracle import lightglue as o_lg
    from oracle import superpoint as o_sp
    a, b = synthetic.synthetic_pair(11, 320)   # b = homography of a: true correspondences
    c, d = synthetic.synthetic_pair(12, 320)   # unrelated to a / b
    images = {"a.jpg": a[:240], "b.jpg": b[:240], "c.jpg": c[:240], "d.jpg": d[:200, :300]}
    names = [Path(n) for n in images]
    conf_lg = {**o_lg.DEFAULT_CONF, **LG_LOWRES_CONF}
    w = o_lg.seeded_weights(conf_lg, seed=2)
    pairs, counts = pairs_from_lowres(names, min_matches=20, lightglue_weights=w, superpoint_weights=sp_weights, images=images,
                                      pair_batch=4, return_counts=True)
    of = {}
    for n, im in images.items():
        f = o_sp.extract(im, sp_weights, SP_LOWRES_CONF)
        of[n] = {"keypoints": f["keypoints"], "descriptors": f["descriptors"]}  # no image_size: extent normalisation
    exp_counts, exp_pairs = [], []
    for i in range(4):
        for j in range(i + 1, 4):
            r = o_lg.match(of[names[i].name], of[names[j].name], w, conf_lg)
            exp_counts.append(len(r["matches"]))
            if len(r["matches"]) > 20:
                exp_pairs.append((names[i], names[j]))
    print("match counts", counts, "oracle", exp_counts)
    assert counts == exp_counts and pairs == exp_pairs
    assert (names[0], names[1]) in pairs


@pytest.mark.parametrize("mode,th", [("nn", 0.0), ("mnn", 0.0), ("snn", 0.9), ("smnn", 0.95)])
@pytest.mark.parametrize("n0,n1", [(700, 650), (512, 777), (130, 129)])
def test_nn_matcher(ctx, mode, th, n0, n1):
    from oracle import nn_match as o_nn
    rng = np.random.default_rng(n0 * 7 + n1)
    a = rng.standard_normal((128, n0)).astype(np.float32); a /= np.linalg.norm(a, axis=0)
    b = rng.standard_normal((128, n1)).astype(np.float32); b /= np.linalg.norm(b, axis=0)
    k = min(n0, n1) // 2
    b[:, :k] = a[:, rng.permutation(n0)[:k]] + 0.3 * rng.standard_normal((128, k)).astype(np.float32)
    b /= np.linalg.norm(b, axis=0)
    a, b = a.astype(np.float16).astype(np.float32), b.astype(np.float16).astype(np.float32)  # as read from features.h5
    idx, dist = ctx.nn_match(a, b, mode, th)
    ridx, rdist = o_nn.kornia_match({"descriptors": a}, {"descriptors": b}, mode, th)
    assert np.array_equal(idx, ridx)
    if len(rdist):
        assert np.abs(dist - rdist).max() < TOL


def test_nn_hloc_golden_and_large_property(ctx, nn_golden):
    """Mutual NN against the in-tree hloc matcher's golden vector (cosine == L2 order on unit vectors), and at
    BASELINE config-5 size (8192 x 256-d) size-independent properties: mutuality, sortedness, idempotence."""
    a, b = nn_golden["plain.desc0"].astype(np.float32), nn_golden["plain.desc1"].astype(np.float32)
    idx, _ = ctx.nn_match(a, b, "mnn")
    m0 = nn_golden["plain.matches0"]
    exp = np.stack([np.nonzero(m0 > -1)[0], m0[m0 > -1]], 1)
    # kornia's match_mnn walks the smaller side (here desc1), so rows come ordered by the second index
    assert {tuple(r) for r in idx} == {tuple(r) for r in exp} and len(idx) == len(exp)
    rng = np.random.default_rng(0)
    d0 = rng.standard_normal((256, 8192)).astype(np.float32); d0 /= np.linalg.norm(d0, axis=0)
    perm = rng.permutation(8192)
    d1 = d0[:, perm] + 0.02 * rng.standard_normal((256, 8192)).astype(np.float32); d1 /= np.linalg.norm(d1, axis=0)
    d0, d1 = d0.astype(np.float16).astype(np.float32), d1.astype(np.float16).astype(np.float32)
    idx, dist = ctx.nn_match(d0, d1, "mnn")
    inv = np.empty(8192, np.int64); inv[perm] = np.arange(8192)
    assert len(idx) == 8192 and np.array_equal(idx[:, 0], np.arange(8192)) and np.array_equal(idx[:, 1], inv)
    back, _ = ctx.nn_match(d1, d0, "mnn")
    assert {tuple(r) for r in idx} == {(j, i) for i, j in back}


def test_pipeline_device_resident_matches_host_path(ctx, sp_weights):
    """extract_dev -> match_dev with features kept in HBM (fp16-rounded like the features.h5 round trip) equals
    the host path extract -> as_half_roundtrip -> match, and both equal the oracle."""
    import torch
    from dim_b200 import _native, synthetic, weights
    from dim_b200.io_h5 import as_half_roundtrip
    from oracle import lightglue as o_lg
    from oracle import superpoint as o_sp
    size, K = 512, 1024
    conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": K}
    g = np.stack(synthetic.synthetic_pair(9, size))
    sp = _sp_net(ctx, sp_weights, conf, 2, size, size)
    w = weights.lightglue_seeded(seed=0)
    lg = _native.LightGlueNet(ctx, w, max_pairs=1, max_kpts=K)
    img = torch.from_numpy(g).cuda()
    kp = torch.zeros(2, K, 2, device="cuda"); sc = torch.zeros(2, K, device="cuda"); de = torch.zeros(2, 256, K, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    sp.extract_dev(img.data_ptr(), 2, size, size, kp.data_ptr(), sc.data_ptr(), de.data_ptr(), cnt.data_ptr(), K, st)
    m = torch.zeros(1, K, 2, dtype=torch.int64, device="cuda"); ms = torch.zeros(1, K, device="cuda")
    nm = torch.zeros(1, dtype=torch.int32, device="cuda"); sl = torch.zeros(1, dtype=torch.int32, device="cuda")
    fd = [_native.FeatsDev(kp[s].data_ptr(), de[s].data_ptr(), cnt[s:s + 1].data_ptr(), K, 0, K, float(size), float(size), 1) for s in range(2)]
    lg.match_dev([fd[0]], [fd[1]], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), sl.data_ptr(), K, st)
    torch.cuda.synchronize()
    n = int(nm[0])
    dev_matches = m[0, :n].cpu().numpy()
    feats = [as_half_roundtrip({**o_sp.extract(x, sp_weights, conf), "image_size": np.array([size, size])}) for x in g]
    # the device path orders keypoints like the oracle only up to top-k ties -> compare through keypoint coordinates
    exp = o_lg.match(feats[0], feats[1], w)
    k0, k1 = kp[0].cpu().numpy(), kp[1].cpu().numpy()
    got = {(tuple(k0[i]), tuple(k1[j])) for i, j in dev_matches}
    want = {(tuple(feats[0]["keypoints"][i]), tuple(feats[1]["keypoints"][j])) for i, j in exp["matches"]}
    assert int(sl[0]) == exp["stop"] and got == want
