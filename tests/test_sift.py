"""SIFT extraction (csrc/sift.cu, dimb_sift_*, SiftNet, the SIFTExtractor plugin) and SIFT image sets
(ImageSetMatcher(extractor="sift", matcher="kornia_matcher")).

The reference is cv2.SIFT_create(...).detectAndCompute of the installed OpenCV, and oracle.sift restates it in numpy.  Keypoints
agree when they lie within 0.01 px, 0.1 degree and 1 % of size of each other; descriptors when every byte is within 1.  Two builds
of OpenCV (its SSE2 baseline against its AVX2 / AVX-512 and IPP paths) agree on all keypoints at n_features 2048 and on 99.94 % at
8000 on a 768 x 1024 image, so the bars below leave room for float rounding near the detector's thresholds, nothing more."""
import ctypes as C

import cv2
import numpy as np
import pytest

from conftest import GOLD

GOLDEN = ["real240x320", "real_odd237x315", "blocks384x512_top512"]
CONF = {"n_layers": 3, "contrast": 0.0004, "edge": 10.0, "sigma": 1.6}  # the sift+kornia_matcher pipeline (config.py)
NET = {"n_octave_layers": 3, "contrast_threshold": 0.0004, "edge_threshold": 10.0, "sigma": 1.6}


def _golden(name):
    return np.load(f"{GOLD}/superpoint_golden.npz")[name + ".image"]


def _synthetic(seed, H, W):
    from dim_b200 import synthetic
    from oracle.sift import to_u8
    return to_u8(synthetic.to_gray_like_reference(synthetic.blocks_image(seed, 256)))[:H, :W].copy()


def _upscale():
    return cv2.resize(_golden("real240x320"), (1024, 768), interpolation=cv2.INTER_LINEAR)


def _check_against(got, ref, what, min_agree=0.995, count_tol=0.005):
    """The bars of this file for features `got` against `ref` (dicts of oracle.sift's layout)."""
    from oracle.sift import agreement
    n_g, n_r = len(got["keypoints"]), len(ref["keypoints"])
    assert abs(n_g - n_r) <= count_tol * n_r, (what, n_g, n_r)
    fa, pairs = agreement(got, ref)
    fb, _ = agreement(ref, got)
    assert fa >= min_agree and fb >= min_agree, (what, fa, fb, n_g, n_r)
    if len(pairs):
        diff = np.abs(got["descriptors"][:, pairs[:, 0]] - ref["descriptors"][:, pairs[:, 1]]).max(0)
        assert np.mean(diff <= 1) >= 0.99, (what, np.mean(diff <= 1))
    return fa, fb


def _tie_count(responses, nf):
    """retainBest(nf) on a deduplicated list: every keypoint at or above the nf-th largest response."""
    if nf <= 0 or len(responses) <= nf:
        return len(responses)
    return int(np.sum(responses >= np.sort(responses)[::-1][nf - 1]))


# ---------------------------------------------------------------------------------------------------------------- no GPU needed

ORACLE_CASES = [("real240x320", 0), ("real_odd237x315", 0), ("blocks384x512_top512", 0), ("real240x320", 50),
                ("real240x320", "boundary"), ("real240x320", "above"), ("synthetic61x93", 0), ("synthetic129x200", 300)]


@pytest.mark.parametrize("name,nf", ORACLE_CASES)
def test_oracle_against_cv2(name, nf):
    """oracle.sift against cv2.SIFT at n_features 0, small, at the boundary (the full count) and above it."""
    from oracle import sift as O
    img = _synthetic(5, *map(int, name[9:].split("x"))) if name.startswith("synthetic") else _golden(name)
    full = O.cv2_extract(img, 0, **CONF)
    nf = {"boundary": len(full["keypoints"]), "above": len(full["keypoints"]) + 100}.get(nf, nf)
    ref = O.cv2_extract(img, nf, **CONF)
    got = O.extract(img, nf, **CONF)
    assert len(ref["keypoints"]) > 0
    _check_against(got, ref, (name, nf))
    # retainBest keeps boundary ties: cv2's count and the oracle's follow the rule on their own uncut responses
    assert len(ref["keypoints"]) == _tie_count(full["response"], nf)
    assert len(got["keypoints"]) == _tie_count(O.extract(img, 0, **CONF)["response"], nf) if nf else True


def test_oracle_tie_rule_matches_cv2_counts():
    """cv2 returns n_features + 1 keypoints for some limits (two orientations of one extremum share a response): its count is
    always the tie rule applied to its uncut responses, and so is the oracle's."""
    from oracle import sift as O
    img = _golden("real240x320")
    full = O.cv2_extract(img, 0, **CONF)["response"]
    over = 0
    for nf in range(40, 1200, 53):
        n = len(O.cv2_extract(img, nf, **CONF)["keypoints"])
        assert n == _tie_count(full, nf), nf
        over += n > nf
    assert over > 0


def test_sift_entries_reject_null_arguments_without_touching_the_gpu():
    """DIMB_ERR_ARG (-3) before any CUDA call."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    conf = _native.SiftConf(2048, 3, 0.0004, 10.0, 1.6, 1, 64, 64)
    h = C.c_void_p()
    assert lib.dimb_sift_create(null, C.byref(conf), C.byref(h)) == -3
    buf = C.c_void_p(16)
    assert lib.dimb_sift_extract_dev(null, buf, 1, 32, 32, buf, buf, None, None, buf, 8, null) == -3
    assert lib.dimb_sift_extract(null, buf, 32, 32, buf, buf, None, None, buf, 8) == -3
    assert lib.dimb_sift_debug_read(null, 0, 0, 0, buf, 4) == -3


def test_plugin_config_and_layouts(monkeypatch):
    """SIFTExtractor: the reference's class attributes and keys, defaults from the sift+kornia_matcher pipeline, and _extract's
    dtypes and layouts (keypoints float32 (N,2), descriptors float64 (128,N), no scores; empty arrays for no keypoints), with the
    device net replaced by a stand-in."""
    from dim_b200 import _native
    from dim_b200.config import Config, confs
    from dim_b200.extractors.sift import SIFT_KEYS, SIFTExtractor, sift_conf
    assert SIFTExtractor.grayscale is True and SIFTExtractor.as_float is False and SIFTExtractor.descriptor_size == 128
    assert {k: SIFTExtractor._default_conf[k] for k in SIFT_KEYS} == {k: confs["sift+kornia_matcher"]["extractor"][k] for k in SIFT_KEYS}
    assert sift_conf(SIFTExtractor._default_conf) == {"n_features": 2048, **NET}
    monkeypatch.setattr(_native.Context, "get", classmethod(lambda cls, device=0: None))

    class Fake:
        def __init__(self, n):
            self.n = n

        def extract(self, image):
            return {"keypoints": np.ones((self.n, 2), np.float32), "descriptors": np.full((128, self.n), 7, np.float32)}

    ext = SIFTExtractor(Config(extractor={"name": "sift", "n_features": 100}, pipeline="sift+kornia_matcher"))
    assert ext._conf["n_features"] == 100 and ext._conf["contrast_threshold"] == 0.0004
    for n in (5, 0):
        ext._net, ext._net_shape = Fake(n), (64, 64)
        f = ext._extract(np.zeros((32, 48), np.uint8))
        assert set(f) == {"keypoints", "descriptors"}
        assert f["keypoints"].dtype == np.float32 and f["keypoints"].shape == (n, 2)
        assert f["descriptors"].dtype == np.float64 and f["descriptors"].shape == (128, n)
    with pytest.raises(ValueError, match="uint8"):
        ext._extract(np.zeros((32, 48), np.float32))


def test_image_set_conf_and_refusals():
    """sp_conf of a SIFT set and every option that is refused, before anything is allocated (no context needed)."""
    from dim_b200.sharded import ImageSetMatcher, sift_set_conf
    assert sift_set_conf({"n_features": 512}) == {"n_features": 512, **NET}
    assert sift_set_conf({"name": "sift", "n_features": 8, "sigma": 2.0})["sigma"] == 2.0
    with pytest.raises(ValueError, match="n_features >= 1"):
        sift_set_conf({"n_features": 0})
    with pytest.raises(ValueError, match="unknown SIFT option"):
        sift_set_conf({"n_features": 8, "max_keypoints": 8})
    sp = {"n_features": 256}
    kw = {"extractor": "sift", "matcher": "kornia_matcher"}
    for matcher in ("lightglue", "superglue"):
        with pytest.raises(ValueError, match=f"matcher '{matcher}'"):
            ImageSetMatcher(None, None, None, 2, 256, 256, sp, {}, extractor="sift", matcher=matcher)
    with pytest.raises(ValueError, match="tiling"):
        ImageSetMatcher(None, None, None, 2, 512, 512, sp, {}, tiling={"tile_size": 256}, **kw)
    with pytest.raises(ValueError, match="tiling"):
        ImageSetMatcher(None, None, None, 2, 1024, 1024, sp, {}, tiling={"tile_size": 512, "tile_selection": "preselection",
                                                                          "tile_preselection_size": 256}, **kw)
    with pytest.raises(ValueError, match="quality"):
        ImageSetMatcher(None, None, None, 2, 256, 256, sp, {}, quality="medium", **kw)
    with pytest.raises(ValueError, match="upright"):
        ImageSetMatcher(None, None, None, 2, 256, 256, sp, {}, upright={"resize_max": 128}, **kw)
    with pytest.raises(ValueError, match="pair_generation"):
        ImageSetMatcher(None, None, None, 2, 256, 256, sp, {}, pair_generation={"strategy": "matching_lowres"}, **kw)
    with pytest.raises(ValueError, match="n_features >= 1"):
        ImageSetMatcher(None, None, None, 2, 256, 256, {"n_features": 0}, {}, **kw)


# ---------------------------------------------------------------------------------------------------------------- on the GPU

def _as_oracle(f):
    return {k: f[k] for k in ("keypoints", "size", "angle", "response", "octave", "descriptors")}


def _net(ctx, nf, H, W, B=1):
    from dim_b200 import _native
    return _native.SiftNet(ctx, n_features=nf, max_batch=B, max_height=H, max_width=W, **NET)


@pytest.mark.gpu
@pytest.mark.parametrize("name,nf", [("real240x320", 0), ("real_odd237x315", 0), ("blocks384x512_top512", 0), ("real240x320", 50),
                                     ("upscale768x1024", 2048), ("upscale768x1024", 8000), ("upscale768x1024", 0),
                                     ("synthetic61x93", 0), ("synthetic129x200", 300)])
def test_device_against_cv2(ctx, name, nf):
    from oracle import sift as O
    if name.startswith("upscale"):
        img = _upscale()
    elif name.startswith("synthetic"):
        img = _synthetic(5, *map(int, name[9:].split("x")))
    else:
        img = _golden(name)
    H, W = img.shape
    got = _net(ctx, nf, H, W).extract(img)
    ref = O.cv2_extract(img, nf, **CONF)
    _check_against(_as_oracle(got), ref, (name, nf))
    assert got["descriptors"].min() >= 0 and got["descriptors"].max() <= 255
    assert np.array_equal(got["descriptors"], np.rint(got["descriptors"]))


@pytest.mark.gpu
@pytest.mark.parametrize("name,nf", [("real240x320", 0), ("real_odd237x315", 500)])
def test_device_against_oracle(ctx, name, nf):
    from oracle import sift as O
    img = _golden(name)
    got = _net(ctx, nf, *img.shape).extract(img)
    ref = O.extract(img, nf, **CONF)
    _check_against(_as_oracle(got), ref, (name, nf))
    fa, pairs = O.agreement(_as_oracle(got), ref)
    oa, ob = got["octave"][pairs[:, 0]], ref["octave"][pairs[:, 1]]
    assert np.array_equal(oa & 0xffff, ob & 0xffff)  # octave and layer; the top byte, the layer offset in 1/255, within 1
    assert np.all(np.abs((oa >> 16) - (ob >> 16)) <= 1)


@pytest.mark.gpu
def test_pyramid_levels_against_float64_restatement(ctx):
    """Every Gaussian and DoG level (debug taps) within 2.5e-4 of the oracle's (float64 taps and sums, 0..255 scale)."""
    from oracle import sift as O
    img = _golden("real_odd237x315")
    H, W = img.shape
    net = _net(ctx, 0, H, W)
    net.extract(img)
    gauss, dog = O.pyramid(img, 3, 1.6)
    for o in range(len(gauss)):
        for i, g in enumerate(gauss[o]):
            assert np.abs(net.debug_read(0, 0, o, i, H, W) - g).max() <= 2.5e-4, ("gauss", o, i)
        for i, d in enumerate(dog[o]):
            assert np.abs(net.debug_read(1, 0, o, i, H, W) - d).max() <= 2.5e-4, ("dog", o, i)


def _dev_extract(net, imgs, cap):
    import torch
    B, H, W = imgs.shape
    d = torch.from_numpy(imgs.astype(np.float32)).cuda()
    kp = torch.full((B, cap, 2), -1.0, device="cuda")
    de = torch.full((B, 128, cap), -1.0, device="cuda")
    fr = torch.full((B, cap, 3), -1.0, device="cuda")
    oc = torch.full((B, cap), -1, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    net.extract_dev(d.data_ptr(), B, H, W, kp.data_ptr(), de.data_ptr(), cnt.data_ptr(), cap, fr.data_ptr(), oc.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in (kp, de, fr, oc, cnt)]


@pytest.mark.gpu
def test_deterministic_across_runs_and_batch_positions(ctx):
    """Bitwise the same output on two runs, and for an image alone and in a batch of 16 (atomic appends, then a total-order sort)."""
    from dim_b200 import synthetic
    base = _golden("real240x320")
    imgs = np.stack([base] + [synthetic.warp_pair(base, k, jitter=20.0) for k in range(1, 16)])
    net = _net(ctx, 0, 240, 320, B=16)
    cap = 3000
    a = _dev_extract(net, imgs, cap)
    b = _dev_extract(net, imgs, cap)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert a[4].min() > 500 and a[4].max() <= cap
    for k in (0, 7, 15):
        one = _dev_extract(net, imgs[k:k + 1], cap)
        for x, y in zip(one, a):
            assert np.array_equal(x[0], y[k]), k
    # float input is converted as convertTo(CV_8U): a fractional image gives the rounded image's features
    frac = _dev_extract(net, imgs[:1] + 0.3, cap)
    assert all(np.array_equal(x[0], y[0]) for x, y in zip(frac, a))


@pytest.mark.gpu
def test_flat_image_has_no_keypoints(ctx):
    from dim_b200.config import Config
    from dim_b200.extractors.sift import SIFTExtractor
    img = np.full((200, 300), 128, np.uint8)
    assert len(_net(ctx, 2048, 200, 300).extract(img)["keypoints"]) == 0
    f = SIFTExtractor(Config(pipeline="sift+kornia_matcher"))._extract(img)
    assert f["keypoints"].shape == (0, 2) and f["descriptors"].shape == (128, 0) and f["descriptors"].dtype == np.float64


@pytest.mark.gpu
def test_n_features_ties(ctx):
    """retainBest on the device: the kept rows are exactly the uncut list's rows with a response at or above the n_features-th,
    in the uncut order (bitwise), and some limits keep more than n_features, as cv2 does."""
    img = _golden("real240x320")
    full = _net(ctx, 0, *img.shape).extract(img)
    over = 0
    for nf in list(range(40, 1200, 53)) + [len(full["keypoints"]) - 1]:
        cut = _net(ctx, nf, *img.shape).extract(img)
        t = np.sort(full["response"])[::-1][nf - 1]
        keep = full["response"] >= t
        assert len(cut["keypoints"]) == _tie_count(full["response"], nf), nf
        for k in ("keypoints", "descriptors", "response", "octave"):
            exp = full[k][:, keep] if k == "descriptors" else full[k][keep]
            assert np.array_equal(cut[k], exp), (nf, k)
        over += len(cut["keypoints"]) > nf
    assert over > 0


def _coord_matches(f0, f1, m):
    return np.concatenate([f0["keypoints"][m[:, 0]], f1["keypoints"][m[:, 1]]], 1)


def _shared(a, b, tol=0.01):
    if len(a) == 0:
        return 1.0
    hit = 0
    for r in a:
        hit += bool(np.any(np.all(np.abs(b - r) <= tol, axis=1)))
    return hit / len(a)


@pytest.mark.gpu
def test_smnn_tables_on_a_warped_pair_match_cv2_features(ctx):
    """smnn 0.85 (the sift+kornia_matcher pipeline) on a warped pair: the matches from device features and from cv2 features agree
    on at least 99 % of matches, as keypoint-coordinate pairs within 0.01 px, both ways."""
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from oracle import sift as O
    img0 = _upscale()[:480, :640].copy()
    img1 = synthetic.warp_pair(img0, 3, jitter=30.0)
    plugin = KorniaMatcher(Config(pipeline="sift+kornia_matcher"))
    net = _net(ctx, 2048, 480, 640)
    dev = [net.extract(x) for x in (img0, img1)]
    ref = [O.cv2_extract(x, 2048, **CONF) for x in (img0, img1)]
    md = _coord_matches(*dev, plugin._match_pairs(*dev))
    mr = _coord_matches(*ref, plugin._match_pairs(*ref))
    assert len(mr) > 100
    assert _shared(md, mr) >= 0.99 and _shared(mr, md) >= 0.99, (len(md), len(mr))


def _set_images():
    from dim_b200 import synthetic
    base = _upscale()[:360, :480].copy()
    return [base] + [synthetic.warp_pair(base, 20 + k, jitter=24.0) for k in range(1, 4)]


def _plugin(nf):
    from dim_b200.config import Config
    from dim_b200.extractors.sift import SIFTExtractor
    return SIFTExtractor(Config(extractor={"n_features": nf}, pipeline="sift+kornia_matcher"))


def _check_store(eng, imgs, nf):
    """The store's features are the plugin's after the float16 cast, bitwise (scores are the ones of a score-less extractor)."""
    ext = _plugin(nf)
    for i, img in enumerate(imgs):
        f = ext._extract(img)
        s = eng.store.get(i)
        assert np.array_equal(s["keypoints"], f["keypoints"].astype(np.float16).astype(np.float32)), i
        assert np.array_equal(s["descriptors"], f["descriptors"].astype(np.float16).astype(np.float32)), i
        assert np.all(s["scores"] == 1) and list(s["image_size"]) == list(img.shape)


@pytest.mark.gpu
def test_image_set_store_tables_verified_and_colmap(ctx, tmp_path):
    import sqlite3

    import torch
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    imgs = _set_images()
    nf = 1024
    pairs = pairs_from_bruteforce(list(range(4)))
    eng = ImageSetMatcher(ctx, None, None, 4, 360, 480, {"n_features": nf}, {"match_mode": "smnn", "th": 0.85}, batch_images=3,
                          batch_pairs=4, extractor="sift", matcher="kornia_matcher", verification={"seed": 3})
    d = torch.from_numpy(np.stack(imgs).astype(np.float32)).cuda()
    tables = eng.run(d, list(range(4)), pairs)
    _check_store(eng, imgs, nf)
    plugin = KorniaMatcher(Config(pipeline="sift+kornia_matcher"))
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(eng.store.get(i), eng.store.get(j))), (i, j)
    assert min(len(t) for t in tables) > 20
    res = eng.run_verified(d, list(range(4)), pairs)
    assert all(np.array_equal(r[0], t) for r, t in zip(res, tables)) and sum(len(r[1]) for r in res) > 0
    db = tmp_path / "sift.db"
    eng.export_colmap(pairs, res, db)
    con = sqlite3.connect(str(db))
    rows = dict(con.execute("SELECT image_id, rows FROM keypoints").fetchall())
    con.close()
    assert rows == {i + 1: eng.store.count(i)[0] for i in range(4)}
    # more keypoints than the store's n_features + SIFT_TIE_ROOM rows is an error at exchange, never a silent cut
    eng.extract(d, list(range(4)))
    eng.sift_counts[2] = eng.cap + 1
    with pytest.raises(RuntimeError, match="image 2"):
        eng.exchange()


@pytest.mark.gpu
def test_image_set_mixed_sizes(ctx):
    import torch
    from dim_b200.sharded import ImageSetMatcher
    from oracle.sift import to_u8
    imgs = [x[:h, :w].copy() for x, (h, w) in zip(_set_images(), [(360, 480), (300, 480), (360, 400), (301, 479)])]
    nf = 700
    eng = ImageSetMatcher(ctx, None, None, 4, [x.shape[0] for x in imgs], [x.shape[1] for x in imgs], {"n_features": nf}, {},
                          batch_images=2, batch_pairs=3, extractor="sift", matcher="kornia_matcher")
    tables = eng.run([torch.from_numpy(x.astype(np.float32)).cuda() for x in imgs], list(range(4)), [(0, 1), (0, 2), (1, 3), (2, 3)])
    _check_store(eng, [to_u8(x) for x in imgs], nf)
    assert min(len(t) for t in tables) > 10
