"""Batched, device-resident LighterGlue (dimb_lg_match_dev for shape-generic LightGlue): the host entry's staging, batch position and
P invariance, the trained goldens and the oracle on seeded shapes, and ImageSetMatcher on given features (extractor=None): LighterGlue,
kornia_matcher and LightGlue sets against the matcher plugins on the store's features."""
import sqlite3

import numpy as np
import pytest

from conftest import LTG_CASES, ltg_case

K = 2048


def _subset(f, n, seed, perm=False):
    """n seeded keypoints of f (in their order, or permuted), with their descriptors (D,N)."""
    rng = np.random.default_rng(seed)
    N = len(f["keypoints"])
    idx = rng.permutation(N)[:n] if perm else np.sort(rng.choice(N, n, replace=False))
    return {**f, "keypoints": f["keypoints"][idx], "descriptors": f["descriptors"][:, idx]}


# ---------------------------------------------------------------------------------------------------------------- no GPU
def test_given_features_configuration_checks():
    """Every refusal of ImageSetMatcher(extractor=None) and of matcher="lighterglue" happens before anything is built."""
    from dim_b200.sharded import ImageSetMatcher, given_features_conf, lighterglue_conf
    assert lighterglue_conf(None) == {"filter_threshold": 0.1} and lighterglue_conf({"filter_threshold": 0.2})["filter_threshold"] == 0.2
    with pytest.raises(ValueError, match="unknown lighterglue option"):
        lighterglue_conf({"depth_confidence": 0.9})
    assert given_features_conf({"max_keypoints": 8, "descriptor_dim": 64}) == (8, 64)
    for bad in ({}, {"max_keypoints": 8}, {"max_keypoints": 0, "descriptor_dim": 64}, {"max_keypoints": 8, "descriptor_dim": 64, "x": 1}):
        with pytest.raises(ValueError, match="sp_conf"):
            given_features_conf(bad)
    sp = {"max_keypoints": 64, "descriptor_dim": 64}
    mk = lambda **kw: ImageSetMatcher(None, None, None, 2, 100, 120, kw.pop("sp_conf", sp), kw.pop("lg_conf", {}), **kw)
    with pytest.raises(ValueError, match="XFeat features only"):
        mk(matcher="lighterglue", extractor="superpoint")
    with pytest.raises(ValueError, match="XFeat features only"):
        mk(matcher="lighterglue", extractor="aliked")
    with pytest.raises(ValueError, match="64-d"):
        mk(matcher="lighterglue", extractor=None, sp_conf={"max_keypoints": 64, "descriptor_dim": 128})
    with pytest.raises(ValueError, match="unknown lighterglue option"):
        mk(matcher="lighterglue", extractor=None, lg_conf={"width_confidence": 0.9})
    for kw in ({"tiling": {"tile_size": 50}}, {"pair_generation": {"strategy": "matching_lowres"}}, {"upright": {"resize_max": 50}},
               {"quality": "medium"}):
        with pytest.raises(ValueError, match="extractor=None"):
            mk(matcher="lighterglue", extractor=None, **kw)
    with pytest.raises(ValueError, match="256 or 128"):
        mk(matcher="lightglue", extractor=None)
    with pytest.raises(ValueError, match="input_dim"):
        mk(matcher="lightglue", extractor=None, sp_conf={"max_keypoints": 64, "descriptor_dim": 128}, lg_conf={"input_dim": 256})
    with pytest.raises(ValueError, match="256-d"):
        mk(matcher="superglue", extractor=None, sp_conf={"max_keypoints": 64, "descriptor_dim": 128})
    with pytest.raises(ValueError, match="extractor must be"):
        mk(matcher="kornia_matcher", extractor="xfeat")


def test_put_features_checks_every_entry_before_the_first_put():
    from dim_b200.sharded import ImageSetMatcher

    class _Store:
        def __init__(self):
            self.puts = []

        def put(self, slot, f):
            self.puts.append(slot)

    m = ImageSetMatcher.__new__(ImageSetMatcher)
    m.extractor, m.D, m.cap, m.sizes, m.slots, m.store = None, 64, 10, [(100, 120), (90, 80)], [0, 1], _Store()
    good = lambda n, size: {"keypoints": np.zeros((n, 2), np.float32), "descriptors": np.zeros((64, n), np.float32), "image_size": size}
    for bad, what in (([good(3, [100, 120]), good(3, [80, 90])], "image_size"), ([good(3, [100, 120]), good(11, [90, 80])], "max_keypoints"),
                      ([good(3, [100, 120]), {**good(3, [90, 80]), "descriptors": np.zeros((128, 3))}], "descriptors"),
                      ([good(3, [100, 120])], "one FeaturesDict")):
        with pytest.raises(ValueError, match=what):
            m.put_features(bad, [0, 1])
        assert m.store.puts == []
    m.put_features([good(3, [100, 120]), good(10, np.array([90, 80]))], [0, 1])
    assert m.store.puts == [0, 1]


def test_lg_match_dev_rejects_a_null_handle():
    from dim_b200 import _native
    lib = _native.load_library()
    f = (_native.FeatsDev * 1)()
    assert lib.dimb_lg_match_dev(None, 1, f, f, None, None, None, None, 8, None) == _native.ERR_ARG
    assert lib.dimb_lg_match_dev(None, 0, f, f, None, None, None, None, 8, None) == _native.ERR_ARG


# ---------------------------------------------------------------------------------------------------------------- on the GPU
class _Dev:
    """One side on the device as dimb_lg_match_dev reads it: float32 keypoints and descriptors (layout 0 (D,N) or 1 (N,D))."""

    def __init__(self, f, layout=0, size=True, round_fp16=False, pad=3):
        import torch
        from dim_b200 import _native
        k = np.ascontiguousarray(f["keypoints"], np.float32)
        d = np.asarray(f["descriptors"], np.float32)
        n = len(k)
        d = d if layout == 0 else d.T
        ld = d.shape[1] + pad if layout == 0 else d.shape[1]
        buf = np.zeros((d.shape[0], ld) if layout == 0 else d.shape, np.float32)
        buf[:, :d.shape[1]] = d
        self.t = [torch.from_numpy(k).cuda().reshape(-1) if n else torch.zeros(2, device="cuda"), torch.from_numpy(buf).cuda(),
                  torch.tensor([n], dtype=torch.int32, device="cuda")]
        s = _native.FeatsDev()
        s.keypoints, s.descriptors, s.n, s.n_cap = self.t[0].data_ptr(), self.t[1].data_ptr(), self.t[2].data_ptr(), n
        s.desc_layout, s.desc_ld, s.round_fp16 = layout, ld if layout == 0 else 0, int(round_fp16)
        if size:
            s.size0, s.size1 = [float(v) for v in f["image_size"]]
        self.s = s


def _host(f, size=True):
    out = {"keypoints": np.asarray(f["keypoints"], np.float32), "descriptors": np.asarray(f["descriptors"], np.float32), "_layout": 0}
    if size:
        out["image_size"] = f["image_size"]
    return out


def _run_dev(net, sides, cap=K, stream=0):
    import torch
    P = len(sides)
    m = torch.full((P, cap, 2), -7, dtype=torch.int64, device="cuda")
    ms = torch.full((P, cap), -7.0, device="cuda")
    nm = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    sl = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    net.match_dev([a.s for a, _ in sides], [b.s for _, b in sides], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), sl.data_ptr(), cap, stream)
    torch.cuda.synchronize()
    m, ms, nm, sl = m.cpu().numpy(), ms.cpu().numpy(), nm.cpu().numpy(), sl.cpu().numpy()
    return [{"matches": m[p, :min(nm[p], cap)], "scores": ms[p, :min(nm[p], cap)], "stop": int(sl[p]), "n": int(nm[p])} for p in range(P)]


def _as_dev_result(r):
    """A LightGlueNet.match result in the form of _run_dev's."""
    return {**r, "n": len(r["matches"])}


def _bitwise(got, exp, what=""):
    assert got["stop"] == exp["stop"], (what, got["stop"], exp["stop"])
    assert got["n"] == len(exp["matches"]), (what, got["n"], len(exp["matches"]))
    assert np.array_equal(got["matches"], exp["matches"]), what
    assert np.array_equal(got["scores"].view(np.uint32), np.asarray(exp["scores"], np.float32).view(np.uint32)), what


def _ltg_net(ctx, w, conf, max_pairs):
    from dim_b200 import _native
    return _native.LightGlueNet(ctx, w, input_dim=conf["input_dim"], descriptor_dim=conf["descriptor_dim"], n_layers=conf["n_layers"],
                                num_heads=conf["num_heads"], depth_confidence=conf["depth_confidence"],
                                width_confidence=conf["width_confidence"], prune_min_kpts=conf.get("prune_min_kpts", 1536),
                                max_pairs=max_pairs, max_kpts=K)


def _mixed_pairs(f0, f1):
    """(feats0, feats1, explicit size?) for the golden pair, its swap, seeded subsets (pruning fires on some sides only), own-extent
    sides and a pair with an empty side."""
    empty = {**f1, "keypoints": np.zeros((0, 2), np.float32), "descriptors": np.zeros((f1["descriptors"].shape[0], 0), np.float32)}
    return [(f0, f1, True), (f1, f0, True), (_subset(f0, 1536, 1), _subset(f1, 1537, 2), True), (_subset(f0, 700, 3), f1, False),
            (_subset(f1, 9, 4), _subset(f0, 2048, 5, perm=True), True), (f0, empty, True), (_subset(f1, 1537, 6, perm=True), f0, False),
            (_subset(f0, 2000, 7), _subset(f1, 1200, 8), True)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("name", LTG_CASES)
def test_host_staging_and_batch_invariance_trained(ctx, ltg_golden, ltg_weights, name, precision):
    """Trained LighterGlue, each golden configuration, mixed pairs: LightGlueNet.match (host (D,N) arrays staged by dimb_lg_match, the
    own extent of a side without a size computed on the host) at P = 8 equals match_dev on device sides (own extent on the device) at
    P = 1, 4 and 8 and LightGlueNet.match one pair at a time, bit for bit - matches, scores, counts and stop layers - and reproduces the
    reference on the golden pair."""
    from oracle.compare import compare_matches
    f0, f1, conf, ref = ltg_case(ltg_golden, name)
    ctx.set_precision(precision)
    try:
        net = _ltg_net(ctx, ltg_weights, conf, 8)
        pairs = _mixed_pairs(f0, f1)
        host = [(_host(a, s), _host(b, s)) for a, b, s in pairs]
        exp = net.match(host)
        for k, pair in enumerate(host):
            _bitwise(_as_dev_result(net.match([pair])[0]), exp[k], (name, precision, "host P = 1", k))
        sides = [(_Dev(a, size=s), _Dev(b, size=s)) for a, b, s in pairs]
        for P in (1, 4, 8):
            for p0 in range(0, len(pairs), P):
                for k, got in enumerate(_run_dev(net, sides[p0:p0 + P])):
                    _bitwise(got, exp[p0 + k], (name, precision, P, p0 + k))
        assert exp[5]["stop"] == 1 and len(exp[5]["matches"]) == 0
        if precision == "exact":  # the fp32-class mode reproduces the reference (FAST is checked against it by test_fast_mode.py)
            rep = compare_matches(exp[0], ref, 0.1, 2e-4)
            assert rep["n"] > 390 and exp[0]["stop"] == ref["stop"]
    finally:
        ctx.set_precision("exact")


@pytest.mark.gpu
def test_input_forms_batch_position_async_and_cap(ctx, ltg_golden, ltg_weights):
    """(D,N) / (N,D) float32, round_fp16, float16 store slots, own-extent and explicit size give one result; a pair's result does not
    depend on its position or on P; match_dev returns before the device is done; a count above cap is reported whole."""
    import torch
    from dim_b200 import _native
    from dim_b200.io_h5 import as_half_roundtrip
    f0, f1, conf, _ = ltg_case(ltg_golden, "lighterglue_default")
    net = _ltg_net(ctx, ltg_weights, conf, 8)
    r0, r1 = as_half_roundtrip({**f0}), as_half_roundtrip({**f1})
    exp = net.match([(_host(r0), _host(r1))])[0]
    forms = [(_Dev(r0), _Dev(r1)), (_Dev(r0, layout=1), _Dev(r1, layout=1)), (_Dev(f0, round_fp16=True), _Dev(f1, round_fp16=True))]
    store = _native.FeatureStoreDev(ctx, 2, K, 64)
    store.put(0, f0)
    store.put(1, f1)
    slot = [store.feats_dev(s, size=[float(v) for v in f["image_size"]]) for s, f in ((0, f0), (1, f1))]

    class _S:
        def __init__(self, s):
            self.s = s
    forms.append((_S(slot[0]), _S(slot[1])))
    for k, got in enumerate(_run_dev(net, forms)):
        _bitwise(got, exp, ("form", k))
    # own extent computed on the device == the host entry's extent == that extent given explicitly
    own = net.match([(_host(r0, False), _host(r1, False))])[0]
    ext = lambda f: {**f, "image_size": (1 + f["keypoints"].max(0)) - f["keypoints"].min(0)}
    for got in _run_dev(net, [(_Dev(r0, size=False), _Dev(r1, size=False)), (_Dev(ext(r0)), _Dev(ext(r1)))]):
        _bitwise(got, own, "own extent")
    # batch position and P
    pairs = _mixed_pairs(r0, r1)[:6]
    sides = [(_Dev(a, size=s), _Dev(b, size=s)) for a, b, s in pairs]
    fwd, rev = _run_dev(net, sides), _run_dev(net, sides[::-1])[::-1]
    for a, b in zip(fwd, rev):
        _bitwise(a, {**b, "matches": b["matches"]}, "position")
    # asynchronous on its stream
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    m = torch.zeros((1, K, 2), dtype=torch.int64, device="cuda")
    ms, nm, sl = torch.zeros((1, K), device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    net.match_dev([forms[0][0].s], [forms[0][1].s], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), sl.data_ptr(), K, s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy and int(nm.item()) == len(exp["matches"]) and np.array_equal(m[0, :len(exp["matches"])].cpu().numpy(), exp["matches"])
    # cap below the count
    got = _run_dev(net, forms[:1], cap=50)[0]
    assert got["n"] == len(exp["matches"]) > 50 and np.array_equal(got["matches"], exp["matches"][:50])
    # argument errors before any launch
    with pytest.raises(_native.DimbError, match=r"code -3"):
        _run_dev(net, forms[:1] * 9)
    big = _Dev(r0)
    big.s.n_cap = K + 1
    with pytest.raises(_native.DimbError, match=r"code -3"):
        _run_dev(net, [(big, forms[0][1])])
    with pytest.raises(_native.DimbError, match=r"code -3"):
        _run_dev(net, forms[:1], cap=0)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(96, 1), (128, 2)])
def test_seeded_shapes_against_oracle(ctx, ltg_golden, shape):
    """Seeded weights: head dim 96 (tensor-core attention, attn_hd128) and 64 (lgx_attention_kernel), adaptive, EXACT: each pair as the
    oracle matches it (stop layer equal, matches equal but at the filter threshold), and P = 4 staged from the host equal to P = 1 on
    device sides bit for bit."""
    from oracle import lightglue as o_lg
    from oracle.compare import compare_matches
    d, h = shape
    f0, f1, _, _ = ltg_case(ltg_golden, "fixed")
    conf = {**o_lg.DEFAULT_CONF, "input_dim": 64, "descriptor_dim": d, "num_heads": h, "n_layers": 4, "depth_confidence": 0.95,
            "width_confidence": 0.99, "prune_min_kpts": 1024}
    w = o_lg.seeded_weights(conf, seed=5)
    net = _ltg_net(ctx, w, conf, 4)
    pairs = _mixed_pairs(f0, f1)[:4]
    exp = net.match([(_host(a, s), _host(b, s)) for a, b, s in pairs])
    for k, (a, b, s) in enumerate(pairs):
        _bitwise(_run_dev(net, [(_Dev(a, size=s), _Dev(b, size=s))])[0], exp[k], (shape, k))
        ref = o_lg.match(*[f if s else {k_: v for k_, v in f.items() if k_ != "image_size"} for f in (a, b)], w, conf)
        compare_matches(exp[k], ref, conf["filter_threshold"], 2e-4)
    assert max(len(e["matches"]) for e in exp) > 0


def _ltg_images(ltg_golden, n):
    """n given-feature images from the two golden XFeat photos: the photos, then seeded subsets / permutations of their keypoints."""
    f = [{"keypoints": ltg_golden[f"kpts{i}"].astype(np.float32), "descriptors": ltg_golden[f"desc{i}"].astype(np.float32),
          "scores": np.linspace(1, 0.5, len(ltg_golden[f"kpts{i}"])).astype(np.float32), "image_size": ltg_golden[f"size{i}"].astype(np.int32)}
         for i in (0, 1)]
    out = list(f)
    for k in range(2, n):
        g = f[k % 2]
        sub = _subset(g, [2048, 1500, 1800, 900, 1200, 2048][k % 6], 40 + k, perm=k % 3 == 0)
        out.append({**sub, "scores": g["scores"][:len(sub["keypoints"])]})
    return out


@pytest.mark.gpu
def test_lighterglue_image_set(ctx, ltg_golden, ltg_weights, tmp_path):
    """ImageSetMatcher(extractor=None, matcher="lighterglue") on 7 golden-derived images, all 21 pairs: the tables of
    LighterGlueMatcher._match_pairs on store.get, at batch_pairs 1 and 4; verified tables, F and counts equal the host
    geometric_verification + gate; export_colmap writes the tables and the store keypoints."""
    from dim_b200.config import Config
    from dim_b200.geometric_verification import geometric_verification, gv_seed
    from dim_b200.io_colmap import image_ids_to_pair_id
    from dim_b200.matchers.lighterglue import LighterGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    n, seed = 7, 3
    feats = _ltg_images(ltg_golden, n)
    H, W = [int(f["image_size"][0]) for f in feats], [int(f["image_size"][1]) for f in feats]
    pairs = pairs_from_bruteforce(list(range(n)))
    sp = {"max_keypoints": K, "descriptor_dim": 64}
    mk = lambda bp, ver=None: ImageSetMatcher(ctx, None, ltg_weights, n, H, W, sp, {}, batch_pairs=bp, matcher="lighterglue", extractor=None,
                                              verification=ver)
    tables = mk(4).run_features(feats, list(range(n)), pairs)
    eng = mk(1, {"seed": seed})
    res = eng.run_features_verified(feats, list(range(n)), pairs)
    plugin = LighterGlueMatcher(Config(matcher={"name": "lighterglue", "weights_dict": ltg_weights}), local_features="xfeat")
    kept = 0
    for k, ((i, j), (raw, ver, F, ninl)) in enumerate(zip(pairs, res)):
        f0, f1 = eng.store.get(store_slot(i, n, 1)), eng.store.get(store_slot(j, n, 1))
        exp = plugin._match_pairs(f0, f1)
        assert np.array_equal(tables[k], exp) and np.array_equal(raw, exp), (i, j, len(tables[k]), len(exp))
        hF, hmask = geometric_verification(f0["keypoints"][exp[:, 0]], f1["keypoints"][exp[:, 1]], "pydegensac", threshold=1.0,
                                           max_iters=10000, seed=gv_seed(seed, k))
        assert ninl == int(hmask.sum()) and (F is None) == (hF is None) and (F is None or np.array_equal(F, hF)), (i, j)
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(exp))
        assert np.array_equal(ver, exp[hmask] if gate else exp[:0]), (i, j)
        kept += bool(gate)
    assert kept >= 3 and max(len(t) for t in tables) > 300
    db = tmp_path / "database.db"
    eng.export_colmap(pairs, res, db)
    con = sqlite3.connect(str(db))
    kp = {r[0]: np.frombuffer(r[3], np.float32).reshape(r[1], r[2]) for r in con.execute("SELECT * FROM keypoints")}
    for i in range(n):
        assert np.array_equal(kp[i + 1][:, :2], eng.store.get(store_slot(i, n, 1))["keypoints"])
    raw = {r[0]: np.frombuffer(r[3], np.uint32).reshape(r[1], r[2]) for r in con.execute("SELECT pair_id, rows, cols, data FROM matches")}
    for (i, j), t in zip(pairs, tables):
        if len(t):
            assert np.array_equal(raw[image_ids_to_pair_id(i + 1, j + 1)], t)
    con.close()


@pytest.mark.gpu
def test_other_matchers_on_given_features(ctx):
    """kornia_matcher (smnn 0.85) on the cfg1 SIFT golden features (128-d) and LightGlue (seeded, 256-d) on SuperPoint-like features
    put from the host: the tables of KorniaMatcher / LightGlueMatcher._match_pairs on the store's features."""
    import os
    from conftest import GOLD
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    g = np.load(os.path.join(GOLD, "cfg1_sift_golden.npz"))
    sift = [{"keypoints": g[f"kpts{i}"].astype(np.float32), "descriptors": g[f"desc{i}"].astype(np.float32), "image_size": g[f"size{i}"]}
            for i in (0, 1)]
    feats = sift + [_subset(sift[0], 1500, 9, perm=True)]
    n = len(feats)
    pairs = pairs_from_bruteforce(list(range(n)))
    H, W = [int(f["image_size"][0]) for f in feats], [int(f["image_size"][1]) for f in feats]
    eng = ImageSetMatcher(ctx, None, None, n, H, W, {"max_keypoints": 2049, "descriptor_dim": 128}, {"match_mode": "smnn", "th": 0.85},
                          batch_pairs=2, matcher="kornia_matcher", extractor=None)
    tables = eng.run_features(feats, list(range(n)), pairs)
    plugin = KorniaMatcher(Config(pipeline="sift+kornia_matcher", matcher={"match_mode": "smnn", "th": 0.85}))
    for (i, j), t in zip(pairs, tables):
        exp = plugin._match_pairs(eng.store.get(store_slot(i, n, 1)), eng.store.get(store_slot(j, n, 1)))
        assert np.array_equal(t, exp), (i, j)
    assert len(tables[0]) > 50
    rng = np.random.default_rng(0)
    sp = []
    for k in range(4):
        N = [700, 512, 640, 300][k]
        d = rng.standard_normal((256, N)).astype(np.float32)
        sp.append({"keypoints": rng.uniform(0, [319, 239], (N, 2)).astype(np.float32), "descriptors": d / np.linalg.norm(d, axis=0),
                   "scores": rng.uniform(0, 1, N).astype(np.float32), "image_size": np.array([240, 320])})
    sp[1] = {**sp[0], "keypoints": sp[0]["keypoints"][:512] + 0.5, "descriptors": sp[0]["descriptors"][:, :512], "scores": sp[0]["scores"][:512]}
    w = weights.lightglue_seeded(seed=0)
    pairs = pairs_from_bruteforce(list(range(4)))
    eng = ImageSetMatcher(ctx, None, w, 4, 240, 320, {"max_keypoints": 1024, "descriptor_dim": 256}, {}, batch_pairs=4, matcher="lightglue",
                          extractor=None)
    tables = eng.run_features(sp, list(range(4)), pairs)
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    for (i, j), t in zip(pairs, tables):
        exp = plugin._match_pairs(eng.store.get(store_slot(i, 4, 1)), eng.store.get(store_slot(j, 4, 1)))
        assert np.array_equal(t, exp), (i, j)
    assert len(tables[0]) > 20
