"""Image sets of mixed sizes in ImageSetMatcher: per-image height / width through extraction (plain, tiled, quality), tile views and
selection, tile preselection (dimb_tile_preselect_pairs_dev), pair generation, verification and the COLMAP export, checked against
the host flows that read each image at its own size.  Every comparison is exact."""
import ctypes as C
import sqlite3

import cv2
import numpy as np
import pytest

F = np.float32
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 1024}
AL_CONF = {"max_num_keypoints": 1024, "detection_threshold": 0.2, "nms_radius": 3}
# landscape, portrait and an odd size; batch_images=2 puts a batch boundary inside the landscape group
MIXED = [(768, 1024), (1024, 768), (768, 1024), (601, 797), (1024, 768), (768, 1024)]
PAIRS = [(i, j) for i in range(len(MIXED)) for j in range(i + 1, len(MIXED))]


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


def test_constructor_rejects_bad_size_forms():
    from dim_b200.sharded import ImageSetMatcher, image_sizes
    assert image_sizes(2, 768, 1024) == [(768, 1024)] * 2
    assert image_sizes(2, [768, 1024], (1024, np.int64(768))) == [(768, 1024), (1024, 768)]
    bad = [(3, [768, 1024], [1024, 768]),     # length != n_images
           (2, [768, 1024], [1024, 768, 5]),
           (2, [768, 1024], 1024),            # sequence and int mixed
           (2, 768, (1024, 768)),
           (2, [768, 0], [1024, 768]),        # sizes below 1
           (2, [768, 1024], [1024, -1]),
           (2, 0, 1024),
           (2, [768.0, 1024], [1024, 768]),   # not ints
           (2, [True, 1024], [1024, 768]),
           (0, [], [])]
    for n, h, w in bad:
        with pytest.raises(ValueError):
            image_sizes(n, h, w)
        with pytest.raises(ValueError):
            ImageSetMatcher(None, {}, {}, n, h, w, SP_CONF, {})


def test_constructor_checks_every_per_size_rule_per_image():
    from dim_b200.sharded import ImageSetMatcher
    hs, ws = [768, 120], [1024, 160]
    with pytest.raises(ValueError, match="16 px"):  # 120 x 160 at "lowest" is 15 x 20
        ImageSetMatcher(None, {}, {}, 2, hs, ws, SP_CONF, {}, quality="lowest")
    with pytest.raises(ValueError, match="32 px"):
        ImageSetMatcher(None, {}, {}, 2, hs, ws, AL_CONF, {}, extractor="aliked", quality="low")
    pre = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 900}
    with pytest.raises(ValueError, match="downscales"):  # 900 > 800, the second image's longest side
        ImageSetMatcher(None, {}, {}, 2, [768, 600], [1024, 800], SP_CONF, {}, tiling=pre)
    with pytest.raises(ValueError, match="to nothing"):  # 1 x 4000 at longest side 2 is 0 x 2
        ImageSetMatcher(None, {}, {}, 2, [768, 1], [1024, 4000], SP_CONF, {}, tiling={**pre, "tile_preselection_size": 2})
    with pytest.raises(ValueError, match="resize_max"):
        ImageSetMatcher(None, {}, {}, 2, [768, 1], [1024, 4000], SP_CONF, {}, pair_generation={"strategy": "matching_lowres", "resize_max": 2})
    with pytest.raises(ValueError, match="2048 tiles"):  # tiles of 32: 768 for 768 x 1024, 16384 for 4096 x 4096
        ImageSetMatcher(None, {}, {}, 2, [768, 4096], [1024, 4096], {**SP_CONF, "fix_sampling": True}, {}, tiling={"tile_size": 32})
    with pytest.raises(ValueError, match="superpoint"):  # the refusals that do not depend on sizes keep their messages
        ImageSetMatcher(None, {}, {}, 2, hs, ws, AL_CONF, {}, extractor="aliked", pair_generation={"strategy": "matching_lowres"})


@pytest.mark.parametrize("tile, overlap", [((512, 384), 64), (1024, 128)])
def test_tile_pairs_for_equals_tile_selection(tile, overlap):
    from dim_b200 import _native, tiling
    from dim_b200.sharded import tile_pairs_for
    sizes = [(1536, 2048), (2048, 1536), (1000, 1300), (1300, 1000), (512, 512)]
    (th, tw), ov = tiling._hw(tile), tiling._hw(overlap)
    counts = {s: len(_native.tile_grid(*s, th, tw, *ov)["origins"]) for s in sizes}
    assert len(set(counts.values())) > 2, counts
    for s0 in sizes:
        for s1 in sizes:
            i0, i1 = np.zeros(s0, F), np.zeros(s1, F)
            for sel in ("grid", "exhaustive"):
                exp = [(int(a), int(b)) for a, b in tiling.tile_selection(i0, i1, sel, tile, overlap)]
                assert tile_pairs_for(sel, counts[s0], counts[s1]) == exp, (s0, s1, sel)
            assert tile_pairs_for("grid", counts[s0]) == tile_pairs_for("grid", counts[s0], counts[s0])


def test_tile_preselect_pairs_dev_rejects_bad_arguments_without_touching_the_gpu():
    """Argument validation comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    feats = (_native.FeatsDev * 2)()
    for f in feats:
        f.keypoints = 0x1000
    no_kpts = (_native.FeatsDev * 2)()
    good_sizes = [768, 1024, 1024, 768] * 2
    good_scales = [0.5, 0.375] * 2

    def pre(ctx=ctx, Q=2, f0=feats, f1=feats, m=dev, nm=dev, cap=64, sizes=good_sizes, tile=(512, 512), ov=64, scales=good_scales, mm=5,
            cnt=dev, fl=dev):
        sz = None if sizes is None else (C.c_int * len(sizes))(*sizes)
        sc = None if scales is None else (C.c_double * len(scales))(*scales)
        return lib.dimb_tile_preselect_pairs_dev(ctx, Q, f0, f1, m, nm, cap, sz, tile[0], tile[1], ov, ov, sc, mm, cnt, fl, null)
    assert pre(ctx=null) == -3 and pre(f0=None) == -3 and pre(f1=None) == -3 and pre(m=null) == -3 and pre(nm=null) == -3
    assert pre(sizes=None) == -3 and pre(scales=None) == -3 and pre(cnt=null) == -3 and pre(fl=null) == -3
    assert pre(f0=no_kpts) == -3 and pre(f1=no_kpts) == -3
    assert pre(Q=0) == -3 and pre(Q=65536) == -3 and pre(cap=0) == -3 and pre(mm=-1) == -3
    assert pre(tile=(0, 512)) == -3 and pre(ov=512) == -3 and pre(tile=(16, 16), ov=0) == -3  # bad grid (too many tiles) on both sides
    for k in range(8):  # a bad size on either side of either pair
        for v in (0, -5, (1 << 20) + 1):
            sizes = list(good_sizes)
            sizes[k] = v
            assert pre(sizes=sizes) == -3, (k, v)
    for k in range(4):
        for v in (0.0, -0.5, float("inf"), float("nan"), 1e-300):  # 1e-300 is 0 in float32
            scales = list(good_scales)
            scales[k] = v
            assert pre(scales=scales) == -3, (k, v)


def test_tile_preselect_pairs_dev_python_wrapper_checks_row_counts():
    from dim_b200 import _native
    c = _native.Context.__new__(_native.Context)  # no device: the row check comes before the library call
    f = _native.FeatsDev()
    with pytest.raises(ValueError, match="one size row"):
        c.tile_preselect_pairs_dev([f, f], [f, f], 0, 0, 8, [(768, 1024, 768, 1024)], 512, 512, 0, 0, [(0.5, 0.5)] * 2, 5, 0, 0)


# ---------------------------------------------------------------------------------------------------------------- on the GPU


def _mixed_rgb(sizes, seed=40):
    """Crops of one blocks scene at small offsets, each warped: images of any sizes that share content."""
    from dim_b200 import synthetic
    scene = synthetic.blocks_image(seed, max(max(s) for s in sizes) + 64)
    out = []
    for k, (H, W) in enumerate(sizes):
        crop = np.ascontiguousarray(scene[8 * k:8 * k + H, 4 * k:4 * k + W])
        out.append(crop if k == 0 else synthetic.warp_pair(crop, seed + k, jitter=0.02 * max(H, W)))
    return out


def _mixed_gray(sizes, seed=40):
    from dim_b200 import synthetic
    return [synthetic.to_gray_like_reference(np.ascontiguousarray(x)).astype(F) for x in _mixed_rgb(sizes, seed)]


def _dev(imgs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x, F)).cuda() for x in imgs]


def _host_features(ext, img, quality="high", tiled=False):
    """The reference's flow per image: _resize_image, _extract (or _extract_by_tile), _resize_features, own image_size, float16."""
    from dim_b200.io_h5 import as_half_roundtrip
    small = ext._resize_image(quality, img)
    f = ext._extract_by_tile(small) if tiled else ext._extract(small)
    f = ext._resize_features(quality, f)
    return as_half_roundtrip({**f, "image_size": np.array(img.shape[:2])})


def _same_features(got, ref, keys=("keypoints", "descriptors", "scores", "image_size")):
    for k in keys:
        assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), k


def _sp_extractor(sp_weights, tile=None, overlap=0, K=1024):
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    if tile is None:
        return SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={**SP_CONF, "max_keypoints": K}))
    return SuperPointExtractor(Config(general={"tile_size": tile, "tile_overlap": overlap},
                                      extractor={**SP_CONF, "fix_sampling": True, "max_keypoints": K, "weights_dict": sp_weights}))


def _lg_plugin(w, features="superpoint"):
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
    return LightGlueMatcher(Config(pipeline=f"{features}+lightglue", matcher={"weights_dict": w}), local_features=features)


def _engine(ctx, sp_weights, w, sizes, conf=SP_CONF, **kw):
    from dim_b200.sharded import ImageSetMatcher
    kw.setdefault("batch_images", 2)
    kw.setdefault("batch_pairs", 4)
    return ImageSetMatcher(ctx, sp_weights, w, len(sizes), [h for h, _ in sizes], [x for _, x in sizes], conf, kw.pop("lg_conf", {}), **kw)


@pytest.fixture(scope="module")
def mixed(ctx, sp_weights):
    from dim_b200 import weights
    imgs = _mixed_gray(MIXED)
    w = weights.lightglue_seeded(seed=0)
    ext = _sp_extractor(sp_weights)
    feats = [_host_features(ext, im) for im in imgs]
    return {"imgs": imgs, "d": _dev(imgs), "w": w, "feats": feats}


def _planted_pair(s0, s1, sc0, sc1, tile, ov, seed):
    """Low-resolution keypoints (float32) and a match table of one pair of different sizes: tile-box edges of both grids (multiples
    of the dyadic scales, so kpt / scale lands on the edge again) matched in order, plus random points."""
    from dim_b200 import _native, tiling
    (th, tw), ovh = tiling._hw(tile), tiling._hw(ov)
    rng = np.random.default_rng(seed)
    pts = []
    for (H, W) in (s0, s1):
        g = _native.tile_grid(H, W, th, tw, *ovh)
        edges = [(ox + dx, oy + dy) for ox, oy in g["origins"] for dx, dy in ((0, 5), (tw, 7), (9, 0), (11, th), (tw // 2, th // 2))]
        rnd = np.stack([rng.uniform(-g["pad_left"] - 8, W + 8, 400), rng.uniform(-g["pad_top"] - 8, H + 8, 400)], 1)
        pts.append(np.concatenate([np.array(edges, np.float64), rnd]))
    n0, n1 = len(pts[0]), len(pts[1])
    e = min(n0, n1) - 400
    m = np.concatenate([np.stack([np.arange(e), np.arange(e)], 1), np.stack([rng.integers(0, n0, 500), rng.integers(0, n1, 500)], 1)])
    return [(pts[0] * sc0).astype(F), (pts[1] * sc1).astype(F)], m.astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("tile, ov", [((512, 512), 64), ((384, 256), 32)])
def test_tile_preselect_pairs_dev_equals_tile_selection(ctx, tile, ov):
    """Pairs of different sizes and scales against tiling.tile_selection on planted matches (CSR blocks of T0 x T1 flags), and on
    pairs of one geometry the counts and flags of dimb_tile_preselect_dev bitwise."""
    import torch
    from dim_b200 import _native, tiling
    (th, tw), ovh = tiling._hw(tile), tiling._hw(ov)
    geo = [((768, 1024), (1024, 768), 0.5, 0.375), ((1000, 1300), (768, 1024), 0.25, 0.5), ((1024, 768), (601, 797), 0.375, 0.25),
           ((768, 1024), (768, 1024), 0.5, 0.5)]
    cases = [_planted_pair(s0, s1, a, b, tile, ov, k) for k, (s0, s1, a, b) in enumerate(geo)]
    cap = max(len(m) for _, m in cases)
    keep, f0, f1 = [], [], []
    d_m = torch.zeros(len(cases), cap, 2, dtype=torch.int64, device="cuda")
    d_nm = torch.tensor([len(m) for _, m in cases], dtype=torch.int32, device="cuda")
    for q, (low, m) in enumerate(cases):
        d_m[q, :len(m)] = torch.from_numpy(m).cuda()
        for side, lst in ((0, f0), (1, f1)):
            t = torch.from_numpy(low[side]).cuda()
            keep.append(t)
            f = _native.FeatsDev()
            f.keypoints = t.data_ptr()
            lst.append(f)
    T = [(len(_native.tile_grid(*s0, th, tw, *ovh)["origins"]), len(_native.tile_grid(*s1, th, tw, *ovh)["origins"])) for s0, s1, _, _ in geo]
    assert any(a != b for a, b in T)
    off = np.cumsum([0] + [a * b for a, b in T])
    for mm in (0, 5):
        counts = torch.full((int(off[-1]),), -1, dtype=torch.int32, device="cuda")
        flags = torch.full((int(off[-1]),), 7, dtype=torch.uint8, device="cuda")
        ctx.tile_preselect_pairs_dev(f0, f1, d_m.data_ptr(), d_nm.data_ptr(), cap, [s0 + s1 for s0, s1, _, _ in geo], th, tw, *ovh,
                                     [(a, b) for _, _, a, b in geo], mm, counts.data_ptr(), flags.data_ptr(), 0)
        counts, flags = counts.cpu().numpy(), flags.cpu().numpy()
        for q, ((s0, s1, a, b), (low, m)) in enumerate(zip(geo, cases)):
            kp0, kp1 = low[0][m[:, 0]] / a, low[1][m[:, 1]] / b
            assert kp0.dtype == F
            lst = tiling.tile_selection(np.zeros(s0, F), np.zeros(s1, F), "preselection", tile, ov, kp0=kp0, kp1=kp1, min_matches_per_tile=mm)
            fq = flags[off[q]:off[q + 1]].reshape(T[q])
            assert [(int(x), int(y)) for x, y in zip(*np.nonzero(fq))] == lst, (mm, q)
            assert len(lst) > 0 and np.array_equal(fq, counts[off[q]:off[q + 1]].reshape(T[q]) > mm)
        # the same pair of one geometry through the single-geometry entry
        q = 3
        (H, W), _, sc, _ = geo[q]
        c1 = torch.full((1, T[q][0] * T[q][1]), -1, dtype=torch.int32, device="cuda")
        fl1 = torch.full((1, T[q][0] * T[q][1]), 7, dtype=torch.uint8, device="cuda")
        ctx.tile_preselect_dev([f0[q]], [f1[q]], d_m[q:].data_ptr(), d_nm[q:].data_ptr(), cap, H, W, th, tw, *ovh, sc, sc, mm, c1.data_ptr(),
                               fl1.data_ptr(), 0)
        assert np.array_equal(c1.cpu().numpy()[0], counts[off[q]:off[q + 1]]) and np.array_equal(fl1.cpu().numpy()[0], flags[off[q]:off[q + 1]])


@pytest.mark.gpu
def test_mixed_set_lightglue_equals_host_flow(ctx, sp_weights, mixed, tmp_path):
    """Every slot equals _extract + as_half_roundtrip with the image's own image_size, every table the plugin's _match_pairs;
    run_verified + export_colmap give every image a camera of its own width and height."""
    s = mixed
    eng = _engine(ctx, sp_weights, s["w"], MIXED, verification={"seed": 3})
    assert eng.H is None and eng.W is None and eng.h2 is None and eng.sizes == MIXED
    tables = eng.run(s["d"], list(range(len(MIXED))), PAIRS)
    for i, f in enumerate(s["feats"]):
        _same_features(eng.store.get(i), f)
    plugin = _lg_plugin(s["w"])
    for (i, j), t in zip(PAIRS, tables):
        assert np.array_equal(t, plugin._match_pairs(s["feats"][i], s["feats"][j])), (i, j)
    assert max(len(t) for (i, j), t in zip(PAIRS, tables) if MIXED[i] == MIXED[j][::-1] and MIXED[i][0] != MIXED[i][1]) > 0
    res = eng.run_verified(s["d"], list(range(len(MIXED))), PAIRS)
    assert all(np.array_equal(r[0], t) for r, t in zip(res, tables)) and sum(len(r[1]) for r in res) > 0
    db = tmp_path / "mixed.db"
    ids = eng.export_colmap(PAIRS, res, db)
    con = sqlite3.connect(str(db))
    cams = {r[0]: (r[1], r[2]) for r in con.execute("SELECT camera_id, width, height FROM cameras")}
    img_cam = {r[0]: r[1] for r in con.execute("SELECT name, camera_id FROM images")}
    con.close()
    for i, (H, W) in enumerate(MIXED):
        assert cams[img_cam[f"image_{i}"]] == (W, H), i
    assert len(ids) == len(MIXED)


@pytest.mark.gpu
def test_mixed_set_superglue_and_kornia(ctx, sp_weights, mixed):
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from oracle import superglue as o_sg
    s = mixed
    w_sg = o_sg.seeded_weights(1)
    sg_conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
    eng = _engine(ctx, sp_weights, w_sg, MIXED, matcher="superglue", lg_conf=sg_conf)
    tables = eng.run(s["d"], list(range(len(MIXED))), PAIRS)
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": w_sg}))
    for (i, j), t in zip(PAIRS, tables):
        assert np.array_equal(t, plugin._match_pairs(s["feats"][i], s["feats"][j])), (i, j)
    assert sum(len(t) for t in tables) > 0
    eng = _engine(ctx, sp_weights, None, MIXED, matcher="kornia_matcher", lg_conf={"match_mode": "smnn", "th": 0.8})
    tables = eng.run(s["d"], list(range(len(MIXED))), PAIRS)
    plugin = KorniaMatcher(Config(matcher={"name": "kornia_matcher", "match_mode": "smnn", "th": 0.8}))
    for (i, j), t in zip(PAIRS, tables):
        assert np.array_equal(t, plugin._match_pairs(s["feats"][i], s["feats"][j])), (i, j)
    assert sum(len(t) for t in tables) > 0


def _al_extractor(al_weights, tile=None, overlap=0):
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    general = {} if tile is None else {"general": {"tile_size": tile, "tile_overlap": overlap}}
    return AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", **AL_CONF, "weights_dict": al_weights},
                                  **general))


@pytest.mark.gpu
def test_mixed_set_aliked_equals_host_flow(ctx, al_weights):
    from dim_b200 import weights
    sizes = [(768, 1024), (1024, 768), (601, 797)]
    imgs = [x.astype(F) for x in _mixed_rgb(sizes, 61)]
    w = weights.lightglue_seeded(input_dim=128, seed=0)
    pairs = [(0, 1), (0, 2), (1, 2)]
    eng = _engine(ctx, al_weights, w, sizes, AL_CONF, extractor="aliked")
    tables = eng.run(_dev(imgs), [0, 1, 2], pairs)
    ext = _al_extractor(al_weights)
    feats = [_host_features(ext, im) for im in imgs]
    for i in range(3):
        _same_features(eng.store.get(i), feats[i])
    plugin = _lg_plugin(w, "aliked")
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
    assert sum(len(t) for t in tables) > 0


TILED_SIZES = [(768, 1024), (512, 640), (1024, 768), (768, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("sel", ["grid", "exhaustive"])
def test_mixed_tiled_superpoint_equals_extract_and_match_by_tile(ctx, sp_weights, sel):
    from dim_b200 import tiling, weights
    imgs = _mixed_gray(TILED_SIZES, 70)
    w = weights.lightglue_seeded(seed=0)
    tiled = {"tile_size": 512, "tile_overlap": 64, "tile_selection": sel}
    pairs = [(i, j) for i in range(4) for j in range(i + 1, 4)]
    eng = _engine(ctx, sp_weights, w, TILED_SIZES, {**SP_CONF, "fix_sampling": True}, batch_images=8, batch_pairs=16, tiling=tiled)
    assert eng.T is None and len(set(eng.tile_counts)) > 1 and eng.view_offsets[-1] == sum(eng.tile_counts[:-1])
    tables = eng.run(_dev(imgs), [0, 1, 2, 3], pairs)
    ext = _sp_extractor(sp_weights, 512, 64)
    feats = [_host_features(ext, im, tiled=True) for im in imgs]
    for i in range(4):
        _same_features(eng.store.get(i), feats[i], ("keypoints", "descriptors", "scores", "tile_idx", "image_size"))
    lists = [[(int(a), int(b)) for a, b in tiling.tile_selection(imgs[i], imgs[j], sel, 512, 64)] for i, j in pairs]
    assert eng._tile_pair_lists(pairs, None) == lists
    plugin = _lg_plugin(w)
    for (i, j), lst, t in zip(pairs, lists, tables):
        assert np.array_equal(t, plugin._match_by_tile(feats[i], feats[j], lst)), (i, j)
    assert sum(len(t) for t in tables) > 0
    explicit = [[(0, eng.tile_counts[j] - 1)] for _, j in pairs]
    got = eng.match(pairs, list(range(len(pairs))), tile_pairs=explicit)
    for k, ((i, j), lst) in enumerate(zip(pairs, explicit)):
        assert np.array_equal(got[k], plugin._match_by_tile(feats[i], feats[j], lst))
    with pytest.raises(ValueError, match="tile indices"):
        eng.match([(1, 0)], [0], tile_pairs=[[(eng.tile_counts[1], 0)]])


@pytest.mark.gpu
def test_mixed_tiled_aliked_equals_extract_and_match_by_tile(ctx, al_weights):
    from dim_b200 import tiling, weights
    sizes = [(768, 1024), (512, 640), (1024, 768)]
    imgs = [x.astype(F) for x in _mixed_rgb(sizes, 71)]
    w = weights.lightglue_seeded(input_dim=128, seed=0)
    pairs = [(0, 1), (0, 2), (1, 2)]
    eng = _engine(ctx, al_weights, w, sizes, AL_CONF, extractor="aliked", batch_images=8, batch_pairs=16,
                  tiling={"tile_size": 512, "tile_overlap": 64, "tile_selection": "exhaustive"})
    assert len(set(eng.tile_counts)) > 1
    tables = eng.run(_dev(imgs), [0, 1, 2], pairs)
    ext = _al_extractor(al_weights, 512, 64)
    feats = [_host_features(ext, im, tiled=True) for im in imgs]
    for i in range(3):
        _same_features(eng.store.get(i), feats[i], ("keypoints", "descriptors", "scores", "tile_idx", "image_size"))
    plugin = _lg_plugin(w, "aliked")
    for (i, j), t in zip(pairs, tables):
        lst = tiling.tile_selection(imgs[i][..., 0], imgs[j][..., 0], "exhaustive", 512, 64)
        assert np.array_equal(t, plugin._match_by_tile(feats[i], feats[j], lst)), (i, j)
    assert sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_mixed_preselection_equals_host_flow(ctx, sp_weights):
    from dim_b200 import _native, tiling, weights
    sizes = [(768, 1024), (1024, 768), (601, 797), (768, 1024)]
    imgs = _mixed_gray(sizes, 80)
    w = weights.lightglue_seeded(seed=0)
    pre = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}
    pairs = [(i, j) for i in range(4) for j in range(i + 1, 4)]
    eng = _engine(ctx, sp_weights, w, sizes, {**SP_CONF, "fix_sampling": True}, batch_images=3, batch_pairs=16, tiling=pre)
    assert eng.pre_h is None and eng.pre.low_sizes[1] == (512, 384)
    tables = eng.run(_dev(imgs), [0, 1, 2, 3], pairs)
    sp_pre = lambda H, W: _native.SuperPointNet(ctx, sp_weights, max_height=H, max_width=W, **tiling.SP_PRESELECTION_CONF)
    lg_pre = _native.LightGlueNet(ctx, w, max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    lists = []
    for i, j in pairs:
        kp0, kp1 = tiling.preselection_matches(imgs[i], imgs[j], 512, sp_pre, lg_pre)
        lists.append([(int(a), int(b)) for a, b in tiling.tile_selection(imgs[i], imgs[j], "preselection", (512, 512), 64, kp0=kp0, kp1=kp1)])
    assert eng._preselect(pairs) == lists
    assert any(0 < len(lst) < eng.tile_counts[i] * eng.tile_counts[j] for (i, j), lst in zip(pairs, lists))
    plugin = _lg_plugin(w)
    for (i, j), lst, t in zip(pairs, lists, tables):
        assert np.array_equal(t, plugin._match_by_tile(eng.store.get(i), eng.store.get(j), lst)), (i, j)
    assert sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_mixed_pair_generation_equals_pairs_from_lowres(ctx, sp_weights):
    """One group enlarged (533 x 800 and 800 x 533 to longest side 1000) and one shrunk (1536 x 2048)."""
    from pathlib import Path

    from dim_b200 import weights
    from dim_b200.pairs_generator import pairs_from_lowres
    from dim_b200.sharded import _lowres_size
    sizes = [(533, 800), (800, 533), (1536, 2048), (533, 800), (1536, 2048)]
    imgs = _mixed_gray(sizes, 90)
    w = weights.lightglue_seeded(seed=0)
    names = [Path(f"{k}.png") for k in range(len(sizes))]
    low = {}
    for p, im in zip(names, imgs):
        _, h, wd = _lowres_size(*im.shape, 1000)
        low[p.name] = cv2.resize(im, (wd, h), interpolation=cv2.INTER_AREA)
    exp_pairs, exp_counts = pairs_from_lowres(names, 1000, 20, lightglue_weights=w, superpoint_weights=sp_weights, images=low, pair_batch=16,
                                              return_counts=True, device=ctx.device)
    exp_pairs = [(int(a.stem), int(b.stem)) for a, b in exp_pairs]
    eng = _engine(ctx, sp_weights, w, sizes, {**SP_CONF, "fix_sampling": True}, batch_images=2, batch_pairs=4,
                  pair_generation={"strategy": "matching_lowres", "resize_max": 1000, "min_matches": 20})
    assert eng.lowres.h is None and eng.lowres.low_sizes[:3] == [(666, 1000), (1000, 666), (750, 1000)]
    eng.extract(_dev(imgs), list(range(len(sizes))))
    eng.exchange()
    assert eng.lowres_pairs() == (exp_pairs, exp_counts)
    assert 0 < len(exp_pairs) and max(exp_counts) > 20


@pytest.mark.gpu
@pytest.mark.parametrize("tiled", [False, True])
def test_mixed_quality_medium_equals_host_flow(ctx, sp_weights, tiled):
    from dim_b200 import weights
    sizes = [(1536, 2048), (2048, 1536), (1201, 1599)] if tiled else MIXED[:4]
    imgs = _mixed_gray(sizes, 95)
    w = weights.lightglue_seeded(seed=0)
    kw = {"tiling": {"tile_size": 512, "tile_overlap": 64, "tile_selection": "grid"}, "batch_images": 8} if tiled else {}
    conf = {**SP_CONF, "fix_sampling": True} if tiled else SP_CONF
    eng = _engine(ctx, sp_weights, w, sizes, conf, quality="medium", **kw)
    assert eng.ext_sizes[:2] == [(sizes[0][0] // 2, sizes[0][1] // 2), (sizes[1][0] // 2, sizes[1][1] // 2)]
    pairs = [(0, 1), (0, 2), (1, 2)]
    tables = eng.run(_dev(imgs), list(range(len(sizes))), pairs)
    ext = _sp_extractor(sp_weights, 512, 64) if tiled else _sp_extractor(sp_weights)
    feats = [_host_features(ext, im, "medium", tiled) for im in imgs]
    keys = ("keypoints", "descriptors", "scores", "tile_idx", "image_size") if tiled else ("keypoints", "descriptors", "scores", "image_size")
    for i in range(len(sizes)):
        _same_features(eng.store.get(i), feats[i], keys)
    plugin = _lg_plugin(w)
    for (i, j), t in zip(pairs, tables):
        if tiled:
            T0, T1 = eng.tile_counts[i], eng.tile_counts[j]
            exp = plugin._match_by_tile(feats[i], feats[j], [(t_, t_) for t_ in range(min(T0, T1))])
        else:
            exp = plugin._match_pairs(feats[i], feats[j])
        assert np.array_equal(t, exp), (i, j)
    assert sum(len(t) for t in tables) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain_pairgen", "preselection"])
def test_uniform_lists_equal_the_int_form(ctx, sp_weights, mode):
    """A set given as lists of one size is a set of one size: the same attributes, launches, slots and tables as the int form, for a
    stacked tensor and for a list of tensors."""
    import torch
    from dim_b200 import weights
    from dim_b200.sharded import ImageSetMatcher
    n, H, W = 4, 768, 1024
    imgs = np.stack(_mixed_gray([(H, W)] * n, 99))
    d = torch.from_numpy(imgs).cuda()
    w = weights.lightglue_seeded(seed=0)
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
    if mode == "preselection":
        kw = {"tiling": {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}}
    else:
        kw = {"pair_generation": {"strategy": "matching_lowres", "resize_max": 512, "min_matches": 0}}
    conf = {**SP_CONF, "fix_sampling": True}
    out = []
    for hw, images in (((H, W), d), (([H] * n, [W] * n), d), (([H] * n, [W] * n), list(d))):
        eng = ImageSetMatcher(ctx, sp_weights, w, n, *hw, conf, {}, batch_images=3, batch_pairs=16, **kw)
        attrs = (eng.H, eng.W, eng.h2, eng.w2, eng.T, eng.G, getattr(eng, "pre_h", None), getattr(eng, "pre_w", None))
        eng.run(images, list(range(n)), pairs)  # warm: scratch grown
        n0 = ctx.launches
        tables = eng.run(images, list(range(n)), pairs)
        launches = ctx.launches - n0
        extra = eng._preselect(pairs) if mode == "preselection" else eng.lowres_pairs()
        out.append((attrs, launches, tables, [eng.store.get(i) for i in range(n)], extra))
    for attrs, launches, tables, slots, extra in out[1:]:
        assert attrs == out[0][0] and launches == out[0][1] and extra == out[0][4]
        assert all(np.array_equal(a, b) for a, b in zip(tables, out[0][2]))
        for a, b in zip(slots, out[0][3]):
            _same_features(a, b, ("keypoints", "descriptors", "scores", "tile_idx", "image_size"))
    assert sum(len(t) for t in out[0][2]) > 0
