"""Tiled matching of image sets: the device tile cut, tile-feature merge, tile views and tile-pair match merge (dimb_tile_*), and
ImageSetMatcher(tiling=...) checked against the reference's host flow - ExtractorBase._extract_by_tile, the features.h5 round trip
(as_half_roundtrip) and MatcherBase._match_by_tile - on the same native networks.  Every comparison is exact."""
import ctypes as C
import sqlite3

import numpy as np
import pytest

# ---------------------------------------------------------------------------------------------------------------- no GPU needed


def test_tile_entries_reject_bad_arguments_without_touching_the_gpu():
    """Argument validation of the dimb_tile_* entries comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU.  The non-NULL
    context / store handles are zeroed dummies that hold no slot."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    fs = C.cast(C.create_string_buffer(512), C.c_void_p)
    dev = C.c_void_p(0x1000)
    out = (C.c_int * 6)()
    assert lib.dimb_tile_grid(1536, 2048, 1024, 1024, 128, 128, out) == 0 and list(out) == [2, 2, 256, 0, 896, 896]
    for bad in ((0, 2048, 1024, 1024, 0, 0), (1536, 2048, 0, 1024, 0, 0), (1536, 2048, 1024, 1024, 1024, 0), (1536, 2048, 1024, 1024, -1, 0),
                (4096, 4096, 16, 16, 0, 0)):  # the last one: 65536 tiles > 2048
        assert lib.dimb_tile_grid(*bad, out) == -3, bad
    assert lib.dimb_tile_grid(1536, 2048, 1024, 1024, 128, 128, None) == -3

    def cut(ctx=ctx, img=dev, B=1, C_=3, tile=1024, ov=128, dst=dev):
        return lib.dimb_tile_cut_dev(ctx, img, B, 1536, 2048, C_, tile, tile, ov, ov, dst, null)
    assert cut(ctx=null) == -3 and cut(img=null) == -3 and cut(dst=null) == -3
    assert cut(B=0) == -3 and cut(C_=2) == -3 and cut(C_=4) == -3 and cut(tile=0) == -3 and cut(ov=1024) == -3 and cut(B=20000) == -3

    slots = (C.c_int * 2)(0, 1)

    def merge(fs=fs, B=2, sl=slots, k=dev, s=dev, d=dev, n=dev, K=64, tile=1024):
        return lib.dimb_tile_merge_dev(fs, B, sl, 1536, 2048, tile, tile, 128, 128, k, s, d, n, K, null)
    assert merge(fs=null) == -3 and merge(sl=None) == -3 and merge(k=null) == -3 and merge(s=null) == -3 and merge(d=null) == -3
    assert merge(n=null) == -3 and merge(B=0) == -3 and merge(K=0) == -3 and merge(tile=-5) == -3
    assert merge() == -3  # the dummy store has no slots

    def views(src=fs, B=2, ss=slots, T=4, dst=fs, ds=slots, m=dev):
        return lib.dimb_tile_views_dev(src, B, ss, T, dst, ds, m, null)
    assert views(src=null) == -3 and views(dst=null) == -3 and views(ss=None) == -3 and views(ds=None) == -3 and views(m=null) == -3
    assert views(B=0) == -3 and views(T=0) == -3 and views(T=4096) == -3 and views() == -3

    off = (C.c_int * 3)(0, 2, 3)
    v = (C.c_int * 3)(0, 1, 2)
    vneg = (C.c_int * 3)(0, -1, 2)

    def mm(ctx=ctx, Q=2, o=off, v0=v, v1=v, maps=dev, ld=64, m=dev, nm=dev, cap=64, d=dev, dn=dev, cap2=128):
        return lib.dimb_tile_match_merge_dev(ctx, Q, o, v0, v1, maps, ld, m, nm, cap, d, dn, cap2, null)
    assert mm(ctx=null) == -3 and mm(o=None) == -3 and mm(v0=None) == -3 and mm(v1=None) == -3 and mm(maps=null) == -3
    assert mm(m=null) == -3 and mm(nm=null) == -3 and mm(d=null) == -3 and mm(dn=null) == -3
    assert mm(Q=0) == -3 and mm(ld=0) == -3 and mm(cap=0) == -3 and mm(cap2=0) == -3 and mm(v1=vneg) == -3
    assert mm(o=(C.c_int * 3)(1, 2, 3)) == -3 and mm(o=(C.c_int * 3)(0, 3, 2)) == -3


def test_tiling_conf_validation():
    from dim_b200.sharded import tiling_conf
    assert tiling_conf(None) is None
    c = tiling_conf({"tile_size": (1024, 768), "tile_overlap": 64})
    assert c["tile_hw"] == (768, 1024) and c["overlap_hw"] == (64, 64) and c["tile_selection"] == "grid"
    assert tiling_conf({"tile_size": 512, "tile_selection": "EXHAUSTIVE"})["tile_selection"] == "exhaustive"
    for bad in ({}, {"tile_size": 0}, {"tile_size": (512,)}, {"tile_size": 512.0}, {"tile_size": 512, "tile_overlap": 512},
                {"tile_size": 512, "tile_overlap": -1}, {"tile_size": 512, "tile_selection": "preselection"}, {"tile_size": 512, "tiles": 4}):
        with pytest.raises(ValueError):
            tiling_conf(bad)


@pytest.mark.parametrize("shape", [(1536, 2048), (1536, 2048, 3), (1000, 1300), (1000, 1300, 3)])
def test_matcher_tile_grid_equals_compute_tiles_by_size(shape):
    from dim_b200 import _native, tiling
    from dim_b200.sharded import tiling_conf
    for size, overlap in ((1024, 128), ((512, 384), 64)):
        conf = tiling_conf({"tile_size": size, "tile_overlap": overlap})
        g = _native.tile_grid(shape[0], shape[1], *conf["tile_hw"], *conf["overlap_hw"])
        tiles, origins, pad = tiling.compute_tiles_by_size(np.zeros(shape, np.float32), size, overlap)
        assert g["origins"] == [origins[k] for k in range(len(origins))] and len(tiles) == len(origins)
        assert (g["pad_top"], g["pad_left"]) == (pad[0], pad[2])
        assert all(t.shape[:2] == conf["tile_hw"] for t in tiles.values())


def test_tile_pair_lists_equal_tile_selection():
    from dim_b200 import tiling
    from dim_b200.sharded import tile_pairs_for
    img = np.zeros((1536, 2048), np.float32)
    for method in ("grid", "exhaustive"):
        assert tile_pairs_for(method, 4) == tiling.tile_selection(img, img, method, 1024, 128)
    odd = np.zeros((1000, 1300), np.float32)
    T = len(tiling.compute_tiles_by_size(odd, (512, 384), 64)[1])
    for method in ("grid", "exhaustive"):
        assert tile_pairs_for(method, T) == tiling.tile_selection(odd, odd, method, (512, 384), 64)


def test_batch_packing_keeps_image_pairs_whole():
    from dim_b200.sharded import pack_tile_batches
    assert pack_tile_batches([4, 4, 4, 4, 4], 8) == [(0, 2), (2, 4), (4, 5)]
    assert pack_tile_batches([3, 0, 5, 2, 8, 1], 8) == [(0, 3), (3, 4), (4, 5), (5, 6)]
    assert pack_tile_batches([], 8) == []
    assert pack_tile_batches([16], 16) == [(0, 1)]
    with pytest.raises(ValueError):
        pack_tile_batches([4, 17, 4], 16)


def test_matcher_refuses_inconsistent_options():
    from dim_b200.sharded import ImageSetMatcher
    tiled = {"tile_size": 512, "tile_overlap": 64}
    with pytest.raises(ValueError, match="fix_sampling"):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, {"max_keypoints": 512, "fix_sampling": False}, {}, tiling=tiled)
    with pytest.raises(ValueError, match="SuperGlue"):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, {"max_num_keypoints": 512}, {}, matcher="superglue", extractor="aliked")
    with pytest.raises(ValueError, match="input_dim"):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, {"max_num_keypoints": 512}, {"input_dim": 256}, extractor="aliked")
    with pytest.raises(ValueError):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, {"max_keypoints": 512}, {}, extractor="disk")
    with pytest.raises(ValueError):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, {"max_keypoints": 512}, {}, tiling={"tile_size": 512, "tile_overlap": 600})


# ---------------------------------------------------------------------------------------------------------------- on the GPU

SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "fix_sampling": True}


def _sp_extractor(sp_weights, tile, overlap, K):
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    return SuperPointExtractor(Config(general={"tile_size": tile, "tile_overlap": overlap},
                                      extractor={**SP_CONF, "max_keypoints": K, "weights_dict": sp_weights}))


def _reference_features(ext, image):
    """as_half_roundtrip(_extract_by_tile(image)) with image_size, and the concatenated count before np.unique."""
    from dim_b200.io_h5 import as_half_roundtrip
    ref = as_half_roundtrip({**ext._extract_by_tile(image), "image_size": np.array(image.shape[:2])})
    concat = len(ext._extract_by_tile(image, select_unique=False)["keypoints"])
    return ref, concat


def _same_features(got, ref):
    for k in ("keypoints", "descriptors", "scores", "tile_idx", "image_size"):
        assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
def test_tile_cut_equals_compute_tiles_by_size(ctx, channels):
    import torch
    from dim_b200 import _native, tiling
    rng = np.random.default_rng(channels)
    for (H, W), tile, ov in (((1536, 2048), 1024, 128), ((1000, 1300), (512, 384), 64)):
        shape = (3, H, W) if channels == 1 else (3, H, W, 3)
        imgs = rng.uniform(0, 255, shape).astype(np.float32)
        th, tw = tiling._hw(tile)
        T = len(_native.tile_grid(H, W, th, tw, ov, ov)["origins"])
        out = torch.full((3 * T, th, tw, channels), -1.0, device="cuda")
        ctx.tile_cut_dev(torch.from_numpy(imgs).cuda().data_ptr(), 3, H, W, channels, th, tw, ov, ov, out.data_ptr(), 0)
        got = out.cpu().numpy()
        for b in range(3):
            tiles, _, _ = tiling.compute_tiles_by_size(imgs[b], tile, ov)
            assert len(tiles) == T
            for t in range(T):
                assert np.array_equal(got[b * T + t], tiles[t].reshape(th, tw, channels)), (b, t)


@pytest.fixture(scope="module")
def big_sp(ctx, sp_weights):
    """A 4096^2 gray blocks image with a constant corner, tiled 512 / 64 (81 tiles of up to 2048 keypoints), through
    ImageSetMatcher.extract + exchange."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.sharded import ImageSetMatcher
    img = synthetic.to_gray_like_reference(synthetic.blocks_image(5, 4096))
    img[:600, :600] = 0.0  # tile 0 lies in it: no keypoints
    eng = ImageSetMatcher(ctx, sp_weights, weights.lightglue_seeded(seed=0), 1, 4096, 4096, {**SP_CONF, "max_keypoints": 2048}, {},
                          batch_images=16, tiling={"tile_size": 512, "tile_overlap": 64})
    eng.extract(torch.from_numpy(img[None]).cuda(), [0])
    eng.exchange()
    return img, eng


@pytest.mark.gpu
def test_superpoint_tile_merge_equals_extract_by_tile(sp_weights, big_sp):
    img, eng = big_sp
    assert eng.T == 81
    ref, concat = _reference_features(_sp_extractor(sp_weights, 512, 64, 2048), img)
    got = eng.store.get(0)
    _same_features(got, ref)
    assert concat > 65536, concat
    assert concat - len(got["keypoints"]) > 0  # cross-tile duplicates were removed
    assert 0 not in set(got["tile_idx"].astype(int).tolist())  # the constant tile yields nothing


@pytest.mark.gpu
def test_tile_views_equal_get_features_by_tile(big_sp):
    from dim_b200 import tiling
    _, eng = big_sp
    merged = eng.store.get(0)
    vmap = eng.vmap.cpu().numpy()
    empty = 0
    for t in range(eng.T):
        ref, idx = tiling.get_features_by_tile(merged, t)
        got = eng.views.get(t)
        for k in ("keypoints", "descriptors", "scores", "image_size"):
            assert np.array_equal(got[k], ref[k]), (t, k)
        assert np.array_equal(got["tile_idx"], np.full(len(idx), t, np.float32))
        assert np.array_equal(vmap[t, :len(idx)], idx), t
        empty += len(idx) == 0
    assert empty >= 1


@pytest.mark.gpu
def test_aliked_tile_merge_equals_extract_by_tile(ctx, al_weights):
    """cfg3 geometry: 2048 x 1536 RGB, tile 1024 / overlap 128, 4096 keypoints per tile; then ALIKED + LightGlue(input_dim 128)
    tables of the grid selection equal _match_by_tile."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(300, 2048, 4)[:1536]
    imgs = np.stack([a, synthetic.warp_pair(a, 1)]).astype(np.float32)
    al_conf = {"max_num_keypoints": 4096, "detection_threshold": 0.2, "nms_radius": 3}
    w_lg = weights.lightglue_seeded(input_dim=128, seed=0)
    tiled = {"tile_size": 1024, "tile_overlap": 128}
    eng = ImageSetMatcher(ctx, al_weights, w_lg, 2, 1536, 2048, al_conf, {}, batch_pairs=8, tiling=tiled, extractor="aliked")
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1], [(0, 1)])
    ext = AlikedExtractor(Config(general={"tile_size": 1024, "tile_overlap": 128},
                                 extractor={"model_name": "aliked-n16rot", **al_conf, "weights_dict": al_weights}))
    feats = []
    for i in range(2):  # ALIKED's sub-pixel keypoints of overlapping tiles do not coincide exactly: np.unique keeps them all
        ref, concat = _reference_features(ext, imgs[i])
        _same_features(eng.store.get(i), ref)
        assert concat == len(ref["keypoints"]) and set(ref["tile_idx"].astype(int).tolist()) == {0, 1, 2, 3}
        feats.append(ref)
    plugin = LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w_lg}), local_features="aliked")
    exp = plugin._match_by_tile(feats[0], feats[1], [(t, t) for t in range(4)])
    assert np.array_equal(tables[0], exp) and len(exp) > 0


@pytest.mark.gpu
def test_image_set_matcher_aliked_untiled_equals_serial_flow(ctx, al_weights):
    """ALIKED without tiling: 3 RGB images, all pairs, batch_images=2 (the extraction crosses a chunk boundary) and batch_pairs=2.
    The store holds AlikedExtractor._extract + as_half_roundtrip of every image, and every table equals the LightGlue plugin's
    _match_pairs (input_dim 128) on those features."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(301, 512)[:384]
    imgs = np.stack([a] + [synthetic.warp_pair(a, 50 + k, jitter=24.0) for k in (1, 2)]).astype(np.float32)
    al_conf = {"max_num_keypoints": 1024, "detection_threshold": 0.2, "nms_radius": 3}
    w_lg = weights.lightglue_seeded(input_dim=128, seed=0)
    pairs = pairs_from_bruteforce([0, 1, 2])
    eng = ImageSetMatcher(ctx, al_weights, w_lg, 3, 384, 512, al_conf, {}, batch_images=2, batch_pairs=2, extractor="aliked")
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    ext = AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", **al_conf, "weights_dict": al_weights}))
    feats = [as_half_roundtrip({**ext._extract(img), "image_size": np.array(img.shape[:2])}) for img in imgs]
    for i in range(3):
        got = eng.store.get(i)
        for k in ("keypoints", "descriptors", "scores"):
            assert got[k].shape == feats[i][k].shape and np.array_equal(got[k], feats[i][k]), (i, k)
    plugin = LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w_lg}), local_features="aliked")
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
    assert min(len(f["keypoints"]) for f in feats) > 100 and sum(len(t) for t in tables) > 0


def _gray_set(n, H=768, W=1024):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(40, max(H, W))[:H, :W]
    imgs = [a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in range(1, n)]
    return np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in imgs]).astype(np.float32)


@pytest.fixture(scope="module")
def lg_set(ctx, sp_weights):
    import torch
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    imgs = _gray_set(3)
    w = weights.lightglue_seeded(seed=0)
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    return {"imgs": imgs, "d": torch.from_numpy(imgs).cuda(), "w": w, "plugin": plugin, "pairs": pairs_from_bruteforce([0, 1, 2])}


def _engine(ctx, sp_weights, s, selection, batch_pairs, **kw):
    from dim_b200.sharded import ImageSetMatcher
    return ImageSetMatcher(ctx, sp_weights, s["w"], 3, 768, 1024, {**SP_CONF, "max_keypoints": 1024}, {}, batch_images=6,
                           batch_pairs=batch_pairs, tiling={"tile_size": 512, "tile_overlap": 64, "tile_selection": selection}, **kw)


def _expected(plugin, eng, pairs, lists):
    return [plugin._match_by_tile(eng.store.get(i), eng.store.get(j), lst) for (i, j), lst in zip(pairs, lists)]


@pytest.mark.gpu
def test_image_set_matcher_tiled_equals_match_by_tile(ctx, sp_weights, lg_set):
    """grid and exhaustive selections, two batch sizes and a permuted pair list: every table equals _match_by_tile on the merged
    (round-tripped) features, which equal _extract_by_tile's."""
    from dim_b200.sharded import tile_pairs_for
    s, pairs = lg_set, lg_set["pairs"]
    ext = _sp_extractor(sp_weights, 512, 64, 1024)
    for selection, bps in (("grid", (4, 9)), ("exhaustive", (16, 40))):
        base = None
        for bp in bps:
            eng = _engine(ctx, sp_weights, s, selection, bp)
            assert eng.T == 4
            tables = eng.run(s["d"], [0, 1, 2], pairs)
            if base is None:
                for i in range(3):
                    _same_features(eng.store.get(i), _reference_features(ext, s["imgs"][i])[0])
                exp = _expected(s["plugin"], eng, pairs, [tile_pairs_for(selection, 4)] * len(pairs))
                assert all(np.array_equal(a, b) for a, b in zip(tables, exp)) and min(len(t) for t in exp) > 0
                base = tables
            else:
                assert all(np.array_equal(a, b) for a, b in zip(tables, base))
            perm = [2, 0, 1]
            res = eng.match([pairs[k] for k in perm], perm)
            assert all(np.array_equal(res[k], base[k]) for k in range(3))


@pytest.mark.gpu
def test_image_set_matcher_explicit_preselection_lists(ctx, sp_weights, lg_set):
    from dim_b200 import _native, tiling
    s, pairs = lg_set, lg_set["pairs"]
    sp_pre = lambda H, W: _native.SuperPointNet(ctx, sp_weights, max_height=H, max_width=W, **tiling.SP_PRESELECTION_CONF)
    lg_pre = _native.LightGlueNet(ctx, s["w"], max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    lists = []
    for i, j in pairs:
        kp0, kp1 = tiling.preselection_matches(s["imgs"][i], s["imgs"][j], 512, sp_pre, lg_pre)
        lists.append(tiling.tile_selection(s["imgs"][i], s["imgs"][j], "preselection", (512, 512), 64, kp0=kp0, kp1=kp1))
    lists[1] = lists[1][:2]  # and one hand-made short list
    eng = _engine(ctx, sp_weights, s, "grid", 16)
    tables = eng.run(s["d"], [0, 1, 2], pairs, tile_pairs=lists)
    exp = _expected(s["plugin"], eng, pairs, lists)
    assert all(np.array_equal(a, b) for a, b in zip(tables, exp))
    with pytest.raises(ValueError):
        eng.match(pairs, [0, 1, 2], tile_pairs=[[(0, 0)]] * 2)
    with pytest.raises(ValueError):
        eng.match(pairs[:1], [0], tile_pairs=[[(0, 4)]])
    with pytest.raises(ValueError):
        _engine(ctx, sp_weights, s, "exhaustive", 8).match(pairs, [0, 1, 2])


@pytest.mark.gpu
def test_image_set_matcher_tiled_superglue(ctx, sp_weights):
    import torch
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from dim_b200.sharded import ImageSetMatcher
    from oracle import superglue as o_sg
    imgs = _gray_set(2, 512, 640)
    w = o_sg.seeded_weights(1)
    conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
    eng = ImageSetMatcher(ctx, sp_weights, w, 2, 512, 640, {**SP_CONF, "max_keypoints": 512}, conf, batch_pairs=8, matcher="superglue",
                          tiling={"tile_size": 384, "tile_overlap": 32, "tile_selection": "grid"})
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1], [(0, 1)])
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": w}))
    exp = plugin._match_by_tile(eng.store.get(0), eng.store.get(1), [(t, t) for t in range(eng.T)])
    assert np.array_equal(tables[0], exp) and len(exp) > 0


@pytest.mark.gpu
def test_match_merge_reports_the_full_count_beyond_cap2(ctx):
    """Three tile pairs over two image pairs with overlapping rows, one tile pair whose count exceeds the table capacity: the merged
    tables are np.unique of the remapped rows; with cap2 below the true count the count stays full and the first cap2 rows are
    written."""
    import torch
    rng = np.random.default_rng(0)
    ld, cap = 64, 16
    maps = np.stack([np.sort(rng.choice(500, ld, replace=False)) for _ in range(4)]).astype(np.int32)
    tabs, counts = [], [12, 40, 9]
    for n in counts:
        r = min(n, cap)
        t0 = np.sort(rng.choice(20, r, replace=False))
        tabs.append(np.stack([t0, rng.integers(0, 20, r)], 1))
    tabs[1][:5] = tabs[0][:5]  # duplicates across the tile pairs of image pair 0 (same views)
    m = np.zeros((3, cap, 2), np.int64)
    for p, t in enumerate(tabs):
        m[p, :len(t)] = t
    v0, v1, off = [0, 0, 2], [1, 1, 3], [0, 2, 3]
    exp = []
    for q in range(2):
        rows = np.concatenate([np.stack([maps[v0[p]][tabs[p][:, 0]], maps[v1[p]][tabs[p][:, 1]]], 1) for p in range(off[q], off[q + 1])])
        exp.append(np.unique(rows, axis=0))
    d_maps, d_m = torch.from_numpy(maps).cuda(), torch.from_numpy(m).cuda()
    d_nm = torch.tensor(counts, dtype=torch.int32, device="cuda")
    for cap2 in (64, len(exp[0]) - 3):
        out = torch.full((2, cap2, 2), -1, dtype=torch.int64, device="cuda")
        n = torch.full((2,), -1, dtype=torch.int32, device="cuda")
        ctx.tile_match_merge_dev(off, v0, v1, d_maps.data_ptr(), ld, d_m.data_ptr(), d_nm.data_ptr(), cap, out.data_ptr(), n.data_ptr(), cap2, 0)
        n, out = n.cpu().numpy(), out.cpu().numpy()
        for q in range(2):
            assert n[q] == len(exp[q])
            k = min(cap2, n[q])
            assert np.array_equal(out[q, :k], exp[q][:k])
    assert len(exp[0]) < counts[0] + cap  # the planted duplicates were dropped


@pytest.mark.gpu
def test_tiled_run_verified_and_colmap_export(ctx, sp_weights, lg_set, tmp_path):
    import torch
    from dim_b200.geometric_verification import gv_seed
    s, pairs = lg_set, lg_set["pairs"]
    eng = _engine(ctx, sp_weights, s, "grid", 8, verification={"seed": 3})
    res = eng.run_verified(s["d"], [0, 1, 2], pairs)
    tables = eng.run(s["d"], [0, 1, 2], pairs)
    P, cap = len(pairs), max(len(t) for t in tables)
    m = torch.zeros(P, cap, 2, dtype=torch.int64, device="cuda")
    for k, t in enumerate(tables):
        m[k, :len(t)] = torch.from_numpy(t)
    nm = torch.tensor([len(t) for t in tables], dtype=torch.int32, device="cuda")
    v = torch.zeros(P, cap, 2, dtype=torch.int64, device="cuda")
    nv, ninl = torch.zeros(P, dtype=torch.int32, device="cuda"), torch.zeros(P, dtype=torch.int32, device="cuda")
    F, mask = torch.zeros(P, 9, device="cuda"), torch.zeros(P, cap, dtype=torch.uint8, device="cuda")
    ctx.gv_verify_dev([eng.store.feats_dev(i) for i, _ in pairs], [eng.store.feats_dev(j) for _, j in pairs], m.data_ptr(), nm.data_ptr(), cap,
                      [gv_seed(3, k) for k in range(P)], 1.0, 10000, 15, 0.2, v.data_ptr(), nv.data_ptr(), F.data_ptr(), mask.data_ptr(),
                      ninl.data_ptr(), 0)
    v, nv, F, ninl = v.cpu().numpy(), nv.cpu().numpy(), F.cpu().numpy(), ninl.cpu().numpy()
    for k, (raw, ver, Fk, n_in) in enumerate(res):
        assert np.array_equal(raw, tables[k]) and np.array_equal(ver, v[k, :nv[k]]) and n_in == ninl[k]
        assert (Fk is None) == (not F[k].any()) and (Fk is None or np.array_equal(Fk.ravel(), F[k]))
    assert max(len(r[1]) for r in res) > 0
    db = tmp_path / "tiled.db"
    eng.export_colmap(pairs, res, db)
    con = sqlite3.connect(str(db))
    rows = dict(con.execute("SELECT image_id, rows FROM keypoints").fetchall())
    con.close()
    assert rows == {i + 1: eng.store.count(i)[0] for i in range(3)} and min(rows.values()) > 1024  # merged: more than one tile's K
