"""SuperPoint and ALIKED at keypoint limits above 16384, and ALIKED's top-k and mean detection modes, end to end.

SuperPoint with max_keypoints > 16384 and ALIKED with an n_limit or a top-k K above 16384 select through the grid-wide top-k of
csrc/detect.cuh (tests/test_topk_select.py checks it bitwise on its own).  Here the extractors are checked against the CPU oracles, the
plugins and the image-set engine against the per-image flow.

ALIKED's top-k mode (detection_threshold <= 0 < max_num_keypoints) is the LightGlue port's DKD branch
``torch.topk(nms_scores.view(b, -1), top_k)`` on the border-zeroed NMS map, with top_k = -1 if detection_threshold > 0 else
max_num_keypoints.  The oracle module restates threshold and mean mode only, so the top-k branch is restated here (`topk_oracle`), from
the reference's DKD code: no golden file of the reference pins it.  When the map has fewer than K nonzero pixels, torch.topk returns
zero-valued pixels in an order it leaves unspecified; the library takes the first ones in row-major order, and `refine_oracle` (the
oracle's refinement and SDDH on given pixel indices) checks the keypoints, dispersities and descriptors of exactly those pixels.

oracle.compare.compare_aliked builds an N x N distance matrix, too large at 20000 keypoints: `pair_aliked` pairs with a k-d tree."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy.spatial import cKDTree

TOL = 1e-4


# ------------------------------------------------------------------ ALIKED oracle pieces
def al_maps(image, w):
    """oracle.aliked.dense_maps of an (H, W, 3) 0..255 image: (feature map (1, 128, H, W), score map (1, 1, H, W))."""
    from oracle import aliked as o_al
    x = torch.tensor(image.transpose(2, 0, 1)[None] / 255.0, dtype=torch.float)
    with torch.no_grad():
        return o_al.dense_maps(x, w, o_al.CFGS["aliked-n16rot"])


def border_zeroed_nms(score, r):
    from oracle import aliked as o_al
    nms = o_al.simple_nms(score, r)
    nms[:, :, :r, :] = 0
    nms[:, :, :, :r] = 0
    nms[:, :, -r:, :] = 0
    nms[:, :, :, -r:] = 0
    return nms


def topk_oracle(score, r, K):
    """DKD's top-k branch: torch.topk of the border-zeroed NMS map (sorted, descending).  Returns pixel indices."""
    return torch.topk(border_zeroed_nms(score, r).reshape(-1), K).indices


@torch.no_grad()
def refine_oracle(feat, score, idx, r, w):
    """oracle.aliked.dkd's sub-pixel refinement and oracle.aliked.sddh on given pixel indices -> FeaturesDict."""
    from oracle import aliked as o_al
    _, _, h, wd = score.shape
    idx = torch.as_tensor(idx, dtype=torch.int64)
    ks = 2 * r + 1
    xs = torch.linspace(-r, r, ks)
    hw_grid = torch.stack(torch.meshgrid([xs, xs], indexing="ij")).view(2, -1).t()[:, [1, 0]]
    patch = F.unfold(score, kernel_size=ks, padding=r)[0].t()[idx]
    xy_nms = torch.stack([idx % wd, torch.div(idx, wd, rounding_mode="trunc")], dim=1)
    max_v = patch.max(dim=1).values[:, None]
    x_exp = ((patch - max_v) / 0.1).exp()
    xy_res = x_exp @ hw_grid / x_exp.sum(dim=1)[:, None]
    d2 = torch.norm((hw_grid[None] - xy_res[:, None]) / r, dim=-1) ** 2
    disp = (x_exp * d2).sum(dim=1) / x_exp.sum(dim=1)
    wh = torch.tensor([wd - 1, h - 1])
    kxy = (xy_nms + xy_res) / wh * 2 - 1
    desc = o_al.sddh(feat, kxy, w, 3, 16)
    return {"keypoints": (wh * (kxy + 1) / 2.0).numpy().astype(np.float32), "descriptors": desc.t().contiguous().numpy().astype(np.float32),
            "scores": disp.numpy().astype(np.float32)}


def pair_aliked(out, ref, max_unpaired, tol_kpt=1e-3):
    """Pairs sub-pixel keypoints by nearest neighbour (k-d tree); at most `max_unpaired` on either side stay unpaired (decisions at
    the cut within fp32 summation-order noise).  Paired dispersities and descriptors within TOL.  Returns the fraction of pairs at the
    same position in both lists."""
    ko, kr = out["keypoints"].astype(np.float64), ref["keypoints"].astype(np.float64)
    if len(ko) == 0 or len(kr) == 0:
        assert len(ko) == len(kr)
        return 1.0
    d, j = cKDTree(kr).query(ko)
    ok = d < tol_kpt
    assert len(set(j[ok].tolist())) == int(ok.sum()), "two keypoints paired with the same oracle keypoint"
    assert (~ok).sum() <= max_unpaired and len(kr) - ok.sum() <= max_unpaired, f"{(~ok).sum()} / {len(kr) - ok.sum()} unpaired"
    a, b = np.flatnonzero(ok), j[ok]
    assert np.abs(out["scores"][a] - ref["scores"][b]).max() < TOL
    assert np.abs(out["descriptors"][:, a] - ref["descriptors"][:, b]).max() < TOL
    return float(np.mean(a == b))


def rgb_image(seed, H, W):
    from dim_b200 import synthetic
    return np.ascontiguousarray(synthetic.blocks_image(seed, max(H, W), 8)[:H, :W]).astype(np.float32)


def test_refine_oracle_equals_dkd(al_weights):
    """The index-given helper reproduces oracle.aliked.extract on the indices threshold mode picks."""
    from oracle import aliked as o_al
    img = rgb_image(5, 96, 128)
    conf = {"model_name": "aliked-n16rot", "max_num_keypoints": 300, "detection_threshold": 0.2, "nms_radius": 2}
    ref = o_al.extract(img, al_weights, conf)
    feat, score = al_maps(img, al_weights)
    nms = border_zeroed_nms(score, 2).reshape(-1)
    idx = torch.nonzero(nms > 0.2)[:, 0]
    if len(idx) > 300:
        idx = idx[score.reshape(-1)[idx].sort(descending=True)[1][:300]]
    got = refine_oracle(feat, score, idx, 2, al_weights)
    assert len(idx) > 20
    for k in ("keypoints", "descriptors", "scores"):
        assert np.array_equal(got[k], ref[k]), k


# ------------------------------------------------------------------ SuperPoint
def sp_gray(seed, H, W, flat_below=None):
    from dim_b200 import synthetic
    g = synthetic.to_gray_like_reference(np.ascontiguousarray(synthetic.blocks_image(seed, max(H, W), 8)[:H, :W])).astype(np.float32)
    if flat_below is not None:
        g[flat_below:] = 128.0
    return g


_SP_REF = {}


def _sp_ref(g, w, conf):
    from oracle import superpoint as o_sp
    key = conf["max_keypoints"]
    if key not in _SP_REF:
        _SP_REF[key] = o_sp.extract(g, w, conf, return_debug=True)
    return _SP_REF[key]


SP_CONF = {"nms_radius": 1, "keypoint_threshold": 0.0001, "remove_borders": 4, "fix_sampling": True}


@pytest.mark.gpu
@pytest.mark.parametrize("K", [20000, 32768])
def test_superpoint_above_16384(ctx, sp_weights, K):
    """2048 x 1536 with C > K against oracle.superpoint.extract; a batch of two images (the second mostly flat, fewer than K
    keypoints) equals the single-image calls; the device entry equals the host entry bitwise."""
    from dim_b200 import _native
    from oracle.compare import compare_superpoint
    conf = {**SP_CONF, "max_keypoints": K}
    g0, g1 = sp_gray(21, 1536, 2048), sp_gray(22, 1536, 2048, flat_below=40)
    ref = _sp_ref(g0, sp_weights, conf)
    C = int(((ref["_nms"][0, 0, 4:-4, 4:-4] if ref["_nms"].ndim == 4 else ref["_nms"][4:-4, 4:-4]) > conf["keypoint_threshold"]).sum())
    assert C > K, C
    net = _native.SuperPointNet(ctx, sp_weights, max_batch=2, max_height=1536, max_width=2048, **conf)
    f0 = net.extract(g0[None])[0]
    nms = ref["_nms"].reshape(1536, 2048)
    rep = compare_superpoint(f0, ref, nms, tol=TOL)
    print("superpoint", K, C, rep["n"], len(rep["boundary_diffs"]))
    assert rep["n"] == K
    fb = net.extract(np.stack([g0, g1]))
    f1 = net.extract(g1[None])[0]
    assert len(fb[1]["keypoints"]) < K == len(fb[0]["keypoints"])
    for a, b in ((fb[0], f0), (fb[1], f1)):
        for k in ("keypoints", "scores", "descriptors"):
            assert np.array_equal(a[k], b[k]), k
    dev = torch.device("cuda", ctx.device)
    imgs = torch.from_numpy(np.stack([g0, g1])).to(dev)
    kp, sc = torch.zeros(2, K, 2, device=dev), torch.zeros(2, K, device=dev)
    de, cnt = torch.zeros(2, 256, K, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
    net.extract_dev(imgs.data_ptr(), 2, 1536, 2048, kp.data_ptr(), sc.data_ptr(), de.data_ptr(), cnt.data_ptr(), K)
    torch.cuda.synchronize()
    kp, sc, de, cnt = kp.cpu().numpy(), sc.cpu().numpy(), de.cpu().numpy(), cnt.cpu().numpy()
    for b in range(2):
        n = cnt[b]
        assert n == len(fb[b]["keypoints"])
        assert np.array_equal(kp[b, :n], fb[b]["keypoints"]) and np.array_equal(sc[b, :n], fb[b]["scores"])
        assert np.array_equal(de[b, :, :n], fb[b]["descriptors"])


# ------------------------------------------------------------------ ALIKED
@pytest.mark.gpu
@pytest.mark.parametrize("H, W, K", [(512, 512, 4096), (1024, 1024, 20000)])
def test_aliked_topk_cut(ctx, al_weights, H, W, K):
    """Top-k mode with C > K, at K <= 16384 and above: the oracle's torch.topk keypoints, in its order."""
    from dim_b200 import _native
    img = rgb_image(31, H, W)
    feat, score = al_maps(img, al_weights)
    C = int((border_zeroed_nms(score, 2) > 0).sum())
    assert C > K, C
    ref = refine_oracle(feat, score, topk_oracle(score, 2, K), 2, al_weights)
    out = _native.AlikedNet(ctx, al_weights, K, -1.0, 2, H, W).extract(img)
    assert len(out["keypoints"]) == K
    same_pos = pair_aliked(out, ref, max_unpaired=32)
    assert same_pos > 0.9, same_pos


@pytest.mark.gpu
@pytest.mark.parametrize("K", [10000, 20000])
def test_aliked_topk_fill(ctx, al_weights, K):
    """Top-k mode with C < K: the first C against the oracle; every tail keypoint comes from a zero pixel of the border-zeroed NMS map,
    the first ones in row-major order, and equals the index-given oracle's."""
    from dim_b200 import _native
    img = rgb_image(32, 256, 256)
    H, W = img.shape[:2]
    feat, score = al_maps(img, al_weights)
    net = _native.AlikedNet(ctx, al_weights, K, 0.0, 2, H, W)
    out = net.extract(img)
    assert len(out["keypoints"]) == K
    # the pixels the kernels chose from: the NMS of the device's own score map (NMS is exact, so this is the map they ran on)
    nms_dev = border_zeroed_nms(torch.from_numpy(net.debug_read(0, (H, W)))[None, None], 2).reshape(-1)
    cand = torch.nonzero(nms_dev > 0)[:, 0]
    C = len(cand)
    assert 0 < C < K
    head = refine_oracle(feat, score, topk_oracle(score, 2, C), 2, al_weights)
    pair_aliked({k: (v[:C] if k != "descriptors" else v[:, :C]) for k, v in out.items()}, head, max_unpaired=8)
    zero = torch.nonzero(nms_dev == 0)[:, 0][:K - C]
    assert len(zero) == K - C and bool((nms_dev[zero] == 0).all())
    tail = refine_oracle(feat, score, zero, 2, al_weights)
    got = {k: (v[C:] if k != "descriptors" else v[:, C:]) for k, v in out.items()}
    assert np.abs(got["keypoints"] - tail["keypoints"]).max() < 1e-3
    assert np.abs(got["scores"] - tail["scores"]).max() < TOL
    assert np.abs(got["descriptors"] - tail["descriptors"]).max() < TOL


@pytest.mark.gpu
def test_aliked_topk_refuses_k_above_pixels(ctx, al_weights):
    from dim_b200 import _native
    net = _native.AlikedNet(ctx, al_weights, 64 * 64 + 1, -1.0, 2, 64, 64)
    with pytest.raises(_native.DimbError, match="exceeds"):
        net.extract(rgb_image(33, 64, 64))
    assert len(_native.AlikedNet(ctx, al_weights, 64 * 64, -1.0, 2, 64, 64).extract(rgb_image(33, 64, 64))["keypoints"]) == 64 * 64


@pytest.mark.gpu
@pytest.mark.parametrize("H, W, thr, K", [(512, 512, -1.0, -1), (2048, 2048, -1.0, -1), (2048, 2048, 0.005, 18000)])
def test_aliked_mean_and_threshold_n_limit(ctx, al_weights, H, W, thr, K):
    """Mean mode (both <= 0: nms > mean(score_map), n_limit 20000) below and above 20000 candidates, and threshold mode with an n_limit
    above 16384 that fires, against oracle.aliked.extract."""
    from dim_b200 import _native
    from oracle import aliked as o_al
    img = rgb_image(34, H, W)
    conf = {"model_name": "aliked-n16rot", "max_num_keypoints": K, "detection_threshold": thr, "nms_radius": 2}
    ref = o_al.extract(img, al_weights, conf, return_debug=True)
    score = torch.from_numpy(ref["_score_map"])[None, None]
    t = float(score.mean()) if thr <= 0 else thr
    C = int((border_zeroed_nms(score, 2) > t).sum())
    n_limit = K if K > 0 else 20000
    print("aliked", H, W, thr, K, "candidates", C)
    if H == 512:
        assert C < n_limit
    else:
        assert C > n_limit > 16384
    out = _native.AlikedNet(ctx, al_weights, K, thr, 2, H, W).extract(img)
    assert abs(len(out["keypoints"]) - len(ref["keypoints"])) <= 16
    assert pair_aliked(out, ref, max_unpaired=32) > 0.9


# ------------------------------------------------------------------ plugins and image sets
@pytest.mark.gpu
def test_aliked_plugin_topk(ctx, al_weights):
    from dim_b200 import _native
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    img = rgb_image(35, 300, 400)
    for conf in ({"max_num_keypoints": 2048, "detection_threshold": -1, "nms_radius": 2},
                 {"max_num_keypoints": -1, "detection_threshold": -1, "nms_radius": 2}):
        ext = AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", **conf, "weights_dict": al_weights}))
        got = ext._extract(img)
        exp = _native.AlikedNet(ctx, al_weights, conf["max_num_keypoints"], conf["detection_threshold"], 2, 300, 400).extract(img)
        for k in ("keypoints", "scores", "descriptors"):
            assert np.array_equal(got[k], exp[k]), (conf, k)
    assert len(got["keypoints"]) > 100


def _nn_plugin():
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    return KorniaMatcher(Config(matcher={"name": "kornia_matcher", "match_mode": "smnn", "th": 0.95}))


@pytest.mark.gpu
@pytest.mark.parametrize("tiled", [False, True])
def test_aliked_topk_set(ctx, al_weights, tiled):
    """An ALIKED top-k set (untiled, and grid-tiled) stores the per-image plugin flow's features, and kornia_matcher's tables equal
    the plugin's on them."""
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.sharded import ImageSetMatcher, tile_pairs_for
    from test_tiled_sets import _reference_features, _same_features
    a = synthetic.blocks_image(36, 512)[:384]
    imgs = np.stack([a] + [synthetic.warp_pair(a, 60 + k, jitter=24.0) for k in (1, 2)]).astype(np.float32)
    al_conf = {"max_num_keypoints": 1500, "detection_threshold": -1.0, "nms_radius": 3}
    kw = {"tiling": {"tile_size": 256, "tile_overlap": 32, "tile_selection": "grid"}} if tiled else {}
    eng = ImageSetMatcher(ctx, al_weights, None, 3, 384, 512, al_conf, {"match_mode": "smnn", "th": 0.95}, batch_images=2,
                          batch_pairs=16 if tiled else 2, extractor="aliked", matcher="kornia_matcher", **kw)
    pairs = [(0, 1), (0, 2), (1, 2)]
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    general = {"tile_size": 256, "tile_overlap": 32} if tiled else {}
    ext = AlikedExtractor(Config(general=general, extractor={"model_name": "aliked-n16rot", **al_conf, "weights_dict": al_weights}))
    plugin = _nn_plugin()
    feats = []
    for i in range(3):
        if tiled:
            ref = _reference_features(ext, imgs[i])[0]
            _same_features(eng.store.get(i), ref)
        else:
            ref = as_half_roundtrip({**ext._extract(imgs[i]), "image_size": np.array(imgs[i].shape[:2])})
            got = eng.store.get(i)
            for k in ("keypoints", "descriptors", "scores"):
                assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), (i, k)
            assert len(ref["keypoints"]) == 1500
        feats.append(ref)
    for (i, j), t in zip(pairs, tables):
        exp = plugin._match_by_tile(feats[i], feats[j], tile_pairs_for("grid", eng.T)) if tiled else plugin._match_pairs(feats[i], feats[j])
        assert np.array_equal(t, exp), (i, j, len(t), len(exp))
    assert sum(len(t) for t in tables) > 20


@pytest.mark.gpu
def test_superpoint_set_above_16384(ctx, sp_weights):
    """A SuperPoint set at max_keypoints 20000 stores SuperPointExtractor's features, and kornia_matcher's tables equal the plugin's."""
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(37, 1024, 8)[:768]
    imgs = np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x))
                     for x in [a] + [synthetic.warp_pair(a, 70 + k, jitter=24.0) for k in (1, 2)]]).astype(np.float32)
    sp_conf = {**SP_CONF, "max_keypoints": 20000}
    eng = ImageSetMatcher(ctx, sp_weights, None, 3, 768, 1024, sp_conf, {"match_mode": "smnn", "th": 0.95}, batch_images=2, batch_pairs=2,
                          matcher="kornia_matcher")
    pairs = [(0, 1), (0, 2), (1, 2)]
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={"name": "superpoint", **sp_conf, "weights_dict": sp_weights}))
    feats = [as_half_roundtrip({**ext._extract(g), "image_size": np.array(g.shape)}) for g in imgs]
    for i in range(3):
        got = eng.store.get(i)
        for k in ("keypoints", "descriptors", "scores"):
            assert got[k].shape == feats[i][k].shape and np.array_equal(got[k], feats[i][k]), (i, k)
    assert min(len(f["keypoints"]) for f in feats) == 20000
    plugin = _nn_plugin()
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
