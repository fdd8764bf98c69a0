"""Tile preselection on the device: the INTER_AREA resize (dimb_resize_area_dev), the own-extent LightGlue size
(dimb_kpts_extent_dev + dimb_feats_dev.size_f32_dev), the tile box count (dimb_tile_preselect_dev), and
ImageSetMatcher(tiling={"tile_selection": "preselection", ...}) checked against the reference's host flow -
cv2.resize, tiling.preselection_matches and tiling.tile_selection - on the same native networks.  Every comparison is exact."""
import ctypes as C

import cv2
import numpy as np
import pytest

# sizes (H, W) -> (H2, W2): the general INTER_AREA order, power-of-two factors, OpenCV's integer-factor path, and identity
RESIZE_CASES = [((1536, 2048), (750, 1000)), ((1536, 2048), (525, 700)), ((1536, 2048), (768, 1024)), ((1000, 1300), (394, 512)),
                ((1000, 1300), (769, 1000)), ((1024, 1024), (512, 512)), ((2048, 2048), (512, 512)), ((768, 1024), (384, 512)),
                ((768, 768), (256, 256)), ((512, 1536), (512, 512)), ((600, 900), (200, 300)), ((1000, 1300), (1000, 1300)),
                ((1000, 1300), (500, 650)), ((1002, 1298), (501, 649)), ((1000, 1030), (500, 515)), ((1000, 1034), (500, 517))]
# the last four are 2 x 2 with W2 % 4 = 2, 1, 3, 1: OpenCV's scalar tail after its 4-lane vector loop


def _fast_factor(s, d):
    """cv::resize's is_area_fast test on one axis: the integer factor, or 0."""
    scale = 1.0 / (d / s)
    i = int(round(scale))
    return i if abs(scale - i) < np.finfo(np.float64).eps else 0


def _area_restated(img, H2, W2):
    """The kernel's accumulation order in numpy float32 (no FMA): OpenCV's resizeArea_ over the tables of dimb_resize_area_tab, or
    resizeAreaFast_ for integer factors; for 2 x 2 its 4-lane vector order over the first floor(W2 / 4) * 4 columns."""
    from dim_b200 import _native
    H, W = img.shape
    if (H2, W2) == (H, W):
        return img.copy()
    fy, fx = _fast_factor(H, H2), _fast_factor(W, W2)
    if fy and fx:
        blk = img[:H2 * fy, :W2 * fx].reshape(H2, fy, W2, fx).transpose(0, 2, 1, 3).reshape(H2, W2, fy * fx)
        s, k, area = np.zeros((H2, W2), np.float32), 0, fy * fx
        while k <= area - 4:
            s = s + (((blk[..., k] + blk[..., k + 1]) + blk[..., k + 2]) + blk[..., k + 3])
            k += 4
        for k in range(k, area):
            s = s + blk[..., k]
        out = s * (np.float32(1) / np.float32(area))
        if (fy, fx) == (2, 2):
            e = W2 // 4 * 4
            out[:, :e] = ((blk[:, :e, 0] + blk[:, :e, 1]) + (blk[:, :e, 2] + blk[:, :e, 3])) * np.float32(0.25)
        return out

    def axis(ssize, dsize):
        di, si, al = _native.resize_area_tab(ssize, dsize)
        assert np.all(np.diff(di) >= 0) and di[0] == 0 and di[-1] == dsize - 1
        return np.searchsorted(di, np.arange(dsize + 1)), si, al
    xo, xs, xa = axis(W, W2)
    yo, ys, ya = axis(H, H2)
    cnt = np.diff(xo)
    out = np.empty((H2, W2), np.float32)
    for dy in range(H2):
        acc = None
        for j in range(yo[dy], yo[dy + 1]):
            row, buf = img[ys[j]], np.zeros(W2, np.float32)
            for k in range(int(cnt.max())):
                ok = k < cnt
                idx = xo[:-1][ok] + k
                buf[ok] = buf[ok] + row[xs[idx]] * xa[idx]
            v = ya[j] * buf
            acc = v if acc is None else acc + v
        out[dy] = acc
    return out


def _images(H, W, seed):
    """One integer-valued and one non-integer float32 gray image of size H x W."""
    from dim_b200 import synthetic
    rng = np.random.default_rng(seed)
    gray = synthetic.to_gray_like_reference(synthetic.blocks_image(seed, max(H, W))[:H, :W])
    return [rng.integers(0, 256, (H, W)).astype(np.float32), np.ascontiguousarray(gray, np.float32)]


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


def test_preselection_entries_reject_bad_arguments_without_touching_the_gpu():
    """Argument validation of the new entries comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    n = C.c_int()
    di, si, al = (C.c_int * 64)(), (C.c_int * 64)(), (C.c_float * 64)()
    assert lib.dimb_resize_area_tab(10, 4, di, si, al, 64, C.byref(n)) == 0 and 4 <= n.value <= 20
    for ss, ds in ((0, 1), (10, 0), (4, 10), (-1, -1)):
        assert lib.dimb_resize_area_tab(ss, ds, di, si, al, 64, C.byref(n)) == -3, (ss, ds)
    assert lib.dimb_resize_area_tab(10, 4, di, si, al, 64, None) == -3
    assert lib.dimb_resize_area_tab(10, 4, di, si, al, 2, C.byref(n)) == -5 and n.value > 2  # capacity: the count is reported

    def resize(ctx=ctx, src=dev, B=1, H=768, W=1024, dst=dev, H2=384, W2=512):
        return lib.dimb_resize_area_dev(ctx, src, B, H, W, dst, H2, W2, null)
    assert resize(ctx=null) == -3 and resize(src=null) == -3 and resize(dst=null) == -3
    assert resize(B=0) == -3 and resize(H=0) == -3 and resize(H2=0) == -3 and resize(W2=0) == -3
    assert resize(H2=769) == -3 and resize(W2=1025) == -3 and resize(B=70000) == -3  # upscaling is refused

    def extent(ctx=ctx, B=2, k=dev, ld=64, n=dev, out=dev):
        return lib.dimb_kpts_extent_dev(ctx, B, k, ld, n, out, null)
    assert extent(ctx=null) == -3 and extent(k=null) == -3 and extent(n=null) == -3 and extent(out=null) == -3
    assert extent(B=0) == -3 and extent(ld=0) == -3

    feats = (_native.FeatsDev * 2)()
    for f in feats:
        f.keypoints = 0x1000
    no_kpts = (_native.FeatsDev * 2)()

    def pre(ctx=ctx, Q=2, f0=feats, f1=feats, m=dev, nm=dev, cap=64, tile=(512, 512), ov=64, sc=0.5, mm=5, cnt=dev, fl=dev):
        return lib.dimb_tile_preselect_dev(ctx, Q, f0, f1, m, nm, cap, 768, 1024, tile[0], tile[1], ov, ov, sc, sc, mm, cnt, fl, null)
    assert pre(ctx=null) == -3 and pre(f0=None) == -3 and pre(f1=None) == -3 and pre(m=null) == -3 and pre(nm=null) == -3
    assert pre(cnt=null) == -3 and pre(fl=null) == -3 and pre(f0=no_kpts) == -3 and pre(f1=no_kpts) == -3
    assert pre(Q=0) == -3 and pre(cap=0) == -3 and pre(tile=(0, 512)) == -3 and pre(ov=512) == -3 and pre(tile=(16, 16), ov=0) == -3
    assert pre(sc=0.0) == -3 and pre(sc=-0.5) == -3 and pre(sc=float("inf")) == -3 and pre(sc=float("nan")) == -3 and pre(mm=-1) == -3


@pytest.mark.parametrize("case", RESIZE_CASES)
def test_resize_area_tables_reproduce_cv2_bitwise(case):
    (H, W), (H2, W2) = case
    for img in _images(H, W, H2):
        ref = cv2.resize(img, (W2, H2), interpolation=cv2.INTER_AREA)
        got = _area_restated(img, H2, W2)
        assert got.dtype == np.float32 and got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_resize_area_tab_matches_opencv_formulas():
    from dim_b200 import _native
    di, si, al = _native.resize_area_tab(10, 4)  # scale 2.5: partial weights at both ends of the cells
    assert di.tolist() == [0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3]
    assert si.tolist() == [0, 1, 2, 2, 3, 4, 5, 6, 7, 7, 8, 9]
    assert np.array_equal(al, np.array([0.4, 0.4, 0.2, 0.2, 0.4, 0.4, 0.4, 0.4, 0.2, 0.2, 0.4, 0.4], np.float32))
    with pytest.raises(ValueError):
        _native.resize_area_tab(4, 10)


def test_tiling_conf_preselection():
    from dim_b200.sharded import tiling_conf
    c = tiling_conf({"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512})
    assert c["tile_selection"] == "preselection" and c["tile_preselection_size"] == 512 and c["min_matches_per_tile"] == 5
    c = tiling_conf({"tile_size": 512, "tile_selection": "PRESELECTION", "tile_preselection_size": 300, "min_matches_per_tile": 0})
    assert c["min_matches_per_tile"] == 0
    base = {"tile_size": 512, "tile_selection": "preselection"}
    for bad in (base, {**base, "tile_preselection_size": 0}, {**base, "tile_preselection_size": 512.0}, {**base, "tile_preselection_size": "512"},
                {**base, "tile_preselection_size": True}, {**base, "tile_preselection_size": 512, "min_matches_per_tile": -1},
                {**base, "tile_preselection_size": 512, "min_matches_per_tile": 2.5}, {**base, "tile_preselection_size": 512, "tiles": 4}):
        with pytest.raises(ValueError):
            tiling_conf(bad)
    for sel in ("grid", "exhaustive"):  # reference configurations carry the keys whatever the selection
        c = tiling_conf({"tile_size": 512, "tile_selection": sel, "tile_preselection_size": 1024, "min_matches_per_tile": 3})
        assert c["tile_selection"] == sel and "tile_preselection_size" not in c


def test_matcher_refuses_inconsistent_preselection_options():
    from dim_b200.sharded import ImageSetMatcher
    pre = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}
    with pytest.raises(ValueError, match="superpoint"):
        ImageSetMatcher(None, {}, {}, 2, 768, 1024, {"max_num_keypoints": 512}, {}, tiling=pre, extractor="aliked")
    with pytest.raises(ValueError, match="preselection_weights"):
        ImageSetMatcher(None, {}, {}, 2, 768, 1024, {"max_keypoints": 512}, {}, tiling=pre, matcher="superglue")
    with pytest.raises(ValueError, match="downscales"):
        ImageSetMatcher(None, {}, {}, 2, 768, 1024, {"max_keypoints": 512}, {}, tiling={**pre, "tile_preselection_size": 1025})


# ---------------------------------------------------------------------------------------------------------------- on the GPU


@pytest.mark.gpu
def test_resize_area_dev_equals_cv2(ctx):
    import torch
    for (H, W), (H2, W2) in RESIZE_CASES:
        imgs = np.stack(_images(H, W, H2) + [_images(H, W, H2 + 1)[1]])
        ref = np.stack([cv2.resize(im, (W2, H2), interpolation=cv2.INTER_AREA) for im in imgs])
        src = torch.from_numpy(imgs).cuda()
        out = torch.full((3, H2, W2), -1.0, device="cuda")
        ctx.resize_area_dev(src.data_ptr(), 3, H, W, out.data_ptr(), H2, W2, 0)
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (H, W, H2, W2)
        for b in range(3):  # one image per call gives the same bits
            one = torch.full((1, H2, W2), -1.0, device="cuda")
            ctx.resize_area_dev(src[b].data_ptr(), 1, H, W, one.data_ptr(), H2, W2, 0)
            assert np.array_equal(one.cpu().numpy()[0].view(np.uint32), got[b].view(np.uint32))


@pytest.mark.gpu
def test_kpts_extent_dev_equals_numpy(ctx):
    import torch
    rng = np.random.default_rng(0)
    ld = 300
    kp = rng.uniform(-3.5, 700.25, (4, ld, 2)).astype(np.float32)
    counts = np.array([ld, 17, 0, 1], np.int32)
    d_kp, d_counts = torch.from_numpy(kp).cuda(), torch.from_numpy(counts).cuda()
    out = torch.full((4, 2), -1.0, device="cuda")
    ctx.kpts_extent_dev(4, d_kp.data_ptr(), ld, d_counts.data_ptr(), out.data_ptr(), 0)
    got = out.cpu().numpy()
    for b, n in enumerate(counts):
        k = kp[b, :n]
        exp = (np.float32(1) + k.max(0)) - k.min(0) if n else np.ones(2, np.float32)
        assert exp.dtype == np.float32 and np.array_equal(got[b], exp), b
    assert np.array_equal(got[3], np.ones(2, np.float32))


def _low_res_features(ctx, sp_weights, imgs, size):
    """tiling.preselection_matches' extraction: cv2 INTER_AREA to the longest side `size`, SuperPoint with SP_PRESELECTION_CONF."""
    from dim_b200 import _native, tiling
    H, W = imgs.shape[1:]
    scale = size / max(W, H)
    W2, H2 = (int(round(x * scale)) for x in (W, H))
    sp = _native.SuperPointNet(ctx, sp_weights, max_height=H2, max_width=W2, **tiling.SP_PRESELECTION_CONF)
    low = [cv2.resize(im, (W2, H2), interpolation=cv2.INTER_AREA) for im in imgs]
    return [sp.extract(np.ascontiguousarray(x, np.float32)[None])[0] for x in low], scale


class _DevSide:
    """Float32 low-resolution features in device memory as a FeatsDev normalised by their own extent (dimb_kpts_extent_dev)."""

    def __init__(self, ctx, f, K=4000):
        import torch
        from dim_b200 import _native
        n = len(f["keypoints"])
        self.kp = torch.zeros(K, 2, device="cuda")
        self.de = torch.zeros(256, K, device="cuda")
        self.kp[:n] = torch.from_numpy(f["keypoints"]).cuda()
        self.de[:, :n] = torch.from_numpy(f["descriptors"]).cuda()
        self.n = torch.tensor([n], dtype=torch.int32, device="cuda")
        self.size = torch.zeros(2, device="cuda")
        ctx.kpts_extent_dev(1, self.kp.data_ptr(), K, self.n.data_ptr(), self.size.data_ptr(), 0)
        self.f = _native.FeatsDev(self.kp.data_ptr(), self.de.data_ptr(), self.n.data_ptr(), K, 0, K, 0.0, 0.0, 0, 0, None, self.size.data_ptr())


@pytest.mark.gpu
def test_lightglue_own_extent_on_device_equals_host(ctx, sp_weights):
    """LightGlue without image_size: match_dev with size_f32_dev gives the host entry's tables, scores and stop layers."""
    import torch
    from dim_b200 import _native, tiling, weights
    imgs = _gray_set(4)
    feats, _ = _low_res_features(ctx, sp_weights, imgs, 512)
    w = weights.lightglue_seeded(seed=0)
    lg = _native.LightGlueNet(ctx, w, max_pairs=3, max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    pairs = [(0, 1), (2, 3), (1, 3)]
    host = lg.match([({**feats[i], "_layout": 0}, {**feats[j], "_layout": 0}) for i, j in pairs])
    sides = [_DevSide(ctx, f) for f in feats]
    m = torch.full((3, 4000, 2), -1, dtype=torch.int64, device="cuda")
    ms = torch.zeros(3, 4000, device="cuda")
    nm, sl = torch.zeros(3, dtype=torch.int32, device="cuda"), torch.zeros(3, dtype=torch.int32, device="cuda")
    lg.match_dev([sides[i].f for i, _ in pairs], [sides[j].f for _, j in pairs], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), sl.data_ptr(), 4000, 0)
    m, ms, nm, sl = m.cpu().numpy(), ms.cpu().numpy(), nm.cpu().numpy(), sl.cpu().numpy()
    for p, h in enumerate(host):
        assert np.array_equal(m[p, :nm[p]], h["matches"]) and np.array_equal(ms[p, :nm[p]], h["scores"]) and sl[p] == h["stop"], p
    assert min(len(h["matches"]) for h in host) > 0


def _host_counts(kp0, kp1, tile_size, overlap, H, W):
    """Per (t0, t1): matches strictly inside both boxes (the loop of tiling.tile_selection, counted)."""
    from dim_b200 import tiling
    _, orig, _ = tiling.compute_tiles_by_size(np.zeros((H, W), np.float32), tile_size, overlap)
    T = len(orig)
    ins = [[tiling.points_in_rect(kp, tiling.get_tile_bounding_box(orig[t], tile_size)) for t in range(T)] for kp in (kp0, kp1)]
    return np.array([[int(np.sum(ins[0][a] & ins[1][b])) for b in range(T)] for a in range(T)], np.int32)


def _planted(H, W, th, tw, ov_hw, scale, seed):
    """Low-resolution keypoints and match tables of four image pairs: random points (negative coordinates in the padding included)
    plus points planted exactly on box edges; the edges alone (matched to themselves); an empty table; random points only.  Edge
    points are multiples of the dyadic scale, so kpt / scale lands exactly on the edge again."""
    from dim_b200 import _native
    g = _native.tile_grid(H, W, th, tw, *ov_hw)
    edges = np.array([(ox + dx, oy + dy) for ox, oy in g["origins"]
                      for dx, dy in ((0, 5), (tw, 7), (9, 0), (11, th), (0, 0), (tw, th), (tw // 2, th // 2))], np.float64)
    rng = np.random.default_rng(seed)

    def rand(k):
        return np.stack([rng.uniform(-g["pad_left"] - 8, W + 8, k), rng.uniform(-g["pad_top"] - 8, H + 8, k)], 1)

    def table(n0, n1, k):
        return np.stack([rng.integers(0, n0, k), rng.integers(0, n1, k)], 1).astype(np.int64)
    e = len(edges)
    ident = np.stack([np.arange(e), np.arange(e)], 1).astype(np.int64)
    cases = [([np.concatenate([edges, rand(600)]), np.concatenate([edges, rand(500)])], np.concatenate([ident, table(e + 600, e + 500, 700)])),
             ([edges, edges], ident), ([rand(50), rand(50)], np.zeros((0, 2), np.int64)), ([rand(300), rand(300)], table(300, 300, 400))]
    return [([(p * scale).astype(np.float32) for p in pts], m) for pts, m in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [((768, 1024), (512, 512), 64, 0.5), ((1000, 1300), (256, 384), 32, 0.375), ((2048, 2048), (256, 256), 0, 0.25)])
def test_device_tile_preselection_equals_tile_selection(ctx, geom):
    """The box count against tiling.tile_selection on planted matches: strict edges, negative origins, an empty table, T up to 64,
    tile_w != tile_h; min_matches_per_tile 5, then a count that occurs (not selected) and one below it (selected)."""
    import torch
    from dim_b200 import _native, tiling
    (H, W), tile_size, overlap, scale = geom
    (th, tw), ov_hw = tiling._hw(tile_size), tiling._hw(overlap)
    T = len(_native.tile_grid(H, W, th, tw, *ov_hw)["origins"])
    cases = _planted(H, W, th, tw, ov_hw, scale, T)
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
    img = np.zeros((H, W), np.float32)
    host = []
    for low, m in cases:
        kp0, kp1 = low[0][m[:, 0]] / scale, low[1][m[:, 1]] / scale  # as preselection_matches maps them back (float32)
        assert kp0.dtype == np.float32
        host.append((kp0, kp1, _host_counts(kp0, kp1, tile_size, overlap, H, W)))
    nz = host[0][2][host[0][2] > 0]
    v = int(np.median(nz))
    assert T >= 4 and v >= 1 and len(host[1][0]) == 7 * T
    for mm in (5, v, v - 1):
        counts = torch.full((len(cases), T * T), -1, dtype=torch.int32, device="cuda")
        flags = torch.full((len(cases), T * T), 7, dtype=torch.uint8, device="cuda")
        ctx.tile_preselect_dev(f0, f1, d_m.data_ptr(), d_nm.data_ptr(), cap, H, W, th, tw, *ov_hw, scale, scale, mm, counts.data_ptr(),
                               flags.data_ptr(), 0)
        counts, flags = counts.cpu().numpy().reshape(-1, T, T), flags.cpu().numpy().reshape(-1, T, T)
        for q, (kp0, kp1, exp) in enumerate(host):
            assert np.array_equal(counts[q], exp), (mm, q)
            lst = tiling.tile_selection(img, img, "preselection", tile_size, overlap, kp0=kp0, kp1=kp1, min_matches_per_tile=mm)
            assert [(int(a), int(b)) for a, b in zip(*np.nonzero(flags[q]))] == lst, (mm, q)
        assert not flags[2].any() and not counts[2].any()  # the empty table
        if mm == v:
            assert not flags[0][counts[0] == v].any()
        if mm == v - 1:
            assert flags[0][counts[0] == v].all()


def _gray_set(n, H=768, W=1024):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(40, max(H, W))[:H, :W]
    imgs = [a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in range(1, n)]
    return np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in imgs]).astype(np.float32)


def _host_lists(ctx, sp_weights, lg_w, imgs, pairs, size, tile_size, overlap):
    """tiling.preselection_matches + tiling.tile_selection per pair, as test_image_set_matcher_explicit_preselection_lists builds them."""
    from dim_b200 import _native, tiling
    sp_pre = lambda H, W: _native.SuperPointNet(ctx, sp_weights, max_height=H, max_width=W, **tiling.SP_PRESELECTION_CONF)
    lg_pre = _native.LightGlueNet(ctx, lg_w, max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    lists = []
    for i, j in pairs:
        kp0, kp1 = tiling.preselection_matches(imgs[i], imgs[j], size, sp_pre, lg_pre)
        lists.append(tiling.tile_selection(imgs[i], imgs[j], "preselection", tile_size, overlap, kp0=kp0, kp1=kp1))
    return lists


SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "fix_sampling": True}
PRESEL = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}


@pytest.fixture(scope="module")
def pre_set(ctx, sp_weights):
    import torch
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    imgs = _gray_set(3)
    w = weights.lightglue_seeded(seed=0)
    pairs = pairs_from_bruteforce([0, 1, 2])
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    lists = _host_lists(ctx, sp_weights, w, imgs, pairs, 512, (512, 512), 64)
    return {"imgs": imgs, "d": torch.from_numpy(imgs).cuda(), "w": w, "plugin": plugin, "pairs": pairs, "lists": lists}


def _engine(ctx, sp_weights, s, batch_pairs, **kw):
    from dim_b200.sharded import ImageSetMatcher
    return ImageSetMatcher(ctx, sp_weights, s["w"], 3, 768, 1024, {**SP_CONF, "max_keypoints": 1024}, {}, batch_images=6,
                           batch_pairs=batch_pairs, tiling=PRESEL, **kw)


@pytest.mark.gpu
def test_image_set_matcher_preselection_equals_host_flow(ctx, sp_weights, pre_set):
    s, pairs, lists = pre_set, pre_set["pairs"], pre_set["lists"]
    assert any(0 < len(lst) < 16 for lst in lists), lists  # preselection actually selects
    base = None
    for bp in (16, 40):
        eng = _engine(ctx, sp_weights, s, bp)
        assert eng.T == 4 and (eng.pre_h, eng.pre_w) == (384, 512)
        tables = eng.run(s["d"], [0, 1, 2], pairs)
        assert eng._preselect(pairs) == lists
        if base is None:
            exp = [s["plugin"]._match_by_tile(eng.store.get(i), eng.store.get(j), lst) for (i, j), lst in zip(pairs, lists)]
            assert all(np.array_equal(a, b) for a, b in zip(tables, exp)) and max(len(t) for t in exp) > 0
            base = tables
        else:
            assert all(np.array_equal(a, b) for a, b in zip(tables, base))
        perm = [2, 0, 1]
        res = eng.match([pairs[k] for k in perm], perm)
        assert all(np.array_equal(res[k], base[k]) for k in range(3))
        explicit = eng.match(pairs, [0, 1, 2], tile_pairs=[[(0, 0)]] * 3)  # explicit lists still override the configured selection
        exp0 = [s["plugin"]._match_by_tile(eng.store.get(i), eng.store.get(j), [(0, 0)]) for i, j in pairs]
        assert all(np.array_equal(explicit[k], exp0[k]) for k in range(3))


@pytest.mark.gpu
def test_preselection_run_verified(ctx, sp_weights, pre_set):
    import torch
    from dim_b200.geometric_verification import gv_seed
    s, pairs = pre_set, pre_set["pairs"]
    eng = _engine(ctx, sp_weights, s, 16, verification={"seed": 3})
    res = eng.run_verified(s["d"], [0, 1, 2], pairs)
    tables = eng.run(s["d"], [0, 1, 2], pairs)
    P, cap = len(pairs), max(1, max(len(t) for t in tables))
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


@pytest.mark.gpu
def test_preselection_with_superglue(ctx, sp_weights):
    import torch
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from dim_b200.sharded import ImageSetMatcher
    from oracle import superglue as o_sg
    imgs = _gray_set(2, 512, 640)
    w_sg, w_lg = o_sg.seeded_weights(1), weights.lightglue_seeded(seed=0)
    conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
    tiled = {"tile_size": (384, 384), "tile_overlap": 32, "tile_selection": "preselection", "tile_preselection_size": 320}
    eng = ImageSetMatcher(ctx, sp_weights, w_sg, 2, 512, 640, {**SP_CONF, "max_keypoints": 512}, conf, batch_pairs=16, matcher="superglue",
                          tiling=tiled, preselection_weights=w_lg)
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1], [(0, 1)])
    lists = _host_lists(ctx, sp_weights, w_lg, imgs, [(0, 1)], 320, (384, 384), 32)
    assert eng._preselect([(0, 1)]) == lists and len(lists[0]) > 0
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": w_sg}))
    exp = plugin._match_by_tile(eng.store.get(0), eng.store.get(1), lists[0])
    assert np.array_equal(tables[0], exp) and len(exp) > 0


@pytest.mark.gpu
def test_preselection_entries_are_asynchronous(ctx):
    """Queued behind a ~0.5 s device spin (after a first call has grown the scratch), each entry returns while the stream is busy."""
    import torch
    from dim_b200 import _native
    H, W, H2, W2 = 1536, 2048, 750, 1000
    img = torch.from_numpy(_images(H, W, 1)[1]).cuda()
    low = torch.zeros(H2, W2, device="cuda")
    kp = torch.from_numpy(np.random.default_rng(0).uniform(0, 500, (64, 2)).astype(np.float32)).cuda()
    n = torch.tensor([64], dtype=torch.int32, device="cuda")
    size = torch.zeros(2, device="cuda")
    f = _native.FeatsDev()
    f.keypoints = kp.data_ptr()
    m = torch.stack([torch.arange(64), torch.arange(64)], 1).to(torch.int64).cuda()[None]
    counts, flags = torch.zeros(1, 16, dtype=torch.int32, device="cuda"), torch.zeros(1, 16, dtype=torch.uint8, device="cuda")
    calls = [lambda st: ctx.resize_area_dev(img.data_ptr(), 1, H, W, low.data_ptr(), H2, W2, st),
             lambda st: ctx.kpts_extent_dev(1, kp.data_ptr(), 64, n.data_ptr(), size.data_ptr(), st),
             lambda st: ctx.tile_preselect_dev([f], [f], m.data_ptr(), n.data_ptr(), 64, 768, 1024, 512, 512, 64, 64, 0.5, 0.5, 5,
                                               counts.data_ptr(), flags.data_ptr(), st)]
    for call in calls:
        call(0)
    torch.cuda.synchronize()
    ref = [low.clone(), size.clone(), flags.clone()]
    low.fill_(-1), size.fill_(-1), flags.fill_(7)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    for call in calls:
        with torch.cuda.stream(s):
            torch.cuda._sleep(1_000_000_000)
        call(s.cuda_stream)
        busy = not s.query()
        s.synchronize()
        assert busy
    for a, b in zip(ref, (low, size, flags)):
        assert torch.equal(a, b)
