"""Extraction quality on the device: cv2.pyrDown / cv2.pyrUp (dimb_pyr_size / dimb_pyr_dev), the keypoint rescale of store slots
(dimb_fstore_rescale_dev) and ImageSetMatcher(quality=...) checked against the reference's host flow (_resize_image, the plugin's
_extract or _extract_by_tile, _resize_features, the float16 cast of features.h5).  Every comparison is exact."""
import ctypes as C

import cv2
import numpy as np
import pytest

LEVELS = {"highest": -1, "high": 0, "medium": 1, "low": 2, "lowest": 3}
# (H, W): even and odd axes, 1- to 3-pixel axes, the reference's 533 x 800 test photos
SIZES = [(64, 64), (533, 800), (33, 47), (1, 1), (1, 2), (2, 1), (3, 3), (2, 5), (5, 2), (3, 7), (7, 9), (8, 11), (13, 6), (1, 17),
         (17, 1), (41, 43), (100, 101), (99, 98)]
F = np.float32


def _reflect101(p, n):
    """cv::borderInterpolate(p, n, BORDER_REFLECT_101)."""
    if n == 1:
        return 0
    while p < 0 or p >= n:
        p = -p if p < 0 else 2 * n - 2 - p
    return p


def _pyr_down(img):
    """pyrDown_ in numpy float32, each product and sum rounded on its own, in the order dimb_pyr_dev uses: horizontal 1 4 6 4 1 sums
    (OpenCV's 4-lane vector order on the columns its SIMD loop covers, the scalar order elsewhere), then the vertical sums (vector
    order on the first floor(W2 * C / 4) * 4 values of a row, scalar order on the rest) and * (1 / 256)."""
    gray = img.ndim == 2
    img = img[:, :, None] if gray else img
    H, W, Cn = img.shape
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    width0 = min(int((W - 3) / 2) + 1, W2)  # C division truncates
    vec_end = 1 + (width0 - 1) // 4 * 4 if Cn == 1 and width0 >= 1 else width0 - 1
    hrow = np.empty((H, W2, Cn), F)
    for x in range(W2):
        s0, s1, s2, s3, s4 = (img[:, _reflect101(2 * x - 2 + k, W)] for k in range(5))
        if 1 <= x < vec_end:
            hrow[:, x] = s2 * F(6) + ((s1 + s3) * F(4) + (s0 + s4))
        else:
            hrow[:, x] = ((s2 * F(6) + (s1 + s3) * F(4)) + s0) + s4
    hr = hrow.reshape(H, W2 * Cn)
    nv = W2 * Cn // 4 * 4
    out = np.empty((H2, W2 * Cn), F)
    for y in range(H2):
        r0, r1, r2, r3, r4 = (hr[_reflect101(2 * y - 2 + k, H)] for k in range(5))
        out[y, :nv] = (((r1 + r3 + r2) * F(4) + (r0 + r4 + (r2 + r2))) * F(1 / 256))[:nv]
        out[y, nv:] = ((((r2 * F(6) + (r1 + r3) * F(4)) + r0) + r4) * F(1 / 256))[nv:]
    out = out.reshape(H2, W2, Cn)
    return out[:, :, 0] if gray else out


def _pyr_up(img):
    """pyrUp_ in numpy float32 as dimb_pyr_dev computes it: 1 6 1 / 4 4 sums with OpenCV's border formulas on the doubled grid, then
    * (1 / 64)."""
    gray = img.ndim == 2
    img = img[:, :, None] if gray else img
    H, W, Cn = img.shape
    hrow = np.empty((H, 2 * W, Cn), F)
    if W == 1:
        hrow[:, 0] = hrow[:, 1] = img[:, 0] * F(8)
    else:
        hrow[:, 0] = img[:, 0] * F(6) + img[:, 1] * F(2)
        hrow[:, 1] = (img[:, 0] + img[:, 1]) * F(4)
        for x in range(1, W - 1):
            hrow[:, 2 * x] = (img[:, x - 1] + img[:, x] * F(6)) + img[:, x + 1]
            hrow[:, 2 * x + 1] = (img[:, x] + img[:, x + 1]) * F(4)
        hrow[:, 2 * W - 2] = img[:, W - 2] + img[:, W - 1] * F(7)
        hrow[:, 2 * W - 1] = img[:, W - 1] * F(8)
    out = np.empty((2 * H, 2 * W, Cn), F)
    row = lambda s: hrow[_reflect101(2 * s, 2 * H) // 2]
    for y in range(H):
        r0, r1, r2 = row(y - 1), hrow[y], row(y + 1)
        out[2 * y] = ((r0 + r1 * F(6)) + r2) * F(1 / 64)
        out[2 * y + 1] = ((r1 + r2) * F(4)) * F(1 / 64)
    return out[:, :, 0] if gray else out


def _cv2_pyr(img, level):
    if level < 0:
        return cv2.pyrUp(img)
    for _ in range(level):
        img = cv2.pyrDown(img)
    return img


def _images(shape, seed):
    """One integer-valued and one non-integer float32 image."""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, shape).astype(F), rng.uniform(0, 255, shape).astype(F)]


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("size", SIZES)
def test_pyramid_restatement_equals_cv2_bitwise(size, channels):
    shape = size if channels == 1 else size + (3,)
    for img in _images(shape, size[0] * 1000 + size[1]):
        assert _bits_equal(_pyr_down(img), cv2.pyrDown(img)), (size, channels)
        assert _bits_equal(_pyr_up(img), cv2.pyrUp(img)), (size, channels)


@pytest.mark.parametrize("channels", [1, 3])
def test_pyramid_restatement_chains_equal_cv2_bitwise(channels):
    for size in ((533, 800), (301, 457), (97, 131)):
        shape = size if channels == 1 else size + (3,)
        for img in _images(shape, size[1]):
            a, b = img, img
            for level in (1, 2, 3):
                a, b = _pyr_down(a), cv2.pyrDown(b)
                assert _bits_equal(a, b), (size, channels, level)


def test_pyr_size_equals_cv2_shapes():
    from dim_b200 import _native
    for H, W in SIZES + [(3000, 4000), (1536, 2048), (1999, 3001)]:
        img = np.zeros((H, W), F)
        for level in (-1, 0, 1, 2, 3):
            assert _native.pyr_size(H, W, level) == _cv2_pyr(img, level).shape, (H, W, level)
    for bad in ((0, 5, 1), (5, 0, 1), (5, 5, -2), (5, 5, 4), ((1 << 20) + 1, 5, 1)):
        with pytest.raises(ValueError):
            _native.pyr_size(*bad)


def test_quality_entries_reject_bad_arguments_without_touching_the_gpu():
    """Argument validation of the new entries comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    h2, w2 = C.c_int(), C.c_int()
    assert lib.dimb_pyr_size(533, 800, 1, C.byref(h2), C.byref(w2)) == 0 and (h2.value, w2.value) == (267, 400)
    assert lib.dimb_pyr_size(533, 800, 1, None, C.byref(w2)) == -3 and lib.dimb_pyr_size(533, 800, 1, C.byref(h2), None) == -3

    def pyr(ctx=ctx, src=dev, B=1, H=533, W=800, ch=1, level=1, dst=dev):
        return lib.dimb_pyr_dev(ctx, src, B, H, W, ch, level, dst, null)
    assert pyr(ctx=null) == -3 and pyr(src=null) == -3 and pyr(dst=null) == -3
    assert pyr(B=0) == -3 and pyr(B=70000) == -3 and pyr(H=0) == -3 and pyr(W=0) == -3 and pyr(W=(1 << 20) + 1) == -3
    assert pyr(ch=2) == -3 and pyr(ch=4) == -3 and pyr(ch=0) == -3 and pyr(level=-2) == -3 and pyr(level=4) == -3
    assert pyr(H=40000, level=-1) == -3  # 80000 output rows in one step
    store = C.cast(C.create_string_buffer(256), C.c_void_p)
    slots = (C.c_int * 2)(0, 1)

    def rescale(fs=store, B=2, s=slots, level=1, H=533, W=800):
        return lib.dimb_fstore_rescale_dev(fs, B, s, level, H, W, null)
    assert rescale(fs=null) == -3 and rescale(s=None) == -3 and rescale(B=0) == -3 and rescale(B=70000) == -3
    assert rescale(level=-2) == -3 and rescale(level=4) == -3 and rescale(H=0) == -3 and rescale(W=0) == -3


def test_quality_conf():
    from dim_b200.sharded import quality_conf
    assert quality_conf() == 0
    for name, level in LEVELS.items():
        assert quality_conf(name) == level and quality_conf(name.upper()) == level and quality_conf(name.capitalize()) == level
    for bad in ("", "med", "ultra", "high ", None, 1, 0, b"high"):
        with pytest.raises(ValueError):
            quality_conf(bad)


def test_matcher_refuses_quality_with_preselection_and_too_small_images():
    from dim_b200.sharded import ImageSetMatcher
    sp = {"max_keypoints": 512}
    pre = {"tile_size": 512, "tile_selection": "preselection", "tile_preselection_size": 256}
    for q in ("highest", "medium", "lowest"):
        with pytest.raises(ValueError, match="preselection"):
            ImageSetMatcher(None, {}, {}, 2, 1024, 1024, sp, {}, tiling=pre, quality=q)
    with pytest.raises(ValueError, match="quality"):
        ImageSetMatcher(None, {}, {}, 2, 1024, 1024, sp, {}, quality="best")
    # SuperPoint needs 16 px per side: 100 -> 50 -> 25 -> 13 at "lowest"
    with pytest.raises(ValueError, match="16 px"):
        ImageSetMatcher(None, {}, {}, 2, 100, 400, sp, {}, quality="lowest")
    with pytest.raises(ValueError, match="32 px"):  # ALIKED needs 32: 120 -> 30 at "low"
        ImageSetMatcher(None, {}, {}, 2, 120, 400, {"max_num_keypoints": 512}, {}, extractor="aliked", quality="low")


class _Stub:
    """An ExtractorBase with a stub _extract that records its input and returns fixed keypoints."""

    @staticmethod
    def make(quality, monkeypatch, tmp_path):
        from dim_b200.config import Config
        from dim_b200.extractors import extractor_base as eb

        class Stub(eb.ExtractorBase):
            def _extract(self, image):
                self.seen = image
                kp = np.array([[0.0, 0.0], [3.0, 1.5], [10.25, 7.0]], F)
                return {"keypoints": kp, "descriptors": np.ones((128, 3), F), "scores": np.full(3, 0.5, F)}

            def _frame2tensor(self, image, device="cuda"):
                return image

        saved = {}
        monkeypatch.setattr(eb, "save_features_h5", lambda path, feats, name, as_half=True: saved.update(feats))
        general = {"output_dir": tmp_path} if quality is None else {"output_dir": tmp_path, "quality": quality}
        return Stub(Config(general=general)), saved


@pytest.mark.parametrize("quality", [None] + list(LEVELS))
def test_mirror_extract_resizes_the_image_and_scales_the_keypoints(quality, monkeypatch, tmp_path):
    """ExtractorBase.extract: _extract sees the cv2-resized image, the keypoints come back * 2^level, image_size is the original's."""
    H, W = 101, 150
    img = np.random.default_rng(3).integers(0, 256, (H, W)).astype(np.uint8)
    path = tmp_path / "im.png"
    cv2.imwrite(str(path), img)
    ext, saved = _Stub.make(quality, monkeypatch, tmp_path)
    ext.extract(path)
    level = LEVELS[quality or "high"]
    assert _bits_equal(ext.seen, _cv2_pyr(img.astype(F), level))
    kp = np.array([[0.0, 0.0], [3.0, 1.5], [10.25, 7.0]], F) * F(2.0 ** level)
    assert np.array_equal(saved["keypoints"], kp) and saved["keypoints"].dtype == F
    assert saved["image_size"].tolist() == [H, W] and np.array_equal(saved["tile_idx"], np.zeros(3, F))


# ---------------------------------------------------------------------------------------------------------------- on the GPU


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
def test_pyr_dev_equals_cv2(ctx, channels):
    import torch
    from dim_b200 import _native
    for H, W in ((533, 800), (301, 457), (64, 64), (33, 47), (7, 9), (1, 17), (3, 1)):
        shape = (H, W) if channels == 1 else (H, W, 3)
        imgs = np.stack(_images(shape, H + W) + [_images(shape, H + W + 1)[1]])
        src = torch.from_numpy(imgs).cuda()
        for level in (-1, 0, 1, 2, 3):
            h2, w2 = _native.pyr_size(H, W, level)
            ref = np.stack([_cv2_pyr(im, level) for im in imgs])
            out = torch.full(ref.shape, -1.0, device="cuda")
            ctx.pyr_dev(src.data_ptr(), 3, H, W, channels, level, out.data_ptr(), 0)
            got = out.cpu().numpy()
            assert ref.shape[1:3] == (h2, w2) and _bits_equal(got, ref), (H, W, channels, level)
            one = torch.full(ref.shape[1:], -1.0, device="cuda")  # one image per call gives the same bits
            ctx.pyr_dev(src[2].data_ptr(), 1, H, W, channels, level, one.data_ptr(), 0)
            assert _bits_equal(one.cpu().numpy(), got[2])


@pytest.mark.gpu
def test_pyr_dev_is_asynchronous(ctx):
    """Queued behind a ~0.5 s device spin (after a first call has grown the scratch), the entry returns while the stream is busy."""
    import torch
    img = torch.from_numpy(_images((1536, 2048), 1)[1]).cuda()
    low = torch.zeros(192, 256, device="cuda")
    ctx.pyr_dev(img.data_ptr(), 1, 1536, 2048, 1, 3, low.data_ptr(), 0)
    torch.cuda.synchronize()
    ref = low.clone()
    low.fill_(-1)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.pyr_dev(img.data_ptr(), 1, 1536, 2048, 1, 3, low.data_ptr(), s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy and torch.equal(ref, low)


@pytest.mark.gpu
def test_fstore_rescale_scales_keypoints_and_sets_the_size(ctx):
    """Stored keypoints * 2^level equal float16(float32 keypoints * 2^level); [H, W] becomes the given size; empty slots stay empty."""
    import torch
    from dim_b200 import _native
    from dim_b200.io_h5 import as_half_roundtrip
    rng = np.random.default_rng(0)
    store = _native.FeatureStoreDev(ctx, 4, 64, 8)
    feats = []
    for s in range(3):
        n = 40 + s
        f = {"keypoints": rng.uniform(0, 500, (n, 2)).astype(F), "descriptors": rng.normal(size=(8, n)).astype(F),
             "scores": rng.uniform(0, 1, n).astype(F), "image_size": np.array([250, 300])}
        f["keypoints"][0] = (0.0, 0.0)
        f["keypoints"][1] = (499.75, 0.5)
        store.put(s, f)
        feats.append(f)
    for level in (-1, 1, 3):
        for s, f in enumerate(feats):
            store.put(s, f)
        store.rescale_dev([0, 2, 3], level, 2001, 2999, torch.cuda.current_stream().cuda_stream)
        for s, f in enumerate(feats):
            got = store.get(s)
            scaled = {**f, "keypoints": f["keypoints"] * F(2.0 ** level), "image_size": np.array([2001, 2999])}
            exp = as_half_roundtrip(scaled if s != 1 else f)
            for k in ("keypoints", "descriptors", "scores", "image_size"):
                assert np.array_equal(got[k], exp[k]), (level, s, k)
        assert store.count(3)[0] == -1


SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 1024}


def _gray_set(n, H, W, seed=40):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(seed, max(H, W))[:H, :W]
    imgs = [a] + [synthetic.warp_pair(a, seed + k, jitter=0.03 * max(H, W)) for k in range(1, n)]
    return np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in imgs]).astype(F)


def _host_features(ext, img, quality, tiled=False):
    """The reference's flow: _resize_image, _extract (or _extract_by_tile), _resize_features, original image_size, float16 cast."""
    from dim_b200.io_h5 import as_half_roundtrip
    small = ext._resize_image(quality, img)
    f = ext._extract_by_tile(small) if tiled else ext._extract(small)
    f = ext._resize_features(quality, f)
    return as_half_roundtrip({**f, "image_size": np.array(img.shape[:2])})


def _same_features(got, ref, keys=("keypoints", "descriptors", "scores", "image_size")):
    for k in keys:
        assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), k


@pytest.fixture(scope="module")
def sp_set(ctx, sp_weights):
    import torch
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.matchers.lightglue import LightGlueMatcher
    imgs = _gray_set(3, 768, 1024)
    w = weights.lightglue_seeded(seed=0)
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={"max_keypoints": SP_CONF["max_keypoints"]}))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    return {"imgs": imgs, "d": torch.from_numpy(imgs).cuda(), "w": w, "ext": ext, "plugin": plugin, "pairs": [(0, 1), (0, 2), (1, 2)]}


def _engine(ctx, sp_weights, s, **kw):
    from dim_b200.sharded import ImageSetMatcher
    n, H, W = s["imgs"].shape
    return ImageSetMatcher(ctx, sp_weights, s["w"], n, H, W, SP_CONF, {}, batch_images=2, batch_pairs=2, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("quality", ["highest", "medium", "low", "lowest"])
def test_image_set_matcher_quality_equals_host_flow(ctx, sp_weights, sp_set, quality):
    """Every slot equals the host flow bitwise (batch_images=2: the extraction crosses a batch boundary), and the match tables equal
    the LightGlue plugin's _match_pairs on the host features."""
    s = sp_set
    eng = _engine(ctx, sp_weights, s, quality=quality)
    tables = eng.run(s["d"], [0, 1, 2], s["pairs"])
    feats = [_host_features(s["ext"], img, quality) for img in s["imgs"]]
    for i in range(3):
        _same_features(eng.store.get(i), feats[i])
    assert sum(len(f["keypoints"]) for f in feats) > 0  # "lowest" extracts from 96 x 128 images
    for (i, j), t in zip(s["pairs"], tables):
        assert np.array_equal(t, s["plugin"]._match_pairs(feats[i], feats[j])), (quality, i, j)
    assert quality not in ("highest", "medium") or sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_image_set_matcher_medium_run_verified_equals_host_features(ctx, sp_weights, sp_set):
    """run_verified at "medium": the raw tables equal the plugin's, and raw, verified, F and counts equal the verification of the
    same host features put into a full-resolution matcher's store."""
    s = sp_set
    gv = {"seed": 5, "min_inliers_per_pair": 8}
    eng = _engine(ctx, sp_weights, s, quality="medium", verification=gv)
    res = eng.run_verified(s["d"], [0, 1, 2], s["pairs"])
    feats = [_host_features(s["ext"], img, "medium") for img in s["imgs"]]
    ref = _engine(ctx, sp_weights, s, verification=gv)
    for i, f in enumerate(feats):
        ref.store.put(ref.slots[i], f)
    exp = ref.match_verified(s["pairs"], list(range(len(s["pairs"]))))
    for k, ((i, j), (raw, ver, F_, n)) in enumerate(zip(s["pairs"], res)):
        assert np.array_equal(raw, s["plugin"]._match_pairs(feats[i], feats[j]))
        r2, v2, F2, n2 = exp[k]
        assert np.array_equal(raw, r2) and np.array_equal(ver, v2) and n == n2
        assert (F_ is None and F2 is None) or np.array_equal(F_, F2)
    assert sum(len(r[1]) for r in res) > 0


@pytest.mark.gpu
def test_image_set_matcher_quality_high_is_unchanged(ctx, sp_weights, sp_set):
    """quality="high" gives the slots, tables and launch count of a matcher built without the argument."""
    s = sp_set
    out = []
    for kw in ({}, {"quality": "high"}, {"quality": "HIGH"}):
        eng = _engine(ctx, sp_weights, s, **kw)
        eng.run(s["d"], [0, 1, 2], s["pairs"])  # warm: scratch grown
        n0 = ctx.launches
        tables = eng.run(s["d"], [0, 1, 2], s["pairs"])
        out.append((ctx.launches - n0, tables, [eng.store.get(i) for i in range(3)]))
    for launches, tables, slots in out[1:]:
        assert launches == out[0][0]
        assert all(np.array_equal(a, b) for a, b in zip(tables, out[0][1]))
        for a, b in zip(slots, out[0][2]):
            _same_features(a, b, ("keypoints", "descriptors", "scores", "tile_idx", "image_size"))


@pytest.mark.gpu
def test_image_set_matcher_aliked_medium_equals_host_flow(ctx, al_weights):
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(301, 1024)[:768]
    imgs = np.stack([a] + [synthetic.warp_pair(a, 60 + k, jitter=24.0) for k in (1, 2)]).astype(F)
    al_conf = {"max_num_keypoints": 1024, "detection_threshold": 0.2, "nms_radius": 3}
    w_lg = weights.lightglue_seeded(input_dim=128, seed=0)
    pairs = [(0, 1), (0, 2), (1, 2)]
    eng = ImageSetMatcher(ctx, al_weights, w_lg, 3, 768, 1024, al_conf, {}, batch_images=2, batch_pairs=2, extractor="aliked",
                          quality="medium")
    assert (eng.h2, eng.w2) == (384, 512)
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    ext = AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", **al_conf, "weights_dict": al_weights}))
    feats = [_host_features(ext, img, "medium") for img in imgs]
    for i in range(3):
        _same_features(eng.store.get(i), feats[i])
    plugin = LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w_lg}), local_features="aliked")
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
    assert min(len(f["keypoints"]) for f in feats) > 100 and sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_image_set_matcher_tiled_medium_equals_extract_by_tile(ctx, sp_weights):
    """Grid tiling at "medium": 1536 x 2048 images resized to 768 x 1024 and cut into 4 tiles of 512 (overlap 64); every merged slot
    equals _extract_by_tile on the cv2-resized image with the keypoints scaled back, and the tables equal _match_by_tile."""
    import torch
    from dim_b200 import weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.sharded import ImageSetMatcher
    imgs = _gray_set(3, 1536, 2048)
    w = weights.lightglue_seeded(seed=0)
    sp = {**SP_CONF, "fix_sampling": True}
    tiling = {"tile_size": 512, "tile_overlap": 64, "tile_selection": "grid"}
    pairs = [(0, 1), (0, 2), (1, 2)]
    eng = ImageSetMatcher(ctx, sp_weights, w, 3, 1536, 2048, sp, {}, batch_images=8, batch_pairs=8, tiling=tiling, quality="medium")
    assert eng.T == 4 and eng.G == 2
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    ext = SuperPointExtractor(Config(general={"tile_size": 512, "tile_overlap": 64}, extractor={**sp, "weights_dict": sp_weights}))
    feats = [_host_features(ext, img, "medium", tiled=True) for img in imgs]
    for i in range(3):
        _same_features(eng.store.get(i), feats[i], ("keypoints", "descriptors", "scores", "tile_idx", "image_size"))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_by_tile(feats[i], feats[j], [(k, k) for k in range(4)])), (i, j)
    assert sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_run_lowres_medium_keeps_the_pairs_of_high(ctx, sp_weights):
    """Pair generation reads the original images: the counts and kept pairs do not depend on quality."""
    import torch
    from dim_b200 import weights
    from dim_b200.sharded import ImageSetMatcher
    imgs = np.concatenate([_gray_set(3, 768, 1024, 40), _gray_set(2, 768, 1024, 90)])
    d = torch.from_numpy(imgs).cuda()
    w = weights.lightglue_seeded(seed=0)
    pg = {"strategy": "matching_lowres", "resize_max": 512, "min_matches": 0}
    out = {}
    for q in ("high", "medium"):
        eng = ImageSetMatcher(ctx, sp_weights, w, 5, 768, 1024, SP_CONF, {}, batch_images=4, batch_pairs=4, pair_generation=pg, quality=q)
        out[q] = eng.run_lowres(d, list(range(5)))
    assert out["medium"][:2] == out["high"][:2] and len(out["high"][0]) > 0
    assert len(out["medium"][2]) == len(out["high"][0])
