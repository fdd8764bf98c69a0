"""The low-resolution passes of ALIKED image sets: the gray rule (pairs_generator.gray_from_rgb), the fused RGB-to-gray INTER_AREA
resize (dimb_resize_area_rgb_dev), and ImageSetMatcher(extractor="aliked") with pair generation, tile preselection and upright
checked against the host flows fed with gray_from_rgb images.  Every comparison is exact."""
import ctypes as C

import cv2
import numpy as np
import pytest

F = np.float32
AL_CONF = {"max_num_keypoints": 1024, "detection_threshold": 0.2, "nms_radius": 3}
UP = {"resize_max": 320, "max_keypoints": 512}


def _gray_rule(rgb):
    """The integer statement of the gray rule."""
    u = np.clip(np.rint(np.asarray(rgb, F)), 0, 255).astype(np.int64)
    return ((9798 * u[..., 0] + 19235 * u[..., 1] + 3735 * u[..., 2] + 16384) >> 15).astype(F)


def _rgb(shape, seed):
    """Non-integral RGB values, some beyond 0..255, some exactly half-way between integers (rounded to even)."""
    rng = np.random.default_rng(seed)
    img = rng.uniform(-20, 280, shape + (3,)).astype(F)
    half = rng.random(img.shape) < 0.1
    img[half] = np.floor(img[half]) + F(0.5)
    return img


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


def test_gray_from_rgb_is_the_integer_rule():
    from dim_b200.pairs_generator import gray_from_rgb
    from dim_b200.synthetic import to_gray_like_reference
    img = _rgb((257, 311), 1)
    assert np.array_equal(gray_from_rgb(img), _gray_rule(img)) and gray_from_rgb(img).dtype == F
    for v in (-0.5, 0.5, 1.5, 2.5, 127.5, 254.5, 255.5, 300.0, -1e9, 1e9):  # half-way values go to the even neighbour; clamped ends
        px = np.full((1, 1, 3), v, F)
        assert gray_from_rgb(px)[0, 0] == _gray_rule(px)[0, 0] == min(max(np.rint(v), 0), 255), v
    # every uint8 value of each channel against the others' extremes
    ramp = np.arange(256, dtype=F)
    for c in range(3):
        for other in (0.0, 255.0):
            px = np.full((1, 256, 3), other, F)
            px[0, :, c] = ramp
            assert np.array_equal(gray_from_rgb(px), _gray_rule(px)), (c, other)
    # R first: not the BGR2GRAY order SuperPoint sets carry
    u8 = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    assert not np.array_equal(gray_from_rgb(img), to_gray_like_reference(u8))


def test_resize_area_rgb_dev_rejects_bad_arguments_without_touching_the_gpu():
    """Argument validation comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)

    def rgb(ctx=ctx, src=dev, B=2, H=300, W=400, dst=dev, H2=150, W2=200):
        return lib.dimb_resize_area_rgb_dev(ctx, src, B, H, W, dst, H2, W2, null)
    assert rgb(ctx=null) == -3 and rgb(src=null) == -3 and rgb(dst=null) == -3
    assert rgb(B=0) == -3 and rgb(B=65536) == -3 and rgb(H=0) == -3 and rgb(W=0) == -3
    assert rgb(H=(1 << 20) + 1) == -3 and rgb(W=(1 << 20) + 1) == -3
    assert rgb(H2=0) == -3 and rgb(W2=0) == -3 and rgb(H2=65536) == -3 and rgb(W2=(1 << 20) + 1) == -3


def test_aliked_low_resolution_passes_need_their_superpoint_weights():
    """The constructor rules of ALIKED sets, all checked before any GPU use (ctx None)."""
    from dim_b200.sharded import ImageSetMatcher
    pg = {"strategy": "matching_lowres"}
    pre = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}
    with pytest.raises(ValueError, match="superpoint_weights"):  # SuperPoint sets: sp_weights is the low-resolution SuperPoint
        ImageSetMatcher(None, {}, {}, 2, 533, 800, {"max_keypoints": 512}, {}, pair_generation=pg, superpoint_weights={})
    for matcher in ("lightglue", "kornia_matcher"):  # lg_weights is an input_dim-128 LightGlue: each pass needs its own weights
        with pytest.raises(ValueError, match="lowres_weights, the superpoint_lightglue"):
            ImageSetMatcher(None, {}, {}, 2, 533, 800, AL_CONF, {}, matcher=matcher, extractor="aliked", pair_generation=pg)
        with pytest.raises(ValueError, match="preselection_weights, the superpoint_lightglue"):
            ImageSetMatcher(None, {}, {}, 2, 768, 1024, AL_CONF, {}, matcher=matcher, extractor="aliked", tiling=pre)
        with pytest.raises(ValueError, match="upright_weights, the superpoint_lightglue"):
            ImageSetMatcher(None, {}, {}, 2, 480, 640, AL_CONF, {}, matcher=matcher, extractor="aliked", upright=UP)
    # the rules that do not depend on the extractor still hold with the weights given
    with pytest.raises(ValueError, match="SuperGlue"):
        ImageSetMatcher(None, {}, {}, 2, 533, 800, AL_CONF, {}, matcher="superglue", extractor="aliked", pair_generation=pg,
                        lowres_weights={})
    with pytest.raises(ValueError, match="quality"):
        ImageSetMatcher(None, {}, {}, 2, 768, 1024, AL_CONF, {}, extractor="aliked", tiling=pre, preselection_weights={}, quality="medium")
    with pytest.raises(ValueError, match="preselection"):
        ImageSetMatcher(None, {}, {}, 2, 768, 1024, AL_CONF, {}, extractor="aliked", tiling=pre, preselection_weights={}, upright=UP,
                        upright_weights={})
    with pytest.raises(ValueError, match="resize_max"):
        ImageSetMatcher(None, {}, {}, 2, [768, 1], [1024, 4000], AL_CONF, {}, extractor="aliked", pair_generation={**pg, "resize_max": 2},
                        lowres_weights={})


# ---------------------------------------------------------------------------------------------------------------- on the GPU

RGB_CASES = [
    ((37, 53), (37, 53)),     # equal size: the gray image itself
    ((64, 88), (32, 44)),     # 2 x 2, output width not a multiple of 4 (OpenCV's vector loop covers 40 columns)
    ((64, 96), (32, 48)),     # 2 x 2, every column in the vector loop
    ((30, 14), (15, 7)),      # 2 x 2, narrower than one vector step past the first
    ((99, 66), (33, 22)),     # 3 x 3
    ((64, 99), (32, 33)),     # 2 x 3
    ((300, 400), (187, 250)),  # non-integer factors
    ((97, 131), (40, 57)),    # non-integer factors, odd sizes
    ((60, 80), (90, 40)),     # one axis enlarged (the bilinear emulation on both axes)
    ((53, 80), (100, 151)),   # both axes enlarged
    ((240, 320), (300, 400)),  # both enlarged by 1.25
]


@pytest.mark.gpu
def test_resize_area_rgb_dev_equals_cv2(ctx):
    import torch
    from dim_b200.pairs_generator import gray_from_rgb
    for (H, W), (H2, W2) in RGB_CASES:
        imgs = np.stack([_rgb((H, W), H * 1000 + W + b) for b in range(3)])
        ref = np.stack([cv2.resize(gray_from_rgb(im), (W2, H2), interpolation=cv2.INTER_AREA) for im in imgs])
        src = torch.from_numpy(imgs).cuda()
        out = torch.full((3, H2, W2), -1.0, device="cuda")
        ctx.resize_area_rgb_dev(src.data_ptr(), 3, H, W, out.data_ptr(), H2, W2, 0)
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (H, W, H2, W2)
        for b in range(3):  # one image per call gives the same bits
            one = torch.full((1, H2, W2), -1.0, device="cuda")
            ctx.resize_area_rgb_dev(src[b].data_ptr(), 1, H, W, one.data_ptr(), H2, W2, 0)
            assert np.array_equal(one.cpu().numpy()[0].view(np.uint32), got[b].view(np.uint32)), (H, W, H2, W2, b)


@pytest.mark.gpu
def test_resize_area_rgb_dev_is_asynchronous(ctx):
    """Queued behind a ~0.5 s device spin (after a first call has grown the scratch), the entry returns while the stream is busy."""
    import torch
    H, W, H2, W2 = 1536, 2048, 750, 1000
    img = torch.from_numpy(_rgb((H, W), 7)).cuda()
    low = torch.zeros(H2, W2, device="cuda")
    ctx.resize_area_rgb_dev(img.data_ptr(), 1, H, W, low.data_ptr(), H2, W2, 0)
    torch.cuda.synchronize()
    ref = low.clone()
    low.fill_(-1)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.resize_area_rgb_dev(img.data_ptr(), 1, H, W, low.data_ptr(), H2, W2, s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy and torch.equal(ref, low)


def _dev(imgs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x, F)).cuda() for x in imgs]


def _aliked(al_weights, tile=None, overlap=0):
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    general = {} if tile is None else {"tile_size": tile, "tile_overlap": overlap}
    return AlikedExtractor(Config(pipeline="aliked+lightglue", general=general,
                                  extractor={"model_name": "aliked-n16rot", **AL_CONF, "weights_dict": al_weights}))


def _plugin(w128):
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
    return LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w128}), local_features="aliked")


def _features(ext, img, tiled=False):
    """as_half_roundtrip of the plugin's features with image_size, as the h5 writer leaves them."""
    from dim_b200.io_h5 import as_half_roundtrip
    f = ext._extract_by_tile(img) if tiled else ext._extract(img)
    return as_half_roundtrip({**f, "image_size": np.array(img.shape[:2])})


# pair generation: five RGB images of two sizes, one scene and an unrelated one; at resize_max 400 the 384 x 512 images are
# down-sampled by 1.28 and the 240 x 320 ones enlarged by 1.25
def _pairgen_set():
    from dim_b200 import synthetic
    a, b = synthetic.blocks_image(50, 512), synthetic.blocks_image(150, 512)
    imgs = [a[:384], synthetic.warp_pair(a[:384], 51, jitter=16.0), a[:240, :320], b[:384], synthetic.warp_pair(b, 52, jitter=16.0)[:240, :320]]
    return [np.ascontiguousarray(x).astype(F) for x in imgs]


@pytest.mark.gpu
def test_aliked_pair_generation_equals_host_flow(ctx, sp_weights, al_weights):
    from pathlib import Path

    from dim_b200 import weights
    from dim_b200.pairs_generator import gray_from_rgb, pairs_from_lowres
    from dim_b200.sharded import ImageSetMatcher, _lowres_size
    imgs, resize_max = _pairgen_set(), 400
    w128, w256 = weights.lightglue_seeded(input_dim=128, seed=0), weights.lightglue_seeded(seed=0)
    names = [Path(f"{k}.png") for k in range(len(imgs))]
    low = {}
    for p, im in zip(names, imgs):
        _, h, w = _lowres_size(*im.shape[:2], resize_max)
        low[p.name] = cv2.resize(gray_from_rgb(im), (w, h), interpolation=cv2.INTER_AREA)
    _, counts = pairs_from_lowres(names, resize_max, 0, lightglue_weights=w256, superpoint_weights=sp_weights, images=low,
                                  return_counts=True, device=ctx.device)
    assert min(counts) < max(counts), counts
    mm = (min(counts) + max(counts)) // 2  # at least one pair kept and one dropped
    pairs = [(i, j) for k, (i, j) in enumerate((i, j) for i in range(5) for j in range(i + 1, 5)) if counts[k] > mm]
    eng = ImageSetMatcher(ctx, al_weights, w128, 5, [im.shape[0] for im in imgs], [im.shape[1] for im in imgs], AL_CONF, {},
                          batch_images=2, batch_pairs=4, extractor="aliked", lowres_weights=w256,
                          pair_generation={"strategy": "matching_lowres", "resize_max": resize_max, "min_matches": mm})
    assert eng.lowres.low_sizes == [(300, 400)] * 5
    got_pairs, got_counts, tables = eng.run_lowres(_dev(imgs), list(range(5)))
    assert (got_pairs, got_counts) == (pairs, counts) and 0 < len(pairs) < 10
    ext, plugin = _aliked(al_weights), _plugin(w128)
    feats = [_features(ext, im) for im in imgs]
    for i in range(5):
        got = eng.store.get(i)
        for k in ("keypoints", "descriptors", "scores", "image_size"):
            assert np.array_equal(got[k], feats[i][k]), (i, k)
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
    assert sum(len(t) for t in tables) > 0


@pytest.mark.gpu
def test_aliked_tiled_preselection_equals_host_flow(ctx, sp_weights, al_weights):
    import torch
    from dim_b200 import _native, synthetic, tiling, weights
    from dim_b200.pairs_generator import gray_from_rgb, pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(40, 1024)[:768]
    imgs = np.stack([a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in (1, 2)]).astype(F)
    grays = [gray_from_rgb(im) for im in imgs]
    w128, w256 = weights.lightglue_seeded(input_dim=128, seed=0), weights.lightglue_seeded(seed=0)
    pairs = pairs_from_bruteforce([0, 1, 2])
    pre = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "preselection", "tile_preselection_size": 512}
    sp_pre = lambda H, W: _native.SuperPointNet(ctx, sp_weights, max_height=H, max_width=W, **tiling.SP_PRESELECTION_CONF)  # noqa: E731
    lg_pre = _native.LightGlueNet(ctx, w256, max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    lists = []
    for i, j in pairs:
        kp0, kp1 = tiling.preselection_matches(grays[i], grays[j], 512, sp_pre, lg_pre)
        lists.append(tiling.tile_selection(grays[i], grays[j], "preselection", (512, 512), 64, kp0=kp0, kp1=kp1))
    assert any(0 < len(lst) < 16 for lst in lists), lists  # preselection actually selects
    eng = ImageSetMatcher(ctx, al_weights, w128, 3, 768, 1024, AL_CONF, {}, batch_images=6, batch_pairs=16, tiling=pre,
                          extractor="aliked", preselection_weights=w256)
    assert eng.T == 4 and (eng.pre_h, eng.pre_w) == (384, 512)
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    assert eng._preselect(pairs) == lists
    ext, plugin = _aliked(al_weights, 512, 64), _plugin(w128)
    feats = [_features(ext, im, tiled=True) for im in imgs]
    for i in range(3):
        got = eng.store.get(i)
        for k in ("keypoints", "descriptors", "scores", "tile_idx", "image_size"):
            assert got[k].shape == feats[i][k].shape and np.array_equal(got[k], feats[i][k]), (i, k)
    for (i, j), lst, t in zip(pairs, lists, tables):
        assert np.array_equal(t, plugin._match_by_tile(feats[i], feats[j], lst)), (i, j)
    assert max(len(t) for t in tables) > 0


# upright: six RGB images of mixed sizes, three of them turned before the search
BASE = [(384, 512), (384, 512), (512, 384), (413, 561), (384, 512), (512, 384)]
TURNED = {1: 90, 3: 180, 5: 270}


def _upright_set(seed=40):
    from dim_b200 import synthetic
    from dim_b200.upright import rotate_image
    scene = synthetic.blocks_image(seed, 700)
    imgs = []
    for k, (H, W) in enumerate(BASE):
        crop = np.ascontiguousarray(scene[8 * k:8 * k + H, 4 * k:4 * k + W])
        rgb = crop if k == 0 else synthetic.warp_pair(crop, seed + k, jitter=0.02 * max(H, W))
        imgs.append(rotate_image(rgb.astype(F), TURNED.get(k, 0)))
    return imgs


@pytest.fixture(scope="module")
def up_set():
    from dim_b200 import weights
    return {"imgs": _upright_set(), "w128": weights.lightglue_seeded(input_dim=128, seed=0), "w256": weights.lightglue_seeded(seed=0)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["untiled", "grid"])
def test_aliked_upright_equals_host_flow(ctx, sp_weights, al_weights, up_set, mode):
    """Rotations and counts equal upright_rotations on the gray images; the stored features equal the plugin on the turned RGB images,
    float16, turned back, float16; the tables equal the engine without upright on the images turned on the host."""
    from dim_b200.pairs_generator import gray_from_rgb, pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    from dim_b200.upright import rotate_back_keypoints, rotate_image, upright_rotations
    imgs, w128, w256 = up_set["imgs"], up_set["w128"], up_set["w256"]
    n = len(imgs)
    pairs = pairs_from_bruteforce(range(n))
    tiled = mode == "grid"
    grid = {"tile_size": 256, "tile_overlap": 32, "tile_selection": "grid"}
    kw = {"tiling": grid, "batch_images": 12, "batch_pairs": 16} if tiled else {"batch_images": 3, "batch_pairs": 6}
    hs, ws = [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]
    # tiling makes the search sample descriptors at fixed positions (quirk A.6): the host flow does the same
    rot, counts = upright_rotations([gray_from_rgb(im) for im in imgs], pairs, UP["resize_max"], UP["max_keypoints"], tiled, w256,
                                    sp_weights, ctx.device)
    eng = ImageSetMatcher(ctx, al_weights, w128, n, hs, ws, AL_CONF, {}, extractor="aliked", upright=UP, upright_weights=w256, **kw)
    tables = eng.run(_dev(imgs), list(range(n)), pairs)
    assert eng.rotations == rot and any(rot)
    assert eng.upright(_dev(imgs), list(range(n)), pairs) == (rot, counts)  # the search alone leaves the store as run left it
    ext =_aliked(al_weights, 256, 32) if tiled else _aliked(al_weights)
    turned = [rotate_image(im, r) for im, r in zip(imgs, rot)]
    keys = ("keypoints", "descriptors", "scores", "image_size") + (("tile_idx",) if tiled else ())
    for i, (im, r) in enumerate(zip(imgs, rot)):
        f = _features(ext, turned[i], tiled)
        exp = {**f, "keypoints": rotate_back_keypoints(f["keypoints"], r, *im.shape[:2]).astype(np.float16).astype(F),
               "image_size": np.array(im.shape[:2], np.int32)}
        got = eng.store.get(i)
        for k in keys:
            assert got[k].shape == exp[k].shape and np.array_equal(got[k], exp[k]), (mode, i, k)
    twin = ImageSetMatcher(ctx, al_weights, w128, n, [t.shape[0] for t in turned], [t.shape[1] for t in turned], AL_CONF, {},
                           extractor="aliked", **kw)
    exp_tables = twin.run(_dev(turned), list(range(n)), pairs)
    for (i, j), g, e in zip(pairs, tables, exp_tables):
        assert np.array_equal(g, e), (mode, i, j)
    assert sum(len(t) for t in tables) > 0
