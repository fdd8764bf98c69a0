"""upright for image sets: the host statement (upright.py: schedule, back-rotation of keypoints and F), dimb_rot90_dev /
dimb_fstore_unrotate_dev, and ImageSetMatcher(upright=...) against the host flow.  Every comparison is exact."""
import ctypes as C
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 512}
UP = {"resize_max": 320, "max_keypoints": 512}


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


def test_schedule_bruteforce_is_one_wave_rooted_at_image_0():
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.upright import upright_schedule
    assert upright_schedule(pairs_from_bruteforce(range(5)), 5) == [[(1, 0), (2, 0), (3, 0), (4, 0)]]


def test_schedule_sequential_is_a_chain():
    from dim_b200.pairs_generator import pairs_from_sequential
    from dim_b200.upright import upright_schedule
    assert upright_schedule(pairs_from_sequential(list(range(5)), 1), 5) == [[(1, 0)], [(2, 1)], [(3, 2)], [(4, 3)]]
    # overlap 2: (0,1) (0,2) (1,2 skipped) (1,3) (2,3 skipped) (2,4) ...
    assert upright_schedule(pairs_from_sequential(list(range(5)), 2), 5) == [[(1, 0), (2, 0)], [(3, 1), (4, 2)]]


def test_schedule_components_isolated_images_and_order():
    from dim_b200.upright import upright_schedule
    # two components (roots 0 and 3), image 6 in no pair, (1, 2) listed after both ends are decided
    pairs = [(0, 1), (3, 4), (0, 2), (1, 2), (4, 5), (5, 3)]
    assert upright_schedule(pairs, 7) == [[(1, 0), (4, 3), (2, 0)], [(5, 4)]]
    # reversed order: the first pair's first image is the root, and one decided end makes the other the target
    assert upright_schedule(pairs[::-1], 7) == [[(3, 5), (4, 5), (2, 1)], [(0, 2)]]
    assert upright_schedule([], 3) == []
    assert upright_schedule([(2, 1), (0, 1)], 3) == [[(1, 2)], [(0, 1)]]


@pytest.mark.parametrize("H, W", [(7, 10), (8, 8), (9, 6), (1, 13), (13, 1), (1, 1), (6, 9)])
def test_rotate_back_keypoints_inverts_cv2_rotate_on_every_pixel(H, W):
    from dim_b200.upright import ROTATIONS, rotate_back_keypoints, rotate_image
    rng = np.random.default_rng(H * 31 + W)
    img = rng.permutation(H * W).astype(F).reshape(H, W)  # each value names its pixel
    for r in ROTATIONS:
        rot = rotate_image(img, r)
        ys, xs = np.mgrid[:rot.shape[0], :rot.shape[1]]
        kp = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)
        back = rotate_back_keypoints(kp, r, H, W).astype(int)
        assert np.array_equal(img[back[:, 1], back[:, 0]], rot.ravel()), r


def test_rotate_back_F_maps_the_epipolar_constraint():
    from dim_b200.upright import ROTATIONS, rotate_back_F, rotate_back_keypoints
    rng = np.random.default_rng(5)
    s0, s1 = (37, 52), (41, 29)
    for r0 in ROTATIONS:
        for r1 in ROTATIONS:
            Fr = rng.normal(size=(3, 3)).astype(F)
            # correspondences in the rotated frames, and the same points in original pixels
            h0, w0 = (s0[1], s0[0]) if r0 in (90, 270) else s0
            h1, w1 = (s1[1], s1[0]) if r1 in (90, 270) else s1
            p0 = np.stack([rng.integers(0, w0, 20), rng.integers(0, h0, 20)], 1).astype(F)
            p1 = np.stack([rng.integers(0, w1, 20), rng.integers(0, h1, 20)], 1).astype(F)
            o0, o1 = rotate_back_keypoints(p0, r0, *s0), rotate_back_keypoints(p1, r1, *s1)
            Fo = rotate_back_F(Fr, r0, s0, r1, s1)
            assert Fo.dtype == F
            hom = lambda p: np.concatenate([p, np.ones((len(p), 1))], 1).astype(np.float64)  # noqa: E731
            got = np.einsum("ni,ij,nj->n", hom(o1), Fo.astype(np.float64), hom(o0))
            exp = np.einsum("ni,ij,nj->n", hom(p1), Fr.astype(np.float64), hom(p0))
            assert np.allclose(got, exp, rtol=1e-5, atol=1e-3), (r0, r1)
            if r0 == r1 == 0:
                assert np.array_equal(Fo, Fr)
    assert rotate_back_F(None, 90, s0, 0, s1) is None


def test_upright_conf():
    from dim_b200.sharded import upright_conf
    assert upright_conf(None) is None
    assert upright_conf({"resize_max": 640}) == {"resize_max": 640, "max_keypoints": 2048}
    assert upright_conf({"resize_max": 1, "max_keypoints": 7}) == {"resize_max": 1, "max_keypoints": 7}
    with pytest.raises(ValueError, match="needs resize_max"):
        upright_conf({})
    with pytest.raises(ValueError, match="unknown upright"):
        upright_conf({"resize_max": 640, "rotations": 4})
    for bad in ({"resize_max": 0}, {"resize_max": 640.0}, {"resize_max": True}, {"resize_max": 640, "max_keypoints": -1},
                {"resize_max": 640, "max_keypoints": 0}):
        with pytest.raises(ValueError, match="int >= 1"):
            upright_conf(bad)


def test_matcher_refusals_with_upright():
    from dim_b200.sharded import ImageSetMatcher
    with pytest.raises(ValueError, match="superpoint"):
        ImageSetMatcher(None, {}, {}, 2, 480, 640, {"max_num_keypoints": 512}, {}, extractor="aliked", upright=UP)
    pre = {"tile_size": 256, "tile_selection": "preselection", "tile_preselection_size": 200}
    with pytest.raises(ValueError, match="preselection"):
        ImageSetMatcher(None, {}, {}, 2, 480, 640, {**SP_CONF, "fix_sampling": True}, {}, tiling=pre, upright=UP)
    with pytest.raises(ValueError, match="to nothing"):  # 1 x 4000 at longest side 2 is 0 x 2
        ImageSetMatcher(None, {}, {}, 2, [480, 1], [640, 4000], SP_CONF, {}, upright={"resize_max": 2})
    for m in ("superglue", "kornia_matcher"):
        with pytest.raises(ValueError, match="upright_weights"):
            ImageSetMatcher(None, {}, {}, 2, 480, 640, SP_CONF, {}, matcher=m, upright=UP)
    with pytest.raises(ValueError, match="unknown upright"):
        ImageSetMatcher(None, {}, {}, 2, 480, 640, SP_CONF, {}, upright={"resize_max": 320, "size": 2})
    # the tile-count limit is checked for the turned size too: with 16 x 32 tiles (H x W) a 1162 x 889 image has 2044 tiles, but
    # the padding of 889 x 1162 gives more than 2048, so only upright refuses it (without upright the check passes and the
    # constructor goes on to read the weights)
    tiled = {"tile_size": (32, 16)}
    with pytest.raises(KeyError):
        ImageSetMatcher(None, {}, {}, 2, [480, 1162], [640, 889], {**SP_CONF, "fix_sampling": True}, {}, tiling=tiled)
    with pytest.raises(ValueError, match="2048 tiles"):
        ImageSetMatcher(None, {}, {}, 2, [480, 1162], [640, 889], {**SP_CONF, "fix_sampling": True}, {}, tiling=tiled, upright=UP)


def test_upright_entries_reject_bad_arguments_without_touching_the_gpu():
    """Argument validation comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    good = (C.c_int * 3)(0, 90, 270)

    def rot(ctx=ctx, src=dev, B=3, H=33, W=47, ch=1, r=good, dst=dev):
        return lib.dimb_rot90_dev(ctx, src, B, H, W, ch, r, dst, null)
    assert rot(ctx=null) == -3 and rot(src=null) == -3 and rot(dst=null) == -3 and rot(r=None) == -3
    assert rot(B=0) == -3 and rot(B=70000) == -3 and rot(H=0) == -3 and rot(W=0) == -3 and rot(W=(1 << 20) + 1) == -3
    assert rot(ch=2) == -3 and rot(ch=0) == -3 and rot(ch=4) == -3
    for bad in (45, -90, 360, 1):
        assert rot(r=(C.c_int * 3)(0, bad, 90)) == -3, bad
    store = C.cast(C.create_string_buffer(256), C.c_void_p)
    slots, hs, ws = (C.c_int * 2)(0, 1), (C.c_int * 2)(480, 640), (C.c_int * 2)(640, 480)

    def unrot(fs=store, B=2, s=slots, r=(C.c_int * 2)(90, 180), h=hs, w=ws):
        return lib.dimb_fstore_unrotate_dev(fs, B, s, r, h, w, null)
    assert unrot(fs=null) == -3 and unrot(s=None) == -3 and unrot(r=None) == -3 and unrot(h=None) == -3 and unrot(w=None) == -3
    assert unrot(B=0) == -3 and unrot(B=70000) == -3 and unrot(r=(C.c_int * 2)(90, 30)) == -3
    assert unrot(h=(C.c_int * 2)(480, 0)) == -3 and unrot(w=(C.c_int * 2)(-1, 480)) == -3


WORKER = r"""
import json, os, sys
sys.path.insert(0, os.environ["DIMB_ROOT"])
import torch.distributed as dist
from dim_b200.sharded import upright_waves
dist.init_process_group("gloo")
rank = dist.get_rank()
calls = []

def count(decisions, rotations):  # a stub of LightGlue: the counts depend on the pair and on the reference's rotation
    calls.extend(decisions)
    return [(t * 7 + a * 3 + rotations[a] // 90 * 5 + k * 11) % 13 for t, a in decisions for k in range(4)]

pairs = [tuple(p) for p in json.loads(os.environ["DIMB_PAIRS"])]
rot, counts = upright_waves(pairs, 9, count, dist)
with open(os.path.join(os.environ["DIMB_OUT"], f"rank{rank}.json"), "w") as f:
    json.dump({"rank": rank, "rot": rot, "counts": {f"{t},{a}": c for (t, a), c in counts.items()}, "calls": calls}, f)
dist.destroy_process_group()
"""


def test_waves_over_two_ranks_equal_one_rank_gloo(tmp_path):
    from dim_b200.pairs_generator import pairs_from_bruteforce, pairs_from_sequential
    from dim_b200.sharded import upright_waves

    def count(decisions, rotations):
        return [(t * 7 + a * 3 + rotations[a] // 90 * 5 + k * 11) % 13 for t, a in decisions for k in range(4)]
    pairs = pairs_from_sequential(list(range(9)), 2) + pairs_from_bruteforce(range(9))
    exp_rot, exp_counts = upright_waves(pairs, 9, count)
    assert len(set(exp_rot)) > 2
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = {**os.environ, "DIMB_ROOT": ROOT, "DIMB_OUT": str(tmp_path), "DIMB_PAIRS": json.dumps(pairs)}
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29598", str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    res = [json.loads((tmp_path / f"rank{k}.json").read_text()) for k in range(2)]
    for d in res:
        assert d["rot"] == exp_rot and d["counts"] == {f"{t},{a}": c for (t, a), c in exp_counts.items()}
    calls = [tuple(c) for d in res for c in d["calls"]]
    assert res[0]["calls"] and res[1]["calls"] and sorted(calls) == sorted(exp_counts)


# ---------------------------------------------------------------------------------------------------------------- on the GPU


def _images(shape, n, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0, 255, shape).astype(F) for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
def test_rot90_dev_equals_cv2_rotate(ctx, channels):
    import torch
    from dim_b200.upright import ROTATIONS, rotate_image
    for H, W in ((33, 47), (64, 64), (48, 32), (301, 457), (1, 17), (17, 1), (1, 1)):
        shape = (H, W) if channels == 1 else (H, W, 3)
        imgs = np.stack(_images(shape, 5, H * 7 + W))
        src = torch.from_numpy(imgs).cuda()
        codes = [90, 0, 270, 180, 90]
        out = torch.full((imgs.size,), -1.0, device="cuda")
        ctx.rot90_dev(src.data_ptr(), 5, H, W, channels, codes, out.data_ptr(), 0)
        got = out.cpu().numpy()
        n = imgs[0].size
        for b, r in enumerate(codes):
            ref = rotate_image(imgs[b], r)
            assert np.array_equal(got[b * n:(b + 1) * n].view(np.uint32), ref.ravel().view(np.uint32)), (H, W, channels, b, r)
        for r in ROTATIONS:  # one image per call gives the same bits
            one = torch.full((n,), -1.0, device="cuda")
            ctx.rot90_dev(src[2].data_ptr(), 1, H, W, channels, [r], one.data_ptr(), 0)
            assert np.array_equal(one.cpu().numpy(), rotate_image(imgs[2], r).ravel()), (H, W, r)


@pytest.mark.gpu
def test_rot90_dev_is_asynchronous(ctx):
    """Queued behind a ~0.5 s device spin (after a first call has grown the scratch), the entry returns while the stream is busy."""
    import torch
    img = torch.from_numpy(_images((1536, 2048), 1, 1)[0]).cuda()
    out = torch.zeros(1536 * 2048, device="cuda")
    ctx.rot90_dev(img.data_ptr(), 1, 1536, 2048, 1, [90], out.data_ptr(), 0)
    torch.cuda.synchronize()
    ref = out.clone()
    out.fill_(-1)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.rot90_dev(img.data_ptr(), 1, 1536, 2048, 1, [90], out.data_ptr(), s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy and torch.equal(ref, out)


@pytest.mark.gpu
def test_fstore_unrotate_dev_equals_numpy(ctx):
    from dim_b200 import _native
    from dim_b200.upright import rotate_back_keypoints
    rng = np.random.default_rng(3)
    store = _native.FeatureStoreDev(ctx, 6, 300, 256)
    sizes = [(480, 640), (640, 480), (333, 517), (517, 333), (1, 40)]
    rots = [90, 180, 270, 0, 90]
    feats = []
    for s, ((H, W), r) in enumerate(zip(sizes, rots)):
        h, w = (W, H) if r in (90, 270) else (H, W)
        n = 250 + s
        kp = np.stack([rng.uniform(0, w - 1, n), rng.uniform(0, h - 1, n)], 1).astype(F)
        kp[:5] = np.round(kp[:5])
        f = {"keypoints": kp, "descriptors": rng.normal(size=(256, n)).astype(F), "scores": rng.uniform(size=n).astype(F),
             "image_size": np.array([h, w])}
        store.put(s, f)
        feats.append(store.get(s))
    store.unrotate_dev(list(range(5)) + [5], rots + [90], [H for H, _ in sizes] + [100], [W for _, W in sizes] + [50])
    for s, ((H, W), r) in enumerate(zip(sizes, rots)):
        got, before = store.get(s), feats[s]
        exp = rotate_back_keypoints(before["keypoints"], r, H, W).astype(np.float16).astype(F)
        assert np.array_equal(got["keypoints"], exp), s
        assert got["image_size"].tolist() == [H, W]
        for k in ("descriptors", "scores", "tile_idx"):
            assert np.array_equal(got[k], before[k]), (s, k)
    assert store.count(5)[0] < 0  # the empty slot stays empty
    with pytest.raises(ValueError, match="one rotation"):
        store.unrotate_dev([0, 1], [90], [4, 4], [4, 4])


# the engine against the host flow: 8 images, 4 of them turned before the search, of mixed sizes
BASE = [(480, 640), (480, 640), (640, 480), (517, 701), (480, 640), (640, 480), (517, 701), (480, 640)]
TURNED = {1: 90, 3: 180, 5: 270, 6: 90}


def _set(seed=40):
    from dim_b200 import synthetic
    from dim_b200.upright import rotate_image
    scene = synthetic.blocks_image(seed, 800)
    imgs = []
    for k, (H, W) in enumerate(BASE):
        crop = np.ascontiguousarray(scene[8 * k:8 * k + H, 4 * k:4 * k + W])
        g = synthetic.to_gray_like_reference(crop if k == 0 else synthetic.warp_pair(crop, seed + k, jitter=0.02 * max(H, W))).astype(F)
        imgs.append(rotate_image(g, TURNED.get(k, 0)))
    return imgs


def _engine(ctx, sp_weights, w, imgs, conf=SP_CONF, up=UP, **kw):
    from dim_b200.sharded import ImageSetMatcher
    kw.setdefault("batch_images", 3)
    kw.setdefault("batch_pairs", 6)
    return ImageSetMatcher(ctx, sp_weights, w, len(imgs), [im.shape[0] for im in imgs], [im.shape[1] for im in imgs], conf,
                           kw.pop("lg_conf", {}), upright=up, **kw)


def _dev(imgs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x, F)).cuda() for x in imgs]


def _turned_back(f, r, H, W):
    from dim_b200.upright import rotate_back_keypoints
    return {**f, "keypoints": rotate_back_keypoints(f["keypoints"], r, H, W).astype(np.float16).astype(F),
            "image_size": np.array([H, W], np.int32)}


@pytest.fixture(scope="module")
def upset(ctx, sp_weights):
    from dim_b200 import weights
    from dim_b200.pairs_generator import pairs_from_bruteforce, pairs_from_sequential
    from dim_b200.upright import upright_rotations
    imgs = _set()
    w = weights.lightglue_seeded(seed=0)
    out = {"imgs": imgs, "d": _dev(imgs), "w": w}
    for name, pairs in (("brute", pairs_from_bruteforce(range(len(imgs)))), ("seq", pairs_from_sequential(list(range(len(imgs))), 2))):
        out[name] = (pairs, upright_rotations(imgs, pairs, UP["resize_max"], UP["max_keypoints"], False, w, sp_weights, ctx.device))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("lists", ["brute", "seq"])
def test_upright_engine_equals_host_flow(ctx, sp_weights, upset, lists):
    """Rotations, per-decision counts, stored features after rotate_back and the match tables equal the host statement."""
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.upright import rotate_image
    s = upset
    pairs, (rot, counts) = s[lists]
    eng = _engine(ctx, sp_weights, s["w"], s["imgs"])
    with pytest.raises(RuntimeError, match="upright"):
        eng.extract(s["d"], list(range(8)))
    tables = eng.run(s["d"], list(range(8)), pairs)
    assert eng.rotations == rot and eng.upright(s["d"], list(range(8)), pairs) == (rot, counts)
    assert any(rot) and len(counts) == 7
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor=SP_CONF))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": s["w"]}))
    feats = []
    for im, r in zip(s["imgs"], rot):
        turned = rotate_image(im, r)
        feats.append(as_half_roundtrip({**ext._extract(turned), "image_size": np.array(turned.shape[:2])}))
    for i, (im, r) in enumerate(zip(s["imgs"], rot)):
        got, exp = eng.store.get(i), _turned_back(feats[i], r, *im.shape)
        for k in ("keypoints", "descriptors", "scores", "image_size"):
            assert np.array_equal(got[k], exp[k]), (i, k)
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(feats[i], feats[j])), (i, j)
    assert sum(len(t) for t in tables) > 0
    with pytest.raises(RuntimeError, match="rotate_back"):
        eng.match(pairs[:1], [0])


def _twin(ctx, sp_weights, w, imgs, rot, **kw):
    """The same engine without upright, run on the images already turned by `rot` on the host."""
    from dim_b200.upright import rotate_image
    turned = [rotate_image(im, r) for im, r in zip(imgs, rot)]
    return _engine(ctx, sp_weights, w, turned, up=None, **kw), _dev(turned)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["verified", "grid", "medium", "kornia"])
def test_upright_engine_equals_the_engine_on_turned_images(ctx, sp_weights, upset, mode, tmp_path):
    """Verification (F through rotate_back_F), grid tiling, quality "medium" and kornia_matcher: the upright engine equals the engine
    without upright on the images the search turned, with its slots rotated back."""
    from dim_b200.upright import rotate_back_F, upright_rotations
    s = upset
    pairs, (rot, counts) = s["brute"]
    if mode == "grid":  # tiling makes the search sample descriptors at fixed positions (quirk A.6): the host flow does the same
        rot, counts = upright_rotations(s["imgs"], pairs, UP["resize_max"], UP["max_keypoints"], True, s["w"], sp_weights, ctx.device)
    kw = {"verified": {"verification": {"seed": 3}}, "medium": {"quality": "medium"},
          "grid": {"tiling": {"tile_size": 256, "tile_overlap": 32, "tile_selection": "grid"}, "batch_images": 12, "batch_pairs": 16},
          "kornia": {"matcher": "kornia_matcher", "lg_conf": {"match_mode": "smnn", "th": 0.9}, "upright_weights": s["w"]}}[mode]
    conf = {**SP_CONF, "fix_sampling": True} if mode == "grid" else SP_CONF
    w = None if mode == "kornia" else s["w"]
    eng = _engine(ctx, sp_weights, w, s["imgs"], conf, **dict(kw))
    kw.pop("upright_weights", None)
    twin, d_turned = _twin(ctx, sp_weights, w, s["imgs"], rot, conf=conf, **kw)
    run = "run_verified" if mode == "verified" else "run"
    got = getattr(eng, run)(s["d"], list(range(8)), pairs)
    exp = getattr(twin, run)(d_turned, list(range(8)), pairs)
    assert eng.rotations == rot
    if mode in ("grid", "kornia"):  # the per-decision counts of the search (fixed sampling; the search's own weights)
        assert eng.upright(s["d"], list(range(8)), pairs) == (rot, counts)
        eng.extract(s["d"], list(range(8)))
        eng.exchange()
        eng.rotate_back()
    keys = ("keypoints", "descriptors", "scores", "tile_idx", "image_size")
    for i, (im, r) in enumerate(zip(s["imgs"], rot)):
        a, b = eng.store.get(i), _turned_back(twin.store.get(i), r, *im.shape)
        for k in keys:
            assert np.array_equal(a[k], b[k]), (mode, i, k)
    for (i, j), g, e in zip(pairs, got, exp):
        if mode != "verified":
            assert np.array_equal(g, e), (mode, i, j)
            continue
        assert np.array_equal(g[0], e[0]) and np.array_equal(g[1], e[1]) and g[3] == e[3], (i, j)
        Fe = rotate_back_F(e[2], rot[i], s["imgs"][i].shape, rot[j], s["imgs"][j].shape)
        assert (g[2] is None) == (Fe is None) and (Fe is None or np.array_equal(g[2], Fe)), (i, j)
    assert sum(len(g if mode != "verified" else g[0]) for g in got) > 0
    if mode == "verified":
        import sqlite3
        eng.export_colmap(pairs, got, tmp_path / "up.db")
        con = sqlite3.connect(str(tmp_path / "up.db"))
        cams = {r[0]: (r[1], r[2]) for r in con.execute("SELECT camera_id, width, height FROM cameras")}
        img_cam = {r[0]: r[1] for r in con.execute("SELECT name, camera_id FROM images")}
        con.close()
        for i, im in enumerate(s["imgs"]):  # the original camera sizes
            assert cams[img_cam[f"image_{i}"]] == (im.shape[1], im.shape[0]), i


@pytest.mark.gpu
def test_upright_run_lowres_searches_the_kept_pairs(ctx, sp_weights, upset):
    from dim_b200.upright import upright_rotations
    s = upset
    pg = {"strategy": "matching_lowres", "resize_max": 400, "min_matches": 20}
    eng = _engine(ctx, sp_weights, s["w"], s["imgs"], {**SP_CONF, "fix_sampling": True}, pair_generation=pg)
    plain = _engine(ctx, sp_weights, s["w"], s["imgs"], {**SP_CONF, "fix_sampling": True}, up=None, pair_generation=pg)
    plain.extract(s["d"], list(range(8)))
    plain.exchange()
    exp_pairs, exp_counts = plain.lowres_pairs()
    pairs, counts, tables = eng.run_lowres(s["d"], list(range(8)))
    assert (pairs, counts) == (exp_pairs, exp_counts) and len(pairs) > 0
    rot, up_counts = upright_rotations(s["imgs"], pairs, UP["resize_max"], UP["max_keypoints"], True, s["w"], sp_weights, ctx.device)
    assert eng.rotations == rot and eng.upright(s["d"], list(range(8)), pairs) == (rot, up_counts)
    twin, d_turned = _twin(ctx, sp_weights, s["w"], s["imgs"], rot, conf={**SP_CONF, "fix_sampling": True})
    exp = twin.run(d_turned, list(range(8)), pairs)
    assert all(np.array_equal(g, e) for g, e in zip(tables, exp))
