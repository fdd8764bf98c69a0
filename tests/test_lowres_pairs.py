"""Low-resolution pair generation on the device: INTER_AREA when an axis is enlarged (dimb_resize_area_linear_tab /
dimb_resize_area_linear_dev) and ImageSetMatcher(pair_generation={"strategy": "matching_lowres", ...}) checked against the host
pairs_generator.pairs_from_lowres on the same native networks and cv2-resized images.  Every comparison is exact."""
import ctypes as C
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest

from conftest import ROOT

# (H, W) -> (H2, W2) with at least one axis enlarged: the reference's own photos (800 x 533 to resize_max 1000), 2x, 1.5x, tiny to
# large, 1-pixel axes, and one axis enlarged with the other reduced (OpenCV then emulates bilinearly on both axes)
LINEAR_CASES = [((533, 800), (666, 1000)), ((100, 100), (200, 200)), ((64, 96), (96, 144)), ((5, 7), (480, 640)), ((7, 5), (480, 640)),
                ((1, 9), (3, 20)), ((9, 1), (20, 3)), ((1, 1), (4, 6)), ((40, 60), (80, 50)), ((40, 60), (30, 90))]


def _linear_restated(img, H2, W2):
    """resizeGeneric_ with HResizeLinear / VResizeLinear in numpy float32 (each product and sum rounded on its own) over the
    coefficients of dimb_resize_area_linear_tab."""
    from dim_b200 import _native
    H, W = img.shape
    xs, xa, xmax = _native.resize_area_linear_tab(W, W2)
    ys, ya, _ = _native.resize_area_linear_tab(H, H2)
    rows = np.empty((H, W2), np.float32)
    for dx in range(W2):
        sx = xs[dx]
        rows[:, dx] = img[:, sx] * xa[dx, 0] + img[:, sx + 1] * xa[dx, 1] if dx < xmax else img[:, sx]
    out = np.empty((H2, W2), np.float32)
    for dy in range(H2):
        sy = ys[dy]
        out[dy] = rows[sy] * ya[dy, 0] + rows[min(sy + 1, H - 1)] * ya[dy, 1]
    return out


def _images(H, W, seed):
    """One integer-valued and one non-integer float32 gray image of size H x W."""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (H, W)).astype(np.float32), rng.uniform(0, 255, (H, W)).astype(np.float32)]


# ---------------------------------------------------------------------------------------------------------------- no GPU needed


@pytest.mark.parametrize("case", LINEAR_CASES)
def test_resize_area_linear_tables_reproduce_cv2_bitwise(case):
    (H, W), (H2, W2) = case
    for img in _images(H, W, H2 * W2):
        ref = cv2.resize(img, (W2, H2), interpolation=cv2.INTER_AREA)
        got = _linear_restated(img, H2, W2)
        assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32)), case


def test_resize_area_linear_tab_formulas():
    from dim_b200 import _native
    si, al, xmax = _native.resize_area_linear_tab(2, 4)  # integer factor 2: OpenCV's INTER_AREA enlarging replicates pixels
    assert si.tolist() == [0, 0, 1, 1] and xmax == 2 and np.array_equal(al, np.array([[1, 0]] * 4, np.float32))
    si, al, xmax = _native.resize_area_linear_tab(3, 4)  # inv 4/3: weights only where a destination cell straddles two sources
    assert si.tolist() == [0, 0, 1, 2] and xmax == 3
    assert np.array_equal(al, np.array([[1, 0], [np.float32(1) - np.float32(2 / 3), np.float32(2 / 3)], [np.float32(1) - np.float32(1 / 3), np.float32(1 / 3)], [1, 0]], np.float32))
    si, al, xmax = _native.resize_area_linear_tab(10, 4)  # a reduced axis of a mixed resize: no border reached
    assert xmax == 4 and si.tolist() == [0, 2, 5, 7]
    with pytest.raises(ValueError):
        _native.resize_area_linear_tab(0, 4)


def test_lowres_entries_reject_bad_arguments_without_touching_the_gpu():
    """Argument validation of the new entries comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    si, al, xmax = (C.c_int * 64)(), (C.c_float * 128)(), C.c_int()
    assert lib.dimb_resize_area_linear_tab(10, 20, si, al, C.byref(xmax)) == 0 and xmax.value == 18
    for ss, ds in ((0, 1), (10, 0), (-1, 4)):
        assert lib.dimb_resize_area_linear_tab(ss, ds, si, al, C.byref(xmax)) == -3, (ss, ds)
    assert lib.dimb_resize_area_linear_tab(10, 20, None, al, C.byref(xmax)) == -3
    assert lib.dimb_resize_area_linear_tab(10, 20, si, None, C.byref(xmax)) == -3
    assert lib.dimb_resize_area_linear_tab(10, 20, si, al, None) == -3

    def resize(ctx=ctx, src=dev, B=1, H=533, W=800, dst=dev, H2=666, W2=1000):
        return lib.dimb_resize_area_linear_dev(ctx, src, B, H, W, dst, H2, W2, null)
    assert resize(ctx=null) == -3 and resize(src=null) == -3 and resize(dst=null) == -3
    assert resize(B=0) == -3 and resize(B=70000) == -3 and resize(H=0) == -3 and resize(W=0) == -3 and resize(H2=0) == -3
    assert resize(W2=0) == -3 and resize(H=1, H2=70000) == -3 and resize(W=(1 << 20) + 1) == -3
    # no axis enlarged: dimb_resize_area_dev's case
    assert resize(H2=533, W2=800) == -3 and resize(H2=300, W2=400) == -3 and resize(H2=533, W2=700) == -3


def test_pair_generation_conf():
    from dim_b200.sharded import pair_generation_conf
    assert pair_generation_conf(None) is None
    assert pair_generation_conf({"strategy": "matching_lowres"}) == {"strategy": "matching_lowres", "resize_max": 1000, "min_matches": 20}
    c = pair_generation_conf({"strategy": "matching_lowres", "resize_max": 640, "min_matches": 0})
    assert c["resize_max"] == 640 and c["min_matches"] == 0
    base = {"strategy": "matching_lowres"}
    for bad in ({}, {"resize_max": 1000}, {**base, "resize_max": 0}, {**base, "resize_max": 1000.0}, {**base, "resize_max": True},
                {**base, "min_matches": -1}, {**base, "min_matches": 2.5}, {**base, "do_geometric_verification": True},
                {**base, "overlap": 2}):
        with pytest.raises(ValueError):
            pair_generation_conf(bad)
    for strategy in ("retrieval", "custom_pairs", "bruteforce", "sequential", "MATCHING_LOWRES"):
        with pytest.raises(ValueError, match="pairs_from_bruteforce or pairs_from_sequential"):
            pair_generation_conf({"strategy": strategy})


def test_matcher_refuses_inconsistent_pair_generation_options():
    from dim_b200.sharded import ImageSetMatcher
    pg = {"strategy": "matching_lowres"}
    with pytest.raises(ValueError, match="superpoint"):
        ImageSetMatcher(None, {}, {}, 2, 533, 800, {"max_num_keypoints": 512}, {}, extractor="aliked", pair_generation=pg)
    for matcher in ("superglue", "kornia_matcher"):
        with pytest.raises(ValueError, match="lowres_weights"):
            ImageSetMatcher(None, {}, {}, 2, 533, 800, {"max_keypoints": 512}, {}, matcher=matcher, pair_generation=pg)
    with pytest.raises(ValueError, match="pairs_from_bruteforce"):
        ImageSetMatcher(None, {}, {}, 2, 533, 800, {"max_keypoints": 512}, {}, pair_generation={"strategy": "retrieval"})
    with pytest.raises(ValueError, match="resize_max"):
        ImageSetMatcher(None, {}, {}, 2, 1, 4000, {"max_keypoints": 512}, {}, pair_generation={**pg, "resize_max": 1})


WORKER = r"""
import json, os, sys
sys.path.insert(0, os.environ["DIMB_ROOT"])
import numpy as np, torch.distributed as dist
from dim_b200.pairs_generator import pairs_from_bruteforce
from dim_b200.sharded import gather_pair_counts, shard_pairs
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n_kpts = [(i * 389) % 700 for i in range(9)]
brute = pairs_from_bruteforce(range(9))
mine = shard_pairs(len(brute), world, rank, [n_kpts[i] * n_kpts[j] for i, j in brute])
local = [(i * 7 + j * 13) % 41 for i, j in (brute[k] for k in mine)]  # this rank's "match counts"
counts = gather_pair_counts(mine, np.array(local, np.int32), len(brute), dist)
kept = [p for p, c in zip(brute, counts) if c > 20]
with open(os.path.join(os.environ["DIMB_OUT"], f"rank{rank}.json"), "w") as f:  # one file per rank: stdout lines can interleave
    json.dump({"rank": rank, "mine": mine, "counts": counts, "kept": kept}, f)
dist.destroy_process_group()
"""


def test_pair_counts_reach_every_rank_gloo(tmp_path):
    """World 2: each rank computes the counts of its share; every rank ends with the same full count array and kept list."""
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = {**os.environ, "DIMB_ROOT": ROOT, "DIMB_OUT": str(tmp_path)}
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29597", str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    res = {d["rank"]: d for d in (json.loads((tmp_path / f"rank{k}.json").read_text()) for k in range(2))}
    assert sorted(res) == [0, 1]
    brute = [(i, j) for i in range(9) for j in range(i + 1, 9)]
    exp = [(i * 7 + j * 13) % 41 for i, j in brute]
    assert res[0]["mine"] and res[1]["mine"] and sorted(res[0]["mine"] + res[1]["mine"]) == list(range(len(brute)))
    for d in res.values():
        assert d["counts"] == exp and [tuple(p) for p in d["kept"]] == [p for p, c in zip(brute, exp) if c > 20]


def test_gather_pair_counts_single_process():
    from dim_b200.sharded import gather_pair_counts
    assert gather_pair_counts([1, 0, 2], [5, 0, 7], 3) == [0, 5, 7]
    assert gather_pair_counts([], [], 0) == []


# ---------------------------------------------------------------------------------------------------------------- on the GPU


@pytest.mark.gpu
def test_resize_area_linear_dev_equals_cv2(ctx):
    import torch
    for (H, W), (H2, W2) in LINEAR_CASES:
        imgs = np.stack(_images(H, W, H2) + [_images(H, W, H2 + 1)[1]])
        ref = np.stack([cv2.resize(im, (W2, H2), interpolation=cv2.INTER_AREA) for im in imgs])
        src = torch.from_numpy(imgs).cuda()
        out = torch.full((3, H2, W2), -1.0, device="cuda")
        ctx.resize_area_linear_dev(src.data_ptr(), 3, H, W, out.data_ptr(), H2, W2, 0)
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (H, W, H2, W2)
        for b in range(3):  # one image per call gives the same bits
            one = torch.full((1, H2, W2), -1.0, device="cuda")
            ctx.resize_area_linear_dev(src[b].data_ptr(), 1, H, W, one.data_ptr(), H2, W2, 0)
            assert np.array_equal(one.cpu().numpy()[0].view(np.uint32), got[b].view(np.uint32))


@pytest.mark.gpu
def test_resize_area_linear_dev_is_asynchronous(ctx):
    """Queued behind a ~0.5 s device spin (after a first call has grown the scratch), the entry returns while the stream is busy."""
    import torch
    H, W, H2, W2 = 533, 800, 666, 1000
    img = torch.from_numpy(_images(H, W, 1)[1]).cuda()
    low = torch.zeros(H2, W2, device="cuda")
    ctx.resize_area_linear_dev(img.data_ptr(), 1, H, W, low.data_ptr(), H2, W2, 0)
    torch.cuda.synchronize()
    ref = low.clone()
    low.fill_(-1)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.resize_area_linear_dev(img.data_ptr(), 1, H, W, low.data_ptr(), H2, W2, s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy and torch.equal(ref, low)


def _scene(H, W, seed):
    """Six gray images: a blocks image, two homography warps of it, an unrelated blocks image with one warp, and a blank image."""
    from dim_b200 import synthetic
    a = synthetic.blocks_image(seed, max(H, W))[:H, :W]
    b = synthetic.blocks_image(seed + 100, max(H, W))[:H, :W]
    rgb = [a, synthetic.warp_pair(a, seed + 1, jitter=16.0), synthetic.warp_pair(a, seed + 2, jitter=24.0), b,
           synthetic.warp_pair(b, seed + 3, jitter=16.0)]
    gray = [synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in rgb] + [np.zeros((H, W), np.float32)]
    return np.stack(gray).astype(np.float32)


def _host(ctx, sp_weights, w, imgs, resize_max, min_matches):
    """pairs_from_lowres(images=...) on the images resized with cv2 as read_lowres does: (kept pairs as (i, j), counts)."""
    from pathlib import Path

    from dim_b200.pairs_generator import pairs_from_lowres
    from dim_b200.sharded import _lowres_size
    _, h, wd = _lowres_size(imgs.shape[1], imgs.shape[2], resize_max)
    names = [Path(f"{k}.png") for k in range(len(imgs))]
    low = {p.name: cv2.resize(im, (wd, h), interpolation=cv2.INTER_AREA) for p, im in zip(names, imgs)}
    pairs, counts = pairs_from_lowres(names, resize_max, min_matches, lightglue_weights=w, superpoint_weights=sp_weights, images=low,
                                      pair_batch=16, return_counts=True, device=ctx.device)
    return [(int(a.stem), int(b.stem)) for a, b in pairs], counts


SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 1024, "fix_sampling": True}
SETS = {"downsample": ((768, 1024), 1000, 40), "enlarge": ((533, 800), 1000, 50)}


@pytest.fixture(scope="module")
def lowres_sets(ctx, sp_weights):
    """Per set: the images and the host counts; min_matches is put between the counts of related and of unrelated pairs."""
    from dim_b200 import weights
    w = weights.lightglue_seeded(seed=0)
    out = {}
    for name, ((H, W), resize_max, seed) in SETS.items():
        imgs = _scene(H, W, seed)
        _, counts = _host(ctx, sp_weights, w, imgs, resize_max, 0)
        related = [counts[k] for k, (i, j) in enumerate((i, j) for i in range(6) for j in range(i + 1, 6)) if {i, j} <= {0, 1, 2} or {i, j} == {3, 4}]
        mm = max(0, min(related) - 1)
        pairs, counts = _host(ctx, sp_weights, w, imgs, resize_max, mm)
        out[name] = {"imgs": imgs, "resize_max": resize_max, "min_matches": mm, "pairs": pairs, "counts": counts, "w": w}
    return out


def _engine(ctx, sp_weights, s, batch_pairs=16, **kw):
    from dim_b200.sharded import ImageSetMatcher
    n, H, W = s["imgs"].shape
    pg = {"strategy": "matching_lowres", "resize_max": s["resize_max"], "min_matches": s["min_matches"]}
    kw.setdefault("lg_weights", s["w"])
    return ImageSetMatcher(ctx, sp_weights, kw.pop("lg_weights"), n, H, W, SP_CONF, kw.pop("lg_conf", {}), batch_images=4,
                           batch_pairs=batch_pairs, pair_generation=pg, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SETS))
def test_lowres_pairs_equal_pairs_from_lowres(ctx, sp_weights, lowres_sets, name):
    import torch
    s = lowres_sets[name]
    pairs, counts = s["pairs"], s["counts"]
    assert 0 < len(pairs) < len(counts), counts  # some pairs kept, some not
    assert all(counts[k] == 0 for k, (i, j) in enumerate((i, j) for i in range(6) for j in range(i + 1, 6)) if j == 5)  # blank image
    d = torch.from_numpy(s["imgs"]).cuda()
    base = None
    for bp in (4, 16):
        eng = _engine(ctx, sp_weights, s, bp)
        up = name == "enlarge"
        assert (eng.lowres.h > s["imgs"].shape[1]) == up
        eng.extract(d, list(range(6)))
        eng.exchange()
        got = eng.lowres_pairs()
        assert got == (pairs, counts), (bp, got, counts)
        base = got if base is None else base
        assert got == base


@pytest.mark.gpu
def test_run_lowres_equals_run_on_kept_pairs(ctx, sp_weights, lowres_sets):
    """run_lowres = lowres_pairs + run(d, ids, kept) of a matcher without pair_generation; verified=True = run_verified."""
    import torch
    from dim_b200.sharded import ImageSetMatcher
    s = lowres_sets["enlarge"]
    d = torch.from_numpy(s["imgs"]).cuda()
    n, H, W = s["imgs"].shape
    eng = _engine(ctx, sp_weights, s, verification={"seed": 3})
    pairs, counts, tables = eng.run_lowres(d, list(range(n)))
    assert (pairs, counts) == (s["pairs"], s["counts"])
    plain = ImageSetMatcher(ctx, sp_weights, s["w"], n, H, W, SP_CONF, {}, batch_images=4, batch_pairs=16, verification={"seed": 3})
    exp = plain.run(d, list(range(n)), pairs)
    assert len(tables) == len(pairs) and all(np.array_equal(a, b) for a, b in zip(tables, exp)) and max(len(t) for t in exp) > 0
    pairs_v, counts_v, res = eng.run_lowres(d, list(range(n)), verified=True)
    exp_v = plain.run_verified(d, list(range(n)), pairs)
    assert (pairs_v, counts_v) == (pairs, counts)
    for (r, v, F, k), (r2, v2, F2, k2) in zip(res, exp_v):
        assert np.array_equal(r, r2) and np.array_equal(v, v2) and k == k2 and ((F is None and F2 is None) or np.array_equal(F, F2))


@pytest.mark.gpu
def test_run_lowres_with_kornia_matcher_and_tiling(ctx, sp_weights, lowres_sets):
    import torch
    from dim_b200.sharded import ImageSetMatcher
    s = lowres_sets["downsample"]
    d = torch.from_numpy(s["imgs"]).cuda()
    n, H, W = s["imgs"].shape
    nn_conf = {"match_mode": "mnn"}
    eng = _engine(ctx, sp_weights, s, lg_weights=None, matcher="kornia_matcher", lg_conf=nn_conf, lowres_weights=s["w"])
    pairs, counts, tables = eng.run_lowres(d, list(range(n)))
    assert (pairs, counts) == (s["pairs"], s["counts"])
    plain = ImageSetMatcher(ctx, sp_weights, None, n, H, W, SP_CONF, nn_conf, batch_images=4, batch_pairs=16, matcher="kornia_matcher")
    exp = plain.run(d, list(range(n)), pairs)
    assert all(np.array_equal(a, b) for a, b in zip(tables, exp)) and max(len(t) for t in exp) > 0
    grid = {"tile_size": (512, 512), "tile_overlap": 64, "tile_selection": "grid"}
    eng = _engine(ctx, sp_weights, s, tiling=grid)
    pairs, counts, tables = eng.run_lowres(d, list(range(n)))
    assert (pairs, counts) == (s["pairs"], s["counts"])
    plain = ImageSetMatcher(ctx, sp_weights, s["w"], n, H, W, SP_CONF, {}, batch_images=4, batch_pairs=16, tiling=grid)
    exp = plain.run(d, list(range(n)), pairs)
    assert all(np.array_equal(a, b) for a, b in zip(tables, exp)) and max(len(t) for t in exp) > 0
