"""Top-k selection at any K (csrc/detect.cuh launch_select) on its own, bitwise against np.lexsort.

Up to K = 16384 production selects in one CTA per image (sp_select_kernel); above, the grid-wide path runs: a radix select of the K-th
largest score over a grid of CTAs per image, an ordered gather of the kept candidates and a stable LSD radix sort.  The self-test entry
dimb_selftest_select runs simple_nms, compaction and either path (the production choice for K, or the grid-wide path at any K) with
every output buffer starting as a sentinel and followed by a tail, as dimb_selftest_detect does (tests/test_detect_kernel.py).

Rule of both paths: every candidate in row-major order if C <= K, else np.lexsort((idx, -score))[:K].  Sort-always (ALIKED's top-k
mode, torch.topk): the kept candidates are sorted even when C <= K, and slots C .. K-1 take the first K - C pixels that are not
candidates, in row-major order, with score 0.

The designed maps are those of test_detect_kernel.py; on top: cuts inside runs of ties spanning many 4096-candidate gather chunks and
2048-key sort tiles, maps differing only in the lowest or only in the highest radix digit, a batch with one image below K and one above,
and the fill.  The CPU tests show the large-K designs are sharp against the mutants the grid path could produce: ties at the cut taken by
the larger index, and an unstable sort that leaves equal scores in an arbitrary (here: reversed) index order."""
import numpy as np
import pytest

import test_detect_kernel as D

SENT, ISENT = D.SENT, D.ISENT


def ref_select(idx, sc, K, sort_all, HW):
    """The selection rule of launch_select (K >= 1)."""
    if not sort_all:
        return D.ref_select(idx, sc, K)
    o = np.lexsort((idx, -sc.astype(np.float64)))[:K]
    si, ss = idx[o], sc[o]
    if len(si) < K:
        fill = np.setdiff1d(np.arange(HW, dtype=np.int32), idx, assume_unique=True)[:K - len(si)]
        si, ss = np.concatenate([si, fill]).astype(np.int32), np.concatenate([ss, np.zeros(len(fill), np.float32)])
    return si, ss


def check_select(out, nms_ref, thr, border, K, cap, sort_all, what):
    """Candidates and selection bitwise per image, every slot past the valid ones and every tail untouched.  Returns the counts."""
    B, H, W = nms_ref.shape
    thr = np.broadcast_to(np.asarray(thr, np.float32), (B,))
    counts = []
    for b in range(B):
        idx, sc = D.ref_candidates(nms_ref[b], thr[b], border)
        counts.append(len(idx))
        assert out["cand_count"][b] == len(idx) and np.array_equal(out["cand_idx"][b, :len(idx)], idx), f"{what}: image {b} candidates"
        si, ss = ref_select(idx, sc, K, sort_all, H * W)
        n = len(si)
        assert out["sel_count"][b] == n, f"{what}: image {b} selected {out['sel_count'][b]} != {n}"
        bad = np.flatnonzero(out["sel_idx"][b, :n] != si)
        assert len(bad) == 0, f"{what}: image {b} selected indices differ at {bad[:5]} (of {n}, C {len(idx)})"
        assert np.array_equal(D._bits(out["sel_score"][b, :n]), D._bits(ss)), f"{what}: image {b} selected scores"
        assert (out["sel_idx"][b, n:] == ISENT).all() and (out["sel_score"][b, n:] == SENT).all(), f"{what}: image {b} stray selections"
    for k in ("nms", "cand_score", "sel_score"):
        assert (out[k + "_tail"] == SENT).all(), f"{what}: write past {k}"
    for k in ("cand_count", "cand_idx", "sel_idx", "sel_count"):
        assert (out[k + "_tail"] == ISENT).all(), f"{what}: write past {k}"
    return counts


def same(a, b):
    """Bitwise equality of two output buffers (float buffers by their bits)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        return np.array_equal(a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    return np.array_equal(a, b)


def quantized(H, W, seed):
    return D.design("quantized", H, W, 0, 64, np.random.default_rng(seed))


def digit_maps(H, W, seed):
    """Scores differing only in the lowest radix digit (16 values around 0.75), and only in the highest (0x30.. 0x3f, low bits fixed)."""
    rng = np.random.default_rng(seed)
    low = np.float32(0.75).view(np.uint32) & np.uint32(0xFFFFFF00)
    high = rng.integers(0x30, 0x40, (H, W)).astype(np.uint32) << np.uint32(24)
    return {"low digit": (low | rng.integers(0, 16, (H, W)).astype(np.uint32)).view(np.float32),
            "high digit": (high | np.uint32(0x123456)).view(np.float32)}


def select_larger_index_ties(idx, sc, K):
    o = np.lexsort((-idx.astype(np.int64), -sc.astype(np.float64)))[:K]
    o = o[np.lexsort((idx[o], -sc[o].astype(np.float64)))]
    return idx[o]


def select_unstable(idx, sc, K):
    """Mutant: the right K, ordered by score with equal scores in descending index order."""
    o = np.lexsort((idx, -sc.astype(np.float64)))[:K]
    return idx[o][np.lexsort((-idx[o].astype(np.int64), -sc[o].astype(np.float64)))]


LARGE_K = (16385, 20000, 65536)


def test_large_k_designs_are_sharp():
    for name, s in {"quantized": quantized(512, 512, 700), **digit_maps(512, 512, 701)}.items():
        idx = np.arange(s.size, dtype=np.int32)
        sc = s.reshape(-1)
        for K in LARGE_K:
            si = ref_select(idx, sc, K, False, s.size)[0]
            srt = np.sort(sc)[::-1]
            assert (srt == srt[K - 1]).sum() > 4096, f"{name} K {K}: the run of ties at the cut spans less than a chunk"
            assert not np.array_equal(si, select_larger_index_ties(idx, sc, K)), f"{name} K {K}"
            assert not np.array_equal(si, select_unstable(idx, sc, K)), f"{name} K {K}"


def test_fill_reference():
    idx = np.array([0, 1, 5, 6], np.int32)
    sc = np.array([0.5, 0.7, 0.7, 0.1], np.float32)
    si, ss = ref_select(idx, sc, 7, True, 9)
    assert si.tolist() == [1, 5, 0, 6, 2, 3, 4] and ss.tolist() == [np.float32(0.7)] * 2 + [0.5, np.float32(0.1), 0, 0, 0]


@pytest.fixture(scope="module")
def st():
    from dim_b200 import _native
    return _native.SelfTest(0)


@pytest.mark.gpu
@pytest.mark.parametrize("sort_all", [False, True])
def test_designs_both_paths(st, sort_all):
    """The designed maps of test_detect_kernel.py at K = 1, 1000, C - 1, C, C + 1: the grid-wide path against np.lexsort, and the
    production choice (sp_select_kernel at these K) bitwise equal to it and, without sort-always, to dimb_selftest_detect."""
    shape = (1, 203, 260)
    for i, name in enumerate(D.DESIGNS):
        s, nms_ref = D._case(shape, [name], 3, 64, 800 + i)
        C = len(D.ref_candidates(nms_ref[0], 0.0005, 4)[0])
        for K in sorted({1, 1000, max(C - 1, 1), max(C, 1), C + 1}):
            what = f"{name} K {K} C {C} sort_all {sort_all}"
            kw = dict(thr=0.0005, border=4, K=K, cap=K + 3, sentinel=SENT)
            grid = st.select(s, 3, sort_all=sort_all, grid=True, **kw)
            check_select(grid, nms_ref, 0.0005, 4, K, K + 3, sort_all, what + " grid")
            cta = st.select(s, 3, sort_all=sort_all, **kw)
            for k in grid:
                if k != "ms":
                    assert same(grid[k], cta[k]), f"{what}: {k} differs between the paths"
            if not sort_all and K <= 16384:  # dimb_selftest_detect keeps sp_select_kernel's limit
                det = st.detect(s, 3, 0, **kw)
                for k in grid:
                    if k != "ms":
                        assert same(grid[k], det[k]), f"{what}: {k} differs from dimb_selftest_detect"


@pytest.mark.gpu
def test_large_k_sizes(st):
    """K above 16384 on a SuperPoint-like map with every pixel a candidate (r = 0, 1024 x 768), and K = C - 1, C, C + 1 with
    C > 16384 (r = 1 on 512 x 512), with and without sort-always."""
    s, nms_ref = D._case((1, 1024, 768), ["softmax_like"], 0, 64, 810)
    for K in LARGE_K:
        for sort_all in (False, True):
            check_select(st.select(s, 0, K, sort_all=sort_all), nms_ref, 0.0, 0, K, K, sort_all, f"K {K} sort_all {sort_all}")
    s, nms_ref = D._case((1, 512, 512), ["uniform"], 1, 64, 811)
    C = len(D.ref_candidates(nms_ref[0], 0.0, 0)[0])
    assert C > 16384
    for K in (C - 1, C, C + 1):
        for sort_all in (False, True):
            out = st.select(s, 1, K, cap=K + 5, sort_all=sort_all)
            check_select(out, nms_ref, 0.0, 0, K, K + 5, sort_all, f"K {K} C {C} sort_all {sort_all}")


@pytest.mark.gpu
def test_large_k_ties_and_radix_digits(st):
    """Cuts inside runs of ties that span many gather chunks and sort tiles (quantized, r = 0), and maps differing only in the lowest
    or only in the highest radix digit."""
    maps = {"quantized": quantized(512, 512, 700), **digit_maps(512, 512, 701)}
    for name, s in maps.items():
        nms_ref = D.ref_nms(s[None], 0)
        for K in LARGE_K + (200001,):
            check_select(st.select(s[None], 0, K), nms_ref, 0.0, 0, K, K, False, f"{name} K {K}")
        check_select(st.select(s[None], 0, 20000, sort_all=True), nms_ref, 0.0, 0, 20000, 20000, True, f"{name} sort_all")
    s = quantized(96, 160, 702)  # the same at small K through the grid-wide path
    for K in (1, 777, 3001, 15360):
        check_select(st.select(s[None], 0, K, grid=True), D.ref_nms(s[None], 0), 0.0, 0, K, K, False, f"quantized grid K {K}")


@pytest.mark.gpu
def test_batch_below_and_above_k(st):
    """B = 2 at K = 20000: image 0 keeps all its candidates (row-major), image 1 is cut; per-image thresholds on the device."""
    s, nms_ref = D._case((2, 256, 256), ["uniform", "uniform"], 0, 64, 820)
    thr = [0.8, 0.1]
    counts = check_select(st.select(s, 0, 20000, thr_per_image=thr), nms_ref, thr, 0, 20000, 20000, False, "batch")
    assert counts[0] < 20000 < counts[1]
    counts = check_select(st.select(s, 0, 20000, thr_per_image=thr, sort_all=True), nms_ref, thr, 0, 20000, 20000, True, "batch sorted")


@pytest.mark.gpu
def test_fill(st):
    """Sort-always with C < K: the first non-candidate pixels (inside the border and in it) fill the tail, on both paths, up to K = H W."""
    s, nms_ref = D._case((1, 128, 128), ["uniform"], 3, 64, 830)
    C = len(D.ref_candidates(nms_ref[0], 0.0, 3)[0])
    for K in (C + 1, 5000, 128 * 128):
        for grid in (False, True):
            out = st.select(s, 3, K, border=3, sort_all=True, grid=grid)
            check_select(out, nms_ref, 0.0, 3, K, K, True, f"fill K {K} grid {grid}")
    s, nms_ref = D._case((1, 256, 256), ["uniform"], 3, 64, 831)
    C = len(D.ref_candidates(nms_ref[0], 0.0, 3)[0])
    assert C < 16385
    check_select(st.select(s, 3, 20000, border=3, sort_all=True), nms_ref, 0.0, 3, 20000, 20000, True, "fill K 20000")


@pytest.mark.gpu
def test_select_refuses_bad_arguments(st):
    from dim_b200 import _native
    s = np.full((1, 16, 16), 0.5, np.float32)
    for kw in [dict(K=0), dict(K=-1), dict(K=100, cap=99), dict(K=257, sort_all=True), dict(K=4, thr=-0.5), dict(K=4, r=9)]:
        kw = {"r": 3, **kw}
        with pytest.raises(_native.DimbError, match=r"code -3\)"):
            st.select(s, **kw)
