"""Verified matching of image sets: dimb_gv_verify_dev (fundamental-matrix RANSAC on device match tables with keypoints from the
float16 feature store, one seed per pair, ordered inlier compaction and the per-pair gate), ImageSetMatcher(verification=...), the
gather of raw / verified tables and F to rank 0, and the COLMAP database written from them.  The device results are compared
bitwise with the single-pair host entry dimb_gv_fundamental on the same (fp16-exact) keypoints and seed: every GV reduction runs in
a fixed order, so a pair's result does not depend on the batch it is verified in."""
import ctypes as C
import os
import sqlite3
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_geometry import check_model, two_view

THR, ITERS = 1.0, 4096


# ---------------------------------------------------------------------------------------------------------------- no GPU needed

def test_gv_seed_is_a_pure_function_of_seed_and_pair_id():
    from dim_b200.geometric_verification import gv_seed
    assert gv_seed(0, 0) == 3298878556 and gv_seed(5, 3) == 1013825697  # the documented mix, pinned
    seeds = [gv_seed(7, k) for k in range(2000)]
    assert seeds == [gv_seed(7, k) for k in range(2000)]
    assert all(isinstance(s, int) and 0 <= s < 2 ** 32 for s in seeds) and len(set(seeds)) == len(seeds)
    assert gv_seed(7 + 2 ** 32, 11) == gv_seed(7, 11) and gv_seed(-1, 4) == gv_seed(2 ** 32 - 1, 4)
    assert gv_seed(1, 11) != gv_seed(2, 11)


def test_verify_dev_rejects_null_handles_and_bad_conf_without_touching_the_gpu():
    """Argument validation of dimb_gv_verify_dev comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU.  Every call below has
    at least one invalid argument; the non-NULL context is a dummy that the validation never dereferences."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    fake = C.create_string_buffer(256)
    ctx = C.cast(fake, C.c_void_p)
    dev = C.c_void_p(0x1000)  # a device-address stand-in: never dereferenced on the host
    f = (_native.FeatsDev * 1)()
    f[0].keypoints = 0x1000
    seeds = (C.c_uint * 1)(0)
    good = _native.GvConf(1.0, 100, 15, 0.2)

    def call(ctx=ctx, P=1, f0=f, f1=f, m=dev, nm=dev, cap=8, sd=seeds, conf=good, outs=(dev,) * 5):
        return lib.dimb_gv_verify_dev(ctx, P, f0, f1, m, nm, cap, sd, C.byref(conf) if conf is not None else None, *outs, null)

    assert call(ctx=null) == -3
    assert call(P=0) == -3 and call(cap=0) == -3
    assert call(f0=None) == -3 and call(f1=None) == -3 and call(sd=None) == -3 and call(conf=None) == -3
    assert call(m=null) == -3 and call(nm=null) == -3
    for k in range(5):
        assert call(outs=tuple(null if j == k else dev for j in range(5))) == -3, k
    for bad in (_native.GvConf(0.0, 100, 15, 0.2), _native.GvConf(-1.0, 100, 15, 0.2), _native.GvConf(float("nan"), 100, 15, 0.2),
                _native.GvConf(1.0, 100, -1, 0.2), _native.GvConf(1.0, 100, 15, -0.1), _native.GvConf(1.0, 100, 15, 1.5),
                _native.GvConf(1.0, 100, 15, float("nan"))):
        assert call(conf=bad) == -3
    nokp = (_native.FeatsDev * 1)()
    assert call(f0=nokp) == -3 and call(f1=nokp) == -3


def test_verification_conf_defaults_and_validation():
    from dim_b200.sharded import verification_conf
    assert verification_conf(None) is None
    c = verification_conf({})
    assert (c["method"], c["threshold"], c["max_iters"], c["seed"], c["min_inliers_per_pair"], c["min_inlier_ratio_per_pair"]) == \
        ("PYDEGENSAC", 1.0, 10000, 0, 15, 0.2)
    assert verification_conf({"method": "none"})["method"] == "NONE"
    for bad in ({"method": "bogus"}, {"threshold": 0}, {"min_inliers_per_pair": -1}, {"min_inlier_ratio_per_pair": 1.5}, {"tresh": 1}):
        with pytest.raises(ValueError):
            verification_conf(bad)


def _fake_results(ids):
    """(raw, verified, F, n_inliers) of pair i, a function of i only (some with F None, one empty, one rejected)."""
    out = []
    for i in ids:
        rng = np.random.default_rng(100 + i)
        raw = rng.integers(0, 2048, (int(rng.integers(0, 60)), 2)).astype(np.int64)
        keep = rng.uniform(size=len(raw)) < 0.7
        ver = raw[keep] if i % 4 != 3 else raw[:0]
        F = rng.standard_normal((3, 3)).astype(np.float32) if i % 3 else None
        out.append((raw, ver, F, int(keep.sum())))
    return out


GATHER_WORKER = r"""
import os, sys
sys.path.insert(0, os.environ["DIMB_ROOT"])
sys.path.insert(0, os.path.join(os.environ["DIMB_ROOT"], "tests"))
import numpy as np, torch.distributed as dist
from dim_b200.sharded import shard_pairs, gather_verified
from test_verify_sets import _fake_results
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 13
costs = [(i * 7919) % 13 + 1 for i in range(n)]
mine = shard_pairs(n, world, rank, costs)
full = gather_verified(mine, _fake_results(mine), n, dist)
if rank == 0:
    single = gather_verified(list(range(n)), _fake_results(range(n)), n, None)
    for i in range(n):
        a, b = full[i], single[i]
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3], i
        assert (a[2] is None) == (b[2] is None) and (a[2] is None or (a[2].dtype == np.float32 and np.array_equal(a[2], b[2]))), i
        assert a[0].dtype == np.int64 and a[1].dtype == np.int64 and a[1].shape[1] == 2
    print("GATHER_VERIFIED_OK", sum(len(r[1]) for r in full))
else:
    assert full is None
dist.destroy_process_group()
"""


def test_gather_verified_single_process():
    from dim_b200.sharded import gather_verified
    res = _fake_results([0, 1, 2, 3])
    out = gather_verified([2, 0, 1, 3], [res[2], res[0], res[1], res[3]], 5)
    assert out[4] is None
    for i in range(4):
        assert np.array_equal(out[i][0], res[i][0]) and np.array_equal(out[i][1], res[i][1]) and out[i][3] == res[i][3]
        assert (out[i][2] is None) == (res[i][2] is None) and (res[i][2] is None or np.array_equal(out[i][2], res[i][2]))


def test_world_size_2_gloo_gathers_verified_results(tmp_path):
    """Two gloo processes deal 13 pairs by cost, gather raw tables, verified tables, F and counts: rank 0 holds what one process
    gets."""
    script = tmp_path / "gather_worker.py"
    script.write_text(GATHER_WORKER)
    env = {**os.environ, "DIMB_ROOT": ROOT}
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29593", str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "GATHER_VERIFIED_OK" in r.stdout


class _HostStore:
    """Stand-in of FeatureStoreDev.get for the COLMAP helper: slot -> FeaturesDict."""

    def __init__(self, feats):
        self.feats = feats

    def get(self, slot):
        return self.feats[slot]


def test_colmap_export_of_a_verified_image_set(tmp_path):
    """Raw tables -> matches, non-empty verified tables and F -> two_view_geometries, gate-rejected pairs absent, a pair listed as
    (high, low) stored low -> high with its columns swapped and F transposed."""
    from dim_b200.io_colmap import image_ids_to_pair_id
    from dim_b200.sharded import export_verified_to_colmap, store_slot
    n, world = 3, 2
    rng = np.random.default_rng(0)
    feats = {}
    for i in range(n):
        feats[store_slot(i, n, world)] = {"keypoints": rng.uniform(0, 100, (10 + i, 2)).astype(np.float32), "image_size": np.array([120, 160])}
    store = _HostStore(feats)
    F01 = np.arange(9, dtype=np.float32).reshape(3, 3) + 1
    F20 = (np.arange(9, dtype=np.float32).reshape(3, 3) + 1) * 10  # pair listed as (2, 0): x0^T F20 x2 = 0
    pairs = [(0, 1), (2, 0), (1, 2)]
    results = [(np.array([[0, 1], [2, 3], [4, 5]]), np.array([[0, 1], [4, 5]]), F01, 2),
               (np.array([[7, 1], [8, 2]]), np.array([[8, 2]]), F20, 1),
               (np.array([[1, 1]]), np.zeros((0, 2), np.int64), None, 1)]  # rejected by the gate
    db_path = tmp_path / "database.db"
    ids = export_verified_to_colmap(store, n, world, pairs, results, db_path, image_names=["a.jpg", "b.jpg", "c.jpg"])
    assert ids == {"a.jpg": 1, "b.jpg": 2, "c.jpg": 3}
    db = sqlite3.connect(str(db_path))
    kp = {r[0]: np.frombuffer(r[3], np.float32).reshape(r[1], r[2]) for r in db.execute("SELECT * FROM keypoints")}
    for i in range(n):
        assert np.array_equal(kp[i + 1], feats[store_slot(i, n, world)]["keypoints"])
    raw = {r[0]: np.frombuffer(r[3], np.uint32).reshape(r[1], r[2]) for r in db.execute("SELECT pair_id, rows, cols, data FROM matches")}
    assert set(raw) == {image_ids_to_pair_id(1, 2), image_ids_to_pair_id(1, 3), image_ids_to_pair_id(2, 3)}
    assert np.array_equal(raw[image_ids_to_pair_id(1, 2)], results[0][0])
    assert np.array_equal(raw[image_ids_to_pair_id(1, 3)], results[1][0][:, ::-1])
    assert np.array_equal(raw[image_ids_to_pair_id(2, 3)], results[2][0])
    tvg = {r[0]: (np.frombuffer(r[3], np.uint32).reshape(r[1], r[2]), r[4], np.frombuffer(r[5], np.float64).reshape(3, 3))
           for r in db.execute("SELECT pair_id, rows, cols, data, config, F FROM two_view_geometries")}
    assert set(tvg) == {image_ids_to_pair_id(1, 2), image_ids_to_pair_id(1, 3)}  # the rejected pair (b, c) is absent
    m, cfg, F = tvg[image_ids_to_pair_id(1, 2)]
    assert np.array_equal(m, results[0][1]) and cfg == 2 and np.array_equal(F, F01.astype(np.float64))
    m, cfg, F = tvg[image_ids_to_pair_id(1, 3)]
    assert np.array_equal(m, [[2, 8]]) and np.array_equal(F, F20.T.astype(np.float64))  # x2^T F20^T x0 = 0: low id -> high id
    db.close()


# ---------------------------------------------------------------------------------------------------------------- on the GPU

def _host_gv(ctx, k0, k1, seed, threshold=THR, iters=ITERS):
    """The single-pair host entry dimb_gv_fundamental: (F [9] float32, mask uint8 [n], n_inliers)."""
    k0, k1 = np.ascontiguousarray(k0, np.float32), np.ascontiguousarray(k1, np.float32)
    n = len(k0)
    F, mask, cnt = np.zeros(9, np.float32), np.zeros(max(n, 1), np.uint8), C.c_int(0)
    ctx.check(ctx.lib.dimb_gv_fundamental(ctx.h, k0.ctypes.data, k1.ctypes.data, n, float(threshold), int(iters), int(seed) & 0xffffffff,
                                          F.ctypes.data, mask.ctypes.data, C.byref(cnt)), "dimb_gv_fundamental")
    return F, mask[:n], cnt.value


class _Case:
    """P two-view pairs in a FeatureStoreDev (float16) with shuffled match indices, as [P][cap][2] device tables (n_matches = the
    pair's size, or `raw`)."""

    def __init__(self, ctx, sizes, cap=1024, raw=None):
        import torch
        from dim_b200 import _native
        self.P, self.cap = len(sizes), cap
        self.store = _native.FeatureStoreDev(ctx, 2 * self.P, max(max(sizes), cap), 128)
        self.m = torch.zeros(self.P, cap, 2, dtype=torch.int64, device="cuda")
        self.nm = torch.zeros(self.P, dtype=torch.int32, device="cuda")
        self.gts, self.tables = [], []
        for p, n in enumerate(sizes):
            k0, k1, gt = two_view(30 + p, n=max(n, 8))
            k0, k1, gt = k0[:n], k1[:n], gt[:n]
            perm = np.random.default_rng(p).permutation(n)
            d = np.zeros((128, n), np.float32)
            self.store.put(2 * p, {"keypoints": k0, "descriptors": d, "image_size": np.array([768, 1024])})
            self.store.put(2 * p + 1, {"keypoints": k1[perm], "descriptors": d, "image_size": np.array([768, 1024])})
            tab = np.stack([np.arange(n), np.argsort(perm)], 1).astype(np.int64)
            rows = min(n, cap)
            self.m[p, :rows] = torch.from_numpy(tab[:rows])
            self.nm[p] = n if raw is None else raw[p]
            self.gts.append(gt)
            self.tables.append(tab)
        self.f0 = [self.store.feats_dev(2 * p) for p in range(self.P)]
        self.f1 = [self.store.feats_dev(2 * p + 1) for p in range(self.P)]

    def matched(self, p):
        """fp16-exact matched keypoints of the first n_raw rows of pair p (store.get: the features.h5 values)."""
        n = min(int(self.nm[p]), self.cap)
        t = self.tables[p][:n]
        return self.store.get(2 * p)["keypoints"][t[:, 0]], self.store.get(2 * p + 1)["keypoints"][t[:, 1]]


def _verify(ctx, f0, f1, m, nm, cap, seeds, stream=0, min_inliers=0, ratio=0.0, threshold=THR, iters=ITERS):
    """One dimb_gv_verify_dev call; returns per pair (verified rows, n_verified, F [9], mask [n_raw], n_inliers) on the host."""
    import torch
    P = len(f0)
    v = torch.full((P, cap, 2), -7, dtype=torch.int64, device="cuda")
    nv = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    F = torch.full((P, 9), -7.0, device="cuda")
    mask = torch.full((P, cap), 7, dtype=torch.uint8, device="cuda")
    ninl = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.gv_verify_dev(f0, f1, m.data_ptr(), nm.data_ptr(), cap, seeds, threshold, iters, min_inliers, ratio, v.data_ptr(), nv.data_ptr(),
                      F.data_ptr(), mask.data_ptr(), ninl.data_ptr(), stream)
    torch.cuda.synchronize()
    return _host(v, nv, F, mask, ninl, nm, cap)


def _host(v, nv, F, mask, ninl, nm, cap):
    v, nv, F, mask, ninl, nm = (t.cpu().numpy() for t in (v, nv, F, mask, ninl, nm))
    out = []
    for p in range(len(nv)):
        n = min(int(nm[p]), cap)
        out.append((v[p], int(nv[p]), F[p].copy(), mask[p, :n].copy(), int(ninl[p])))
    return out


def _same(a, b):
    assert a[1] == b[1] and a[4] == b[4] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
    assert np.array_equal(a[0][:a[1]], b[0][:b[1]])


@pytest.fixture(scope="module")
def case(ctx):
    return _Case(ctx, [700, 800, 900, 750, 1000])


@pytest.mark.gpu
def test_store_input_known_geometry_equals_host_entry(ctx, case):
    """Keypoints straight from the float16 store: mask, F and count bitwise equal to the host entry on the fp16-exact matched
    keypoints with the same seed; the model recovers the known geometry; the verified table is raw[mask] in order."""
    from dim_b200.geometric_verification import gv_seed
    seeds = [gv_seed(3, p) for p in range(case.P)]
    res = _verify(ctx, case.f0, case.f1, case.m, case.nm, case.cap, seeds)
    for p in range(case.P):
        ver, nv, F, mask, ninl = res[p]
        k0, k1 = case.matched(p)
        hF, hmask, hn = _host_gv(ctx, k0, k1, seeds[p])
        assert np.array_equal(F, hF) and np.array_equal(mask, hmask) and ninl == hn, p
        check_model(F.reshape(3, 3), mask.astype(bool), k0, k1, case.gts[p])
        raw = case.tables[p]
        assert nv == ninl == mask.sum() and np.array_equal(ver[:nv], raw[mask.astype(bool)])


@pytest.mark.gpu
def test_batch_independence(ctx, case):
    """The same pairs verified one per call, three per call, all at once and in reversed order: identical per-pair outputs."""
    import torch
    from dim_b200.geometric_verification import gv_seed
    seeds = [gv_seed(11, 100 + p) for p in range(case.P)]
    full = _verify(ctx, case.f0, case.f1, case.m, case.nm, case.cap, seeds, min_inliers=15, ratio=0.2)
    for p in range(case.P):
        one = _verify(ctx, case.f0[p:p + 1], case.f1[p:p + 1], case.m[p:p + 1], case.nm[p:p + 1], case.cap, seeds[p:p + 1], min_inliers=15,
                      ratio=0.2)
        _same(one[0], full[p])
    for b0 in range(0, case.P, 3):
        sl = slice(b0, b0 + 3)
        part = _verify(ctx, case.f0[sl], case.f1[sl], case.m[sl], case.nm[sl], case.cap, seeds[sl], min_inliers=15, ratio=0.2)
        for k, r in enumerate(part):
            _same(r, full[b0 + k])
    rev = list(range(case.P))[::-1]
    idx = torch.tensor(rev, device="cuda")
    back = _verify(ctx, [case.f0[k] for k in rev], [case.f1[k] for k in rev], case.m[idx].contiguous(), case.nm[idx].contiguous(), case.cap,
                   [seeds[k] for k in rev], min_inliers=15, ratio=0.2)
    for j, k in enumerate(rev):
        _same(back[j], full[k])


@pytest.mark.gpu
def test_gates_and_edges(ctx):
    """< 8 matches: all ones, F zeros, n_inliers = n_raw, rejected by the default gate and kept by 0 / 0; too few inliers and a
    low ratio each reject while mask / F / count are still written; n_matches > cap uses cap rows; float32 keypoints with
    round_fp16 = 1 give the store path's results."""
    import torch
    from dim_b200 import _native
    from dim_b200.geometric_verification import gv_seed
    cs = _Case(ctx, [5, 600, 900], cap=1024)
    seeds = [gv_seed(0, p) for p in range(cs.P)]
    free = _verify(ctx, cs.f0, cs.f1, cs.m, cs.nm, cs.cap, seeds)                       # gates 0 / 0: every pair kept
    dflt = _verify(ctx, cs.f0, cs.f1, cs.m, cs.nm, cs.cap, seeds, min_inliers=15, ratio=0.2)
    ver, nv, F, mask, ninl = free[0]
    assert mask.all() and len(mask) == 5 and not F.any() and ninl == 5 and nv == 5 and np.array_equal(ver[:5], cs.tables[0])
    assert dflt[0][1] == 0 and dflt[0][4] == 5 and dflt[0][3].all()
    for p in (1, 2):
        assert free[p][1] == free[p][4] > 15
        _same(dflt[p], free[p])
    ninl = free[1][4]
    few = _verify(ctx, cs.f0, cs.f1, cs.m, cs.nm, cs.cap, seeds, min_inliers=ninl + 1)
    assert few[1][1] == 0 and few[1][4] == ninl and np.array_equal(few[1][2], free[1][2]) and np.array_equal(few[1][3], free[1][3])
    assert few[2][1] == (free[2][4] if free[2][4] >= ninl + 1 else 0)
    low = _verify(ctx, cs.f0, cs.f1, cs.m, cs.nm, cs.cap, seeds, ratio=1.0)  # two_view has outliers: n_inliers < n_raw
    for p in (1, 2):
        assert free[p][4] < len(free[p][3]) and low[p][1] == 0 and low[p][4] == free[p][4] and np.array_equal(low[p][2], free[p][2])
    assert low[0][1] == 5  # all ones: ratio 1 holds
    # n_matches beyond cap: the first cap rows are verified
    small = _Case(ctx, [900], cap=500, raw=[900])
    r = _verify(ctx, small.f0, small.f1, small.m, small.nm, small.cap, seeds[:1])[0]
    k0, k1 = small.matched(0)
    assert len(k0) == 500 and len(r[3]) == 500
    hF, hmask, hn = _host_gv(ctx, k0, k1, seeds[0])
    assert np.array_equal(r[2], hF) and np.array_equal(r[3], hmask) and r[4] == hn == r[1]
    # float32 keypoints rounded to fp16 on the device == the float16 store slots
    keep, f0, f1 = [], [], []
    for p in range(cs.P):
        fs = []
        for s in (2 * p, 2 * p + 1):
            n = cs.store.count(s)[0]
            kp = np.full((cs.cap, 2), np.nan, np.float32)
            src = two_view(30 + p, n=max(n, 8))[:2]
            kp[:n] = src[0][:n] if s % 2 == 0 else src[1][:n][np.random.default_rng(p).permutation(n)]
            t = torch.from_numpy(kp).cuda()
            keep.append(t)
            fs.append(_native.FeatsDev(t.data_ptr(), 0, 0, cs.cap, 0, 0, 0.0, 0.0, 1, 0, None))
        f0.append(fs[0])
        f1.append(fs[1])
    r32 = _verify(ctx, f0, f1, cs.m, cs.nm, cs.cap, seeds, min_inliers=15, ratio=0.2)
    for p in range(cs.P):
        _same(r32[p], dflt[p])


@pytest.mark.gpu
def test_verify_dev_is_asynchronous(ctx, case):
    """Queued behind a ~0.5 s device spin, the call returns while the stream is still busy; results are right after a synchronise."""
    import torch
    from dim_b200.geometric_verification import gv_seed
    seeds = [gv_seed(3, p) for p in range(case.P)]
    ref = _verify(ctx, case.f0, case.f1, case.m, case.nm, case.cap, seeds)  # also grows the scratch to this call's size
    P, cap = case.P, case.cap
    v = torch.zeros(P, cap, 2, dtype=torch.int64, device="cuda")
    nv = torch.zeros(P, dtype=torch.int32, device="cuda")
    F = torch.zeros(P, 9, device="cuda")
    mask = torch.zeros(P, cap, dtype=torch.uint8, device="cuda")
    ninl = torch.zeros(P, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.gv_verify_dev(case.f0, case.f1, case.m.data_ptr(), case.nm.data_ptr(), cap, seeds, THR, ITERS, 0, 0.0, v.data_ptr(), nv.data_ptr(),
                      F.data_ptr(), mask.data_ptr(), ninl.data_ptr(), s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    assert busy
    for a, b in zip(_host(v, nv, F, mask, ninl, case.nm, cap), ref):
        _same(a, b)


def _image_set(matcher):
    from dim_b200 import synthetic, weights
    from oracle import superglue as o_sg
    if matcher == "superglue":
        size = 320
        a, b = synthetic.synthetic_pair(11, size)
        c, d = synthetic.synthetic_pair(12, size)
        imgs = np.stack([a, b, c, d, synthetic.synthetic_pair(13, size)[0]]).astype(np.float32)
        conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
        return imgs, size, o_sg.seeded_weights(1), conf
    size = 384
    imgs = []
    for p in range(3):
        imgs += list(synthetic.synthetic_pair(70 + p, size))
    return np.stack(imgs[:5]).astype(np.float32), size, weights.lightglue_seeded(seed=0), {}


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", ["lightglue", "superglue"])
def test_image_set_matcher_verified(ctx, sp_weights, matcher):
    """5 images, all 10 pairs: raw tables == run(); each verified table == the plugin's table filtered by the host
    geometric_verification mask (seed gv_seed(seed, pair id)) and the gate, with the same F; batch_pairs 1 == 4; method NONE gives
    verified == raw; verification=None allocates nothing new and run() is unchanged."""
    import torch
    from dim_b200.config import Config
    from dim_b200.geometric_verification import geometric_verification, gv_seed
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    imgs, size, w, conf = _image_set(matcher)
    K, seed = 512, 3
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": K}
    pairs = pairs_from_bruteforce(list(range(5)))
    d_imgs = torch.from_numpy(imgs).cuda()
    mk = lambda bp, ver: ImageSetMatcher(ctx, sp_weights, w, 5, size, size, sp_conf, conf, batch_images=3, batch_pairs=bp, matcher=matcher,
                                         verification=ver)
    plain = mk(4, None)
    assert plain.gv is None and not hasattr(plain, "v") and not hasattr(plain, "host_out")
    tables = plain.run(d_imgs, list(range(5)), pairs)
    eng = mk(4, {"seed": seed})
    res = eng.run_verified(d_imgs, list(range(5)), pairs)
    assert [np.array_equal(a, b) for a, b in zip(eng.run(d_imgs, list(range(5)), pairs), tables)] == [True] * 10
    if matcher == "superglue":
        plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": w}))
    else:
        plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    kept = 0
    for k, ((i, j), (raw, ver, F, ninl)) in enumerate(zip(pairs, res)):
        assert np.array_equal(raw, tables[k]) and raw.dtype == ver.dtype == np.int64
        f0, f1 = eng.store.get(store_slot(i, 5, 1)), eng.store.get(store_slot(j, 5, 1))
        exp = plugin._match_pairs(f0, f1)
        assert np.array_equal(raw, exp), (i, j)
        hF, hmask = geometric_verification(f0["keypoints"][exp[:, 0]], f1["keypoints"][exp[:, 1]], "pydegensac", threshold=1.0,
                                           max_iters=10000, seed=gv_seed(seed, k))
        assert ninl == int(hmask.sum()) and (F is None) == (hF is None) and (F is None or np.array_equal(F, hF)), (i, j)
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(exp))
        assert np.array_equal(ver, exp[hmask] if gate else exp[:0]), (i, j, len(ver), gate)
        kept += bool(gate)
    assert kept >= 1 and max(len(r[1]) for r in res) > 20, [len(r[1]) for r in res]
    one = mk(1, {"seed": seed}).run_verified(d_imgs, list(range(5)), pairs)
    for a, b in zip(one, res):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3]
        assert (a[2] is None) == (b[2] is None) and (a[2] is None or np.array_equal(a[2], b[2]))
    none = mk(4, {"method": "NONE"})
    assert not hasattr(none, "v")
    for (raw, ver, F, ninl), t in zip(none.run_verified(d_imgs, list(range(5)), pairs), tables):
        assert np.array_equal(raw, t) and np.array_equal(ver, t) and F is None and ninl == len(t)
