"""Batched, device-resident SuperGlue (dimb_sg_match_dev): P pairs per call from device features, [P][cap][2] match tables, no host
synchronisation.  Against the oracle (indices identical up to match-threshold flips, scores within 2e-4), against the single-pair
host entry dimb_sg_match on identical inputs (indices identical, scores within 1e-5), from the device feature store, and through
sharded.ImageSetMatcher(matcher="superglue")."""
import ctypes as C

import numpy as np
import pytest

MAXK = 320   # max_kpts of the batched handle
SEED = 1     # weights seed (that of the golden "small" case)
SENT = -7    # sentinel of untouched output rows


def _pairs():
    """Six pairs of mixed shapes: m != n, 480x640 and 640x480 images, the golden `small` arguments, a pair at max_kpts, a pair with
    no keypoints on one side, a 1 x 1 pair."""
    import os
    from conftest import GOLD
    from oracle.gen_golden import lg_pair
    seed, m, n, h, w = [int(x) for x in np.load(os.path.join(GOLD, "superglue_golden.npz"))["small.args"]]
    f0, f1 = lg_pair(5, 40, 30, 256, (200, 240))
    f1 = {k: (v[:0] if k != "image_size" else v) for k, v in f1.items()}
    f1["descriptors"] = np.zeros((256, 0), np.float32)
    return [lg_pair(11, 150, 100, 256, (480, 640)), lg_pair(12, 120, 160, 256, (640, 480)), lg_pair(seed, m, n, 256, (h, w)),
            lg_pair(13, MAXK, MAXK - 37, 256, (480, 640)), (f0, f1), lg_pair(14, 1, 1, 256, (100, 120))]


class _DevSide:
    """float32 device copy of a FeaturesDict with NaN padding past n (never read) and the dimb_sg_feats_dev describing it."""

    def __init__(self, f, round_fp16=1, pad=3):
        import torch
        from dim_b200 import _native
        n = f["keypoints"].shape[0]
        cap = min(n + pad, MAXK) if n < MAXK else n
        w = max(cap, 1)
        nan = float("nan")
        self.kp = torch.full((w, 2), nan, device="cuda")
        self.de = torch.full((256, w), nan, device="cuda")
        self.sc = torch.full((w,), nan, device="cuda")
        self.kp[:n] = torch.from_numpy(np.ascontiguousarray(f["keypoints"], np.float32))
        self.de[:, :n] = torch.from_numpy(np.ascontiguousarray(f["descriptors"], np.float32))
        self.sc[:n] = torch.from_numpy(np.ascontiguousarray(f["scores"], np.float32))
        self.cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
        h, wd = [int(v) for v in f["image_size"]]
        self.s = _native.SgFeatsDev(self.kp.data_ptr(), self.de.data_ptr(), self.sc.data_ptr(), self.cnt.data_ptr(), cap, w, 0, round_fp16,
                                    h, wd, None)


def _run(net, sides, cap=MAXK, stream=0):
    """sides: list of (_DevSide, _DevSide).  Returns (list of {matches, scores}, n_matches, raw tables)."""
    import torch
    P = len(sides)
    m = torch.full((P, cap, 2), SENT, dtype=torch.int64, device="cuda")
    ms = torch.full((P, cap), float(SENT), device="cuda")
    nm = torch.full((P,), SENT, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    net.match_dev([a.s for a, _ in sides], [b.s for _, b in sides], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), cap, stream)
    torch.cuda.synchronize()
    m, ms, nm = m.cpu().numpy(), ms.cpu().numpy(), nm.cpu().numpy()
    out = [{"matches": m[p, :min(nm[p], cap)].copy(), "scores": ms[p, :min(nm[p], cap)].copy()} for p in range(P)]
    return out, nm, (m, ms)


def _same(a, b, tol):
    assert np.array_equal(a["matches"], b["matches"]), (len(a["matches"]), len(b["matches"]))
    if len(a["scores"]):
        assert np.abs(a["scores"] - b["scores"]).max() <= tol


@pytest.fixture(scope="module")
def sg_case():
    from oracle import superglue as o_sg
    return o_sg.seeded_weights(SEED), _pairs()


@pytest.fixture(scope="module")
def sg_net(ctx, sg_case):
    from dim_b200 import _native
    return _native.SuperGlueNet(ctx, sg_case[0], max_kpts=MAXK, max_pairs=6)


@pytest.fixture(scope="module")
def batch(sg_net, sg_case):
    sides = [(_DevSide(a), _DevSide(b)) for a, b in sg_case[1]]
    out, nm, _ = _run(sg_net, sides)
    return sides, out, nm


def test_sg_dev_entries_reject_null_handles_without_touching_the_gpu():
    """Argument validation of the device entries comes before any CUDA call: DIMB_ERR_ARG (-3) without a GPU."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    f = _native.SgFeatsDev()
    assert lib.dimb_sg_match_dev(null, 1, C.byref(f), C.byref(f), null, null, null, 1, null) == -3
    assert lib.dimb_sg_match_dev(null, 1, None, None, null, null, null, 1, null) == -3
    assert lib.dimb_fstore_sg_feats_dev(null, 0, C.byref(f)) == -3
    assert lib.dimb_fstore_sg_feats_dev(null, 0, None) == -3


@pytest.mark.gpu
def test_batch_matches_oracle(sg_case, batch):
    """Six pairs of mixed shapes in ONE call (float32 inputs rounded to fp16 on the device) against the oracle on the features.h5
    round trip of the same features."""
    from dim_b200.io_h5 import as_half_roundtrip
    from oracle import superglue as o_sg
    from oracle.compare import compare_matches
    wts, pairs = sg_case
    _, out, nm = batch
    for p, (f0, f1) in enumerate(pairs):
        ref = o_sg.match(as_half_roundtrip(f0), as_half_roundtrip(f1), wts)
        exp = {"matches": ref["matches"], "scores": ref["matching_scores0"][ref["matches"][:, 0]], "stop": 0}
        rep = compare_matches({**out[p], "stop": 0}, exp, 0.2, 2e-4)
        print(p, rep["n"], "matches, max score delta", rep["max_dscore"], rep["boundary_diffs"])
        assert out[p]["matches"].dtype == np.int64
    assert nm[4] == 0  # no keypoints on one side: nothing matched, the other pairs undisturbed
    assert min(nm[k] for k in (0, 1, 2, 3)) > 20


@pytest.mark.gpu
def test_batch_equals_host_entry(sg_net, sg_case, batch):
    """The host entry (stage one pair, same engine with P = 1) on the fp16-rounded features gives the batch's tables."""
    from dim_b200.io_h5 import as_half_roundtrip
    _, out, _ = batch
    for p, (f0, f1) in enumerate(sg_case[1]):
        host = sg_net.match(as_half_roundtrip(f0), as_half_roundtrip(f1))
        _same(out[p], host, 1e-5)


@pytest.mark.gpu
def test_no_cross_pair_leakage_and_workspace_reuse(sg_net, batch):
    """Permuted pairs in a full batch, then a smaller batch on the same handle: every pair's result is unchanged."""
    sides, out, _ = batch
    perm = [3, 5, 0, 4, 2, 1]
    res, _, _ = _run(sg_net, [sides[k] for k in perm])
    for j, k in enumerate(perm):
        _same(res[j], out[k], 1e-6)
    small = [2, 0, 4]
    res, _, _ = _run(sg_net, [sides[k] for k in small])
    for j, k in enumerate(small):
        _same(res[j], out[k], 1e-6)


@pytest.mark.gpu
def test_capacity_reports_full_count_and_writes_cap_rows(sg_net, batch):
    """cap below the match count: n_matches holds the full count, the first cap rows are those of the uncapped call, and nothing past
    a pair's rows is written (rows of a pair with fewer matches than cap, and a guard after the last pair)."""
    import torch
    sides, out, nm_full = batch
    sel = [3, 5]
    cap = int(nm_full[3]) // 2
    assert cap >= 10 and nm_full[5] < cap
    guard = 16
    m = torch.full((2 * cap + guard, 2), SENT, dtype=torch.int64, device="cuda")
    ms = torch.full((2 * cap + guard,), float(SENT), device="cuda")
    nm = torch.full((2,), SENT, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sg_net.match_dev([sides[k][0].s for k in sel], [sides[k][1].s for k in sel], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), cap)
    torch.cuda.synchronize()
    m, ms, nm = m.cpu().numpy(), ms.cpu().numpy(), nm.cpu().numpy()
    assert list(nm) == [nm_full[3], nm_full[5]]
    for j, k in enumerate(sel):
        rows = min(int(nm[j]), cap)
        blk, sblk = m[j * cap:(j + 1) * cap], ms[j * cap:(j + 1) * cap]
        assert np.array_equal(blk[:rows], out[k]["matches"][:rows])
        assert np.abs(sblk[:rows] - out[k]["scores"][:rows]).max(initial=0) <= 1e-6
        assert np.all(blk[rows:] == SENT) and np.all(sblk[rows:] == SENT)
    assert np.all(m[2 * cap:] == SENT) and np.all(ms[2 * cap:] == SENT)


@pytest.mark.gpu
def test_feature_store_path_equals_plugin(ctx, sg_case):
    """Host put into the device feature store, sg_feats_dev, match_dev == SuperGlueMatcher._match_pairs on store.get (the features.h5
    contract)."""
    import torch
    from dim_b200 import _native
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    wts, pairs = sg_case
    use = [pairs[k] for k in (0, 1, 2, 3)]
    store = _native.FeatureStoreDev(ctx, 2 * len(use), MAXK, 256)
    for p, (a, b) in enumerate(use):
        store.put(2 * p, a)
        store.put(2 * p + 1, b)
    net = _native.SuperGlueNet(ctx, wts, max_kpts=store.cap, max_pairs=len(use))
    P, cap = len(use), store.cap
    m = torch.full((P, cap, 2), SENT, dtype=torch.int64, device="cuda")
    ms = torch.zeros((P, cap), device="cuda")
    nm = torch.zeros((P,), dtype=torch.int32, device="cuda")
    net.match_dev([store.sg_feats_dev(2 * p) for p in range(P)], [store.sg_feats_dev(2 * p + 1) for p in range(P)], m.data_ptr(),
                  ms.data_ptr(), nm.data_ptr(), cap)
    torch.cuda.synchronize()
    m, nm = m.cpu().numpy(), nm.cpu().numpy()
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": wts}))
    for p in range(P):
        exp = plugin._match_pairs(store.get(2 * p), store.get(2 * p + 1))
        assert np.array_equal(m[p, :nm[p]], exp), (p, nm[p], len(exp))
        assert len(exp) > 20


@pytest.mark.gpu
def test_match_dev_is_asynchronous(sg_net, batch):
    """Queued behind a ~0.5 s device spin, the call returns while the stream is still busy; results are right after a synchronise."""
    import torch
    sides, out, _ = batch
    P, cap = len(sides), MAXK
    m = torch.full((P, cap, 2), SENT, dtype=torch.int64, device="cuda")
    ms = torch.full((P, cap), float(SENT), device="cuda")
    nm = torch.full((P,), SENT, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    sg_net.match_dev([a.s for a, _ in sides], [b.s for _, b in sides], m.data_ptr(), ms.data_ptr(), nm.data_ptr(), cap, s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    m, ms, nm = m.cpu().numpy(), ms.cpu().numpy(), nm.cpu().numpy()
    assert busy
    for p in range(len(sides)):
        _same({"matches": m[p, :nm[p]], "scores": ms[p, :nm[p]]}, out[p], 1e-6)


@pytest.mark.gpu
def test_argument_errors_and_fast_mode(sg_net, sg_case, batch):
    from dim_b200 import _native
    from dim_b200.io_h5 import as_half_roundtrip
    sides, _, _ = batch
    with pytest.raises(_native.DimbError, match=r"code -3"):  # P > max_pairs
        _run(sg_net, sides + sides[:1])
    big = _DevSide(sg_case[1][3][0], pad=0)
    big.s.n_cap = MAXK + 1
    with pytest.raises(_native.DimbError, match=r"code -3"):  # n_cap > max_kpts
        _run(sg_net, [(big, sides[0][1])])
    no_scores = _DevSide(sg_case[1][0][0])
    no_scores.s.scores = None
    with pytest.raises(_native.DimbError, match=r"code -3"):  # NULL scores
        _run(sg_net, [(no_scores, sides[0][1])])
    fast = _native.Context(0, precision="fast")
    net = _native.SuperGlueNet(fast, sg_case[0], max_kpts=MAXK, max_pairs=6)
    res, _, _ = _run(net, sides)
    for p, (f0, f1) in enumerate(sg_case[1]):
        host = net.match(as_half_roundtrip(f0), as_half_roundtrip(f1))
        assert np.array_equal(res[p]["matches"], host["matches"]), p


@pytest.mark.gpu
def test_image_set_matcher_superglue(ctx, sp_weights, sg_case):
    """ImageSetMatcher(matcher="superglue") in one process on 5 synthetic 320 x 320 images (0 and 1: a homography pair), all 10 pairs:
    every table equals the SuperGlue plugin on the store's features."""
    import torch
    from dim_b200 import synthetic
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    size, K = 320, 512
    a, b = synthetic.synthetic_pair(11, size)
    c, d = synthetic.synthetic_pair(12, size)
    e = synthetic.synthetic_pair(13, size)[0]
    imgs = np.stack([a, b, c, d, e]).astype(np.float32)
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": K}
    wts = sg_case[0]
    sg_conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
    pairs = pairs_from_bruteforce(list(range(5)))
    eng = ImageSetMatcher(ctx, sp_weights, wts, 5, size, size, sp_conf, sg_conf, batch_images=3, batch_pairs=4, matcher="superglue")
    tables = eng.run(torch.from_numpy(imgs).cuda(), list(range(5)), pairs)
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": wts}))
    assert len(tables) == 10
    for (i, j), t in zip(pairs, tables):
        exp = plugin._match_pairs(eng.store.get(store_slot(i, 5, 1)), eng.store.get(store_slot(j, 5, 1)))
        assert t.dtype == np.int64 and np.array_equal(t, exp), (i, j, len(t), len(exp))
    assert len(tables[0]) > 20, len(tables[0])
