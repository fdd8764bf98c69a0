"""degensac, the third geometric-verification estimator (csrc/gv.cu, gv_math.cuh): lo-ransac's waves plus DEGENSAC's dominant-plane
test (H from F and three points over five triplets) and plane-and-parallax recovery of F.  The arithmetic is tested on the CPU through
the self-test library (dimb_gv_h_from_f3_host, dimb_gv_degenerate_host, dimb_gv_plane_parallax_host, dimb_gv_degensac_host); the GPU
tests check the device estimator on the same scenes, against OpenCV's USAC_ACCURATE, across batching, and through
ImageSetMatcher(verification={"estimator": "degensac"})."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_geometry import check_model
from test_gv_lo import OUTLIER_SCENES, SEEDS, scene, true_F

# (plane fraction, outlier fraction) at n = 4000.  Bars on the off-plane recall over SEEDS: mean >= 0.95 and no seed below 0.8.  At
# 0.99 / 50 % only about 23 of 2000 off-plane matches are inliers, so a 2-point draw is all-inlier with probability ~1.3e-4 and the
# 1024 draws of a plane-and-parallax step find one about 1 time in 8: there the bar is the measured host figure (mean 0.748, min 0.267),
# still above lo-ransac (0.592 / 0.067) and OpenCV USAC_ACCURATE (0.532 / 0.174) on the same points.
PLANE_SCENES = {"0.98/50%": (0.98, 0.5), "0.99/50%": (0.99, 0.5), "0.99/20%": (0.99, 0.2)}
PLANE_BARS = {"0.98/50%": (0.95, 0.8), "0.99/50%": (0.70, 0.2), "0.99/20%": (0.95, 0.8)}


def _lib():
    from dim_b200 import _native
    return _native.load_selftest_library()


def deg_host(k0, k1, seed, threshold=1.0, max_iters=10000, confidence=0.9999):
    """dimb_gv_degensac_host: (rc, F (3,3), mask bool, hypotheses run)."""
    F, mask, nh = np.zeros(9, np.float32), np.zeros(len(k0), np.uint8), C.c_int(0)
    rc = _lib().dimb_gv_degensac_host(k0.ctypes.data, k1.ctypes.data, len(k0), threshold, max_iters, confidence, seed, F.ctypes.data,
                                      mask.ctypes.data, C.byref(nh))
    return rc, F.reshape(3, 3), mask.astype(bool), nh.value


def plane_scene(s, name):
    pl, out = PLANE_SCENES[name]
    return scene(s, n=4000, plane=pl, out_frac=out)


def check_plane(name, results):
    """check_model on every seed and the off-plane recall bars of `name`; returns the per-seed off-plane recalls."""
    off = []
    for s, (F, mask) in zip(SEEDS, results):
        k0, k1, gt, onp = plane_scene(s, name)
        check_model(F, mask, k0, k1, gt)
        off.append((mask & gt & ~onp).sum() / (gt & ~onp).sum())
    mean_bar, min_bar = PLANE_BARS[name]
    print(name, "off-plane recall", np.round(off, 3), "mean", round(float(np.mean(off)), 3))
    assert np.mean(off) >= mean_bar and min(off) >= min_bar, (name, off)
    return np.array(off)


def true_H():
    """The homography of scene()'s plane z = 6 + 0.3 x (pixels, image 0 -> image 1): K (R - t n^T / d) K^-1 with n^T X = d."""
    a = 0.09
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    t = np.array([0.6, 0.05, 0.1])
    K = np.array([[800.0, 0, 512.0], [0, 800.0, 384.0], [0, 0, 1]])
    n, d = np.array([-0.3, 0.0, 1.0]), 6.0
    H = K @ (R + np.outer(t, n) / d) @ np.linalg.inv(K)
    return H / np.linalg.norm(H)


def _apply(H, k):
    h = np.concatenate([k, np.ones((len(k), 1))], 1) @ H.T
    return h[:, :2] / h[:, 2:]


# ---------------------------------------------------------------------------------------------------------------- no GPU needed

def test_true_homography_of_the_scene():
    k0, k1, _, onp = scene(0, n=400, plane=0.5, out_frac=0.0, noise=0.0)
    assert np.abs(_apply(true_H(), k0[onp]) - k1[onp]).max() < 1e-3


def test_h_from_f_and_three_points():
    """On noise-free plane points, H from the true F and any three of them maps every on-plane point to float tolerance, and
    equals the plane's homography up to scale and sign; three collinear points are rejected."""
    lib = _lib()
    k0, k1, _, onp = scene(1, n=300, plane=0.6, out_frac=0.0, noise=0.0)
    on = np.flatnonzero(onp)
    F = true_F().astype(np.float32).ravel()
    rng = np.random.default_rng(3)
    Ht = true_H()
    for _ in range(20):
        idx = rng.choice(on, 3, replace=False).astype(np.int32)
        H = np.zeros(9, np.float32)
        assert lib.dimb_gv_h_from_f3_host(F.ctypes.data, k0.ctypes.data, k1.ctypes.data, len(k0), idx.ctypes.data, H.ctypes.data) == 1
        H = H.reshape(3, 3).astype(np.float64)
        assert np.abs(_apply(H, k0[on]) - k1[on]).max() < 0.02
        assert min(np.linalg.norm(H - Ht), np.linalg.norm(H + Ht)) < 1e-3
    line = np.ascontiguousarray(np.stack([np.linspace(100, 900, 3), np.linspace(50, 650, 3)], 1).astype(np.float32))
    kk0, kk1 = np.concatenate([line, k0]).astype(np.float32), np.concatenate([line, k1]).astype(np.float32)
    H = np.zeros(9, np.float32)
    idx = np.array([0, 1, 2], np.int32)
    assert lib.dimb_gv_h_from_f3_host(F.ctypes.data, kk0.ctypes.data, kk1.ctypes.data, len(kk0), idx.ctypes.data, H.ctypes.data) == 0


def test_five_triplets_cover_every_five_subset():
    tri = [{0, 1, 2}, {3, 4, 5}, {0, 1, 6}, {3, 4, 6}, {2, 5, 6}]
    for sub in itertools.combinations(range(7), 5):
        assert any(t <= set(sub) for t in tri), sub


def h_from_f3_ref(F, x, xp):
    """Hartley & Zisserman Result 13.6 in float64: H = A - e' (M^-1 b)^T (x, xp: (3,2) pixels)."""
    e = np.linalg.svd(F.T)[2][-1]
    A = np.cross(e, F.T).T  # [e']_x F
    X, Xp = np.concatenate([x, np.ones((3, 1))], 1), np.concatenate([xp, np.ones((3, 1))], 1)
    b = np.array([np.cross(Xp[i], A @ X[i]) @ np.cross(Xp[i], e) / np.sum(np.cross(Xp[i], e) ** 2) for i in range(3)])
    return A - np.outer(e, np.linalg.solve(X, b))


def degenerate_ref(F, a0, a1, threshold):
    """The five-triplet test in float64 with the smallest margin of any count decision to the 2 x threshold bar: (flagged, margin)."""
    flagged, margin = False, np.inf
    for t in ([0, 1, 2], [3, 4, 5], [0, 1, 6], [3, 4, 6], [2, 5, 6]):
        err = np.linalg.norm(_apply(h_from_f3_ref(F, a0[t], a1[t]), a0) - a1, axis=1)
        flagged |= (err < 2 * threshold).sum() >= 5
        margin = min(margin, np.abs(np.delete(err, t) - 2 * threshold).min())
    return flagged, margin


@pytest.mark.parametrize("k", range(8))
def test_degeneracy_test_flags_five_or_more_coplanar_points(k):
    """Noise-free 7-samples with k points on the plane (at random positions in the sample), on the true F: a sample with k >= 5 is
    always flagged; every sample is flagged exactly when the float64 test flags it (three points off the plane span a virtual plane
    that two more sample points can lie near), and the H returned maps 5 or more sample points within 2 px."""
    lib = _lib()
    k0, k1, _, onp = scene(2, n=600, plane=0.5, out_frac=0.0, noise=0.0)
    on, off = np.flatnonzero(onp), np.flatnonzero(~onp)
    F = true_F().astype(np.float32).ravel()
    rng = np.random.default_rng(10 + k)
    flagged = 0
    for _ in range(30):
        idx = np.concatenate([rng.choice(on, k, replace=False), rng.choice(off, 7 - k, replace=False)])
        idx = rng.permutation(idx).astype(np.int32)
        H = np.zeros(9, np.float32)
        t = lib.dimb_gv_degenerate_host(F.ctypes.data, k0.ctypes.data, k1.ctypes.data, len(k0), idx.ctypes.data, 1.0, H.ctypes.data)
        ref, margin = degenerate_ref(true_F(), k0[idx].astype(np.float64), k1[idx].astype(np.float64), 1.0)
        if margin > 1e-2:
            assert (t >= 0) == ref, (k, t, ref)
        flagged += t >= 0
        if t >= 0:
            assert (np.linalg.norm(_apply(H.reshape(3, 3).astype(np.float64), k0[idx]) - k1[idx], axis=1) < 2.0).sum() >= 5
        if k >= 5:
            assert t >= 0
    if k < 5:
        assert flagged <= 10, flagged  # general position is the rule


def test_plane_and_parallax_recovers_the_true_F():
    lib = _lib()
    k0, k1, _, onp = scene(4, n=400, plane=0.5, out_frac=0.0, noise=0.0)
    off = np.flatnonzero(~onp)
    H = true_H().astype(np.float32).ravel()
    Ft = true_F()
    rng = np.random.default_rng(5)
    for _ in range(20):
        i, j = rng.choice(off, 2, replace=False)
        F = np.zeros(9, np.float32)
        assert lib.dimb_gv_plane_parallax_host(H.ctypes.data, k0.ctypes.data, k1.ctypes.data, len(k0), int(i), int(j), F.ctypes.data) == 1
        F = F.reshape(3, 3).astype(np.float64)
        F /= np.linalg.norm(F)
        assert min(np.linalg.norm(F - Ft), np.linalg.norm(F + Ft)) < 2e-3
        assert np.linalg.svd(F, compute_uv=False)[2] < 1e-5


@pytest.mark.parametrize("name", list(PLANE_SCENES))
def test_degensac_host_on_dominant_planes(name):
    res = []
    for s in SEEDS:
        k0, k1, _, _ = plane_scene(s, name)
        rc, F, mask, nh = deg_host(k0, k1, s)
        assert rc == 0 and 1024 <= nh <= 10000
        res.append((F, mask))
    check_plane(name, res)


@pytest.mark.parametrize("name", list(OUTLIER_SCENES))
def test_degensac_host_recovers_the_inliers(name):
    """lo-ransac's criteria on its outlier scenes: check_model on every seed."""
    for s in SEEDS:
        k0, k1, gt, _ = scene(s, **OUTLIER_SCENES[name])
        rc, F, mask, nh = deg_host(k0, k1, s)
        assert rc == 0 and 1024 <= nh <= 10000
        check_model(F, mask, k0, k1, gt)


def test_degensac_arguments_are_checked_before_any_cuda_call():
    """DIMB_ERR_ARG (-3) without a GPU: degensac (3) with confidence outside (0, 1) or max_iters < 1, and the unknown estimators 2
    and 4, from dimb_gv_estimate and dimb_gv_verify_dev (the dummy context is never dereferenced); verification_conf refuses the same.
    2 stays unknown: it was refused before degensac existed."""
    from dim_b200 import _native
    from dim_b200.sharded import verification_conf
    lib = _native.load_library()
    ctx = C.cast(C.create_string_buffer(256), C.c_void_p)
    dev = C.c_void_p(0x1000)
    k = np.zeros((16, 2), np.float32)
    F, mask, cnt, nh = np.zeros(9, np.float32), np.zeros(16, np.uint8), C.c_int(), C.c_int()
    f = (_native.FeatsDev * 1)()
    f[0].keypoints = 0x1000
    seeds = (C.c_uint * 1)(0)
    assert _native.gv_estimator("degensac") == 3
    bad = [_native.GvConf(1.0, 100, 15, 0.2, 3, 0.0), _native.GvConf(1.0, 100, 15, 0.2, 3, 1.0),
           _native.GvConf(1.0, 100, 15, 0.2, 3, float("nan")), _native.GvConf(1.0, 0, 15, 0.2, 3, 0.99),
           _native.GvConf(1.0, 100, 15, 0.2, 2, 0.99), _native.GvConf(1.0, 100, 15, 0.2, 4, 0.99)]
    for conf in bad:
        assert lib.dimb_gv_estimate(ctx, k.ctypes.data, k.ctypes.data, 16, C.byref(conf), 0, F.ctypes.data, mask.ctypes.data, C.byref(cnt),
                                    C.byref(nh)) == -3
        assert lib.dimb_gv_verify_dev(ctx, 1, f, f, dev, dev, 8, seeds, C.byref(conf), dev, dev, dev, dev, dev, None) == -3
    assert deg_host(k, k, 0, confidence=1.0)[0] == -3 and deg_host(k, k, 0, max_iters=0)[0] == -3
    assert verification_conf({"estimator": "degensac", "confidence": 0.99})["estimator"] == "degensac"
    for bad in ({"estimator": "magsac"}, {"estimator": "degensac", "confidence": 1.0}, {"estimator": "degensac", "max_iters": 0}):
        with pytest.raises(ValueError):
            verification_conf(bad)


# ---------------------------------------------------------------------------------------------------------------- on the GPU

@pytest.mark.gpu
def test_degensac_geometric_verification(ctx):
    """geometric_verification(estimator="degensac"): on the outlier scenes lo-ransac's device criteria (every seed at 33, 65 and 75 %,
    up to 2 misses of 12 at 80 %) with >= 0.97 of USAC_ACCURATE's inliers; on the plane scenes the host drive's bars and a higher mean
    off-plane recall than USAC_ACCURATE; the same answer for the same seed."""
    import cv2
    from dim_b200.geometric_verification import geometric_verification
    kw = dict(method="pydegensac", threshold=1.0, confidence=0.9999, max_iters=10000, estimator="degensac")
    for name, sc in OUTLIER_SCENES.items():
        missed = []
        for s in SEEDS:
            k0, k1, gt, _ = scene(s, **sc)
            F, mask = geometric_verification(k0, k1, seed=s, **kw)
            if s < 2:
                F2, mask2 = geometric_verification(k0, k1, seed=s, **kw)
                assert np.array_equal(F, F2) and np.array_equal(mask, mask2)
            try:
                check_model(F, mask, k0, k1, gt)
                _, inl = cv2.findFundamentalMat(k0, k1, cv2.USAC_ACCURATE, 1.0, 0.9999, 10000)
                cvm = inl.ravel() > 0
                assert (mask & cvm).sum() >= 0.97 * cvm.sum(), (name, s)
            except AssertionError:
                missed.append((s, round(float((mask & gt).sum() / gt.sum()), 3)))
        print(name, "seeds that missed (seed, recall):", missed)
        assert len(missed) <= (2 if name == "80%" else 0), (name, missed)
    for name in PLANE_SCENES:
        off = check_plane(name, [geometric_verification(*plane_scene(s, name)[:2], seed=s, **kw) for s in SEEDS])
        cv_off = []
        for s in SEEDS:
            k0, k1, gt, onp = plane_scene(s, name)
            _, inl = cv2.findFundamentalMat(k0, k1, cv2.USAC_ACCURATE, 1.0, 0.9999, 10000)
            cv_off.append((inl.ravel().astype(bool) & gt & ~onp).sum() / (gt & ~onp).sum())
        print(name, "USAC_ACCURATE off-plane recall mean", round(float(np.mean(cv_off)), 3))
        assert off.mean() > np.mean(cv_off), (name, off.mean(), np.mean(cv_off))


def _verify(ctx, case, order, seeds, stream=None, sleep=False):
    """dimb_gv_verify_dev with degensac on the pairs `order` of a test_gv_lo._StoreCase; per pair (verified rows, n_verified, F, mask,
    n_inliers).  With `sleep` the call is queued behind a device spin and must return while it is busy."""
    import torch
    P, cap = len(order), case.cap
    idx = torch.tensor(order, device="cuda")
    m, nm = case.m[idx].contiguous(), case.nm[idx].contiguous()
    v = torch.full((P, cap, 2), -7, dtype=torch.int64, device="cuda")
    nv, ninl = torch.full((P,), -7, dtype=torch.int32, device="cuda"), torch.full((P,), -7, dtype=torch.int32, device="cuda")
    F, mask = torch.full((P, 9), -7.0, device="cuda"), torch.full((P, cap), 7, dtype=torch.uint8, device="cuda")
    s = stream or torch.cuda.current_stream()
    torch.cuda.synchronize()
    if sleep:
        with torch.cuda.stream(s):
            torch.cuda._sleep(1_000_000_000)
    ctx.gv_verify_dev([case.f0[k] for k in order], [case.f1[k] for k in order], m.data_ptr(), nm.data_ptr(), cap, [seeds[k] for k in order],
                      1.0, 10000, 15, 0.2, v.data_ptr(), nv.data_ptr(), F.data_ptr(), mask.data_ptr(), ninl.data_ptr(), s.cuda_stream,
                      "degensac", 0.9999)
    busy = not s.query()
    torch.cuda.synchronize()
    if sleep:
        assert busy
    v, nv, F, mask, ninl, nm = (t.cpu().numpy() for t in (v, nv, F, mask, ninl, nm))
    return [(v[j, :nv[j]].copy(), int(nv[j]), F[j].copy(), mask[j, :nm[j]].copy(), int(ninl[j])) for j in range(P)]


@pytest.mark.gpu
def test_verify_dev_degensac_equals_the_host_entry_and_ignores_batching(ctx):
    """dimb_gv_verify_dev with degensac on a batch mixing outlier ratios and plane scenes: per pair bitwise equal to dimb_gv_estimate
    with the same seed, and the same with one pair per call and with permuted positions; asynchronous."""
    import torch
    from dim_b200.geometric_verification import gv_seed
    from test_gv_lo import PLANE_SCENE, _same, _StoreCase
    specs = [(1500, {}), (1500, {"out_frac": 0.65}), (1500, {"plane": 0.98, "out_frac": 0.5}), (5, {}), (1500, PLANE_SCENE),
             (1500, {"out_frac": 0.8}), (900, {"plane": 0.99, "out_frac": 0.5})]
    cs = _StoreCase(ctx, specs)
    seeds = [gv_seed(11, p) for p in range(cs.P)]
    full = _verify(ctx, cs, list(range(cs.P)), seeds)
    hyps = []
    for p in range(cs.P):
        k0, k1 = cs.matched(p)
        hF, hmask, nh = ctx.gv_estimate(k0, k1, 1.0, 10000, seeds[p], "degensac", 0.9999)
        hyps.append(nh)
        ver, nv, F, mask, ninl = full[p]
        assert np.array_equal(mask.astype(bool), hmask) and ninl == hmask.sum(), p
        assert (hF is None and not F.any()) or np.array_equal(F, hF.ravel()), p
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(k0))
        assert nv == (ninl if gate else 0) and np.array_equal(ver, cs.tables[p][hmask] if gate else cs.tables[p][:0])
        _same(_verify(ctx, cs, [p], seeds)[0], full[p])
    assert hyps[3] == 0 and full[3][3].all() and hyps[0] == 1024 and max(hyps) == 10000, hyps
    perm = list(np.random.default_rng(4).permutation(cs.P))
    for j, r in enumerate(_verify(ctx, cs, perm, seeds)):
        _same(r, full[perm[j]])
    for a, b in zip(_verify(ctx, cs, list(range(cs.P)), seeds, stream=torch.cuda.Stream(), sleep=True), full):
        _same(a, b)


def _check_verified_set(res, raw_tables, kpts, seed):
    """Each verified table == the raw table filtered by the host degensac mask (seed gv_seed(seed, pair id)) plus the gate."""
    from dim_b200.geometric_verification import geometric_verification, gv_seed
    kept = 0
    for k, (raw, ver, F, ninl) in enumerate(res):
        assert np.array_equal(raw, raw_tables[k])
        k0, k1 = kpts(k)
        hF, hmask = geometric_verification(k0[raw[:, 0]], k1[raw[:, 1]], "pydegensac", threshold=1.0, max_iters=10000, seed=gv_seed(seed, k),
                                           estimator="degensac")
        assert ninl == int(hmask.sum()) and (F is None) == (hF is None) and (F is None or np.array_equal(F, hF)), k
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(raw))
        assert np.array_equal(ver, raw[hmask] if gate else raw[:0]), k
        kept += bool(gate)
    assert kept >= 1


@pytest.mark.gpu
def test_image_set_matcher_degensac(ctx, sp_weights):
    """ImageSetMatcher(verification={"estimator": "degensac"}) on 5 images, all 10 pairs: verified tables as the host degensac mask
    plus the gate; batch_pairs 1 == 4."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    size, seed = 384, 3
    imgs = []
    for p in range(3):
        imgs += list(synthetic.synthetic_pair(70 + p, size))
    imgs = np.stack(imgs[:5]).astype(np.float32)
    w = weights.lightglue_seeded(seed=0)
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 512}
    pairs = pairs_from_bruteforce(list(range(5)))
    d_imgs = torch.from_numpy(imgs).cuda()
    mk = lambda bp: ImageSetMatcher(ctx, sp_weights, w, 5, size, size, sp_conf, {}, batch_images=3, batch_pairs=bp,
                                    verification={"seed": seed, "estimator": "degensac"})
    eng = mk(4)
    res = eng.run_verified(d_imgs, list(range(5)), pairs)
    feats = {i: eng.store.get(store_slot(i, 5, 1)) for i in range(5)}
    _check_verified_set(res, [r[0] for r in res], lambda k: (feats[pairs[k][0]]["keypoints"], feats[pairs[k][1]]["keypoints"]), seed)
    for a, b in zip(mk(1).run_verified(d_imgs, list(range(5)), pairs), res):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3]
        assert (a[2] is None) == (b[2] is None) and (a[2] is None or np.array_equal(a[2], b[2]))


@pytest.mark.gpu
def test_tiled_image_set_degensac(ctx, sp_weights):
    """A tiled set (3 images 768 x 1024, 512-pixel tiles): the merged tables verified by degensac equal the host degensac mask on the
    merged slots plus the gate; batch_pairs 4 == 8."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(40, 1024)[:768, :1024]
    imgs = [a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in range(1, 3)]
    imgs = np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in imgs]).astype(np.float32)
    d = torch.from_numpy(imgs).cuda()
    pairs, seed = pairs_from_bruteforce([0, 1, 2]), 5
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "fix_sampling": True, "max_keypoints": 1024}
    mk = lambda bp: ImageSetMatcher(ctx, sp_weights, weights.lightglue_seeded(seed=0), 3, 768, 1024, sp_conf, {}, batch_images=6,
                                    batch_pairs=bp, tiling={"tile_size": 512, "tile_overlap": 64, "tile_selection": "grid"},
                                    verification={"seed": seed, "estimator": "degensac"})
    eng = mk(8)
    res = eng.run_verified(d, [0, 1, 2], pairs)
    tables = eng.run(d, [0, 1, 2], pairs)
    _check_verified_set(res, tables, lambda k: (eng.store.get(pairs[k][0])["keypoints"], eng.store.get(pairs[k][1])["keypoints"]), seed)
    for x, y in zip(mk(4).run_verified(d, [0, 1, 2], pairs), res):
        assert np.array_equal(x[1], y[1]) and x[3] == y[3]
