"""lo-ransac, the second geometric-verification estimator (csrc/gv.cu, gv_math.cuh): 7-point hypotheses in waves of 1024, local
optimisation of each wave's new best model and confidence stopping.  The arithmetic is tested on the CPU through the self-test
library's host drive (dimb_gv_lo_host, dimb_gv_seven_point_host); the GPU tests check the device estimator on the same scenes, against
OpenCV's USAC_ACCURATE, across batching, and through ImageSetMatcher(verification={"estimator": "lo-ransac"})."""
import ctypes as C

import numpy as np
import pytest

from test_geometry import check_model

SEEDS = range(12)
OUTLIER_SCENES = {"33%": {}, "65%": {"out_frac": 0.65}, "75%": {"out_frac": 0.75}, "80%": {"out_frac": 0.8}}
PLANE_SCENE = {"plane": 0.99, "out_frac": 0.2}


def scene(seed, n=1500, plane=0.0, out_frac=1 / 3, noise=0.3):
    """Points seen by two cameras (test_geometry.two_view's geometry); a fraction `plane` of them on one tilted plane; each
    correspondence replaced by a random point with probability `out_frac`.  Returns k0, k1, true-inlier mask, on-plane mask."""
    rng = np.random.default_rng(seed)
    f, c = 800.0, np.array([512.0, 384.0])
    X = np.stack([3 * rng.uniform(-1, 1, n), 2 * rng.uniform(-1, 1, n), 6 + 2 * rng.uniform(-1, 1, n)], 1)
    onp = rng.uniform(size=n) < plane
    X[onp, 2] = 6 + 0.3 * X[onp, 0]
    a = 0.09
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    t = np.array([0.6, 0.05, 0.1])
    k0 = f * X[:, :2] / X[:, 2:] + c
    Xc = X @ R.T + t
    k1 = f * Xc[:, :2] / Xc[:, 2:] + c + noise * rng.uniform(-1, 1, (n, 2))
    gt = np.ones(n, bool)
    out = rng.uniform(size=n) < out_frac
    k1[out] = c + rng.uniform(-1, 1, (int(out.sum()), 2)) * np.array([500, 380])
    gt[out] = False
    return k0.astype(np.float32), k1.astype(np.float32), gt, onp


def true_F():
    """The fundamental matrix of scene()'s cameras (x1^T F x0 = 0), unit Frobenius norm."""
    a = 0.09
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    t = np.array([0.6, 0.05, 0.1])
    K = np.array([[800.0, 0, 512.0], [0, 800.0, 384.0], [0, 0, 1]])
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K)
    return F / np.linalg.norm(F)


def lo_host(k0, k1, seed, threshold=1.0, max_iters=10000, confidence=0.9999):
    """dimb_gv_lo_host: (rc, F (3,3), mask bool, hypotheses run)."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    F, mask, nh = np.zeros(9, np.float32), np.zeros(len(k0), np.uint8), C.c_int(0)
    rc = lib.dimb_gv_lo_host(k0.ctypes.data, k1.ctypes.data, len(k0), threshold, max_iters, confidence, seed, F.ctypes.data,
                             mask.ctypes.data, C.byref(nh))
    return rc, F.reshape(3, 3), mask.astype(bool), nh.value


def sampson(F, k0, k1):
    h0 = np.concatenate([k0, np.ones((len(k0), 1))], 1).astype(np.float64)
    h1 = np.concatenate([k1, np.ones((len(k1), 1))], 1).astype(np.float64)
    e = np.einsum("ni,ij,nj->n", h1, F, h0)
    l0, l1 = h0 @ F.T, h1 @ F
    return e ** 2 / (l0[:, 0] ** 2 + l0[:, 1] ** 2 + l1[:, 0] ** 2 + l1[:, 1] ** 2)


def check_plane_scene(masks):
    """The 99 %-plane scene over SEEDS: check_model on every seed, mean recall of the off-plane inliers >= 0.9."""
    off = []
    for s, (F, mask) in zip(SEEDS, masks):
        k0, k1, gt, onp = scene(s, **PLANE_SCENE)
        check_model(F, mask, k0, k1, gt)
        off.append((mask & gt & ~onp).sum() / (gt & ~onp).sum())
    assert np.mean(off) >= 0.9, off


# ---------------------------------------------------------------------------------------------------------------- no GPU needed

def test_seven_point_solver_on_exact_correspondences():
    """gv::seven_point on noise-free correspondences of known cameras, 20 random 7-subsets: one model is the true F up to scale and
    sign, and every model is singular and satisfies the 7 epipolar constraints."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    k0, k1, gt, _ = scene(0, n=400, out_frac=0.0, noise=0.0)
    Ft = true_F()
    rng = np.random.default_rng(7)
    for _ in range(20):
        idx = rng.choice(len(k0), 7, replace=False)
        a0, a1 = np.ascontiguousarray(k0[idx]), np.ascontiguousarray(k1[idx])
        out = np.zeros((3, 9), np.float32)
        m = lib.dimb_gv_seven_point_host(a0.ctypes.data, a1.ctypes.data, out.ctypes.data)
        assert 1 <= m <= 3
        errs = []
        for F in out[:m].astype(np.float64).reshape(m, 3, 3):
            F = F / np.linalg.norm(F)
            errs.append(min(np.linalg.norm(F - Ft), np.linalg.norm(F + Ft)))
            s = np.linalg.svd(F, compute_uv=False)
            assert s[2] < 1e-4 * s[0]                                  # det ~ 0: rank 2
            assert np.all(sampson(F, a0, a1) < 1e-4), sampson(F, a0, a1)  # x1^T F x0 = 0 on the sample (squared pixels)
        assert min(errs) < 1e-3, errs


@pytest.mark.parametrize("name", list(OUTLIER_SCENES))
def test_lo_host_recovers_the_inliers(name):
    """The host drive at 1 px, confidence 0.9999 and max_iters 10000 keeps >= 0.98 of the true inliers on every seed, lets few
    outliers through and returns a rank-2 model (check_model)."""
    for s in SEEDS:
        k0, k1, gt, _ = scene(s, **OUTLIER_SCENES[name])
        rc, F, mask, nh = lo_host(k0, k1, s)
        assert rc == 0 and 1024 <= nh <= 10000
        check_model(F, mask, k0, k1, gt)


def test_lo_host_on_a_dominant_plane():
    res = []
    for s in SEEDS:
        k0, k1, _, _ = scene(s, **PLANE_SCENE)
        rc, F, mask, _ = lo_host(k0, k1, s)
        assert rc == 0
        res.append((F, mask))
    check_plane_scene(res)


def test_lo_host_confidence_stopping():
    """Stopping at confidence 0.9999, max_iters 10000: a well-matched pair stops after the first wave; at 65 % outliers the bound
    exceeds max_iters, so exactly max_iters run (the last wave partial); confidence 0.5 stops earlier; never more than max_iters."""
    for s in range(4):
        k0, k1, _, _ = scene(s)
        assert lo_host(k0, k1, s)[3] == 1024
        k0, k1, _, _ = scene(s, out_frac=0.65)
        assert lo_host(k0, k1, s)[3] == 10000
        assert lo_host(k0, k1, s, confidence=0.5)[3] < 10000
        assert lo_host(k0, k1, s, max_iters=1500)[3] == 1500
        assert lo_host(k0, k1, s, max_iters=700)[3] == 700
    k0, k1, _, _ = scene(0)
    assert lo_host(k0, k1, 0, max_iters=300)[3] == 300
    assert lo_host(k0, k1, 0, confidence=1.0)[0] == -3 and lo_host(k0, k1, 0, max_iters=0)[0] == -3


def test_verification_conf_estimator():
    from dim_b200.sharded import verification_conf
    c = verification_conf({})
    assert c["estimator"] == "ransac8" and c["confidence"] == 0.9999
    assert verification_conf({"estimator": "lo-ransac", "confidence": 0.99})["estimator"] == "lo-ransac"
    assert verification_conf({"confidence": 1.5})["confidence"] == 1.5  # read by lo-ransac only
    for bad in ({"estimator": "magsac"}, {"estimator": "lo-ransac", "confidence": 1.0}, {"estimator": "lo-ransac", "confidence": 0},
                {"estimator": "lo-ransac", "max_iters": 0}):
        with pytest.raises(ValueError):
            verification_conf(bad)


def test_estimator_arguments_are_checked_before_any_cuda_call():
    """DIMB_ERR_ARG (-3) without a GPU for an unknown estimator and, with lo-ransac, confidence outside (0, 1) or max_iters < 1, from
    dimb_gv_estimate and dimb_gv_verify_dev; the non-NULL context is a dummy that the validation never dereferences."""
    from dim_b200 import _native
    from dim_b200.geometric_verification import geometric_verification
    lib = _native.load_library()
    fake = C.create_string_buffer(256)
    ctx = C.cast(fake, C.c_void_p)
    dev = C.c_void_p(0x1000)
    k = np.zeros((16, 2), np.float32)
    F, mask, cnt, nh = np.zeros(9, np.float32), np.zeros(16, np.uint8), C.c_int(), C.c_int()
    f = (_native.FeatsDev * 1)()
    f[0].keypoints = 0x1000
    seeds = (C.c_uint * 1)(0)
    bad = [_native.GvConf(1.0, 100, 15, 0.2, 2, 0.99), _native.GvConf(1.0, 100, 15, 0.2, -1, 0.99),
           _native.GvConf(1.0, 100, 15, 0.2, 1, 0.0), _native.GvConf(1.0, 100, 15, 0.2, 1, 1.0),
           _native.GvConf(1.0, 100, 15, 0.2, 1, float("nan")), _native.GvConf(1.0, 0, 15, 0.2, 1, 0.99),
           _native.GvConf(0.0, 100, 15, 0.2, 1, 0.99)]
    for conf in bad:
        assert lib.dimb_gv_estimate(ctx, k.ctypes.data, k.ctypes.data, 16, C.byref(conf), 0, F.ctypes.data, mask.ctypes.data, C.byref(cnt),
                                    C.byref(nh)) == -3
        assert lib.dimb_gv_verify_dev(ctx, 1, f, f, dev, dev, 8, seeds, C.byref(conf), dev, dev, dev, dev, dev, None) == -3
    assert lib.dimb_gv_estimate(ctx, k.ctypes.data, k.ctypes.data, 16, None, 0, F.ctypes.data, mask.ctypes.data, C.byref(cnt), None) == -3
    with pytest.raises(ValueError, match="estimator"):
        geometric_verification(k[:5], k[:5], estimator="bogus")


# ---------------------------------------------------------------------------------------------------------------- on the GPU

@pytest.mark.gpu
def test_lo_ransac_geometric_verification(ctx):
    """geometric_verification(estimator="lo-ransac") on the outlier scenes and the plane scene: the recall and outlier criteria and
    check_model, >= 0.97 of OpenCV USAC_ACCURATE's inliers, and the same answer for the same seed.  Every seed must pass at 33, 65 and
    75 % outliers and on the plane scene; at 80 % outliers (about 300 inliers in 1500) the device estimator may miss on 2 seeds of 12:
    near that breakdown point its float order (fused multiply-adds) can lead it to a wrong local optimum where the host drive does not."""
    import cv2
    from dim_b200.geometric_verification import geometric_verification
    kw = dict(method="pydegensac", threshold=1.0, confidence=0.9999, max_iters=10000, estimator="lo-ransac")
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
    check_plane_scene([geometric_verification(*scene(s, **PLANE_SCENE)[:2], seed=s, **kw) for s in SEEDS])
    k0, k1, _, _ = scene(0)
    F, mask = geometric_verification(k0[:7], k1[:7], **kw)
    assert F is None and mask.all()


class _StoreCase:
    """Scenes with mixed outlier ratios (and one pair below 8 matches) in a FeatureStoreDev (float16), match tables with shuffled
    indices as [P][cap][2] device tables."""

    def __init__(self, ctx, specs, cap=1600):
        import torch
        from dim_b200 import _native
        self.P, self.cap = len(specs), cap
        self.store = _native.FeatureStoreDev(ctx, 2 * self.P, cap, 128)
        self.m = torch.zeros(self.P, cap, 2, dtype=torch.int64, device="cuda")
        self.nm = torch.zeros(self.P, dtype=torch.int32, device="cuda")
        self.tables = []
        for p, (n, kw) in enumerate(specs):
            k0, k1, _, _ = scene(50 + p, n=max(n, 8), **kw)
            k0, k1 = k0[:n], k1[:n]
            perm = np.random.default_rng(p).permutation(n)
            d = np.zeros((128, n), np.float32)
            self.store.put(2 * p, {"keypoints": k0, "descriptors": d, "image_size": np.array([768, 1024])})
            self.store.put(2 * p + 1, {"keypoints": k1[perm], "descriptors": d, "image_size": np.array([768, 1024])})
            tab = np.stack([np.arange(n), np.argsort(perm)], 1).astype(np.int64)
            self.m[p, :n] = torch.from_numpy(tab)
            self.nm[p] = n
            self.tables.append(tab)
        self.f0 = [self.store.feats_dev(2 * p) for p in range(self.P)]
        self.f1 = [self.store.feats_dev(2 * p + 1) for p in range(self.P)]

    def matched(self, p):
        t = self.tables[p]
        return self.store.get(2 * p)["keypoints"][t[:, 0]], self.store.get(2 * p + 1)["keypoints"][t[:, 1]]

    def verify(self, ctx, order, seeds, stream=None, sleep=False):
        """dimb_gv_verify_dev with lo-ransac on the pairs `order` (in that order); per pair (verified rows, n_verified, F, mask,
        n_inliers) on the host.  With `sleep` the call is queued behind a device spin on `stream` and must return while it is busy."""
        import torch
        P, cap = len(order), self.cap
        idx = torch.tensor(order, device="cuda")
        m, nm = self.m[idx].contiguous(), self.nm[idx].contiguous()
        v = torch.full((P, cap, 2), -7, dtype=torch.int64, device="cuda")
        nv, ninl = torch.full((P,), -7, dtype=torch.int32, device="cuda"), torch.full((P,), -7, dtype=torch.int32, device="cuda")
        F, mask = torch.full((P, 9), -7.0, device="cuda"), torch.full((P, cap), 7, dtype=torch.uint8, device="cuda")
        s = stream or torch.cuda.current_stream()
        torch.cuda.synchronize()
        if sleep:
            with torch.cuda.stream(s):
                torch.cuda._sleep(1_000_000_000)
        ctx.gv_verify_dev([self.f0[k] for k in order], [self.f1[k] for k in order], m.data_ptr(), nm.data_ptr(), cap, [seeds[k] for k in order],
                          1.0, 10000, 15, 0.2, v.data_ptr(), nv.data_ptr(), F.data_ptr(), mask.data_ptr(), ninl.data_ptr(), s.cuda_stream,
                          "lo-ransac", 0.9999)
        busy = not s.query()
        torch.cuda.synchronize()
        if sleep:
            assert busy
        v, nv, F, mask, ninl, nm = (t.cpu().numpy() for t in (v, nv, F, mask, ninl, nm))
        return [(v[j, :nv[j]].copy(), int(nv[j]), F[j].copy(), mask[j, :nm[j]].copy(), int(ninl[j])) for j in range(P)]


def _same(a, b):
    assert a[1] == b[1] and a[4] == b[4] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]) and np.array_equal(a[0], b[0])


@pytest.mark.gpu
def test_verify_dev_lo_ransac_equals_the_host_entry_and_ignores_batching(ctx):
    """dimb_gv_verify_dev with lo-ransac on a batch mixing outlier ratios: per pair bitwise equal to dimb_gv_estimate on the
    fp16-exact matched keypoints with the same seed, and the same with one pair per call and with permuted positions; asynchronous."""
    from dim_b200.geometric_verification import gv_seed
    specs = [(1500, {}), (1500, {"out_frac": 0.65}), (1200, {"out_frac": 0.75}), (1500, {"out_frac": 0.8}), (5, {}),
             (1500, PLANE_SCENE), (900, {"out_frac": 0.5})]
    cs = _StoreCase(ctx, specs)
    seeds = [gv_seed(9, p) for p in range(cs.P)]
    full = cs.verify(ctx, list(range(cs.P)), seeds)
    hyps = []
    for p in range(cs.P):
        k0, k1 = cs.matched(p)
        hF, hmask, nh = ctx.gv_estimate(k0, k1, 1.0, 10000, seeds[p], "lo-ransac", 0.9999)
        hyps.append(nh)
        ver, nv, F, mask, ninl = full[p]
        assert np.array_equal(mask.astype(bool), hmask) and ninl == hmask.sum(), p
        assert (hF is None and not F.any()) or np.array_equal(F, hF.ravel()), p
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(k0))
        assert nv == (ninl if gate else 0) and np.array_equal(ver, cs.tables[p][hmask] if gate else cs.tables[p][:0])
        _same(cs.verify(ctx, [p], seeds)[0], full[p])
    assert hyps[4] == 0 and full[4][3].all() and hyps[0] == 1024 and max(hyps) == 10000, hyps
    perm = list(np.random.default_rng(3).permutation(cs.P))
    for j, r in enumerate(cs.verify(ctx, perm, seeds)):
        _same(r, full[perm[j]])
    import torch
    for a, b in zip(cs.verify(ctx, list(range(cs.P)), seeds, stream=torch.cuda.Stream(), sleep=True), full):
        _same(a, b)


def _check_verified_set(res, raw_tables, kpts, seed, plugin_tables=None):
    """Each verified table == the raw table filtered by the host lo-ransac mask (seed gv_seed(seed, pair id)) plus the gate."""
    from dim_b200.geometric_verification import geometric_verification, gv_seed
    kept = 0
    for k, (raw, ver, F, ninl) in enumerate(res):
        assert np.array_equal(raw, raw_tables[k])
        if plugin_tables is not None:
            assert np.array_equal(raw, plugin_tables[k]), k
        k0, k1 = kpts(k)
        hF, hmask = geometric_verification(k0[raw[:, 0]], k1[raw[:, 1]], "pydegensac", threshold=1.0, max_iters=10000, seed=gv_seed(seed, k),
                                           estimator="lo-ransac")
        assert ninl == int(hmask.sum()) and (F is None) == (hF is None) and (F is None or np.array_equal(F, hF)), k
        gate = ninl >= 15 and np.float32(ninl) >= np.float32(0.2) * np.float32(len(raw))
        assert np.array_equal(ver, raw[hmask] if gate else raw[:0]), k
        kept += bool(gate)
    assert kept >= 1


@pytest.mark.gpu
def test_image_set_matcher_lo_ransac(ctx, sp_weights):
    """ImageSetMatcher(verification={"estimator": "lo-ransac"}) on 5 images, all 10 pairs: tables as LightGlueMatcher._match_pairs,
    verified tables as the host lo-ransac mask plus the gate; batch_pairs 1 == 4; the default verification == explicit ransac8."""
    import torch
    from dim_b200 import synthetic, weights
    from dim_b200.config import Config
    from dim_b200.matchers.lightglue import LightGlueMatcher
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
    mk = lambda bp, ver: ImageSetMatcher(ctx, sp_weights, w, 5, size, size, sp_conf, {}, batch_images=3, batch_pairs=bp, verification=ver)
    eng = mk(4, {"seed": seed, "estimator": "lo-ransac"})
    res = eng.run_verified(d_imgs, list(range(5)), pairs)
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w}), local_features="superpoint")
    feats = {i: eng.store.get(store_slot(i, 5, 1)) for i in range(5)}
    expected = [plugin._match_pairs(feats[i], feats[j]) for i, j in pairs]
    _check_verified_set(res, [r[0] for r in res], lambda k: (feats[pairs[k][0]]["keypoints"], feats[pairs[k][1]]["keypoints"]), seed,
                        expected)
    for a, b in zip(mk(1, {"seed": seed, "estimator": "lo-ransac"}).run_verified(d_imgs, list(range(5)), pairs), res):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3]
        assert (a[2] is None) == (b[2] is None) and (a[2] is None or np.array_equal(a[2], b[2]))
    dflt = mk(4, {"seed": seed}).run_verified(d_imgs, list(range(5)), pairs)
    for a, b in zip(dflt, mk(4, {"seed": seed, "estimator": "ransac8"}).run_verified(d_imgs, list(range(5)), pairs)):
        assert np.array_equal(a[1], b[1]) and a[3] == b[3] and (a[2] is None or np.array_equal(a[2], b[2]))


@pytest.mark.gpu
def test_tiled_image_set_lo_ransac(ctx, sp_weights):
    """A tiled set (3 images 768 x 1024, 512-pixel tiles): the merged tables verified by lo-ransac equal the host lo-ransac mask on
    the merged slots plus the gate; batch_pairs 4 (one image pair's 4 tile pairs per batch) == 8."""
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
                                    verification={"seed": seed, "estimator": "lo-ransac"})
    eng = mk(8)
    res = eng.run_verified(d, [0, 1, 2], pairs)
    tables = eng.run(d, [0, 1, 2], pairs)
    _check_verified_set(res, tables, lambda k: (eng.store.get(pairs[k][0])["keypoints"], eng.store.get(pairs[k][1])["keypoints"]), seed)
    for x, y in zip(mk(4).run_verified(d, [0, 1, 2], pairs), res):
        assert np.array_equal(x[1], y[1]) and x[3] == y[3]
