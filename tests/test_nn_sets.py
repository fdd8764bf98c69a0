"""Batched, device-resident brute-force NN matching (dimb_nn_match_batch_dev) and ImageSetMatcher(matcher="kornia_matcher").  The
engine is compared bitwise with the single-pair entries dimb_nn_match_dev / dimb_nn_match (same kernels, P = 1) and with the kornia
oracle; the image-set matcher's tables exactly with KorniaMatcher._match_pairs / _match_by_tile on the store's features."""
import ctypes as C

import numpy as np
import pytest

CAP = 768                                      # keypoint capacity of the store
COUNTS = [700, 129, 2, 1, 0, CAP, 300, 650]    # live keypoints of slots 0..7
PAIRS = [(4, 0), (0, 1), (1, 0), (2, 3), (3, 2), (5, 7), (6, 5), (0, 7), (1, 6)]  # empty, n0 > n1, n0 < n1, tiny, at capacity
MODES = [("nn", 0.0), ("mnn", 0.0), ("snn", 0.9), ("smnn", 0.95)]
SENT = -7


def test_batch_entry_rejects_a_null_context_without_touching_the_gpu():
    """DIMB_ERR_ARG (-3) for a NULL context before any CUDA call (the other argument checks need a context: see
    test_batch_entry_rejects_bad_arguments)."""
    from dim_b200 import _native
    lib = _native.load_library()
    null = C.c_void_p()
    f = (_native.FeatsDev * 1)()
    buf = C.c_void_p(16)
    assert lib.dimb_nn_match_batch_dev(null, 1, f, f, 256, 3, 0.8, buf, buf, buf, 8, null) == -3
    assert lib.dimb_nn_match_batch_dev(null, 1, None, None, 256, 3, 0.8, null, null, null, 8, null) == -3


def test_kornia_conf_and_image_set_matcher_option_checks():
    """KorniaMatcher's keys and defaults; a bad mode raises the plugin's NotImplementedError, an unknown key ValueError, and tile
    preselection needs its LightGlue weights - all before anything is allocated (no context needed)."""
    from dim_b200.sharded import ImageSetMatcher, kornia_conf
    assert kornia_conf({}) == {"match_mode": "smnn", "th": 0.8}
    assert kornia_conf(None) == {"match_mode": "smnn", "th": 0.8}
    assert kornia_conf({"match_mode": "mnn", "th": 1}) == {"match_mode": "mnn", "th": 1.0}
    with pytest.raises(NotImplementedError, match=r"^xnn is not supported\. Try one of \['nn', 'mnn', 'snn', 'smnn'\]$"):
        kornia_conf({"match_mode": "xnn"})
    with pytest.raises(ValueError, match="unknown kornia_matcher option"):
        kornia_conf({"ratio": 0.8})
    sp = {"max_keypoints": 512}
    with pytest.raises(NotImplementedError):
        ImageSetMatcher(None, {}, None, 2, 512, 512, sp, {"match_mode": "xnn"}, matcher="kornia_matcher")
    with pytest.raises(ValueError, match="unknown kornia_matcher option"):
        ImageSetMatcher(None, {}, None, 2, 512, 512, sp, {"filter_threshold": 0.1}, matcher="kornia_matcher")
    with pytest.raises(ValueError, match="preselection_weights"):
        ImageSetMatcher(None, {}, None, 2, 1024, 1024, sp, {}, matcher="kornia_matcher",
                        tiling={"tile_size": 512, "tile_selection": "preselection", "tile_preselection_size": 256})
    with pytest.raises(ValueError, match="matcher must be"):
        ImageSetMatcher(None, {}, None, 2, 512, 512, sp, {}, matcher="kornia")


# ---------------------------------------------------------------------------------------------------------------- on the GPU

def _slot_feats(seed=0, D=256):
    """Eight feature sets sharing noisy views of one pool of descriptors (so that every mode finds matches), float16-exact once
    stored."""
    rng = np.random.default_rng(seed)
    pool = rng.standard_normal((D, 900)).astype(np.float32)
    out = []
    for n in COUNTS:
        d = pool[:, rng.permutation(900)[:n]] + 0.35 * rng.standard_normal((D, n)).astype(np.float32)
        d /= np.maximum(np.linalg.norm(d, axis=0), 1e-6)
        out.append({"keypoints": rng.uniform(0, 500, (n, 2)).astype(np.float32), "descriptors": d.astype(np.float32),
                    "image_size": np.array([512, 512])})
    return out


@pytest.fixture(scope="module")
def nn_store(ctx):
    from dim_b200 import _native
    feats = _slot_feats()
    store = _native.FeatureStoreDev(ctx, len(COUNTS), CAP, 256)
    for s, f in enumerate(feats):
        store.put(s, f)
    return store, feats


def _batch(ctx, f0, f1, mode, th, cap=CAP, D=256, stream=0):
    """One dimb_nn_match_batch_dev call; returns per pair (idx, dist, full count) and the raw [P][cap] buffers."""
    import torch
    P = len(f0)
    idx = torch.full((P, cap, 2), SENT, dtype=torch.int64, device="cuda")
    dist = torch.full((P, cap), float(SENT), device="cuda")
    n = torch.full((P,), SENT, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.nn_match_batch_dev(f0, f1, D, mode, th, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), cap, stream)
    torch.cuda.synchronize()
    idx, dist, n = idx.cpu().numpy(), dist.cpu().numpy(), n.cpu().numpy()
    return [(idx[p, :min(n[p], cap)].copy(), dist[p, :min(n[p], cap)].copy(), int(n[p])) for p in range(P)], (idx, dist)


def _single_dev(ctx, store, s0, s1, mode, th):
    """dimb_nn_match_dev on the two slots with their counts read on the host."""
    import torch
    n0, n1 = (max(store.count(s)[0], 0) for s in (s0, s1))
    a, b = store.feats_dev(s0), store.feats_dev(s1)
    idx = torch.full((CAP, 2), SENT, dtype=torch.int64, device="cuda")
    dist = torch.full((CAP,), float(SENT), device="cuda")
    n = torch.full((1,), SENT, dtype=torch.int32, device="cuda")
    ctx.nn_match_dev(a.descriptors, n0, b.descriptors, n1, 256, mode, th, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), CAP, f16=True,
                     ld0=a.desc_ld, ld1=b.desc_ld)
    torch.cuda.synchronize()
    k = int(n.cpu()[0])
    return idx.cpu().numpy()[:k], dist.cpu().numpy()[:k], k


def _bitwise(a, b):
    ia, da, na = a
    ib, db, nb = b
    assert na == nb and np.array_equal(ia, ib) and np.array_equal(da.view(np.uint32), db.view(np.uint32)), (na, nb)


def _oracle(f0, f1, mode, th):
    """oracle.nn_match's restatement of kornia's modes on the distance matrix of torch.cdist computed in float64 and rounded to
    float32: the reference then does not depend on the accuracy of the host BLAS's float32 matrix product, which torch.cdist uses."""
    import torch
    from oracle import nn_match as o_nn
    d1, d2 = (torch.tensor(np.ascontiguousarray(f["descriptors"].T), dtype=torch.float64) for f in (f0, f1))
    dm = torch.cdist(d1, d2).float() if len(d1) and len(d2) else None
    dist, idx = o_nn.MODES[mode](d1.float(), d2.float(), *((th,) if mode in ("snn", "smnn") else ()), dm=dm)
    return idx.numpy().astype(np.int64).reshape(-1, 2), dist.numpy().astype(np.float32).reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,th", MODES)
def test_batch_equals_single_pair_entry_and_oracle(ctx, nn_store, mode, th):
    """One mixed batch of store pairs (counts 0, 1, 2, 129, 300, 650, 700 and capacity; n0 > n1 and n0 < n1; 129, 300, 650 and 700 end
    inside a 128-column tile): per pair bitwise the single-pair device entry with host-read counts, and the kornia oracle's indices
    (distances within 1e-4)."""
    store, _ = nn_store
    out, _ = _batch(ctx, [store.feats_dev(a) for a, _ in PAIRS], [store.feats_dev(b) for _, b in PAIRS], mode, th)
    for p, (s0, s1) in enumerate(PAIRS):
        _bitwise(out[p], _single_dev(ctx, store, s0, s1, mode, th))
        ridx, rdist = _oracle(store.get(s0), store.get(s1), mode, th)
        assert np.array_equal(out[p][0], ridx), (p, len(out[p][0]), len(ridx))
        if len(rdist):
            assert np.abs(out[p][1] - rdist).max() < 1e-4, p
    assert out[0][2] == 0 and sum(o[2] for o in out) > 100


@pytest.mark.gpu
def test_batch_entry_rejects_bad_arguments(ctx, nn_store):
    """With a real context every bad argument on its own gives DIMB_ERR_ARG (-3) and writes nothing: NULL pair arrays or outputs,
    P < 1, cap < 1, D < 1, a mode outside 0..3, and per side NULL descriptors, a NULL count, n_cap < 0 or desc_layout != 0."""
    import torch
    from dim_b200 import _native
    store, _ = nn_store
    lib = ctx.lib
    idx = torch.full((1, CAP, 2), SENT, dtype=torch.int64, device="cuda")
    dist = torch.full((1, CAP), float(SENT), device="cuda")
    n = torch.full((1,), SENT, dtype=torch.int32, device="cuda")

    def side(**kw):
        f = store.feats_dev(0)
        for k, v in kw.items():
            setattr(f, k, v)
        return (_native.FeatsDev * 1)(f)

    good = side()
    ok = dict(P=1, f0=good, f1=side(), D=256, mode=3, idx=idx.data_ptr(), dist=dist.data_ptr(), n=n.data_ptr(), cap=CAP)

    def call(a):
        return lib.dimb_nn_match_batch_dev(ctx.h, a["P"], a["f0"], a["f1"], a["D"], a["mode"], 0.8, a["idx"], a["dist"], a["n"], a["cap"],
                                           None)
    torch.cuda.synchronize()
    for bad in ({"f0": None}, {"f1": None}, {"idx": None}, {"dist": None}, {"n": None}, {"P": 0}, {"cap": 0}, {"D": 0}, {"mode": 4},
                {"mode": -1}, {"f1": side(descriptors=None)}, {"f0": side(n=None)}, {"f1": side(n_cap=-1)}, {"f0": side(desc_layout=1)}):
        assert call({**ok, **bad}) == -3, bad
    torch.cuda.synchronize()
    assert int(n.cpu()[0]) == SENT and bool((idx == SENT).all()) and bool((dist == SENT).all())
    assert call(ok) == 0  # the same arguments without the fault run
    torch.cuda.synchronize()
    assert int(n.cpu()[0]) > 0


class _F32Side:
    """float32 device copy (D, n_cap) of a feature set's descriptors, NaN past n (never read), with its FeatsDev."""

    def __init__(self, f, round_fp16, pad=5):
        import torch
        from dim_b200 import _native
        d = np.ascontiguousarray(f["descriptors"], np.float32)
        n = d.shape[1]
        self.de = torch.full((d.shape[0], n + pad), float("nan"), device="cuda")
        self.de[:, :n] = torch.from_numpy(d)
        self.cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
        self.f = _native.FeatsDev(None, self.de.data_ptr(), self.cnt.data_ptr(), n + pad, 0, n + pad, 0.0, 0.0, round_fp16, 0, None, None)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_float32_inputs_equal_host_entry(nn_store, precision):
    """Float32 extractor-style inputs: round_fp16 = 0 equals dimb_nn_match on the same arrays (three MMAs in EXACT), round_fp16 = 1
    equals it on the fp16-rounded arrays (one MMA), in both precision modes."""
    from dim_b200 import _native
    c = _native.Context(0, precision=precision)
    _, feats = nn_store
    pairs = [(0, 1), (1, 0), (5, 7), (2, 6), (4, 6)]
    for r16 in (0, 1):
        sides = [(_F32Side(feats[a], r16), _F32Side(feats[b], r16)) for a, b in pairs]
        for mode, th in MODES:
            out, _ = _batch(c, [x.f for x, _ in sides], [y.f for _, y in sides], mode, th)
            for p, (a, b) in enumerate(pairs):
                d0, d1 = feats[a]["descriptors"], feats[b]["descriptors"]
                if r16:
                    d0, d1 = d0.astype(np.float16).astype(np.float32), d1.astype(np.float16).astype(np.float32)
                idx, dist = c.nn_match(d0, d1, mode, th)
                _bitwise(out[p], (idx, dist, len(idx)))


@pytest.mark.gpu
def test_permuted_and_resplit_batches_across_workspace_growth(nn_store):
    """On a fresh context (its scratch grows, then is reused smaller): a two-pair batch, the reversed full batch, then a three-pair
    batch give every pair the outputs of the full batch, in every mode."""
    from dim_b200 import _native
    store, _ = nn_store
    c = _native.Context(0)
    for mode, th in MODES:
        base, _ = _batch(c, [store.feats_dev(a) for a, _ in PAIRS], [store.feats_dev(b) for _, b in PAIRS], mode, th)
        fresh = _native.Context(0)
        for sel in ([5, 1], list(range(len(PAIRS)))[::-1], [2, 7, 0]):
            res, _ = _batch(fresh, [store.feats_dev(PAIRS[k][0]) for k in sel], [store.feats_dev(PAIRS[k][1]) for k in sel], mode, th)
            for j, k in enumerate(sel):
                _bitwise(res[j], base[k])


@pytest.mark.gpu
def test_cap_below_the_count(ctx, nn_store):
    """cap below a pair's match count: d_n holds the full count, the first cap rows are those of the uncapped call, nothing past a
    pair's rows is written."""
    store, _ = nn_store
    sel = [PAIRS[1], PAIRS[3], PAIRS[7]]
    f0, f1 = [store.feats_dev(a) for a, _ in sel], [store.feats_dev(b) for _, b in sel]
    full, _ = _batch(ctx, f0, f1, "nn", 0.0)
    cap = full[0][2] // 3
    assert cap > 10 and full[1][2] < cap
    out, (idx, dist) = _batch(ctx, f0, f1, "nn", 0.0, cap=cap)
    for p in range(len(sel)):
        rows = min(full[p][2], cap)
        assert out[p][2] == full[p][2]
        assert np.array_equal(out[p][0], full[p][0][:rows]) and np.array_equal(out[p][1], full[p][1][:rows])
        assert np.all(idx[p, rows:] == SENT) and np.all(dist[p, rows:] == SENT)


@pytest.mark.gpu
def test_batch_dev_is_asynchronous(ctx, nn_store):
    """Queued behind a ~0.5 s device spin (scratch already grown by a first call), the call returns while the stream is still busy;
    the results are right after a synchronise."""
    import torch
    store, _ = nn_store
    f0, f1 = [store.feats_dev(a) for a, _ in PAIRS], [store.feats_dev(b) for _, b in PAIRS]
    base, _ = _batch(ctx, f0, f1, "smnn", 0.95)
    P = len(PAIRS)
    idx = torch.full((P, CAP, 2), SENT, dtype=torch.int64, device="cuda")
    dist = torch.full((P, CAP), float(SENT), device="cuda")
    n = torch.full((P,), SENT, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000_000)
    ctx.nn_match_batch_dev(f0, f1, 256, "smnn", 0.95, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), CAP, s.cuda_stream)
    busy = not s.query()
    s.synchronize()
    idx, dist, n = idx.cpu().numpy(), dist.cpu().numpy(), n.cpu().numpy()
    assert busy
    for p in range(P):
        _bitwise((idx[p, :n[p]], dist[p, :n[p]], int(n[p])), base[p])


# ---------------------------------------------------------------------------------------------------------------- ImageSetMatcher

def _plugin(mode, th):
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    return KorniaMatcher(Config(matcher={"name": "kornia_matcher", "match_mode": mode, "th": th}))


@pytest.mark.gpu
def test_image_set_matcher_superpoint_untiled(ctx, sp_weights):
    """5 synthetic images, all 10 pairs, smnn (the plugin's defaults) and mnn in batches of 4 and 3: every table equals
    KorniaMatcher._match_pairs on the store's features."""
    import torch
    from dim_b200 import synthetic
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot
    size = 320
    a, b = synthetic.synthetic_pair(11, size)
    c, d = synthetic.synthetic_pair(12, size)
    imgs = torch.from_numpy(np.stack([a, b, c, d, synthetic.synthetic_pair(13, size)[0]]).astype(np.float32)).cuda()
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 512}
    pairs = pairs_from_bruteforce(list(range(5)))
    for conf, bp in (({}, 4), ({"match_mode": "mnn"}, 3)):
        eng = ImageSetMatcher(ctx, sp_weights, None, 5, size, size, sp_conf, conf, batch_images=3, batch_pairs=bp, matcher="kornia_matcher")
        tables = eng.run(imgs, list(range(5)), pairs)
        plugin = _plugin(eng.nn_conf["match_mode"], eng.nn_conf["th"])
        for (i, j), t in zip(pairs, tables):
            exp = plugin._match_pairs(eng.store.get(store_slot(i, 5, 1)), eng.store.get(store_slot(j, 5, 1)))
            assert t.dtype == np.int64 and np.array_equal(t, exp), (conf, i, j, len(t), len(exp))
        assert len(tables[0]) > 20, len(tables[0])


@pytest.mark.gpu
def test_image_set_matcher_aliked_untiled(ctx, al_weights):
    """ALIKED (128-d) without tiling, 3 RGB images, all pairs: every table equals the plugin's on the store's features."""
    import torch
    from dim_b200 import synthetic
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    a = synthetic.blocks_image(301, 512)[:384]
    imgs = np.stack([a] + [synthetic.warp_pair(a, 50 + k, jitter=24.0) for k in (1, 2)]).astype(np.float32)
    al_conf = {"max_num_keypoints": 1024, "detection_threshold": 0.2, "nms_radius": 3}
    pairs = pairs_from_bruteforce([0, 1, 2])
    eng = ImageSetMatcher(ctx, al_weights, None, 3, 384, 512, al_conf, {"match_mode": "smnn", "th": 0.9}, batch_images=2, batch_pairs=2,
                          extractor="aliked", matcher="kornia_matcher")
    tables = eng.run(torch.from_numpy(imgs).cuda(), [0, 1, 2], pairs)
    plugin = _plugin("smnn", 0.9)
    for (i, j), t in zip(pairs, tables):
        assert np.array_equal(t, plugin._match_pairs(eng.store.get(i), eng.store.get(j))), (i, j)
    assert sum(len(t) for t in tables) > 20


def _gray_set(n, H, W):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(40, max(H, W))[:H, :W]
    imgs = [a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in range(1, n)]
    return np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in imgs]).astype(np.float32)


@pytest.mark.gpu
def test_image_set_matcher_tiled_and_verified(ctx, sp_weights):
    """Tiled grid and exhaustive selections: the tables equal KorniaMatcher._match_by_tile on the merged slots; run_verified's raw
    tables are those tables and its verified results equal dimb_gv_verify_dev run on them."""
    import torch
    from dim_b200.geometric_verification import gv_seed
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, tile_pairs_for
    imgs = torch.from_numpy(_gray_set(3, 512, 640)).cuda()
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 512}
    pairs = pairs_from_bruteforce([0, 1, 2])
    plugin = _plugin("smnn", 0.8)
    for sel in ("grid", "exhaustive"):
        eng = ImageSetMatcher(ctx, sp_weights, None, 3, 512, 640, sp_conf, {}, batch_pairs=16, matcher="kornia_matcher",
                              tiling={"tile_size": 384, "tile_overlap": 32, "tile_selection": sel}, verification={"seed": 3})
        tables = eng.run(imgs, [0, 1, 2], pairs)
        for (i, j), t in zip(pairs, tables):
            exp = plugin._match_by_tile(eng.store.get(i), eng.store.get(j), tile_pairs_for(sel, eng.T))
            assert np.array_equal(t, exp), (sel, i, j, len(t), len(exp))
        assert min(len(t) for t in tables) > 0
    res = eng.run_verified(imgs, [0, 1, 2], pairs)
    P, cap = len(pairs), max(len(t) for t in tables)
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
