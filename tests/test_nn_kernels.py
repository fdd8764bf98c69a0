"""The brute-force NN engine (csrc/nn_kernels.cuh) on its own, against a float64 reference of kornia's matcher.

tests/test_nn_sets.py and test_gpu_parity.py compare the engine with the kornia oracle on random unit descriptors, which almost never
tie.  The descriptors this matcher gets from ORB (D = 32 bytes) and SIFT (D = 128, integral values) are integers stored in fp16: every
squared distance is then an exact integer on the device, equal distances are common, and the device owes kornia's answer bitwise.
Here the self-test library runs the engine's pieces (dimb_selftest_nn_stats: prep, top-2 GEMM and merge of both directions on either
engine; dimb_selftest_nn_select: the mode logic on planted row statistics), with outputs that start as a sentinel and are followed by
a tail, and the product entries run end to end.

The reference (ref_stats) works in float64: the exact squared distance s, the float32 distance f = float32(sqrt(s)) (correctly
rounded), best = the first index among the smallest f (torch.min's rule), second = the second-smallest f counting ties; ref_tables
puts kornia's nn / mnn / snn / smnn logic on top.  On the CPU it is pinned to oracle/nn_match.py and to torch.cdist + torch.min.

Exactness classes:
  integer  integer values with |a|^2 + |b|^2 < 2^24 for every pair: the norms, the fp16 products, their fp32 sums and a2 + |b|^2 are
           exact, so d1, d2, i1 and the match tables equal the reference bitwise.
  float    compared in the squared domain against bar(a, b) = c * (|a|^2 + |b|^2) + 2^-23 sqrt(Dp) (|a| + |b|); see bar_coeff.
"""
import ctypes as C

import numpy as np
import pytest

SENT = -777.0
ISENT = int(np.float32(SENT).view(np.int32))
ERR_ARG = -3
NUM_SMS = 132  # SMs of an H100 SXM: the CPU test of the plans asks gemm_plan for the card this engine runs on
MODES = ["nn", "mnn", "snn", "smnn"]


# ------------------------------------------------------------------ references
def ref_stats(A, B):
    """A (n0, D), B (n1, D) float64 (the values the device reads) -> dict: s (n0, n1) squared distances (exact for integer inputs),
    f float32 distances, d1 / d2 float32, i1 int (first index among the smallest f).  check_float_stats takes the margins of its
    decisions from s."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    s = (A * A).sum(1)[:, None] + (B * B).sum(1)[None, :] - 2.0 * (A @ B.T)
    f = np.sqrt(np.maximum(s, 0.0)).astype(np.float32)
    n0, n1 = s.shape
    i1 = np.argmin(f, axis=1) if n1 else np.zeros(n0, np.int64)
    r = np.arange(n0)
    d1 = f[r, i1] if n1 else np.full(n0, np.inf, np.float32)
    fm = f.copy()
    if n1:
        fm[r, i1] = np.inf
    d2 = fm.min(1) if n1 else np.full(n0, np.inf, np.float32)
    return {"s": s, "f": f, "d1": d1.astype(np.float32), "d2": d2.astype(np.float32), "i1": i1.astype(np.int64)}


def ref_tables(fw, bw, n0, n1, mode, th):
    """kornia's DescriptorMatcher(mode, th) on the row statistics of both directions -> (idx (S, 2) int64, dist (S,) float32)."""
    empty = np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    if n0 == 0 or n1 == 0 or (mode == "snn" and n1 < 2) or (mode == "smnn" and (n0 < 2 or n1 < 2)):
        return empty
    th32 = np.float32(th)
    with np.errstate(invalid="ignore", divide="ignore"):
        rf = fw["d1"] / fw["d2"]
        rb = bw["d1"] / bw["d2"]
    i = np.arange(n0)
    if mode == "nn":
        return np.stack([i, fw["i1"]], 1), fw["d1"].copy()
    if mode == "mnn":
        if n0 <= n1:
            keep = bw["i1"][fw["i1"]] == i
            return np.stack([i, fw["i1"]], 1)[keep], fw["d1"][keep]
        j = np.arange(n1)
        keep = fw["i1"][bw["i1"]] == j
        return np.stack([bw["i1"], j], 1)[keep], bw["d1"][keep]
    if mode == "snn":
        keep = rf <= th32
        return np.stack([i, fw["i1"]], 1)[keep], rf[keep].astype(np.float32)
    j = fw["i1"]
    keep = (rf <= th32) & (rb[j] <= th32) & (bw["i1"][j] == i)
    return np.stack([i, j], 1)[keep], np.maximum(rf, rb[j])[keep].astype(np.float32)


def bar_coeff(D, kind):
    """c of bar(a, b) = c (|a|^2 + |b|^2) + 2^-23 sqrt(Dp) (|a| + |b|) for the squared distance the device forms from float inputs,
    kind: 'split' (fp32 inputs, three MMAs), 'fast' (fp32 inputs, one MMA on the fp16 hi planes), 'f16' (fp16 inputs, one MMA).

    The device forms s = fma(-2, dot, a2 + b2).  |a.b| <= sum |a_k b_k| <= (|a|^2 + |b|^2) / 2 =: N / 2.
      dot: the fp16 x fp16 products are exact in fp32; the tensor cores add them into an fp32 accumulator that may truncate, so every
           addition can lose 2^-23 of the running sum, which never exceeds sum |a_k b_k|: m Dp 2^-23 N / 2 for the 2 dot, with m = 1
           MMA per product, or 3 for the split (hi hi + hi lo + lo hi).  The split drops lo lo and rounds lo to fp16 (2^-22 relative,
           or 2^-25 absolute where lo is subnormal): 2^-21 N plus the additive 2^-23 sqrt(Dp) (|a| + |b|) term.
      fast: the dot comes from hi = fp16(x) alone: each factor is off by 2^-11 relative (or 2^-25 absolute where subnormal), each
           product by 2^-10: 2^-10 N for the 2 dot, while the norms come from the fp32 values.
      norms: D fp32 squares (2^-24 each), summed in 32-wide shuffle trees (5 levels) and then over Dp / 32 chunks: (Dp / 32 + 7) 2^-24 N.
      a2 + b2 and the fma: 2^-24 N and 2^-24 |s| <= 2^-23 N.
      sqrt: the device reports d = float32(sqrt(s)), and the test squares it: 2^-22 |s| <= 2^-21 N."""
    Dp = -(-D // 64) * 64
    m = 3 if kind == "split" else 1
    c = m * Dp * 2.0 ** -23 + (Dp / 32 + 7) * 2.0 ** -24 + 2.0 ** -24 + 2.0 ** -23 + 2.0 ** -21
    if kind == "split":
        c += 2.0 ** -21
    if kind == "fast":
        c += 2.0 ** -10
    return c


def bars(A, B, kind):
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    D = A.shape[1]
    na, nb = (A * A).sum(1), (B * B).sum(1)
    return bar_coeff(D, kind) * (na[:, None] + nb[None, :]) + 2.0 ** -23 * np.sqrt(-(-D // 64) * 64) * (
        np.sqrt(na)[:, None] + np.sqrt(nb)[None, :])


def check_float_stats(ref, d1, d2, i1, bar, what):
    """d1 / d2 / i1 of the device (one direction, live rows) against the float64 reference within bar [n0][n1]: i1 may name another
    column only when its squared distance is within the bars of the best's; d1^2 is within the bar of the s of i1, d2^2 between the
    smallest s - bar and s + bar of the other columns.  Returns the worst |d1^2 - s| as a share of its bar."""
    s = ref["s"]
    n0 = s.shape[0]
    r = np.arange(n0)
    assert np.all((i1 >= 0) & (i1 < s.shape[1])), what
    hi_all = (s + bar).min(1)
    assert np.all(s[r, i1] - bar[r, i1] <= hi_all), (what, np.nonzero(s[r, i1] - bar[r, i1] > hi_all)[0][:5])
    e1 = np.abs(d1.astype(np.float64) ** 2 - np.maximum(s[r, i1], 0))
    share = e1 / bar[r, i1]
    assert np.all(share <= 1.0), (what, share.max(), np.argmax(share))
    if s.shape[1] > 1:
        so, bo = s.copy(), bar.copy()
        so[r, i1] = np.inf
        lo2, hi2 = (so - bo).min(1), (so + bo).min(1)
        q = d2.astype(np.float64) ** 2
        assert np.all((q >= lo2) & (q <= hi2)), (what, np.nonzero((q < lo2) | (q > hi2))[0][:5])
    return float(share.max(initial=0.0))


# ------------------------------------------------------------------ data
def bytes_desc(rng, D, n, hi=256):
    return rng.integers(0, hi, (n, D)).astype(np.float64)


def sum_of_squares(target, D):
    """D byte values whose squares add up to target (greedy with a four-square tail)."""
    v = []
    rest = target
    while rest > 0 and len(v) < D - 4:
        x = min(255, int(np.sqrt(rest)))
        if rest - x * x < 0:
            x -= 1
        # keep a remainder that four squares can reach
        v.append(x)
        rest -= x * x
    for a in range(int(np.sqrt(rest)) + 1):
        for b in range(a + 1):
            for c in range(b + 1):
                d2 = rest - a * a - b * b - c * c
                if d2 >= 0 and int(np.sqrt(d2)) ** 2 == d2:
                    v += [a, b, c, int(np.sqrt(d2))]
                    out = np.zeros(D)
                    out[:len(v)] = v
                    assert int((out * out).sum()) == target
                    return out
    raise AssertionError(target)


def planted_ties(rng, D=32, n0=300, n1=2200):
    """Byte descriptors with exact ties planted at every place the engine decides one: a duplicate of the best in the same 32-column
    chunk, in another chunk of the same 128-column tile, in another tile, in another merge lane and in the same lane one loop step
    later (columns j and j + 1024), with the duplicate before or after the original; ties for second place; triple ties; duplicate
    query rows (ties in the backward direction, so that mnn fails mutuality as kornia does); and queries equal to two candidates (d1 =
    d2 = 0).  Returns A (n0, D), B (n1, D)."""
    B = bytes_desc(rng, D, n1)
    A = bytes_desc(rng, D, n0)
    offs = [1, 5, 31, 32, 40, 96, 127, 128, 300, 1023, 1024, 1056, 2048 - 64]
    q = 0
    for o in [o for o in offs if o < n1]:
        for before in (False, True):
            j = int(rng.integers(0, n1 - o))
            a, b = (j + o, j) if before else (j, j + o)
            B[b] = B[a]
            A[q] = np.clip(B[a] + rng.integers(-2, 3, D), 0, 255)
            q += 1
    for _ in range(12):  # tie for second: a near copy of one column, two equal columns a little further
        j, k, m = rng.choice(n1, 3, replace=False)
        A[q] = B[j]
        B[k] = np.clip(B[j] + np.eye(D)[0] * 3, 0, 255) if B[j][0] < 250 else np.clip(B[j] - np.eye(D)[0] * 3, 0, 255)
        B[m] = B[k]
        q += 1
    for _ in range(8):  # triple tie for the best
        j, k, m = rng.choice(n1, 3, replace=False)
        B[k] = B[j]
        B[m] = B[j]
        A[q] = np.clip(B[j] + rng.integers(-1, 2, D), 0, 255)
        q += 1
    for _ in range(10):  # a query equal to two candidates
        j, k = rng.choice(n1, 2, replace=False)
        B[k] = B[j]
        A[q] = B[j]
        q += 1
    for _ in range(10):  # duplicate query rows: a backward tie
        A[q] = A[q - 30]
        q += 1
    for _ in range(10):  # the same pattern near the end of the rows (last tile)
        A[n0 - 1 - _] = A[_]
    return A, B


# ------------------------------------------------------------------ CPU: the reference against kornia's restatement and torch
def test_reference_matches_oracle_and_torch_without_ties():
    """On random float data (no ties), ref_stats equals torch.cdist + torch.min / topk values and ref_tables the oracle's tables."""
    import torch
    from oracle import nn_match as O
    rng = np.random.default_rng(0)
    for D, n0, n1 in [(128, 150, 220), (256, 90, 60), (3, 40, 41)]:
        A = rng.standard_normal((n0, D)).astype(np.float32).astype(np.float64)
        B = rng.standard_normal((n1, D)).astype(np.float32).astype(np.float64)
        fw, bw = ref_stats(A, B), ref_stats(B, A)
        dm = torch.cdist(torch.tensor(A), torch.tensor(B))  # float64
        v, i = torch.min(dm, 1)
        assert np.array_equal(i.numpy(), fw["i1"])
        assert np.allclose(v.numpy(), fw["d1"], rtol=1e-6)
        vals, _ = torch.topk(dm, 2, 1, largest=False)
        assert np.allclose(vals[:, 1].numpy(), fw["d2"], rtol=1e-6)
        for mode, th in [("nn", 0), ("mnn", 0), ("snn", 0.95), ("smnn", 0.98)]:
            idx, dist = ref_tables(fw, bw, n0, n1, mode, th)
            oi, od = O.kornia_match({"descriptors": A.T}, {"descriptors": B.T}, mode, th)
            assert np.array_equal(idx, oi), (D, mode)
            assert np.allclose(dist, od, rtol=1e-5), (D, mode)


def test_reference_matches_oracle_on_planted_ties():
    """On byte descriptors with planted ties the float32 squared distances torch forms are exact.  torch's CPU float32 sqrt (in
    torch.sqrt and torch.cdist) is not correctly rounded: it is within one ulp of ref_stats' distances, which are (the device's sqrtf
    is IEEE).  On those distances torch.min gives ref_stats' best bitwise (the first index), and kornia's mode logic (oracle/nn_match.py
    given the distance matrix) gives ref_tables' tables bitwise: nn and mnn everywhere, snn / smnn at th < 1, where a tied best (ratio
    1) is rejected.  torch.topk does not return the first index among ties: only its values are compared."""
    import torch
    from oracle import nn_match as O
    rng = np.random.default_rng(1)
    n0, n1 = 200, 1500
    A, B = planted_ties(rng, 32, n0, n1)
    fw, bw = ref_stats(A, B), ref_stats(B, A)
    a, b = torch.tensor(A, dtype=torch.float32), torch.tensor(B, dtype=torch.float32)
    s = (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.T
    assert np.array_equal(s.numpy().astype(np.float64), fw["s"])
    for t in (torch.sqrt(s), torch.cdist(a, b)):
        assert np.abs(t.numpy().view(np.int32).astype(np.int64) - fw["f"].view(np.int32)).max() <= 1
    assert np.array_equal(torch.sqrt(s.double()).float().numpy(), fw["f"])
    dm = torch.from_numpy(fw["f"])
    v, i = torch.min(dm, 1)
    assert np.array_equal(i.numpy(), fw["i1"]) and np.array_equal(v.numpy(), fw["d1"])
    vals, _ = torch.topk(dm, 2, 1, largest=False)
    assert np.array_equal(vals[:, 1].numpy(), fw["d2"])
    assert np.sum(fw["d1"] == fw["d2"]) >= 30
    for mode, th in [("nn", 0), ("mnn", 0), ("snn", 0.9), ("smnn", 0.95)]:
        idx, dist = ref_tables(fw, bw, n0, n1, mode, th)
        args = (th,) if mode in ("snn", "smnn") else ()
        od, oi = O.MODES[mode](a, b, *args, dm=dm)
        assert np.array_equal(idx, oi.numpy()) and np.array_equal(dist, od.numpy().reshape(-1)), mode
    for mode in ("mnn",):  # n0 > n1: mnn's swapped order
        od, oi = O.MODES[mode](b[:150], a, dm=dm.t()[:150])
        idx, dist = ref_tables(ref_stats(B[:150], A), ref_stats(A, B[:150]), 150, n0, mode, 0)
        assert np.array_equal(idx, oi.numpy()) and np.array_equal(dist, od.numpy().reshape(-1))
    # torch.topk's index at a tie is not kornia's first index: [3, 7] for a tie over {3, 5, 7} on the CPU
    t = torch.tensor([[9.0, 9, 9, 1, 9, 1, 9, 1]])
    assert torch.min(t, 1).indices.item() == 3 and torch.topk(t, 2, 1, largest=False).values.tolist() == [[1.0, 1.0]]


def test_sqrt_collision_vectors():
    """The byte vectors of the collision cases: squared distances 4197200 and 4197201 from the zero query, equal float32 distances."""
    a, b = sum_of_squares(4197201, 128), sum_of_squares(4197200, 128)
    assert np.float32(np.sqrt(4197200.0)) == np.float32(np.sqrt(4197201.0))
    assert a.max() <= 255 and b.max() <= 255
    # the first colliding pair of integers: below 2^22 distinct integers keep distinct float32 square roots
    r = np.sqrt(np.arange(4190000, 4197202, dtype=np.float64)).astype(np.float32)
    assert np.nonzero(r[1:] == r[:-1])[0][0] + 4190000 == 4197200


def test_bar_cases_reach_both_gemm_plans():
    """The host-count cases of test_stats_integer_shapes reach both the resident-B and the streamed-B plans of the top-2 GEMM on an
    H100 SXM (132 SMs).  This is shape coverage: the tiles come from the counts as the host-count engine forms them, and gemm_plan is
    the plan rule the launch applies; the plan is not read back from a launch."""
    from dim_b200 import _native
    resb = set()
    for D, n0, n1 in SHAPE_CASES:
        for split in (0, 1):
            Dp = -(-D // 64) * 64
            resb.add(_native.gemm_plan(0, 128, split, True, Dp // 64, -(-n0 // 128), -(-n1 // 128), NUM_SMS)[0])
    assert resb == {0, 1}


def test_selftest_entries_reject_bad_arguments_without_touching_the_gpu():
    """DIMB_ERR_ARG for a NULL context before any CUDA call."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    null = C.c_void_p()
    f = (_native.FeatsDev * 1)()
    buf = np.zeros(16, np.float32)
    p = _native._ptr(buf)
    assert lib.dimb_selftest_nn_stats(null, 1, f, f, 32, 0, 0, 1, 128, 0.0, p, p, p, p, p) == ERR_ARG
    assert lib.dimb_selftest_nn_select(null, 0, 0.8, 1, 128, p, p, p, p, 8, 0.0, p, p, p) == ERR_ARG


# ------------------------------------------------------------------ GPU helpers
D_LIST = [1, 3, 32, 63, 64, 65, 128, 129, 256, 320]
SHAPE_CASES = [(D, 33, 129) for D in D_LIST] + [(D, 129, 33) for D in D_LIST] + [
    (32, 1, 2), (32, 2, 1), (32, 31, 32), (32, 32, 33), (32, 33, 31), (32, 127, 128), (32, 128, 129), (32, 129, 127),
    (32, 1023, 1025), (32, 1024, 1024), (32, 1025, 1023), (32, 4100, 1025), (32, 1025, 4100), (128, 4100, 4100), (320, 1025, 4100),
    (256, 2048, 2048), (320, 300, 300)]


class Sides:
    """Device sides (FeatsDev) of descriptors given as (n, D) arrays; the tensors stay alive with the object."""

    def __init__(self):
        self.keep = []

    def side(self, X, kind="f16", ld=None, n=None, n_cap=None):
        """kind 'f16' (fp16 array), 'f32', or 'round' (fp32 array with round_fp16).  Columns past the rows hold NaN.  n: the device
        count (default the rows); n_cap: the capacity (default the rows)."""
        import torch
        from dim_b200 import _native
        X = np.asarray(X)
        m, D = X.shape
        ld = ld or max(m, 1)
        dt = torch.float16 if kind == "f16" else torch.float32
        buf = torch.full((D, ld), float("nan"), dtype=dt, device="cuda")
        if m:
            buf[:, :m] = torch.from_numpy(np.ascontiguousarray(X.T.astype(np.float32))).to("cuda", dt)
        cnt = torch.tensor([m if n is None else n], dtype=torch.int32, device="cuda")
        self.keep += [buf, cnt]
        f = _native.FeatsDev()
        f.descriptors, f.n, f.n_cap, f.desc_layout, f.desc_ld = buf.data_ptr(), cnt.data_ptr(), m if n_cap is None else n_cap, 0, ld
        f.f16, f.round_fp16 = int(kind == "f16"), int(kind == "round")
        return f


def seen(X, kind):
    """The values the device reads from X under kind."""
    X = np.asarray(X, np.float32)
    return (X.astype(np.float16) if kind in ("f16", "round") else X).astype(np.float64)


@pytest.fixture(scope="module")
def st():
    from dim_b200 import _native
    return _native.SelfTest(0)


def stats(st, A, B, kind="f16", split=0, host=True, mode="nn", **kw):
    sd = Sides()
    return st.nn_stats([sd.side(A, kind, **kw)], [sd.side(B, kind)], A.shape[1], mode, split, host)


def check_untouched(res, n_live, what):
    """Rows past each side's live count and the tails keep the sentinel."""
    for s, n in enumerate(n_live):
        for k in ("d1", "d2"):
            assert np.all(res[k][s, n:] == np.float32(SENT)), (what, k, s)
        assert np.all(res["i1"][s, n:] == ISENT), (what, s)
    for k in ("d1", "d2"):
        assert np.all(res[k + "_tail"] == np.float32(SENT)), what
    assert np.all(res["i1_tail"] == ISENT) and np.all(res["n_live_tail"] == ISENT), what


def check_exact(res, A, B, what, p=0, refs=None):
    """Both directions of pair p bitwise equal to the float64 reference (refs: precomputed (forward, backward)); returns them."""
    fw, bw = refs or (ref_stats(A, B), ref_stats(B, A))
    n0, n1 = len(A), len(B)
    for s, r, n in ((2 * p, fw, n0), (2 * p + 1, bw, n1)):
        assert res["n_live"][s] == n, (what, s)
        assert np.array_equal(res["d1"][s, :n].view(np.int32), r["d1"].view(np.int32)), (what, s, "d1")
        assert np.array_equal(res["d2"][s, :n].view(np.int32), r["d2"].view(np.int32)), (what, s, "d2")
        bad = np.nonzero(res["i1"][s, :n] != r["i1"])[0]
        assert len(bad) == 0, (what, s, "i1", bad[:5], res["i1"][s, bad[:5]], r["i1"][bad[:5]])
    return fw, bw


# ------------------------------------------------------------------ GPU: row statistics
@pytest.mark.gpu
@pytest.mark.parametrize("D,n0,n1", SHAPE_CASES)
def test_stats_integer_shapes(st, D, n0, n1):
    """Integer descriptors (bytes up to D = 128, 0..15 above, so |a|^2 + |b|^2 < 2^24) with planted duplicates: d1, d2, i1 of both
    directions bitwise equal to the reference on both engines and with one and three MMAs; rows past the counts and the tails
    untouched.  The entry's plan (computed with gemm_plan from the engine's NNShape, not read back from the launch) agrees with
    gemm_plan on tiles derived here from the counts and the device's SM count: shape coverage, not an observation of the launch."""
    from dim_b200 import _native
    rng = np.random.default_rng(D * 7919 + n0 * 31 + n1)
    hi = 256 if D <= 128 else 16
    A, B = bytes_desc(rng, D, n0, hi), bytes_desc(rng, D, n1, hi)
    if n1 > 2:  # a few exact duplicates of columns, and queries on them
        for _ in range(min(n0, 8)):
            j, k = rng.choice(n1, 2, replace=False)
            B[max(j, k)] = B[min(j, k)]
            A[rng.integers(n0)] = B[j]
    out, refs = None, (ref_stats(A, B), ref_stats(B, A))
    for host in (True, False):
        for split in (0, 1):
            res = stats(st, A, B, "f16", split, host)
            what = (D, n0, n1, host, split)
            check_exact(res, A, B, what, refs=refs)
            check_untouched(res, [n0, n1], what)
            if host:
                Dp = -(-D // 64) * 64
                for d, (m, n) in enumerate(((n0, n1), (n1, n0))):
                    exp = _native.gemm_plan(0, 128, split, True, Dp // 64, -(-m // 128), -(-n // 128), device_sms())
                    assert tuple(res["plan"][d]) == exp
            if out is not None:
                for k in ("d1", "d2", "i1"):
                    assert np.array_equal(res[k], out[k]), (what, k)
            out = res


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_stats_planted_ties(st):
    """Exact ties at every place the engine decides one (planted_ties), with more than 1024 partners so that a merge lane loops over
    several chunks: bitwise equal to the reference in both directions on both engines."""
    rng = np.random.default_rng(5)
    for D, n0, n1 in [(32, 300, 2200), (128, 250, 1100)]:
        A, B = planted_ties(rng, D, n0, n1)
        for host in (True, False):
            res = stats(st, A, B, "f16", 0, host)
            fw, _ = check_exact(res, A, B, (D, host))
            check_untouched(res, [n0, n1], (D, host))
        assert np.sum(fw["d1"] == fw["d2"]) >= 30


@pytest.mark.gpu
@pytest.mark.parametrize("split", [0, 1])
def test_stats_sqrt_collision(st, split):
    """Squared distances 4197201 (earlier column) and 4197200 (later column) share one float32 distance, so kornia's best is the
    earlier column; placed in one 32-column chunk, in two chunks of a tile, and in two tiles.  Every other column is farther."""
    far, near = sum_of_squares(4197201, 128), sum_of_squares(4197200, 128)
    n1 = 300
    B = np.full((n1, 128), 255.0)
    A = np.zeros((4, 128))
    places = [(5, 6), (6, 40), (3, 200)]
    for q, (j, k) in enumerate(places):
        Bq = B.copy()
        Bq[j], Bq[k] = far, near
        res = stats(st, A[:1], Bq, "f16", split, True)
        fw = ref_stats(A[:1], Bq)
        assert fw["i1"][0] == j
        assert res["i1"][0, 0] == j, (places[q], int(res["i1"][0, 0]))
        assert res["d1"][0, 0] == fw["d1"][0] and res["d2"][0, 0] == fw["d2"][0]
    # the later column first in the row order, and both inside one chunk of the second tile
    B[130], B[131] = far, near
    res = stats(st, A, B, "f16", split, False)
    check_exact(res, A, B, "collision batch")


@pytest.mark.gpu
def test_nn_match_dev_sqrt_collision(ctx):
    """The product entry on the collision case: kornia's nn table keeps the earlier column."""
    import torch
    far, near = sum_of_squares(4197201, 128), sum_of_squares(4197200, 128)
    B = np.full((64, 128), 255.0)
    B[10], B[11] = far, near
    A = np.zeros((1, 128))
    d0 = torch.from_numpy(A.T.astype(np.float16).copy()).cuda()
    d1 = torch.from_numpy(B.T.astype(np.float16).copy()).cuda()
    idx = torch.full((4, 2), -1, dtype=torch.int64, device="cuda")
    dist = torch.zeros(4, device="cuda")
    n = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.nn_match_dev(d0.data_ptr(), 1, d1.data_ptr(), 64, 128, "nn", 0.0, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), 4, f16=True)
    torch.cuda.synchronize()
    assert n.item() == 1 and idx[0].tolist() == [0, 10], idx[0].tolist()
    assert dist[0].item() == float(np.float32(np.sqrt(4197201.0)))


FLOAT_CASES = {
    "superpoint_unit256": lambda rng: _unit(rng, 256, 700, 900),
    "aliked_unit128": lambda rng: _unit(rng, 128, 900, 500),
    "unnormalised_1e3": lambda rng: tuple(x * 1e3 for x in _unit(rng, 128, 400, 600)),
    "near_duplicates_1e-3": lambda rng: _near(rng, 256, 500, 700),
}


def _unit(rng, D, n0, n1):
    pool = rng.standard_normal((max(n0, n1), D))
    A = pool[rng.permutation(len(pool))[:n0]] + 0.4 * rng.standard_normal((n0, D))
    B = pool[rng.permutation(len(pool))[:n1]] + 0.4 * rng.standard_normal((n1, D))
    return [X / np.linalg.norm(X, axis=1, keepdims=True) for X in (A, B)]


def _near(rng, D, n0, n1):
    B = rng.standard_normal((n1, D))
    B /= np.linalg.norm(B, axis=1, keepdims=True)
    A = B[rng.integers(0, n1, n0)] + 1e-3 * rng.standard_normal((n0, D))
    return A, B


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FLOAT_CASES))
def test_stats_float_within_bars(st, case):
    """Float descriptors as fp32 with three MMAs (EXACT) and one (FAST), and as fp16 with one MMA: d1, d2, i1 of both directions within
    the bars of bar_coeff; both engines bitwise equal.  Prints the worst |d1^2 - s| of each class as a share of its bar."""
    rng = np.random.default_rng(list(FLOAT_CASES).index(case) + 100)
    A, B = FLOAT_CASES[case](rng)
    for kind, split, cls in (("f32", 1, "split"), ("f32", 0, "fast"), ("f16", 0, "f16")):
        As, Bs = seen(A, kind), seen(B, kind)
        res = stats(st, A, B, kind, split, True)
        other = stats(st, A, B, kind, split, False)
        for k in ("d1", "d2", "i1"):
            assert np.array_equal(res[k], other[k]), (case, cls, k)
        check_untouched(res, [len(A), len(B)], (case, cls))
        worst = 0.0
        for s, (X, Y) in enumerate(((As, Bs), (Bs, As))):
            n = len(X)
            worst = max(worst, check_float_stats(ref_stats(X, Y), res["d1"][s, :n], res["d2"][s, :n], res["i1"][s, :n], bars(X, Y, cls),
                                                 (case, cls, s)))
        print(f"\n{case} {cls}: worst |d1^2 - s| / bar = {worst:.3g}")


# ------------------------------------------------------------------ GPU: batch bookkeeping
@pytest.mark.gpu
def test_stats_batch_bookkeeping(st):
    """P = 40 pairs of mixed counts on the device-count engine, each equal to its own single-pair call; a device count above n_cap is
    clamped, a negative one is 0; n = 1 under snn / smnn and an empty partner leave the pair empty; nothing is written past a side's
    live rows."""
    rng = np.random.default_rng(11)
    counts = [0, 1, 2, 31, 32, 33, 127, 128, 129, 300, 1023, 1024, 1025, 700]
    pairs = [(int(rng.choice(counts)), int(rng.choice(counts))) for _ in range(40)]
    pairs[:4] = [(0, 50), (50, 0), (1, 40), (40, 1)]
    data = [(bytes_desc(rng, 32, a), bytes_desc(rng, 32, b)) for a, b in pairs]
    for mode in MODES:
        sd = Sides()
        f0 = [sd.side(A, "f16") for A, _ in data]
        f1 = [sd.side(B, "f16") for _, B in data]
        # pair 4: a count above its capacity (clamped); pair 5: a negative count (0)
        f0[4] = sd.side(data[4][0], "f16", n=len(data[4][0]) + 500)
        f1[5] = sd.side(data[5][1], "f16", n=-3)
        res = st.nn_stats(f0, f1, 32, mode, 0, False)
        live = []
        for p, (A, B) in enumerate(data):
            n0, n1 = len(A), (0 if p == 5 else len(B))
            empty = n0 == 0 or n1 == 0 or (mode == "snn" and n1 < 2) or (mode == "smnn" and (n0 < 2 or n1 < 2))
            live += [0, 0] if empty else [n0, n1]
            assert res["n_live"][2 * p] == live[-2] and res["n_live"][2 * p + 1] == live[-1], (mode, p)
            if not empty:
                check_exact(res, A, B[:n1], (mode, p), p)
                one = stats(st, A, B, "f16", 0, False, mode)
                for k in ("d1", "d2", "i1"):
                    assert np.array_equal(res[k][2 * p, :n0], one[k][0, :n0]) and np.array_equal(res[k][2 * p + 1, :n1], one[k][1, :n1])
        check_untouched(res, live, mode)


# ------------------------------------------------------------------ GPU: select on planted statistics
def _select_case(st, mode, th, fw, bw, cap=None):
    """fw / bw: (d1, d2, i1) of one pair's directions -> the kernel's table and count; also checks against ref_tables."""
    n0, n1 = len(fw[0]), len(bw[0])
    NPp = max(n0, n1, 1)
    d1, d2 = np.full((2, NPp), np.nan, np.float32), np.full((2, NPp), np.nan, np.float32)
    i1 = np.zeros((2, NPp), np.int32)
    for s, (a, b, c) in enumerate((fw, bw)):
        d1[s, :len(a)], d2[s, :len(a)], i1[s, :len(a)] = a, b, c
    cap = cap or max(n0, 1)
    out = st.nn_select(mode, th, [n0, n1], d1, d2, i1, cap)
    f = {"d1": np.asarray(fw[0], np.float32), "d2": np.asarray(fw[1], np.float32), "i1": np.asarray(fw[2])}
    b = {"d1": np.asarray(bw[0], np.float32), "d2": np.asarray(bw[1], np.float32), "i1": np.asarray(bw[2])}
    ri, rd = ref_tables(f, b, n0, n1, mode, th)
    cnt = out["count"][0]
    assert cnt == len(ri), (mode, th, cnt, len(ri))
    k = min(cnt, cap)
    assert np.array_equal(out["idx"][0, :k], ri[:k]) and np.array_equal(out["dist"][0, :k].view(np.int32), rd[:k].view(np.int32))
    assert np.all(out["idx"][0, k:] == int(SENT)) and np.all(out["dist"][0, k:] == np.float32(SENT))
    assert np.all(out["idx_tail"] == int(SENT)) and np.all(out["dist_tail"] == np.float32(SENT)) and np.all(out["count_tail"] == ISENT)
    return out, ri


@pytest.mark.gpu
def test_select_ratio_boundaries(st):
    """snn / smnn: a ratio exactly th (3 / 5 and th / 1 against th = float32(0.6)) is accepted and one ulp above is rejected; 0 / 0
    is rejected at every th, 1 and +inf included; a +inf second gives ratio 0."""
    th32 = np.float32(0.6)
    th, up = float(th32), np.nextafter(th32, np.float32(1.0))
    fw = ([3.0, up, 0.0, 2.0, 0.0, th], [5.0, 1.0, 0.0, np.inf, 4.0, 1.0], [0, 1, 2, 3, 4, 5])
    bw = ([3.0, 3.0, 0.0, 1.0, 0.0, 1.0], [5.0, 5.0, 0.0, 3.0, 1.0, 2.0], [0, 1, 2, 3, 4, 5])
    assert np.float32(3.0) / np.float32(5.0) == th32 and up / np.float32(1.0) > th32
    for mode in ("snn", "smnn"):
        for t in (th, 1.0, np.inf):
            _, ri = _select_case(st, mode, t, fw, bw)
            assert 2 not in ri[:, 0], (mode, t)  # 0 / 0
        _, ri = _select_case(st, mode, th, fw, bw)
        assert ri[:, 0].tolist() == [0, 3, 4, 5], (mode, ri)


@pytest.mark.gpu
def test_select_smnn_distance_and_mnn_order(st):
    """smnn reports max(forward ratio, backward ratio); mnn iterates the smaller side and reports the backward distance when n0 > n1,
    and the forward one when n0 <= n1 (n0 == n1 included)."""
    fw = ([1.0, 4.0, 2.0], [4.0, 5.0, 8.0], [1, 0, 2])
    bw = ([4.0, 1.0, 2.0], [5.0, 2.0, 4.0], [1, 0, 2])
    out, _ = _select_case(st, "smnn", 0.9, fw, bw)
    assert out["count"][0] == 3 and out["dist"][0, 0] == np.float32(0.5)  # max(1/4, 1/2)
    for n0, n1 in ((3, 2), (2, 3), (3, 3)):
        rng = np.random.default_rng(n0 * 10 + n1)
        f = (rng.random(n0).astype(np.float32), np.ones(n0, np.float32), rng.integers(0, n1, n0))
        b = (rng.random(n1).astype(np.float32) + 2, np.ones(n1, np.float32), rng.integers(0, n0, n1))
        _select_case(st, "mnn", 0.0, f, b)
    # every row mutual with n0 > n1: the rows of the smaller side in ascending order, with its distances
    f = ([1.0, 2.0, 3.0], [9.0] * 3, [1, 0, 0])
    b = ([5.0, 6.0], [9.0] * 2, [1, 0])
    out, ri = _select_case(st, "mnn", 0.0, f, b)
    assert ri.tolist() == [[1, 0], [0, 1]] and out["dist"][0, :2].tolist() == [5.0, 6.0]


@pytest.mark.gpu
def test_select_many_rows_and_cap(st):
    """More than 1024 rows (the compaction spans passes) in every mode, and cap below the count: the count stays full and nothing past
    cap is written."""
    rng = np.random.default_rng(3)
    n0, n1 = 3000, 2500
    f = (rng.random(n0).astype(np.float32), (rng.random(n0) + 0.5).astype(np.float32), rng.integers(0, n1, n0))
    b = (rng.random(n1).astype(np.float32), (rng.random(n1) + 0.5).astype(np.float32), rng.integers(0, n0, n1))
    for i in range(0, n1, 3):  # make many rows mutual
        b[2][f[2][i]] = i
    for mode in MODES:
        out, ri = _select_case(st, mode, 0.8, f, b)
        assert len(ri) > (1024 if mode in ("nn", "snn") else 50), (mode, len(ri))
        out, _ = _select_case(st, mode, 0.8, f, b, cap=len(ri) // 3 + 1)


# ------------------------------------------------------------------ GPU: the product entries
def _entry_tables(ctx, entry, A, B, mode, th, kind):
    """One match table from a product entry: 'host' dimb_nn_match, 'dev' dimb_nn_match_dev (ld > n), 'batch' dimb_nn_match_batch_dev."""
    import torch
    n0, n1, D = len(A), len(B), A.shape[1]
    cap = max(n0, n1, 1)
    if entry == "host":
        return ctx.nn_match(np.asarray(A.T, np.float32), np.asarray(B.T, np.float32), mode, th)
    idx = torch.full((cap, 2), -5, dtype=torch.int64, device="cuda")
    dist = torch.full((cap,), -5.0, device="cuda")
    n = torch.full((1,), -5, dtype=torch.int32, device="cuda")
    sd = Sides()
    if entry == "dev":
        f0, f1 = sd.side(A, kind, ld=n0 + 17), sd.side(B, kind, ld=n1 + 5)
        ctx.nn_match_dev(f0.descriptors, n0, f1.descriptors, n1, D, mode, th, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), cap,
                         f16=kind == "f16", ld0=n0 + 17, ld1=n1 + 5)
    else:
        f0, f1 = sd.side(A, kind, n_cap=n0 + 40), sd.side(B, "f16" if kind == "round" else kind)
        ctx.nn_match_batch_dev([f0], [f1], D, mode, th, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), cap)
    torch.cuda.synchronize()
    k = n.item()
    return idx[:k].cpu().numpy(), dist[:k].cpu().numpy()


@pytest.fixture(scope="module")
def ctx_exact():
    from dim_b200 import _native
    return _native.Context(0, "exact")


@pytest.fixture(scope="module")
def ctx_fast():
    from dim_b200 import _native
    return _native.Context(0, "fast")


@pytest.mark.gpu
@pytest.mark.parametrize("entry,kind", [("host", "f32"), ("dev", "f16"), ("dev", "f32"), ("batch", "f16"), ("batch", "f32"),
                                        ("batch", "round")])
def test_entries_on_planted_ties_bitwise(ctx_exact, ctx_fast, entry, kind):
    """Every entry and input kind on byte descriptors with planted ties (integer class): the tables of all four modes equal the float64
    reference bitwise, in EXACT and FAST."""
    rng = np.random.default_rng(21)
    A, B = planted_ties(rng, 32, 300, 1300)
    fw, bw = ref_stats(A, B), ref_stats(B, A)
    for c in (ctx_exact, ctx_fast):
        for mode, th in [("nn", 0.0), ("mnn", 0.0), ("snn", 0.9), ("smnn", 0.95), ("snn", 1.0)]:
            ri, rd = ref_tables(fw, bw, len(A), len(B), mode, th)
            gi, gd = _entry_tables(c, entry, A, B, mode, th, kind)
            assert np.array_equal(gi, ri) and np.array_equal(gd.view(np.int32), rd.view(np.int32)), (entry, kind, mode, th)
    # n0 > n1 for mnn's swapped order
    fw, bw = ref_stats(B[:200], A[:150]), ref_stats(A[:150], B[:200])
    ri, rd = ref_tables(fw, bw, 200, 150, "mnn", 0.0)
    gi, gd = _entry_tables(ctx_exact, entry, B[:200], A[:150], "mnn", 0.0, kind)
    assert np.array_equal(gi, ri) and np.array_equal(gd, rd)


@pytest.mark.gpu
def test_host_entry_picks_the_split_from_the_values(ctx_exact, st):
    """dimb_nn_match in EXACT runs one MMA on fp16-exact float32 and three once a single value is not fp16: its nn distances equal
    the self-test's split 0 / split 1 statistics bitwise, and the two differ on the second input."""
    rng = np.random.default_rng(4)
    A, B = _unit(rng, 128, 200, 300)
    A, B = A.astype(np.float16).astype(np.float32), B.astype(np.float16).astype(np.float32)
    A[:50] = B[:50] + np.float32(1e-2) * A[:50]
    A, B = A.astype(np.float16).astype(np.float32), B.astype(np.float16).astype(np.float32)
    _, d_exact16 = ctx_exact.nn_match(A.T, B.T, "nn")
    s0 = stats(st, A, B, "f32", 0, True)
    assert np.array_equal(d_exact16, s0["d1"][0, :200])
    B2 = B.copy()
    B2[:, 0] += np.float32(2.0 ** -20)  # not fp16 any more
    assert np.any(B2.astype(np.float16).astype(np.float32) != B2)
    _, d_split = ctx_exact.nn_match(A.T, B2.T, "nn")
    s1, s0b = stats(st, A, B2, "f32", 1, True), stats(st, A, B2, "f32", 0, True)
    assert np.array_equal(d_split, s1["d1"][0, :200])
    assert not np.array_equal(s1["d1"][0, :200], s0b["d1"][0, :200])


# ------------------------------------------------------------------ GPU: ORB and SIFT image sets end to end
@pytest.mark.gpu
@pytest.mark.parametrize("extractor", ["orb", "sift"])
def test_store_tables_of_device_features_bitwise(ctx, extractor):
    """Device ORB / SIFT features of synthetic images go through the feature store into nn_match_batch_dev in all four modes: every
    table equals the float64 reference bitwise.  Prints how many rows had an exactly tied best."""
    import torch
    from dim_b200 import _native, synthetic
    from oracle.orb import to_u8
    base = to_u8(synthetic.to_gray_like_reference(synthetic.blocks_image(7, 512)))[:360, :480].copy()
    imgs = [base] + [synthetic.warp_pair(base, 30 + k, jitter=24.0) for k in range(3)]
    if extractor == "orb":
        net = _native.OrbNet(ctx, n_features=3000, max_batch=1, max_height=360, max_width=480)
        D = 32
    else:
        net = _native.SiftNet(ctx, n_features=3000, max_batch=1, max_height=360, max_width=480)
        D = 128
    feats = [net.extract(x) for x in imgs]
    cap = max(len(f["keypoints"]) for f in feats)
    store = _native.FeatureStoreDev(ctx, len(imgs), cap, D)
    for s, f in enumerate(feats):
        store.put(s, {"keypoints": f["keypoints"], "descriptors": f["descriptors"], "image_size": np.array([360, 480])})
    pairs = [(0, 1), (1, 0), (0, 2), (2, 3), (3, 1), (1, 1)]
    f0 = [store.feats_dev(a) for a, _ in pairs]
    f1 = [store.feats_dev(b) for _, b in pairs]
    P = len(pairs)
    ties = 0
    for mode, th in [("nn", 0.0), ("mnn", 0.0), ("snn", 0.8), ("smnn", 0.9)]:
        idx = torch.full((P, cap, 2), -5, dtype=torch.int64, device="cuda")
        dist = torch.full((P, cap), -5.0, device="cuda")
        n = torch.zeros(P, dtype=torch.int32, device="cuda")
        ctx.nn_match_batch_dev(f0, f1, D, mode, th, idx.data_ptr(), dist.data_ptr(), n.data_ptr(), cap)
        torch.cuda.synchronize()
        for p, (a, b) in enumerate(pairs):
            A = np.asarray(feats[a]["descriptors"], np.float64).T
            B = np.asarray(feats[b]["descriptors"], np.float64).T
            assert np.array_equal(A, A.astype(np.float16).astype(np.float64)) and A.max() <= 255
            fw, bw = ref_stats(A, B), ref_stats(B, A)
            if mode == "nn":
                ties += int(np.sum(np.sum(fw["f"] == fw["d1"][:, None], 1) > 1))
            ri, rd = ref_tables(fw, bw, len(A), len(B), mode, th)
            k = n[p].item()
            assert k == len(ri), (extractor, mode, p)
            assert np.array_equal(idx[p, :k].cpu().numpy(), ri), (extractor, mode, p)
            assert np.array_equal(dist[p, :k].cpu().numpy().view(np.int32), rd.view(np.int32)), (extractor, mode, p)
    print(f"\n{extractor}: {ties} query rows with an exactly tied best over {len(pairs)} pairs")


@pytest.mark.gpu
def test_selftest_entries_reject_bad_arguments(st):
    """With a real context, every argument check of the two entries returns DIMB_ERR_ARG before any CUDA call: host counts with P != 1,
    split or host_counts outside 0..1, an NPp other than the engine's, a host-count pair kornia leaves empty, a side the batch entry
    refuses; and in select n_live above NPp or negative, and a live row's i1 outside [0, NPp), which keeps planted statistics in
    bounds."""
    from dim_b200 import _native
    lib = st.lib
    sd = Sides()
    rng = np.random.default_rng(0)
    A, B = bytes_desc(rng, 32, 40), bytes_desc(rng, 32, 50)
    f0, f1 = sd.side(A), sd.side(B)
    one = sd.side(A[:1])
    bad = _native.FeatsDev.from_buffer_copy(f0)
    bad.desc_layout = 1
    buf = np.zeros(2 * 2 * 128 + _native.DET_TAIL, np.float32)
    p = _native._ptr(buf)

    def stats_rc(P, a0, a1, mode=0, split=0, host=1, NPp=128):
        return lib.dimb_selftest_nn_stats(st.h, P, (_native.FeatsDev * P)(*a0), (_native.FeatsDev * P)(*a1), 32, mode, split, host, NPp, 0.0,
                                          p, p, p, p, p)

    assert stats_rc(1, [f0], [f1]) == 0  # the valid call the others vary
    assert stats_rc(2, [f0, f0], [f1, f1], host=1) == ERR_ARG
    assert stats_rc(1, [f0], [f1], split=2) == ERR_ARG and stats_rc(1, [f0], [f1], split=-1) == ERR_ARG
    assert stats_rc(1, [f0], [f1], host=2) == ERR_ARG
    assert stats_rc(1, [f0], [f1], NPp=256) == ERR_ARG and stats_rc(1, [f0], [f1], NPp=0) == ERR_ARG
    assert stats_rc(1, [one], [f1], mode=3) == ERR_ARG  # smnn with one row: the host-count entries return before the engine
    assert stats_rc(1, [f0], [one], mode=2) == ERR_ARG  # snn with one candidate
    assert stats_rc(1, [bad], [f1]) == ERR_ARG and stats_rc(1, [f0], [f1], mode=4) == ERR_ARG

    NPp = 4
    live = np.array([3, 2], np.int32)
    d = np.ones((2, NPp), np.float32)
    i1 = np.zeros((2, NPp), np.int32)
    out = np.zeros(2 * 8 + _native.DET_TAIL, np.int64)
    q = _native._ptr

    def select_rc(live, i1, NPp=NPp):
        return lib.dimb_selftest_nn_select(st.h, 1, 0.8, 1, NPp, q(live), q(d), q(d), q(i1), 8, 0.0, q(out), q(buf), q(buf))

    assert select_rc(live, i1) == 0
    assert select_rc(np.array([5, 2], np.int32), i1) == ERR_ARG and select_rc(np.array([-1, 2], np.int32), i1) == ERR_ARG
    for s, r, v in ((0, 2, NPp), (1, 1, -1)):
        j = i1.copy()
        j[s, r] = v
        assert select_rc(live, j) == ERR_ARG, (s, r, v)
    j = i1.copy()
    j[1, 3] = 99  # past side 1's live rows: not read, not checked
    assert select_rc(live, j) == 0
