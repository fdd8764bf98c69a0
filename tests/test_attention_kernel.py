"""Flash attention (csrc/attention.cuh) on its own, against a float64 softmax(scale Q K^T) V of the same fp32 operands.

The kernels run through their production launches in the self-test library (dimb_selftest_attention): lg_attn_kernel (LightGlue /
SuperGlue: 4 heads x 64, self and cross, several sides with their own live counts and stopped pairs) and
lgx_attn_tc_kernel (the shape-generic path: head dim padded to 128, operands packed by hd128_attend as production packs them, the
cross form and, where the live counts are equal, the self form).  Padding rows hold a large finite value, as the stale rows of earlier
layers do in production, and the output buffer starts as a sentinel, so the mask (the packers' for the shape-generic path) and the rows
that must not be written are checked as well as the values.

Logits are designed: query rows are (A, A, b_i, noise) and key rows (u_hi, u_lo, w_j, noise), so the logit of (i, j) is
A (u_hi + u_lo) + b_i w_j + noise.  Every operand is fp16-exact and every partial sum a multiple of 2^-12 below 2^11, so Q K^T is exact
in fp32 and the cases test the online softmax, not operand rounding.  The key term u sets each 64-key block's maximum (one key per block
sits exactly on it); the row term b_i w_j (at most 0.9 log2 units, zero on the block-maximum keys) makes rows differ without moving
those maxima.

The CPU tests run a numpy model of the kernel's arithmetic (fp32 running state, exp2 with the scale folded in, fp16 hi / lo split of P,
lazy rescaling) on the same cases.  They show that the designed cases force the rescale branch where intended, that the bounds the GPU
tests use leave room for the kernel's own rounding, and that a rescale bug would break those bounds."""
import os

import numpy as np
import pytest

LOG2E = 1.4426950408889634
BLK = 64                # keys per block of the kernel
A = 8.0                 # query scale: logit = A * u + b w + noise
PAD = 1e3               # stale value in every Q / K row and V^T column past the live count
OUT_PAD = -777.0        # output buffer content before the call (fp16-exact)
# max |O - ref| / max |V_live|.  Largest measured on an H100 80GB HBM3 (700 W): EXACT 8.2e-7 (offset), FAST 6.8e-4 (jump_late);
# the numpy model below predicts 7.5e-7 for EXACT.
EXACT_TOL = 2e-6
FAST_TOL = 2e-3
LAZIES = (0.0, 8.0, 15.0)
PATTERNS = ["random", "ramp_below", "ramp_above", "jump_late", "max_first", "one_hot", "uniform", "offset"]
# (nq, nk): every edge of the 128-row query tile and of the 64-key block, no keys, one key, long rows
SHAPES = [(1, 1), (1, 2048), (127, 63), (127, 1000), (128, 64), (128, 0), (129, 65), (129, 191), (300, 2048), (300, 1), (129, 1),
          (300, 191)]
HD128 = [(66, 1), (96, 2), (128, 1), (66, 2), (96, 1), (128, 2)]  # (head dim, heads) of the generic kernel, cycled over SHAPES


def c2_of(hd):
    """log2 units per raw logit: the kernel evaluates softmax(scale * s) as exp2(s * scale * log2 e)."""
    return hd ** -0.5 * LOG2E


def _q32(x, step=2.0 ** -5):
    return np.round(np.asarray(x, np.float64) / step) * step


def design(pattern, nq, nk, hd, rng):
    """One head: q [nq][hd], k [nk][hd], v [nk][hd] float32 and the index of the hot key (one_hot) or None."""
    if pattern == "random":
        f = lambda *s: rng.standard_normal(s).astype(np.float32)
        return f(nq, hd), f(nk, hd), f(nk, hd), None
    c2 = c2_of(hd)
    nb = -(-nk // BLK)
    L = np.zeros(nk)                 # designed logit of each key, log2 units
    top = np.zeros(nk, bool)         # keys that sit exactly on their block's maximum (no row term)
    hot = None

    def blocks(M):                   # block b peaks at M[b] (one key at a random live position), the others 1..7 units below
        for b in range(nb):
            lo, hi = b * BLK, min(nk, b * BLK + BLK)
            L[lo:hi] = M[b] - rng.uniform(1, 7, hi - lo)
            j = rng.integers(lo, hi)
            L[j], top[j] = M[b], True

    if pattern == "ramp_below":      # the maximum climbs on every block but ends 7.9 units above block 0's: no rescale at lazy 8
        blocks(7.9 * np.arange(nb) / max(nb - 1, 1))
    elif pattern == "ramp_above":    # 8.1 units per block: a rescale on every block at lazy 8
        blocks(8.1 * np.arange(nb))
    elif pattern == "steep":         # 16.5 units per block: overflows P's fp16 hi plane unless lazy <= 15
        blocks(16.5 * np.arange(nb))
    elif pattern == "offset":        # shifted by 100 units (exp of it overflows fp32), the maximum growing by 2 per block
        blocks(100.0 + 2.0 * np.arange(nb))
    elif pattern == "max_first":     # the maximum in block 0, never exceeded
        L[:] = rng.uniform(-7, -1, nk)
        if nk:
            j = rng.integers(0, min(nk, BLK))
            L[j], top[j] = 0.0, True
    elif pattern == "jump_late":     # the maximum at nk - 1, next to the mask: 14.5 units up (no rescale at lazy 15, P = 2^14.5)
        L[:] = rng.uniform(-4, 0, nk)
        if nk:
            L[-1], top[-1] = 14.5, True
    elif pattern == "one_hot":       # one key 30 units above the rest: the output is its V row
        L[:] = rng.uniform(-1, 0, nk)
        if nk:
            hot = int(rng.integers(nk // 2, nk))
            L[hot], top[hot] = 31.0, True
    elif pattern == "uniform":       # all logits equal: the output is the mean of the live V rows
        L[:] = 3.0
        top[:] = True
    else:
        raise ValueError(pattern)
    u = _q32(L / c2 / A)
    u_hi = u.astype(np.float16).astype(np.float64)
    w = np.where(top, 0.0, _q32(rng.uniform(-1, 1, nk) * 0.9 / c2))
    b = rng.integers(-8, 9, nq) / 8.0
    q, k = np.zeros((nq, hd)), np.zeros((nk, hd))
    q[:, 0], q[:, 1], q[:, 2] = A, A, b
    k[:, 0], k[:, 1], k[:, 2] = u_hi, u - u_hi, w
    if pattern != "uniform":
        q[:, 3:] = rng.integers(-2, 3, (nq, hd - 3)) / 64.0
        k[:, 3:] = rng.integers(-2, 3, (nk, hd - 3)) / 64.0
    v = rng.standard_normal((nk, hd)).astype(np.float16)
    return q.astype(np.float32), k.astype(np.float32), v.astype(np.float32), hot


def reference(q, k, v, scale):
    """float64 softmax(scale q k^T) v of the fp32 operands; zeros for an empty key set (lightglue.py:103-104)."""
    if k.shape[0] == 0:
        return np.zeros((q.shape[0], v.shape[1]))
    s = (q.astype(np.float64) @ k.astype(np.float64).T) * scale
    p = np.exp(s - s.max(1, keepdims=True))
    return (p / p.sum(1, keepdims=True)) @ v.astype(np.float64)


# ------------------------------------------------------------------ numpy model of the kernel's arithmetic
def split(x):
    h = np.asarray(x, np.float32).astype(np.float16)
    return h.astype(np.float32), (np.asarray(x, np.float32) - h.astype(np.float32)).astype(np.float16).astype(np.float32)


def kernel_model(q, k, v, scale, lazy, exact=True, alpha_on_o=True):
    """The per-block online softmax of attn_tile for every query row: logits in fp32, fp32 running maximum / sum, P = exp2(s c2 - m c2)
    rounded to fp32 and split into fp16 hi / lo planes (hi only in FAST), lazy rescaling.  Returns (O, rescales after block 0 per row).
    alpha_on_o=False leaves the rescale factor off O but not off l (a model of a rescale bug)."""
    f32 = np.float32
    qh, ql = split(q)
    kh, kl = split(k)
    vh, vl = split(v)
    d64 = lambda a, b: a.astype(np.float64) @ b.astype(np.float64).T
    s = (d64(qh, kh) + d64(qh, kl) + d64(ql, kh) if exact else d64(qh, kh)).astype(f32)
    c2 = f32(f32(scale) * f32(LOG2E))
    nq, nk = s.shape
    m_run = np.full(nq, -np.inf, f32)
    l = np.zeros(nq, f32)
    o = np.zeros((nq, v.shape[1]))
    rescales = np.zeros(nq, int)
    with np.errstate(invalid="ignore", over="ignore"):
        for j0 in range(0, nk, BLK):
            sc = s[:, j0:j0 + BLK]
            m_blk = np.maximum(m_run, sc.max(1))
            grow = (m_blk - m_run).astype(f32) * c2 > f32(lazy)
            m_new = np.where(grow, m_blk, m_run)
            alpha = np.where(grow, np.exp2(((m_run - m_new) * c2).astype(f32)), f32(1)).astype(f32)
            rescales += grow & (j0 > 0)
            mc = (m_new * c2).astype(f32)
            m_run = m_new
            p =np.exp2((sc.astype(np.float64) * np.float64(c2) - mc[:, None]).astype(f32)).astype(f32)
            l = (l * alpha + p.sum(1, dtype=f32)).astype(f32)
            if alpha_on_o:
                o *= alpha[:, None]
            ph, pl = split(p)
            vb_h, vb_l = vh[j0:j0 + BLK].astype(np.float64), vl[j0:j0 + BLK].astype(np.float64)
            o += ph @ (vb_h + vb_l) + pl @ vb_h if exact else ph @ vb_h
        out = o / l[:, None] if nk else np.zeros_like(o)
    return out.astype(f32), rescales


def rel_err(o, ref, v):
    return float(np.abs(o.astype(np.float64) - ref).max() / np.abs(v).max()) if len(o) and len(v) else 0.0


# ------------------------------------------------------------------ CPU: the cases do what they are meant to
@pytest.mark.parametrize("nk", [1000, 2048])
def test_model_rescale_counts(nk):
    """At lazy 8 ramp_above rescales on every block after the first and ramp_below on none, so the GPU cases provably run the
    rescale branch; at lazy 0 ramp_below rescales on every block too (its maximum does climb)."""
    nb = -(-nk // BLK)
    for hd in (64, 66, 96, 128):
        rng = np.random.default_rng(nk + hd)
        q, k, v, _ = design("ramp_above", 32, nk, hd, rng)
        assert (kernel_model(q, k, v, hd ** -0.5, 8.0)[1] == nb - 1).all()
        assert (kernel_model(q, k, v, hd ** -0.5, 15.0)[1] == (nb - 1) // 2).all()
        q, k, v, _ = design("ramp_below", 32, nk, hd, rng)
        assert (kernel_model(q, k, v, hd ** -0.5, 8.0)[1] == 0).all()
        assert (kernel_model(q, k, v, hd ** -0.5, 0.0)[1] == nb - 1).all()
        q, k, v, _ = design("jump_late", 32, nk, hd, rng)
        assert (kernel_model(q, k, v, hd ** -0.5, 8.0)[1] == 1).all() and (kernel_model(q, k, v, hd ** -0.5, 15.0)[1] == 0).all()


def test_model_meets_the_bounds():
    """The kernel's own arithmetic stays inside the bounds the GPU tests assert, on every pattern, lazy and precision, with room."""
    worst = {}
    for pattern in PATTERNS:
        for nq, nk in [(64, 1000), (32, 2048), (16, 65)]:
            for hd in (64, 96):
                q, k, v, _ = design(pattern, nq, nk, hd, np.random.default_rng(nq + nk + hd))
                ref = reference(q, k, v, hd ** -0.5)
                for lazy in LAZIES:
                    for exact in (True, False):
                        e = rel_err(kernel_model(q, k, v, hd ** -0.5, lazy, exact)[0], ref, v)
                        worst[pattern, exact] = max(worst.get((pattern, exact), 0.0), e)
    print({f"{p} {'exact' if x else 'fast'}": f"{e:.1e}" for (p, x), e in worst.items()})
    assert all(e < EXACT_TOL / 2 for (p, x), e in worst.items() if x)
    assert all(e < FAST_TOL / 2 for (p, x), e in worst.items() if not x)


def test_model_rescale_bug_breaks_the_bound():
    """Leaving alpha off O (but not off l) misses the reference by more than 100 x the EXACT bound on ramp_above: a rescale bug in the
    kernel cannot pass the GPU tests."""
    q, k, v, _ = design("ramp_above", 64, 1000, 64, np.random.default_rng(3))
    ref = reference(q, k, v, 0.125)
    assert rel_err(kernel_model(q, k, v, 0.125, 8.0)[0], ref, v) < EXACT_TOL
    assert rel_err(kernel_model(q, k, v, 0.125, 8.0, alpha_on_o=False)[0], ref, v) > 100 * EXACT_TOL


def test_model_lazy_above_15_overflows_fp16():
    """Why DIMB_ATTN_LAZY is bounded by 15: with a maximum growing by 16.5 log2 units per block, lazy 17 lets P (up to 2^lazy) overflow
    its fp16 hi plane and the rows turn NaN; lazy 15 keeps them within the EXACT bound."""
    q, k, v, _ = design("steep", 32, 256, 64, np.random.default_rng(4))
    ref = reference(q, k, v, 0.125)
    assert np.isnan(kernel_model(q, k, v, 0.125, 17.0)[0]).all()
    assert np.isnan(kernel_model(q, k, v, 0.125, float("nan"))[0]).all()
    assert rel_err(kernel_model(q, k, v, 0.125, 15.0)[0], ref, v) < EXACT_TOL


# ------------------------------------------------------------------ GPU
def _selftest(env=None):
    """A self-test context; env switches are read when a context is created, so those get a context of their own."""
    from dim_b200 import _native
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return _native.SelfTest(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def st():
    return _selftest()


def lg_case(pattern, n, cross, rng):
    """Variant 0 operands Q, K, V [S][4][NP][64] for live counts n[S].  Self: side s attends over its own n[s] rows.  Cross: the even
    side of a pair gets query rows and the odd side key rows, so the even side sees the designed logits over the odd side's keys."""
    S = len(n)
    NP = max(-(-max(n) // 128) * 128, 128)
    Q, K, V = (np.zeros((S, 4, NP, 64), np.float32) for _ in range(3))
    hot = {}
    for h in range(4):
        for s in range(S):
            if cross and s % 2 == 0:
                q, k, v, hot[s, h] = design(pattern, n[s], n[s + 1], 64, rng)
                Q[s, h, :n[s]], Q[s + 1, h, :n[s + 1]], V[s + 1, h, :n[s + 1]] = q, k, v
                V[s, h, :n[s]] = rng.standard_normal((n[s], 64)).astype(np.float16)
            elif not cross:
                q, k, v, hot[s, h] = design(pattern, n[s], n[s], 64, rng)
                Q[s, h, :n[s]], K[s, h, :n[s]], V[s, h, :n[s]] = q, k, v
    return Q, K, V, hot


def check_lg(out, Q, K, V, n, stopped, cross, pattern, hot, tol):
    """Per live side and head: max |O - ref| / max |V_live| <= tol, exact zeros without keys, closed forms where designed; rows past
    the live count and every row of a stopped pair untouched; nothing NaN.  Returns the largest relative error."""
    assert not np.isnan(out).any()
    worst = 0.0
    for s in range(len(n)):
        if stopped[s // 2]:
            assert (out[s] == OUT_PAD).all(), f"stopped side {s} written"
            continue
        assert (out[s, n[s]:] == OUT_PAD).all(), f"side {s}: rows >= {n[s]} written"
        ks = s ^ 1 if cross else s
        for h in range(4):
            o = out[s, :n[s], 64 * h:64 * h + 64]
            keys = (Q if cross else K)[ks, h, :n[ks]]
            vl = V[ks, h, :n[ks]]
            if n[ks] == 0:
                assert (o == 0).all(), f"side {s} head {h}: no keys must give zeros"
                continue
            e = rel_err(o, reference(Q[s, h, :n[s]], keys, vl, 0.125), vl)
            assert e <= tol, f"side {s} head {h}: {e:.2e}"
            worst = max(worst, e)
            designed = not cross or s % 2 == 0
            if designed and pattern == "one_hot":
                assert np.abs(o - vl[hot[s, h]]).max() <= tol * np.abs(vl).max()
            if designed and pattern == "uniform":
                assert np.abs(o - vl.astype(np.float64).mean(0)).max() <= tol * np.abs(vl).max()
    return worst


def _lg_live_counts(i, nq, nk):
    """Pair i % 2 runs with live counts (nq, nk); the other pair (700 / 129 rows) is stopped."""
    n = [nq, nk, 700, 129] if i % 2 == 0 else [700, 129, nq, nk]
    return n, [0, 1] if i % 2 == 0 else [1, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("cross", [False, True], ids=["self", "cross"])
def test_lg_attention(st, pattern, cross):
    """lg_attn_kernel (LightGlue / SuperGlue) over every shape, lazy threshold and precision."""
    for i, (nq, nk) in enumerate(SHAPES):
        n, stopped = _lg_live_counts(i, nq, nk)
        Q, K, V, hot = lg_case(pattern, n, cross, np.random.default_rng(i))
        for precision, tol in (("exact", EXACT_TOL), ("fast", FAST_TOL)):
            st.set_precision(precision)
            for lazy in LAZIES:
                out = st.attention(0, Q, None if cross else K, V, n, stopped=stopped, cross=cross, lazy=lazy, pad=PAD, out_pad=OUT_PAD)
                check_lg(out, Q, K, V, n, stopped, cross, pattern, hot, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
def test_hd128_attention(st, pattern):
    """lgx_attn_tc_kernel with its packers (the shape-generic path, head dim padded to 128) over every shape, lazy threshold and
    precision."""
    for i, (nq, nk) in enumerate(SHAPES):
        hd, H = HD128[i % len(HD128)]
        rng = np.random.default_rng(100 + i)
        parts = [design(pattern, nq, nk, hd, rng) for _ in range(H)]
        Q, K, V = (np.concatenate([p[j] for p in parts], 1) for j in range(3))
        for precision, tol in (("exact", EXACT_TOL), ("fast", FAST_TOL)):
            st.set_precision(precision)
            for lazy in LAZIES:
                out = st.attention(1, Q, K, V, (nq, nk), heads=H, lazy=lazy, pad=PAD, out_pad=OUT_PAD)
                assert not np.isnan(out).any()
                assert (out[nq:] == OUT_PAD).all(), "rows >= nq written"
                for h, (q, k, v, hot) in enumerate(parts):
                    o = out[:nq, h * hd:(h + 1) * hd]
                    if nk == 0:
                        assert (o == 0).all()
                        continue
                    e = rel_err(o, reference(q, k, v, hd ** -0.5), v)
                    assert e <= tol, f"{precision} lazy {lazy} hd {hd} head {h}: {e:.2e}"
                    if pattern == "one_hot":
                        assert np.abs(o - v[hot]).max() <= tol * np.abs(v).max()
                    if pattern == "uniform":
                        assert np.abs(o - v.astype(np.float64).mean(0)).max() <= tol * np.abs(v).max()


@pytest.mark.gpu
def test_attention_is_bitwise_repeatable(st):
    """Two identical calls give identical bits (no race between the TMA ring, the two consumer warpgroups and the stores)."""
    st.set_precision("exact")
    n, stopped = [300, 2048, 129, 700], [0, 0]
    Q, K, V, _ = lg_case("ramp_above", n, False, np.random.default_rng(7))
    a, b = (st.attention(0, Q, K, V, n, stopped=stopped, lazy=8.0, pad=PAD, out_pad=OUT_PAD) for _ in range(2))
    assert np.array_equal(a, b)
    q, k, v, _ = design("random", 300, 1000, 96, np.random.default_rng(8))
    a, b = (st.attention(1, q, k, v, (300, 1000), heads=1, lazy=8.0, pad=PAD, out_pad=OUT_PAD) for _ in range(2))
    assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("value", ["17", "nan", "inf", "-1", "x"])
def test_attn_lazy_environment_is_bounded(value):
    """DIMB_ATTN_LAZY outside [0, 15] (or not a number) keeps the default threshold: a maximum growing by 16.5 log2 units per block
    stays finite and within the EXACT bound instead of overflowing P's fp16 hi plane."""
    st = _selftest({"DIMB_ATTN_LAZY": value})
    n, stopped = [128, 256, 256, 128], [0, 0]
    Q, K, V, hot = lg_case("steep", n, False, np.random.default_rng(9))
    out = st.attention(0, Q, K, V, n, stopped=stopped, lazy=-1.0, pad=PAD, out_pad=OUT_PAD)
    check_lg(out, Q, K, V, n, stopped, False, "steep", hot, EXACT_TOL)
    assert np.array_equal(out, st.attention(0, Q, K, V, n, stopped=stopped, lazy=8.0, pad=PAD, out_pad=OUT_PAD))


@pytest.mark.gpu
def test_attn_lazy_environment_is_used():
    """A valid DIMB_ATTN_LAZY is what lazy = -1 runs with."""
    st = _selftest({"DIMB_ATTN_LAZY": "0"})
    n, stopped = [300, 1000, 129, 700], [0, 0]
    Q, K, V, _ = lg_case("ramp_below", n, False, np.random.default_rng(10))
    a, b = (st.attention(0, Q, K, V, n, stopped=stopped, lazy=lz, pad=PAD, out_pad=OUT_PAD) for lz in (-1.0, 0.0))
    assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("lazy", [15.5, 16.0, float("nan"), float("inf")])
def test_attention_refuses_lazy_out_of_range(st, lazy):
    from dim_b200 import _native
    n = [128, 128]
    Q, K, V, _ = lg_case("random", n, False, np.random.default_rng(11))
    with pytest.raises(_native.DimbError, match=r"code -3\)"):
        st.attention(0, Q, K, V, n, stopped=[0], lazy=lazy)
