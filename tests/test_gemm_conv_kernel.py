"""The persistent tensor-core GEMM / 3x3-conv kernel (csrc/gemm.cuh, tc_gemm_pers_kernel) on its own, against float64 references.

The kernel runs through its production launches in the self-test library: dimb_selftest_gemm (launch_gemm with the fp32 store epilogue,
including the 32-wide-K mode of the LightGlue linears) and dimb_selftest_conv3x3 (the SuperPoint layer: make_conv_layer's weight layout,
run_conv3's NHWC tensor maps and the bias + ReLU + 2x2 max pool epilogue, csrc/conv3x3.cuh).  Operand rows past M / N and the image after
the last one hold a large finite guard, and the output buffers start as a sentinel, so TMA out-of-bounds fill, halo reads across image
boundaries, unwritten outputs and stray writes all show.

Which ring depths and whether the weights stay resident (RESB) is decided by pers_plan from the shapes and the precision; the tests
reach every plan the production call sites produce by choosing shapes, never by forcing one.  The CPU tests check the plan invariants
at every call site and a numpy model of the arithmetic (fp16 hi / lo operand split without lo * lo, fp32 accumulation rounded toward
zero per 16-deep MMA, output rounded to the stored planes) against the bounds the GPU tests use.

Cases:
  designed  activations small integers / 8, weights small integers / 64: every operand is exact in fp16 and every partial sum a multiple
            of 2^-9 below 2^14, so the float64 result is exact in fp32 in any order.  EXACT must equal it bitwise, FAST must equal its
            fp16 rounding (conv) or itself (GEMM) bitwise.
  shift     output channel o reads only tap o % 9 of input channel o % cin: a wrong tap, halo or channel block names itself.
  random    normal operands with non-zero lo planes, checked element by element against a bound scaled by sum_k |a_k b_k|: these catch
            a lost lo plane, which the designed cases cannot.
"""
import numpy as np
import pytest

GUARD = 1e3          # operand rows / the image past the end: finite (the ReLU maps NaN to 0) and below the fp16 clamp of split_f32
SENTINEL = -777.0    # output buffers before the call (fp16-exact; the ReLU output is never negative)
SMEM_MAX = 232448    # opt-in shared memory per block on sm_90
STG_BYTES = 2 * 64 * 68 * 4  # accumulator staging of the two consumer warpgroups (gemm.cuh kStgBytes)
# Per-element bound: |out - ref| <= REL * sum_k |a_k b_k| + ABS * sum_k (|a_k| + |b_k|) + ACC * (sum of |partial sums|) + OUT * |ref|
# + 2^-24.
#   REL: operand split (EXACT: hi + lo carry ~22 bits, lo * lo dropped; FAST: hi only, 2^-11 per operand).
#   ABS: an operand's lo plane is fp16-subnormal below ~2^-3 and rounds to 2^-25 absolute.
#   ACC: the fp32 accumulation, per MMA: the tensor cores round the accumulator toward zero, so these errors do not cancel and grow with
#        K; one ulp (2^-23) of every partial sum the MMAs produce (see bound()).
#   OUT: the stored output: fp32 (GEMM), hi + lo fp16 planes (EXACT conv), hi only (FAST conv, half an fp16 ulp).
# Largest observed |err| / bound (test_report_error_ratios) on an NVIDIA H100 80GB HBM3 at a 700 W power limit: EXACT conv 0.29,
# EXACT GEMM 0.29, FAST conv 0.13, FAST GEMM 0.22; the numpy model predicts at most 0.33.  This file ran in 66 s there (CPU tests
# included).  Without the ACC term the EXACT GEMM at K = 2048 reached 1.13: the round-toward-zero model reproduces that (1.30).
ACC = 2.0 ** -23
BOUNDS = {  # precision -> (REL, ABS, OUT for the GEMM, OUT for the conv)
    "exact": (2.0 ** -20, 2.0 ** -24, 2.0 ** -23, 2.0 ** -21),
    "fast": (2.0 ** -10, 2.0 ** -24, 2.0 ** -23, 2.0 ** -10),
}
SP_CONVS = [(64, 64), (64, 128), (128, 128), (128, 256)]  # (cin, cout) of the SuperPoint 3x3 convolutions
CONV_HW = [(2, 2), (3, 5), (16, 16), (37, 45)]


# ------------------------------------------------------------------ launch plans of the production call sites
def _sites():
    """(name, conv mode, bn, num_kb, Epi::kConstB, m_tiles choices, n_tiles choices) of every launch_gemm call site, from the code."""
    many = (1, 2, 3, 8, 40, 131, 400)
    return [
        ("superpoint conv 64->64 (1b, 2a, 2b)", 1, 64, 9, True, many, (1,)),          # superpoint.cu run_conv3<64>
        ("superpoint conv 64->128 (3a)", 1, 128, 9, True, many, (1,)),               # run_conv3<128>
        ("superpoint conv 128->128 (3b, 4a, 4b)", 1, 128, 18, True, many, (1,)),
        ("superpoint conv 128->256 (Pa, Da)", 1, 128, 18, True, many, (2,)),
        ("superpoint 1x1 (Pb, Db)", 0, 128, 4, True, many, (1, 2)),                  # run_conv1_f32
        ("lightglue linears K 128 / 256 / 512", 0, 128, (2, 4, 8), True, many, (1, 2, 4)),  # lg_gemm, lg.qk
        ("lightglue BN 256 (DIMB_BN256)", 0, 256, (4, 8), True, many, (1, 2)),
        ("lightglue K32 (DIMB_K32)", 3, 256, (8, 16), True, many, (1, 2)),
        ("lightglue / superglue vT", 0, 128, 4, True, (2,), (1, 4, 16, 64)),
        ("lightglue final_proj, sim; superglue scores", 0, 128, 4, False, many, (1, 2, 16)),
        ("superglue linears", 0, 128, (4, 8), True, many, (2, 4, 6)),
        ("nn matcher", 0, 128, (2, 4), True, many, (1, 8, 32)),
        ("nn matcher, batched", 0, 128, (2, 4), False, many, (1, 8, 32)),
        ("aliked sddh", 0, 128, (2, 32), True, many, (1,)),
    ]


def _plan(conv, bn, split, const_b, nkb, mt, nt, sms):
    from dim_b200 import _native
    resb, sa, sb, smem, grid = _native.gemm_plan(conv, bn, split, const_b, nkb, mt, nt, sms)
    return bool(resb), sa, sb, smem, grid


def _geometry(conv, bn, split):
    """A-stage and B-tile pitches of PersGeom<bn, split, conv> in bytes."""
    pl = 2 if split else 1
    row = 64 if conv == 3 else 128
    abox = (10 * 16 * 128 if conv == 1 else 128 * row)
    return pl * (-(-abox // 1024) * 1024), pl * bn * row


def production_plans(sms):
    """{(bn, split, conv, resb, sa, sb)} over every call site, both precisions and the tile counts a call can have."""
    out = set()
    for _, conv, bn, nkbs, const_b, mts, nts in _sites():
        for nkb in (nkbs if isinstance(nkbs, tuple) else (nkbs,)):
            for split in (True, False):
                for mt in mts:
                    for nt in nts:
                        resb, sa, sb, _, _ = _plan(conv, bn, split, const_b, nkb, mt, nt, sms)
                        out.add((bn, split, conv, resb, sa, sb))
    return out


@pytest.mark.parametrize("sms", [114, 132])
def test_plan_invariants_at_every_call_site(sms):
    """Shared memory within the opt-in limit, at least one A stage, enough B slots for the conv schedule (the consumer holds the three
    dy taps of a stage before releasing any), the mbarriers in the 1 KB before the staging buffer, RESB only for a constant B panel on a
    grid that pins every CTA to one n-tile, and swizzle-atom aligned stage pitches."""
    for name, conv, bn, nkbs, const_b, mts, nts in _sites():
        for nkb in (nkbs if isinstance(nkbs, tuple) else (nkbs,)):
            for split in (True, False):
                astage, btile = _geometry(conv, bn, split)
                assert astage % 1024 == 0 and btile % 1024 == 0, name
                for mt in mts:
                    for nt in nts:
                        resb, sa, sb, smem, grid = _plan(conv, bn, split, const_b, nkb, mt, nt, sms)
                        what = f"{name}: split {split} num_kb {nkb} tiles {mt} x {nt} on {sms} SMs"
                        slots = nkb if resb else sb
                        assert smem == sa * astage + slots * btile + 2048 + STG_BYTES, what  # the Python geometry is the kernel's
                        assert smem <= SMEM_MAX, what
                        assert 1 <= sa <= 8, what
                        if not resb:
                            assert sb >= (3 if conv == 1 else 1), what
                        assert 8 * (2 * sa + 2 * slots) <= 1024, what
                        assert 1 <= grid <= min(sms, mt * nt), what
                        if resb:
                            assert const_b and grid % nt == 0 and sb == 0 and sa >= 2, what


def test_plan_table():
    """The plans of the SuperPoint convolutions and the LightGlue linears on 132 SMs at a full-size tile count (EXACT / FAST)."""
    want = {  # (conv, bn, num_kb, n_tiles): (EXACT (resb, sa, sb), FAST (resb, sa, sb))
        (1, 64, 9, 1): ((False, 2, 6), (True, 5, 0)),
        (1, 128, 9, 1): ((False, 1, 4), (True, 2, 0)),
        (1, 128, 18, 1): ((False, 1, 4), (False, 2, 9)),
        (1, 128, 18, 2): ((False, 1, 4), (False, 2, 9)),
        (0, 128, 4, 2): ((False, 2, 3), (True, 7, 0)),
        (0, 128, 8, 2): ((False, 2, 3), (True, 3, 0)),
        (0, 256, 4, 2): ((False, 1, 2), (True, 3, 0)),
        (3, 256, 8, 2): ((False, 3, 4), (True, 7, 0)),
    }
    for (conv, bn, nkb, nt), (ex, fa) in want.items():
        assert _plan(conv, bn, True, True, nkb, 400, nt, 132)[:3] == ex
        assert _plan(conv, bn, False, True, nkb, 400, nt, 132)[:3] == fa


def test_plan_refuses_unknown_instantiations():
    from dim_b200 import _native
    for args in [(1, 256, 1, 1, 9, 1, 1, 132), (3, 128, 1, 1, 8, 1, 1, 132), (2, 128, 1, 1, 4, 1, 1, 132), (0, 128, 1, 1, 0, 1, 1, 132)]:
        with pytest.raises(_native.DimbError):
            _native.gemm_plan(*args)


# ------------------------------------------------------------------ references and the model of the arithmetic
def im2col(x, swap_taps=False):
    """NHWC [B][H][W][cin] -> [B*H*W][9*cin] float64, column tap*cin + c with tap = 3 dy + dx (zero padding 1), as the weights are laid
    out ([cout][tap*cin + c]).  swap_taps: tap = 3 dx + dy (a model of a dx / dy mix-up)."""
    B, H, W, C = x.shape
    xp = np.pad(np.asarray(x, np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
    cols = np.empty((B, H, W, 9, C))
    for dy in range(3):
        for dx in range(3):
            cols[:, :, :, (3 * dx + dy) if swap_taps else (3 * dy + dx)] = xp[:, dy:dy + H, dx:dx + W]
    return cols.reshape(B * H * W, 9 * C)


def wmat(w):
    """OIHW [cout][cin][3][3] -> [cout][tap*cin + c] float64."""
    return np.asarray(w, np.float64).transpose(0, 2, 3, 1).reshape(w.shape[0], -1)


def split(x):
    """fp16 hi / lo planes of fp32 values, as split_f32 makes them (values clamped to +-65504)."""
    x = np.clip(np.asarray(x, np.float32), -65504, 65504)
    h = x.astype(np.float16).astype(np.float32)
    return h.astype(np.float64), (x - h).astype(np.float16).astype(np.float64)


def store(y, precision, conv):
    """The value the caller reads back: fp32 (GEMM); hi + lo fp16 planes (EXACT conv) or hi only (FAST conv)."""
    y = np.asarray(y, np.float32)
    if not conv:
        return y.astype(np.float64)
    h = y.astype(np.float16)
    if precision == "fast":
        return h.astype(np.float64)
    return h.astype(np.float64) + (y - h.astype(np.float32)).astype(np.float16).astype(np.float64)


def rz32(x):
    """float64 -> float32 rounded toward zero."""
    r = np.asarray(x, np.float64).astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(x)
    return np.where(over, np.nextafter(r, np.float32(0)), r)


def model(a, b, precision, drop_lo=False, drop_block=None):
    """The kernel's arithmetic on A [M][K], B [N][K]: per 16-deep MMA step the products hi*hi (+ hi*lo + lo*hi in EXACT; lo*lo never),
    each MMA's sum added to the fp32 accumulator and rounded toward zero, as the tensor cores' fp32 accumulation does.  drop_lo: A's lo
    plane lost; drop_block: one 64-wide K block skipped (models of bugs).  Returns the fp32 accumulator as float64."""
    ah, al = split(a)
    bh, bl = split(b)
    if drop_lo:
        al = np.zeros_like(al)
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    planes = [(ah, bh)] + ([(ah, bl), (al, bh)] if precision == "exact" else [])
    for k0 in range(0, a.shape[1], 16):
        if drop_block is not None and k0 // 64 == drop_block:
            continue
        for pa, pb in planes:
            acc = rz32(acc + pa[:, k0:k0 + 16] @ pb[:, k0:k0 + 16].T)
    return acc.astype(np.float64)


def bound(a, b, ref, precision, conv):
    """Per-element bound: the operand split and the stored output (BOUNDS), plus the fp32 accumulation: every MMA adds its 16-deep sum
    to the accumulator with an error below one ulp of the new partial sum (2^-23 of it), one add per plane and k16 step."""
    rel, ab, out_gemm, out_conv = BOUNDS[precision]
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    part, steps = np.zeros((a.shape[0], b.shape[0])), np.zeros((a.shape[0], b.shape[0]))
    for k0 in range(0, a.shape[1], 16):
        part += a[:, k0:k0 + 16] @ b[:, k0:k0 + 16].T
        steps += np.abs(part)
    planes = 3 if precision == "exact" else 1
    a, b = np.abs(a), np.abs(b)
    return (rel * (a @ b.T) + ab * (a.sum(1)[:, None] + b.sum(1)[None, :]) + ACC * planes * steps
            + (out_conv if conv else out_gemm) * np.abs(ref) + 2.0 ** -24)


def pool2(v, B, H, W):
    """2x2 max pool (floor) of [B*H*W][C] -> [B][H/2][W/2][C]."""
    v = v.reshape(B, H, W, -1)[:, :H // 2 * 2, :W // 2 * 2]
    return v.reshape(B, H // 2, 2, W // 2, 2, -1).max((2, 4))


def conv_reference(x, w, bias, pool, precision):
    """(float64 reference, per-element bound) of relu(conv3x3(x) + bias), pooled; the bound of a pooled value is its window's largest."""
    B, H, W, _ = x.shape
    a, bm = im2col(x), wmat(w)
    pre = a @ bm.T + np.asarray(bias, np.float64)
    ref, tol = np.maximum(pre, 0), bound(a, bm, pre, precision, True)
    if pool:
        return pool2(ref, B, H, W), pool2(tol, B, H, W)
    return ref.reshape(B, H, W, -1), tol.reshape(B, H, W, -1)


def conv_model(x, w, bias, pool, precision, **mut):
    B, H, W, _ = x.shape
    swap = mut.pop("swap_taps", False)
    acc = model(im2col(x, swap), wmat(w), precision, **mut)
    y = store(np.maximum((acc.astype(np.float32) + np.asarray(bias, np.float32)).astype(np.float32), 0), precision, True)
    return pool2(y, B, H, W) if pool else y.reshape(B, H, W, -1)


def ratio(out, ref, tol):
    return float((np.abs(np.asarray(out, np.float64) - ref) / tol).max())


# ------------------------------------------------------------------ cases
def conv_case(kind, B, H, W, cin, cout, rng):
    """x [B][H][W][cin], w [cout][cin][3][3], bias [cout] of one kind; image b is offset by 4 b (designed) or 3 b (random), so a halo read
    from the wrong image is large."""
    if kind == "designed":
        x = rng.integers(-8, 9, (B, H, W, cin)) / 8.0 + 4.0 * np.arange(B)[:, None, None, None]
        w = rng.integers(-4, 5, (cout, cin, 3, 3)) / 64.0
        bias = rng.integers(-64, 65, cout) / 64.0
    elif kind == "shift":
        x = rng.integers(-8, 9, (B, H, W, cin)) / 8.0 + 4.0 * np.arange(B)[:, None, None, None]
        w = np.zeros((cout, cin, 3, 3))
        o = np.arange(cout)
        w[o, o % cin, (o % 9) // 3, (o % 9) % 3] = (1 + o % 3) / 64.0
        bias = np.ones(cout)
    else:
        x = rng.standard_normal((B, H, W, cin)) + 3.0 * np.arange(B)[:, None, None, None]
        w = rng.standard_normal((cout, cin, 3, 3)) * 0.05
        bias = rng.standard_normal(cout) * 0.1
    return x.astype(np.float32), w.astype(np.float32), bias.astype(np.float32)


def gemm_case(kind, M, N, K, rng, with_bias):
    if kind == "designed":
        a, b = rng.integers(-8, 9, (M, K)) / 8.0, rng.integers(-4, 5, (N, K)) / 64.0
        bias = rng.integers(-64, 65, N) / 64.0
    else:
        a, b, bias = rng.standard_normal((M, K)), rng.standard_normal((N, K)), rng.standard_normal(N)
    return a.astype(np.float32), b.astype(np.float32), bias.astype(np.float32) if with_bias else None


# ------------------------------------------------------------------ CPU: the model meets the bounds, and bugs break them
def test_designed_cases_are_exact_in_fp32():
    """Every partial sum of a designed case is a multiple of 2^-9 below 2^14, so the fp32 model equals the float64 reference bitwise (in
    any accumulation order) and so must the kernel; FAST differs from it only by the fp16 rounding of the stored conv output."""
    rng = np.random.default_rng(0)
    for kind in ("designed", "shift"):
        x, w, bias = conv_case(kind, 2, 6, 7, 128, 256, rng)
        a, bm = im2col(x), wmat(w)
        assert np.abs(a).max() * np.abs(bm).max() * a.shape[1] + np.abs(bias).max() < 2.0 ** 14
        for precision in ("exact", "fast"):
            for pool in (False, True):
                ref, _ = conv_reference(x, w, bias, pool, precision)
                want = ref if precision == "exact" else ref.astype(np.float16).astype(np.float64)
                assert np.array_equal(conv_model(x, w, bias, pool, precision), want)
    a, b, bias = gemm_case("designed", 300, 65, 2048, rng, True)
    ref = a.astype(np.float64) @ b.astype(np.float64).T + bias
    for precision in ("exact", "fast"):
        assert np.array_equal((model(a, b, precision).astype(np.float32) + bias).astype(np.float64), ref)


def test_model_meets_the_bounds():
    """The model of the kernel's arithmetic stays within half of every bound the GPU tests use, on the random cases."""
    rng = np.random.default_rng(1)
    worst = {}
    for precision in ("exact", "fast"):
        for cin, cout in SP_CONVS:
            for pool in (False, True):
                x, w, bias = conv_case("random", 2, 5, 7, cin, cout, rng)
                ref, tol = conv_reference(x, w, bias, pool, precision)
                worst[precision, "conv"] = max(worst.get((precision, "conv"), 0), ratio(conv_model(x, w, bias, pool, precision), ref, tol))
        for M, N, K in [(130, 65, 256), (64, 128, 2048), (128, 256, 576)]:
            a, b, bias = gemm_case("random", M, N, K, rng, True)
            ref = a.astype(np.float64) @ b.astype(np.float64).T
            out = store(model(a, b, precision), precision, False)
            worst[precision, "gemm"] = max(worst.get((precision, "gemm"), 0), ratio(out, ref, bound(a, b, ref, precision, False)))
    print({f"{p} {k}": f"{v:.3f}" for (p, k), v in worst.items()})
    assert all(v <= 0.5 for v in worst.values()), worst


def test_model_bugs_break_the_exact_bound():
    """A lost lo plane, a skipped K block and a dx / dy mix-up each miss the reference by more than 10 x the EXACT bound."""
    rng = np.random.default_rng(2)
    x, w, bias = conv_case("random", 2, 9, 11, 128, 128, rng)
    ref, tol = conv_reference(x, w, bias, False, "exact")
    assert ratio(conv_model(x, w, bias, False, "exact"), ref, tol) < 1
    assert ratio(conv_model(x, w, bias, False, "exact", drop_lo=True), ref, tol) > 10
    assert ratio(conv_model(x, w, bias, False, "exact", drop_block=5), ref, tol) > 10
    assert ratio(conv_model(x, w, bias, False, "exact", swap_taps=True), ref, tol) > 10
    a, b, _ = gemm_case("random", 200, 65, 512, rng, False)
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    tol = bound(a, b, ref, "exact", False)
    assert ratio(model(a, b, "exact", drop_lo=True), ref, tol) > 10
    assert ratio(model(a, b, "exact", drop_block=3), ref, tol) > 10


# ------------------------------------------------------------------ GPU
EXECUTED = set()   # (bn, split, conv, resb, sa, sb) of every tensor-core launch the GPU tests ran
WORST = {}         # (precision, "gemm" / "conv") -> largest |err| / bound of the random cases


def _selftest():
    from dim_b200 import _native
    return _native.SelfTest(0)


@pytest.fixture(scope="module")
def st():
    return _selftest()


def _record(plan, bn, precision, conv):
    resb, sa, sb, smem, grid = plan
    assert resb in (0, 1) and sa >= 1 and smem <= SMEM_MAX and grid >= 1
    EXECUTED.add((bn, precision == "exact", conv, bool(resb), sa, sb))


def run_conv(st, kind, B, H, W, cin, cout, pool, precision, seed):
    """One conv case on the context `st`, checked completely; returns the output."""
    st.set_precision(precision)
    x, w, bias = conv_case(kind, B, H, W, cin, cout, np.random.default_rng(seed))
    out, tail, plan = st.conv3x3(x, w, bias, pool, guard=GUARD, sentinel=SENTINEL)
    what = f"{kind} {precision} B{B} {H}x{W} {cin}->{cout} pool {pool} plan {plan}"
    assert (tail == SENTINEL).all(), f"{what}: write past the last output image"
    assert (out != SENTINEL).all(), f"{what}: {int((out == SENTINEL).sum())} outputs not written"
    ref, tol = conv_reference(x, w, bias, pool, precision)
    if kind == "random":
        r = ratio(out, ref, tol)
        WORST[precision, "conv"] = max(WORST.get((precision, "conv"), 0.0), r)
        assert r <= 1, f"{what}: |err| / bound = {r:.2f}"
    else:
        want = ref if precision == "exact" else ref.astype(np.float16).astype(np.float64)
        bad = np.argwhere(out != want)
        if len(bad):
            b, y, xx, o = bad[0]
            raise AssertionError(f"{what}: {len(bad)} outputs differ, first at image {b} ({y}, {xx}) channel {o}"
                                 + (f" (tap dy {o % 9 // 3} dx {o % 9 % 3} of input channel {o % cin})" if kind == "shift" else "")
                                 + f": {out[b, y, xx, o]} != {want[b, y, xx, o]}")
    _record(plan, 64 if cout == 64 else 128, precision, 1)
    return out


def run_gemm(st, kind, M, N, K, bn, precision, seed, k32=False, with_bias=True):
    st.set_precision(precision)
    a, b, bias = gemm_case(kind, M, N, K, np.random.default_rng(seed), with_bias)
    out, tail, plan = st.gemm(a, b, bn, bias=bias, k32=k32, guard=GUARD)
    what = f"{kind} {precision} {M}x{N}x{K} bn {bn}{' k32' if k32 else ''} plan {plan}"
    assert (tail == GUARD).all(), f"{what}: write past row M"
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    full = ref + (bias if bias is not None else 0)
    if kind == "random":
        r = ratio(out, full, bound(a, b, full, precision, False))
        WORST[precision, "gemm"] = max(WORST.get((precision, "gemm"), 0.0), r)
        assert r <= 1, f"{what}: |err| / bound = {r:.2f}"
    else:
        bad = np.argwhere(out != full)
        assert not len(bad), f"{what}: {len(bad)} outputs differ, first at {tuple(bad[0])}"
    _record(plan, bn, precision, 3 if k32 else 0)
    return out


PRECISIONS = ["exact", "fast"]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cin,cout", SP_CONVS)
def test_conv3x3(st, cin, cout, precision):
    """Every SuperPoint (cin, cout) pair, with and without pool, at 2 x 2 up to 37 x 45 (odd sizes included), two images: designed,
    shift and random cases."""
    for i, (H, W) in enumerate(CONV_HW):
        for pool in (False, True):
            for kind in ("designed", "shift", "random"):
                run_conv(st, kind, 2, H, W, cin, cout, pool, precision, seed=100 * i + 2 * pool + len(kind))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cin,cout", SP_CONVS)
def test_conv3x3_persistent(st, cin, cout, precision):
    """More tiles than SMs (2 x 96 x 100: 168 tiles per n-tile), so CTAs carry their rings and barrier phases across tiles."""
    pool = cout != 128
    for kind in ("designed", "random"):
        run_conv(st, kind, 2, 96, 100, cin, cout, pool, precision, seed=7 + len(kind))


# (M, N, K, bn, k32): M off the 128 grid, N = 65 (the scalar store branch, as convPb), N = 1024 at BN 128 (8 n-tiles: the grid is cut to a
# multiple of 8), more than 2 x SMs tiles, K too long for resident weights, 32-wide K blocks, and K = 128 (resident in EXACT)
GEMM_SHAPES = [
    (300, 200, 128, 64, False), (128, 256, 576, 256, False), (1000, 768, 512, 128, False), (128, 128, 64, 128, False),
    (300, 65, 256, 128, False), (2181, 1024, 256, 128, False), (34637, 128, 256, 128, False), (1000, 128, 2048, 128, False),
    (1000, 512, 512, 256, True), (777, 256, 256, 256, True), (1000, 512, 256, 256, False), (1000, 512, 512, 256, False),
    (500, 256, 128, 128, False), (1000, 256, 512, 128, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("m,n,k,bn,k32", GEMM_SHAPES)
def test_tensor_core_gemm(st, m, n, k, bn, k32, precision):
    """C = A B^T + bias through the production launch: random operands against the per-element bound, designed ones bitwise."""
    for kind in ("random", "designed"):
        run_gemm(st, kind, m, n, k, bn, precision, seed=m + n + k, k32=k32)


def _case_plans(sms):
    """{(bn, split, conv, resb, sa, sb)} the GPU cases of this file launch on `sms` SMs."""
    out = set()
    for split in (True, False):
        for cin, cout in SP_CONVS:
            bn = 64 if cout == 64 else 128
            for B, H, W in [(2, h, w) for h, w in CONV_HW] + [(2, 96, 100)]:
                mt = B * -(-W // 16) * -(-H // 8)
                resb, sa, sb, _, _ = _plan(1, bn, split, True, 9 * cin // 64, mt, -(-cout // bn), sms)
                out.add((bn, split, 1, resb, sa, sb))
        for m, n, k, bn, k32 in GEMM_SHAPES:
            conv = 3 if k32 else 0
            resb, sa, sb, _, _ = _plan(conv, bn, split, True, k // (32 if k32 else 64), -(-m // 128), -(-n // bn), sms)
            out.add((bn, split, conv, resb, sa, sb))
    return out


@pytest.mark.parametrize("sms", [114, 132])
def test_cases_reach_every_production_plan(sms):
    """The GPU cases are chosen so that, on an H100 PCIe (114 SMs) or SXM (132 SMs), they launch every plan a production call site
    can: test_coverage_of_production_plans then checks the plans that actually ran."""
    missing = production_plans(sms) - _case_plans(sms)
    assert not missing, sorted(missing)


@pytest.mark.gpu
def test_gemm_without_bias(st):
    for precision in PRECISIONS:
        run_gemm(st, "random", 300, 65, 256, 128, precision, seed=5, with_bias=False)


@pytest.mark.gpu
def test_bitwise_repeatable(st):
    """Two identical calls give identical bits: a persistent RESB GEMM (FAST, 8 n-tiles on a cut grid) and a persistent non-RESB conv
    (EXACT 128 -> 256)."""
    st.set_precision("fast")
    a, b, bias = gemm_case("random", 2181, 1024, 256, np.random.default_rng(11), True)
    r1, r2 = (st.gemm(a, b, 128, bias=bias, guard=GUARD) for _ in range(2))
    assert r1[2][0] == 1 and np.array_equal(r1[0], r2[0])
    st.set_precision("exact")
    x, w, bias = conv_case("random", 2, 96, 100, 128, 256, np.random.default_rng(12))
    c1, c2 = (st.conv3x3(x, w, bias, False, guard=GUARD, sentinel=SENTINEL) for _ in range(2))
    assert c1[2][0] == 0 and np.array_equal(c1[0], c2[0])


@pytest.mark.gpu
def test_coverage_of_production_plans():
    """Every (bn, split, conv, resb, sa, sb) the production call sites produce on this device has been run by the tests above."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    want = production_plans(sms)
    print(f"{len(EXECUTED)} plans executed on {sms} SMs:", sorted(EXECUTED))
    missing = want - EXECUTED
    assert not missing, f"production plans never executed: {sorted(missing)}"


@pytest.mark.gpu
def test_report_error_ratios():
    """The largest |err| / bound of the random cases, per precision and kernel mode (recorded in the header of this file)."""
    import torch
    props = torch.cuda.get_device_properties(0)
    print(f"{props.name}: largest |err| / bound", {f"{p} {k}": f"{v:.3g}" for (p, k), v in sorted(WORST.items())})
    assert all(v <= 1 for v in WORST.values())
