"""The 16 x 16-pixel tiles of the SuperPoint 64 -> 64 channel 3x3 convolutions (csrc/gemm.cuh CONV mode 2) against float64 references
and, bitwise, against the 8 x 16-pixel tiles (mode 1) on the same inputs.

Mode 2 runs every output element through the same wgmma sequence as mode 1 ((dx, channel block), dy, k16, then hi * hi, hi * lo, lo * hi),
so the two tile shapes must agree bit for bit.  run_conv3 picks mode 2 by shape (conv3x3.cuh conv_mode): 64 output channels and at
least two 16 x 16 tiles per SM, in either precision; the GPU cases pass the tile shape explicitly through the self-test
entry (dimb_selftest_conv3x3), and one case checks the production choice.  The reference, the bound model and the case kinds (designed,
shift, random) are those of test_gemm_conv_kernel.py.
"""
import numpy as np
import pytest

import test_gemm_conv_kernel as K

STG2_BYTES = 2 * 64 * 20 * 4  # mode 2 accumulator staging of the two consumer warpgroups: [64 rows][16 + 4 columns] fp32 each
BENCH_SHAPES = [(66, 1024, 1024), (66, 512, 512)]  # conv1b; conv2a and conv2b of the bench.py step
MANY = (1, 2, 3, 8, 40, 131, 264, 400, 67584, 135168)


def _geometry2(split):
    """A-stage and B-tile pitches of PersGeom<64, split, 2>: one (16 + 2) x 16-pixel box of 128-byte rows per plane."""
    pl = 2 if split else 1
    return pl * (-(-(18 * 16 * 128) // 1024) * 1024), pl * 64 * 128


def _mode(cout, B, H, W, sms):
    from dim_b200 import _native
    return _native.conv_mode(cout, B, H, W, sms)


def production_plans2(sms):
    """{(bn, split, conv, resb, sa, sb)} of the mode 2 launches run_conv3 can make on `sms` SMs."""
    out = set()
    for split in (True, False):
        for mt in MANY:
            if _mode(64, mt, 16, 16, sms) == 2:  # mt images of one tile each
                resb, sa, sb, _, _ = K._plan(2, 64, split, True, 9, mt, 1, sms)
                out.add((64, split, 2, resb, sa, sb))
    return out


# ------------------------------------------------------------------ CPU: plans and the selection rule
@pytest.mark.parametrize("sms", [114, 132])
def test_mode2_plan_invariants(sms):
    """The rules of test_plan_invariants_at_every_call_site for mode 2, with its smaller staging buffer: shared memory within the opt-in
    limit and equal to the geometry, at least one A stage, at least three B slots (one per dy tap of a stage), the mbarriers in their 1 KB, RESB
    only on a grid pinned to the n-tile, atom-aligned pitches."""
    for split in (True, False):
        astage, btile = _geometry2(split)
        assert astage % 1024 == 0 and btile % 1024 == 0
        for mt in MANY:
            resb, sa, sb, smem, grid = K._plan(2, 64, split, True, 9, mt, 1, sms)
            what = f"split {split} tiles {mt} on {sms} SMs"
            slots = 9 if resb else sb
            assert smem == sa * astage + slots * btile + 2048 + STG2_BYTES, what
            assert smem <= K.SMEM_MAX, what
            assert 1 <= sa <= 8, what
            if not resb:
                assert sb >= 3, what
            assert 8 * (2 * sa + 2 * slots) <= 1024, what
            assert 1 <= grid <= min(sms, mt), what
            if resb:
                assert sb == 0 and sa >= 2, what


def test_mode2_plan_table():
    """EXACT: two 36 KB-per-plane A stages and four B slots, weights streamed; FAST: weights resident, three A stages."""
    assert K._plan(2, 64, True, True, 9, 135168, 1, 132)[:3] == (False, 2, 4)
    assert K._plan(2, 64, False, True, 9, 135168, 1, 132)[:3] == (True, 3, 0)


def test_mode2_refuses_other_widths():
    from dim_b200 import _native
    for args in [(2, 128, 1, 1, 9, 1, 1, 132), (2, 256, 1, 1, 9, 1, 1, 132), (1, 256, 1, 1, 9, 1, 1, 132), (3, 128, 1, 1, 8, 1, 1, 132)]:
        with pytest.raises(_native.DimbError):
            _native.gemm_plan(*args)


@pytest.mark.parametrize("sms", [114, 132])
def test_tile_selection(sms):
    """16 x 16 tiles for the 64-channel layers when they give at least two tiles per SM: the bench shapes (and image-set batches) take
    them; every size of test_gemm_conv_kernel.py and the 128-channel layers keep 8 x 16."""
    for B, H, W in BENCH_SHAPES + [(8, 1024, 1024), (4, 768, 1024)]:
        assert _mode(64, B, H, W, sms) == 2, (B, H, W)
        assert _mode(128, B, H, W, sms) == 1, (B, H, W)
    for H, W in K.CONV_HW + [(96, 100)]:
        assert _mode(64, 2, H, W, sms) == 1, (H, W)
    # the boundary: one tile row of exactly 2 x sms tiles (the last one partial), and one tile fewer
    assert _mode(64, 1, 16, 16 * 2 * sms - 15, sms) == 2
    assert _mode(64, 1, 16, 16 * (2 * sms - 1), sms) == 1


@pytest.mark.parametrize("sms", [114, 132])
def test_cases_reach_every_mode2_plan(sms):
    """The GPU cases below launch every plan mode 2 has in production (test_coverage_of_mode2_plans checks the ones that ran)."""
    missing = production_plans2(sms) - _case_plans2(sms)
    assert not missing, sorted(missing)


# ------------------------------------------------------------------ GPU
EXECUTED2 = set()
# (B, H, W): partial tiles in both directions (H mod 16 != 0, odd W), a single partial tile, and more 16 x 16 tiles than SMs (160)
TILE16_HW = [(2, 37, 45), (1, 5, 7), (3, 33, 17), (2, 115, 155)]


def _case_plans2(sms):
    out = set()
    for split in (True, False):
        for B, H, W in TILE16_HW:
            resb, sa, sb, _, _ = K._plan(2, 64, split, True, 9, B * -(-W // 16) * -(-H // 16), 1, sms)
            out.add((64, split, 2, resb, sa, sb))
    return out


@pytest.fixture(scope="module")
def st():
    return K._selftest()


def run_tiles(st, kind, B, H, W, pool, precision, seed, check_reference=True):
    """One 64 -> 64 conv case on 16 x 16 and on 8 x 16 tiles: both complete and bitwise equal, the 16 x 16 output checked against the
    float64 reference as test_gemm_conv_kernel.run_conv checks it."""
    st.set_precision(precision)
    x, w, bias = K.conv_case(kind, B, H, W, 64, 64, np.random.default_rng(seed))
    out16, tail16, plan16, mode16 = st.conv3x3_tiles(x, w, bias, pool, 16, guard=K.GUARD, sentinel=K.SENTINEL)
    out8, tail8, _, mode8 = st.conv3x3_tiles(x, w, bias, pool, 8, guard=K.GUARD, sentinel=K.SENTINEL)
    what = f"{kind} {precision} B{B} {H}x{W} pool {pool} plan {plan16}"
    assert (mode16, mode8) == (2, 1), what
    assert (tail16 == K.SENTINEL).all() and (tail8 == K.SENTINEL).all(), f"{what}: write past the last output image"
    assert (out16 != K.SENTINEL).all(), f"{what}: {int((out16 == K.SENTINEL).sum())} outputs not written"
    bad = np.argwhere(out16.view(np.uint32) != out8.view(np.uint32))
    if len(bad):
        b, y, xx, o = bad[0]
        raise AssertionError(f"{what}: {len(bad)} outputs differ from the 8 x 16 tiles, first at image {b} ({y}, {xx}) channel {o}: "
                             f"{out16[b, y, xx, o]} != {out8[b, y, xx, o]}")
    if check_reference:
        ref, tol = K.conv_reference(x, w, bias, pool, precision)
        if kind == "random":
            r = K.ratio(out16, ref, tol)
            assert r <= 1, f"{what}: |err| / bound = {r:.2f}"
        else:
            want = ref if precision == "exact" else ref.astype(np.float16).astype(np.float64)
            bad = np.argwhere(out16 != want)
            assert not len(bad), f"{what}: {len(bad)} outputs differ from the reference, first at {tuple(bad[0])}"
    resb, sa, sb, smem, grid = plan16
    assert resb in (0, 1) and sa >= 1 and smem <= K.SMEM_MAX and grid >= 1, what
    EXECUTED2.add((64, precision == "exact", 2, bool(plan16[0]), plan16[1], plan16[2]))
    return out16


@pytest.mark.gpu
@pytest.mark.parametrize("precision", K.PRECISIONS)
@pytest.mark.parametrize("pool", [False, True])
def test_tile16_matches_reference_and_8x16(st, precision, pool):
    """Designed, shift and random cases at partial-tile sizes and at more tiles than SMs."""
    for i, (B, H, W) in enumerate(TILE16_HW):
        for kind in ("designed", "shift", "random"):
            run_tiles(st, kind, B, H, W, pool, precision, seed=300 + 10 * i + 2 * pool + len(kind))


@pytest.mark.gpu
def test_production_choice(st):
    """Through the production entry (tile 0): at two tiles per SM a 64 -> 64 conv runs on 16 x 16 tiles, bitwise as 8 x 16 does, in
    both precisions; one tile fewer and it stays on 8 x 16."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B, H, W = 1, 16, 16 * 2 * sms - 15  # exactly 2 x sms tiles, the last one partial
    x, w, bias = K.conv_case("random", B, H, W, 64, 64, np.random.default_rng(5))
    for precision, plan in (("exact", (0, 2, 4)), ("fast", (1, 3, 0))):
        st.set_precision(precision)
        out0, _, plan0, mode0 = st.conv3x3_tiles(x, w, bias, True, 0, guard=K.GUARD, sentinel=K.SENTINEL)
        out8, _, _, _ = st.conv3x3_tiles(x, w, bias, True, 8, guard=K.GUARD, sentinel=K.SENTINEL)
        assert mode0 == 2 and plan0[:3] == plan, precision
        assert np.array_equal(out0.view(np.uint32), out8.view(np.uint32)), precision
        assert st.conv3x3_tiles(x[:, :, :W - 16], w, bias, True, 0, guard=K.GUARD, sentinel=K.SENTINEL)[3] == 1, precision


@pytest.mark.gpu
def test_tile16_bitwise_repeatable(st):
    st.set_precision("exact")
    x, w, bias = K.conv_case("random", 2, 115, 155, 64, 64, np.random.default_rng(13))
    r1, r2 = (st.conv3x3_tiles(x, w, bias, True, 16, guard=K.GUARD, sentinel=K.SENTINEL)[0] for _ in range(2))
    assert np.array_equal(r1.view(np.uint32), r2.view(np.uint32))


@pytest.mark.gpu
def test_coverage_of_mode2_plans():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    missing = production_plans2(sms) - EXECUTED2
    print(f"mode 2 plans executed on {sms} SMs:", sorted(EXECUTED2))
    assert not missing, f"mode 2 production plans never executed: {sorted(missing)}"
