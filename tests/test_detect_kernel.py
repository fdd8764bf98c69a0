"""Keypoint detection (csrc/detect.cuh) and the SuperPoint head kernels (csrc/sp_head.cuh) on their own, against exact references.

Every extractor ends in the same machinery: simple_nms (the bit-mask kernel sp_nms2_kernel for radii 1..5, the first cut sp_nms_kernel
for radius 0 and radii 6..8), threshold + border compaction in row-major order, and top-k selection
(radix select, a tie rank over blocks of 1024 candidates, a bitonic sort).  The self-test library runs them through the launch helpers
SuperPoint and ALIKED call (dimb_selftest_detect), with every output buffer starting as a sentinel and followed by a tail, so unwritten
slots and stray writes both show.  These are exact operations, so the GPU tests compare bitwise:
  NMS         oracle.superpoint.simple_nms (the reference's float32 max-pools);
  compaction  np.nonzero((nms > thr) & inside_border), row-major;
  selection   every candidate in row-major order if K < 0 or C <= K, else np.lexsort((idx, -score))[:K]: the K largest, ties at the
              cut broken by the smaller pixel index, ordered by score descending, then index ascending.
The head kernels get float bounds: sp_softmax_d2s_kernel against a float64 softmax of the fp32 logits, sp_describe_kernel against
oracle.superpoint.sample_descriptors run in float64 on the float64-normalised dense map.

Designed score maps, each for what it forces:
  softmax_like  a softmax of random 65-way logits, depth-to-space: what production sees.
  uniform       random in (0, 1): few ties.
  quantized     8 levels k / 8: plateaus, equal neighbours everywhere, many ties at the top-k cut.
  chains        peaks rising by one step every r pixels along rows, away from a tile edge or the image border (and peaks r + 1 ..
                2r + 1 apart): a pixel's final mask depends on the score 5r away, through suppression in round one and new maxima
                in round two, so a halo of 5r - 1 or a single round gets these wrong.
  chains_t      the same along columns, across the horizontal tile edges.
  plateau_edge  a constant block straddling every tile corner.
  constant      one value everywhere.
  subnormal     values near 1e-40 next to normal ones (softmax scores do underflow, and the build does not flush to zero).
The CPU tests show the designs are sharp: a tiled NMS with a 5r - 1 halo, a one-round NMS, top-k with the opposite tie order or a tie
rank restarting every 1024 candidates, and a >= threshold all differ from the references on them."""
import numpy as np
import pytest
import torch

SENT = -777.0                                  # every output buffer before the call
ISENT = int(np.float32(SENT).view(np.int32))   # ... its int buffers hold the sentinel's bits
SMEM_MAX = 232448                              # opt-in shared memory per block on sm_90
SEL_BLOCK = 1024                               # candidates per tie-rank block of sp_select_kernel
DESIGNS = ["softmax_like", "uniform", "quantized", "chains", "chains_t", "plateau_edge", "constant", "subnormal"]
# (B, H, W): below one tile, one tile, tile edges in both axes, long thin maps, an ALIKED-style size not a multiple of 8, 4095 pixels
# and 4 * 4096 + 7 pixels (compaction chunk edges)
NMS_SHAPES = [(1, 16, 16), (1, 64, 64), (1, 72, 136), (1, 16, 1000), (1, 1000, 16), (1, 203, 260), (1, 63, 65), (1, 37, 443)]
# Head bounds, against float64 references of the same fp32 inputs.
#   softmax: |gpu - ref| <= SM_REL (1 + |l - max l|) ref + 2^-126.  The fp32 difference l - max l rounds by up to half an ulp, which
#   exp turns into a relative error of |l - max l| 2^-24; expf (2 ulp), the 65-term sum (7 levels, all terms positive) and the division
#   add about 8 ulp = 2^-21.  2^-126 absolute: a result below the smallest normal is not judged relatively.
#   describe: |gpu - ref| <= DESC_ABS + DESC_COORD max(w, h) per element of the unit descriptors.  The grid coordinates are computed in
#   fp32 at magnitudes up to max(w, h), about 2 ulp = max(w, h) 2^-22 off, which moves each component by that times the difference of
#   two unit vectors' components (below 1); the two normalisations and the bilinear sum add a few 2^-24 to each component.
# Largest measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: softmax 0.65 of the relative term (random logits, sd 5);
# descriptors 6.6e-6 on 192 x 256 cells (0.1 of the bound, align_corners) and 1.4e-7 on the 2 x 2 and 3 x 5 grids.
SM_REL = 2.0 ** -21
DESC_ABS = 2e-6
DESC_COORD = 2.0 ** -22


# ------------------------------------------------------------------ references
def ref_nms(scores, r):
    """oracle.superpoint.simple_nms per image: [B][H][W] float32."""
    from oracle import superpoint as o_sp
    return np.stack([o_sp.simple_nms(torch.from_numpy(np.ascontiguousarray(s)), r).numpy() for s in scores])


def _pool(x, r):
    """(2r + 1)^2 window max, separable, -inf outside the map."""
    H, W = x.shape
    p = np.full((H, W + 2 * r), -np.inf, x.dtype)
    p[:, r:r + W] = x
    m = p[:, :W].copy()
    for d in range(1, 2 * r + 1):
        m = np.maximum(m, p[:, d:d + W])
    q = np.full((H + 2 * r, W), -np.inf, x.dtype)
    q[r:r + H] = m
    o = q[:H].copy()
    for d in range(1, 2 * r + 1):
        o = np.maximum(o, q[d:d + H])
    return o


def np_nms(s, r, rounds=2):
    """An independent numpy simple_nms of one [H][W] map: max_mask, then `rounds` suppression rounds (the reference runs two)."""
    z = np.zeros_like(s)
    mm = s == _pool(s, r)
    for _ in range(rounds):
        sup = _pool(mm.astype(np.float32), r) > 0
        ss = np.where(sup, z, s)
        mm = mm | ((ss == _pool(ss, r)) & ~sup)
    return np.where(mm, s, z)


def tiled_nms(s, r, tile, halo):
    """np_nms computed tile by tile, each on its tile plus `halo` pixels (cut at the image): the kernels' decomposition."""
    H, W = s.shape
    out = np.zeros_like(s)
    for y0 in range(0, H, tile):
        for x0 in range(0, W, tile):
            ya, xa = max(0, y0 - halo), max(0, x0 - halo)
            part = np_nms(s[ya:min(H, y0 + tile + halo), xa:min(W, x0 + tile + halo)], r)
            out[y0:y0 + tile, x0:x0 + tile] = part[y0 - ya:y0 - ya + tile, x0 - xa:x0 - xa + tile]
    return out


def ref_candidates(nms, thr, border, ge=False):
    """Pixel indices and scores of nms > thr (>= with ge) at least `border` pixels inside, row-major."""
    H, W = nms.shape
    inside = np.zeros((H, W), bool)
    inside[border:H - border, border:W - border] = True
    idx = np.flatnonzero(((nms >= thr) if ge else (nms > thr)) & inside).astype(np.int32)
    return idx, nms.reshape(-1)[idx]


def ref_select(idx, sc, K):
    """The top-k rule of sp_select_kernel."""
    if K < 0 or len(idx) <= K:
        return idx, sc
    o = np.lexsort((idx, -sc.astype(np.float64)))[:K]
    return idx[o], sc[o]


def select_larger_index_ties(idx, sc, K):
    """Mutant: ties at the cut broken by the larger pixel index."""
    if K < 0 or len(idx) <= K:
        return idx, sc
    o = np.lexsort((-idx.astype(np.int64), -sc.astype(np.float64)))[:K]
    o = o[np.lexsort((idx[o], -sc[o].astype(np.float64)))]
    return idx[o], sc[o]


def select_blockwise_tie_rank(idx, sc, K):
    """Mutant of sp_select_kernel: the rank among ties at the cut restarts in every block of 1024 candidates (s_tiepos not carried), so
    each block writes its first ties into the same slots and the last block's win."""
    if K < 0 or len(idx) <= K:
        return idx, sc
    T = np.sort(sc)[::-1][K - 1]
    greater = np.flatnonzero(sc > T)
    need = K - len(greater)
    slots = {}
    for b0 in range(0, len(idx), SEL_BLOCK):
        ties = b0 + np.flatnonzero(sc[b0:b0 + SEL_BLOCK] == T)
        for rank, i in enumerate(ties[:need]):
            slots[rank] = i
    chosen = np.concatenate([greater, np.array([slots[k] for k in sorted(slots)], np.int64)]).astype(np.int64)
    o = chosen[np.lexsort((idx[chosen], -sc[chosen].astype(np.float64)))]
    return idx[o], sc[o]


# ------------------------------------------------------------------ designed score maps
def design(name, H, W, r, tile, rng):
    """One positive float32 [H][W] score map; `tile` is the NMS tile the kernel under test runs with."""
    if name == "softmax_like":
        hc, wc = -(-H // 8), -(-W // 8)
        lg = rng.normal(0.0, 2.0, (hc * wc, 65))
        lg[:, 64] += 4.0
        p = np.exp(lg - lg.max(1, keepdims=True))
        p = (p / p.sum(1, keepdims=True))[:, :64].astype(np.float32)
        return np.ascontiguousarray(p.reshape(hc, wc, 8, 8).transpose(0, 2, 1, 3).reshape(8 * hc, 8 * wc)[:H, :W])
    if name == "uniform":
        return rng.uniform(2.0 ** -24, 1.0, (H, W)).astype(np.float32)
    if name == "quantized":
        return (rng.integers(1, 9, (H, W)) / 8.0).astype(np.float32)
    if name == "constant":
        return np.full((H, W), 0.5, np.float32)
    if name == "subnormal":
        s = rng.uniform(1e-41, 1e-39, (H, W))
        normal = ((np.arange(H)[:, None] // 8 + np.arange(W)[None] // 8) % 2 == 1) & (np.arange(H)[:, None] >= H // 4)
        return np.where(normal, rng.uniform(0.0, 1.0, (H, W)), s).astype(np.float32)
    if name == "plateau_edge":
        s = rng.uniform(0.0, 0.5, (H, W))
        corners = [(y, x) for y in range(0, H, tile) for x in range(0, W, tile)] + [(H // 2, W // 2)]
        for y, x in corners:
            s[max(0, y - r - 1):y + r + 2, max(0, x - r - 1):x + r + 2] = 0.75
        return s.astype(np.float32)
    if name == "chains":
        return chains(H, W, r, tile, rng)
    if name == "chains_t":
        return np.ascontiguousarray(chains(W, H, r, tile, rng).T)
    raise ValueError(name)


def chains(H, W, r, tile, rng):
    """Background below 0.01 with ramps of six peaks along rows: the lowest sits on the last (first) column of a tile or on the left
    (right) border, and each next one is r pixels further right (left) and 0.08 higher, so the final mask of the lowest depends on the
    highest, 5r away in the next tile.  Ramps in one row start two tiles apart (a ramp is longer than a 32-pixel tile at r >= 7), rows
    4r + 3 apart; between some of them, peaks r + 1 .. 2r + 1 apart (suppressed in round one, maxima in round two)."""
    s = rng.uniform(0.001, 0.01, (H, W))
    step = max(r, 1)

    def ramp(y, x, dx, gaps):
        for k, d in enumerate(np.cumsum([0] + list(gaps))):
            if 0 <= x + dx * d < W:
                s[y, x + dx * d] = 0.3 + 0.08 * k

    rows = sorted({0, H - 1} | set(range(2 * r + 1, H, 4 * r + 3)))
    for i, y in enumerate(rows):
        right = i % 2 == 0
        starts = ([0] + list(range(tile - 1, W, tile))) if right else ([W - 1] + list(range(tile, W, tile)))
        for x in starts[(i // 2) % 2::2]:
            ramp(y, x, 1 if right else -1, [step] * 5)
        if i % 3 == 2 and y + 2 * r + 1 < H:
            ramp(y + 2 * r + 1, int(rng.integers(0, W)), 1, rng.integers(r + 1, 2 * r + 2, 5))
    return s.astype(np.float32)


def _tile(r, cut):
    from dim_b200 import _native
    return _native.nms_plan(r, cut)[1]


# ------------------------------------------------------------------ CPU: the references agree and the designs are sharp
PLAN_TABLE = {  # (r, cut) -> (kernel, tile, threads, smem bytes)
    **{(r, 1): (1, 64, 1024, b) for r, b in enumerate([74880, 99900, 128520, 160740, 196560])},
    **{(r, 1): (1, 32, 1024, b) for r, b in zip(range(5, 9), [122508, 154008, 189108, 227808])},
    **{(r, 2): (2, 64, 512, b) for r, b in zip(range(1, 6), [72816, 82656, 92496, 130624, 143184])},
}


def test_nms_plan_table():
    """The plans of both kernels at radii 0..8 are pinned, fit the opt-in shared memory, follow the kernels' layouts, and cut 0 (the
    production choice) takes the bit-mask kernel exactly for radii 1..5."""
    from dim_b200 import _native
    for (r, cut), want in PLAN_TABLE.items():
        got = _native.nms_plan(r, cut)
        assert got == want, (r, cut, got)
        assert got[3] <= SMEM_MAX
        if cut == 1:  # five planes of S x (S | 1): four float, two byte masks
            S = got[1] + 10 * r
            assert got[3] == S * (S | 1) * 18
        assert _native.nms_plan(r, 0) == PLAN_TABLE[r, 2 if 1 <= r <= 5 else 1]
    assert _native.nms_plan(5, 1)[1] == 32 and (64 + 50) * (115) * 18 > SMEM_MAX  # radius 5 needs the 32-pixel tile


@pytest.mark.parametrize("r, cut", [(-1, 1), (9, 1), (9, 0), (0, 2), (6, 2), (8, 2), (3, 3), (3, -1)])
def test_nms_plan_refuses(r, cut):
    from dim_b200 import _native
    with pytest.raises(_native.DimbError, match=r"code -3\)"):
        _native.nms_plan(r, cut)


def test_entries_refuse_a_null_context():
    """Every new entry checks its arguments before any CUDA call."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    buf = np.zeros(64 * 1024, np.float32)
    p = _native._ptr(buf)
    assert lib.dimb_selftest_detect(None, p, 1, 16, 16, 3, 0, 0.0, None, 0, -1, 256, SENT, *([p] * 7), None) == -3
    assert lib.dimb_selftest_sp_softmax(None, p, 1, 2, 2, SENT, p) == -3
    assert lib.dimb_selftest_sp_describe(None, p, p, p, p, 1, 2, 2, 4, 0, SENT, p, p, p) == -3
    assert lib.dimb_selftest_nms_plan(3, 0, None) == -3


@pytest.mark.parametrize("name", DESIGNS)
def test_references_agree(name):
    """oracle simple_nms (torch max-pools) and the numpy simple_nms agree bitwise on every design at every radius."""
    for r in range(9):
        for H, W in [(72, 136), (37, 45)]:
            s = design(name, H, W, r, 32 if r >= 5 else 64, np.random.default_rng(r))
            assert np.array_equal(ref_nms(s[None], r)[0].view(np.uint32), np_nms(s, r).view(np.uint32)), (name, r, H, W)


@pytest.mark.parametrize("r", range(1, 9))
def test_chains_reach_the_halo_edge(r):
    """On chains, the tiled NMS equals the global one with the kernels' 5r halo and differs with 5r - 1, on every tile the kernels use
    at radius r, and one suppression round differs from two."""
    for cut in ((1, 2) if r <= 5 else (1,)):
        tile = _tile(r, cut)
        for name in ("chains", "chains_t"):
            s = design(name, 2 * tile + 8, 2 * tile + 8, r, tile, np.random.default_rng(r))
            ref = np_nms(s, r)
            assert np.array_equal(tiled_nms(s, r, tile, 5 * r), ref)
            assert not np.array_equal(tiled_nms(s, r, tile, 5 * r - 1), ref), f"{name} radius {r}, tile {tile}: halo 5r - 1 not reached"
            assert not np.array_equal(np_nms(s, r, rounds=1), ref), f"{name} radius {r}: one round suffices"


def test_tie_mutants_differ_on_quantized():
    """With ties spanning more than one 1024-candidate block at the cut, the opposite tie order and a tie rank restarting per block both
    change the selection."""
    s = design("quantized", 128, 128, 0, 64, np.random.default_rng(0))
    idx, sc = ref_candidates(ref_nms(s[None], 0)[0], 0.0, 0)
    K = int((sc > 0.5).sum()) + 1500  # the cut falls inside the 0.5 level, whose ~2048 ties spread over all 16 blocks
    assert (sc == 0.5).sum() > 1500 and len(idx) == 128 * 128
    want = ref_select(idx, sc, K)
    for mutant in (select_larger_index_ties, select_blockwise_tie_rank):
        got = mutant(idx, sc, K)
        assert not (np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])), mutant.__name__


def test_threshold_mutant_differs():
    """nms >= thr instead of nms > thr changes the candidates when the threshold equals a score."""
    nms = ref_nms(design("quantized", 72, 136, 2, 64, np.random.default_rng(1))[None], 2)[0]
    assert not np.array_equal(ref_candidates(nms, 0.5, 0)[0], ref_candidates(nms, 0.5, 0, ge=True)[0])


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def st():
    from dim_b200 import _native
    return _native.SelfTest(0)


_REF = {}


def _case(shape, names, r, tile, seed):
    """Scores [B][H][W] (image b from design names[b]) and their reference NMS, cached across kernels."""
    key = (shape, tuple(names), r, tile, seed)
    if key not in _REF:
        B, H, W = shape
        s = np.stack([design(n, H, W, r, tile, np.random.default_rng(seed + 7 * b)) for b, n in enumerate(names)])
        _REF[key] = s, ref_nms(s, r)
    return _REF[key]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_detect(out, nms_ref, thr, border, K, cap, what):
    """nms bitwise; per image the candidates, then the selection, bitwise, with every slot past the valid ones untouched; tails
    untouched.  Returns the candidate counts."""
    B = nms_ref.shape[0]
    assert np.array_equal(_bits(out["nms"]), _bits(nms_ref)), f"{what}: nms differs at {np.argwhere(_bits(out['nms']) != _bits(nms_ref))[:5]}"
    thr = np.broadcast_to(np.asarray(thr, np.float32), (B,))
    counts = []
    for b in range(B):
        idx, sc = ref_candidates(nms_ref[b], thr[b], border)
        C = len(idx)
        counts.append(C)
        assert out["cand_count"][b] == C, f"{what}: image {b} candidates {out['cand_count'][b]} != {C}"
        assert np.array_equal(out["cand_idx"][b, :C], idx), f"{what}: image {b} candidate indices"
        assert np.array_equal(_bits(out["cand_score"][b, :C]), _bits(sc)), f"{what}: image {b} candidate scores"
        assert (out["cand_idx"][b, C:] == ISENT).all() and (out["cand_score"][b, C:] == SENT).all(), f"{what}: image {b} stray candidates"
        si, ss = ref_select(idx, sc, K)
        n = min(len(si), cap)
        assert out["sel_count"][b] == len(si), f"{what}: image {b} selected {out['sel_count'][b]} != {len(si)}"
        assert np.array_equal(out["sel_idx"][b, :n], si[:n]), f"{what}: image {b} selected indices"
        assert np.array_equal(_bits(out["sel_score"][b, :n]), _bits(ss[:n])), f"{what}: image {b} selected scores"
        assert (out["sel_idx"][b, n:] == ISENT).all() and (out["sel_score"][b, n:] == SENT).all(), f"{what}: image {b} stray selections"
    for k in ("nms", "cand_score", "sel_score"):
        assert (out[k + "_tail"] == SENT).all(), f"{what}: write past {k}"
    for k in ("cand_count", "cand_idx", "sel_idx", "sel_count"):
        assert (out[k + "_tail"] == ISENT).all(), f"{what}: write past {k}"
    return counts


NMS_KERNELS = [(1, r) for r in range(9)] + [(2, r) for r in range(1, 6)] + [(0, r) for r in (0, 3, 5, 6, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("cut, r", NMS_KERNELS, ids=[f"cut{c}-r{r}" for c, r in NMS_KERNELS])
def test_nms(st, cut, r):
    """One simple_nms kernel at one radius, over every shape and design (and a batch of three designs), bitwise; candidates and the
    keep-all selection checked on the way.  cut 0 checks the production dispatch."""
    from dim_b200 import _native
    plan = _native.nms_plan(r, cut)
    tile = plan[1]
    cases = [(shape, [n]) for shape in NMS_SHAPES for n in DESIGNS]
    cases += [((3, 72, 136), ["chains", "quantized", "subnormal"]), ((3, 203, 260), ["softmax_like", "plateau_edge", "constant"])]
    for i, (shape, names) in enumerate(cases):
        s, nms_ref = _case(shape, names, r, tile, i)
        out = st.detect(s, r, cut, thr=0.0, border=0, K=-1, cap=shape[1] * shape[2], sentinel=SENT)
        assert out["plan"] == plan
        check_detect(out, nms_ref, 0.0, 0, -1, shape[1] * shape[2], f"cut {cut} r {r} {shape} {names}")


@pytest.mark.gpu
def test_threshold_equal_to_a_score_and_per_image_thresholds(st):
    """A threshold equal to a score keeps only the strictly greater; thresholds read on the device (ALIKED's path) apply per image and
    replace the scalar one."""
    shape, names = (3, 203, 260), ["quantized", "quantized", "softmax_like"]
    s, nms_ref = _case(shape, names, 2, 64, 100)
    out = st.detect(s, 2, 0, thr=0.5, border=4, K=-1, cap=203 * 260, sentinel=SENT)
    check_detect(out, nms_ref, 0.5, 4, -1, 203 * 260, "thr 0.5")
    per = np.array([0.25, 0.625, 0.0005], np.float32)
    out = st.detect(s, 2, 0, thr=0.9, thr_per_image=per, border=2, K=300, cap=300, sentinel=SENT)
    check_detect(out, nms_ref, per, 2, 300, 300, "per-image thresholds")


@pytest.mark.gpu
def test_borders(st):
    """Border 0, 4, r, and one that leaves no candidate: count 0 and nothing written."""
    r = 3
    for shape in [(1, 63, 65), (2, 37, 443)]:
        s, nms_ref = _case(shape, ["softmax_like"] * shape[0], r, 64, 200)
        for border in (0, 4, r, min(shape[1], shape[2]) // 2 + 1):
            out = st.detect(s, r, 0, thr=0.0, border=border, K=1000, cap=1000, sentinel=SENT)
            counts = check_detect(out, nms_ref, 0.0, border, 1000, 1000, f"{shape} border {border}")
            if border > min(shape[1:]) // 2:
                assert counts == [0] * shape[0]


@pytest.mark.gpu
def test_top_k_sizes(st):
    """K = -1, 1, 1000, C - 1, C, C + 1 on SuperPoint-like maps, and K = 16384 with C much larger (r = 0 on 1024 x 768)."""
    shape = (2, 203, 260)
    s, nms_ref = _case(shape, ["softmax_like", "uniform"], 3, 64, 300)
    C = min(len(ref_candidates(nms_ref[b], 0.0005, 4)[0]) for b in range(2))
    assert 1000 < C < 16384
    for K in (-1, 1, 1000, C - 1, C, C + 1):
        cap = K if K > 0 else 203 * 260
        check_detect(st.detect(s, 3, 0, thr=0.0005, border=4, K=K, cap=cap, sentinel=SENT), nms_ref, 0.0005, 4, K, cap, f"K {K}")
    s, nms_ref = _case((1, 1024, 768), ["softmax_like"], 0, 64, 301)
    out = st.detect(s, 0, 0, thr=0.0, border=0, K=16384, cap=16384, sentinel=SENT)
    assert check_detect(out, nms_ref, 0.0, 0, 16384, 16384, "K 16384")[0] == 1024 * 768


@pytest.mark.gpu
def test_top_k_ties_and_radix_digits(st):
    """Ties at the cut spanning many 1024-candidate blocks (quantized, r = 0: every pixel a candidate), scores differing only in the
    lowest radix digit or only in the highest, at cuts inside a run of ties and at non-power-of-two K."""
    rng = np.random.default_rng(400)
    maps = {"quantized": design("quantized", 96, 160, 0, 64, rng)}
    low = np.float32(0.75).view(np.uint32) & np.uint32(0xFFFFFF00)
    maps["low digit"] = (low | rng.integers(0, 16, (96, 160)).astype(np.uint32)).view(np.float32)
    high = rng.integers(0x30, 0x40, (96, 160)).astype(np.uint32) << np.uint32(24)
    maps["high digit"] = (high | np.uint32(0x123456)).view(np.float32)
    for name, s in maps.items():
        nms_ref = ref_nms(s[None], 0)
        sc = np.sort(s.reshape(-1))[::-1]
        for K in (1, 777, 3001, 8191, 9000, 15360):
            assert (sc == sc[K - 1]).sum() > 1, f"{name} K {K}: the cut is not inside a run of ties"
            check_detect(st.detect(s[None], 0, 0, thr=0.0, border=0, K=K, cap=K, sentinel=SENT), nms_ref, 0.0, 0, K, K, f"{name} K {K}")


@pytest.mark.gpu
def test_keep_all_beyond_cap(st):
    """K = -1 with more candidates than slots: sel_count is the candidate count and nothing is written past cap."""
    s, nms_ref = _case((1, 64, 64), ["uniform"], 0, 64, 500)
    out = st.detect(s, 0, 0, thr=0.0, border=0, K=-1, cap=100, sentinel=SENT)
    check_detect(out, nms_ref, 0.0, 0, -1, 100, "K -1, cap 100")
    assert out["sel_count"][0] == 4096


@pytest.mark.gpu
def test_production_size(st):
    """As bench.py runs it: 2 x 2048 x 1536, r = 3, threshold 0.0005, border 4, K = 2048."""
    s, nms_ref = _case((2, 2048, 1536), ["softmax_like"] * 2, 3, 64, 600)
    out = st.detect(s, 3, 0, thr=0.0005, border=4, K=2048, cap=2048, sentinel=SENT)
    check_detect(out, nms_ref, 0.0005, 4, 2048, 2048, "production size")


@pytest.mark.gpu
def test_detect_refuses_bad_arguments(st):
    from dim_b200 import _native
    s = np.full((1, 16, 16), 0.5, np.float32)
    for kw in [dict(r=9), dict(r=6, cut=2), dict(r=0, cut=2), dict(r=3, cut=3), dict(r=3, K=0), dict(r=3, K=-2), dict(r=3, K=16385),
               dict(r=3, K=100, cap=99), dict(r=3, thr=-0.5), dict(r=3, thr=float("nan")), dict(r=3, border=-1),
               dict(r=3, thr_per_image=[-1.0])]:
        with pytest.raises(_native.DimbError, match=r"code -3\)"):
            st.detect(s, **kw)


# ------------------------------------------------------------------ SuperPoint heads
def ref_softmax(logits, B, h, w):
    """float64 softmax of the fp32 logits, dustbin dropped, depth-to-space: [B][8h][8w]."""
    lg = logits.astype(np.float64)
    p = np.exp(lg - lg.max(1, keepdims=True))
    p = (p / p.sum(1, keepdims=True))[:, :64]
    return p.reshape(B, h, w, 8, 8).transpose(0, 1, 3, 2, 4).reshape(B, 8 * h, 8 * w)


def softmax_bound(logits, ref, B, h, w):
    gap = (logits.max(1, keepdims=True) - logits)[:, :64].astype(np.float64)
    gap = gap.reshape(B, h, w, 8, 8).transpose(0, 1, 3, 2, 4).reshape(B, 8 * h, 8 * w)
    return SM_REL * (1.0 + gap) * ref + 2.0 ** -126


def softmax_logits(kind, n, rng):
    if kind == "random":
        return rng.normal(0.0, 5.0, (n, 65)).astype(np.float32)
    if kind == "equal":
        return np.full((n, 65), rng.normal(), np.float32)
    if kind == "large":  # near +-80: exp of the raw logits would overflow / underflow fp32
        return (rng.choice([-80.0, 80.0], (n, 65)) + rng.normal(0.0, 1.0, (n, 65))).astype(np.float32)
    if kind == "dustbin":  # 100 above the rest: every score e^-100 or less, subnormal in fp32
        lg = rng.normal(0.0, 1.0, (n, 65))
        lg[:, 64] = lg.max(1) + 100.0
        return lg.astype(np.float32)
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "equal", "large", "dustbin"])
def test_sp_softmax(st, kind):
    worst = 0.0
    for h, w in [(2, 2), (3, 5), (192, 256)]:
        B = 2
        lg = softmax_logits(kind, B * h * w, np.random.default_rng(h * w))
        got, tail = st.sp_softmax(lg, B, h, w, sentinel=SENT)
        ref = ref_softmax(lg, B, h, w)
        bound = softmax_bound(lg, ref, B, h, w)
        err = np.abs(got.astype(np.float64) - ref)
        assert (err <= bound).all(), f"{kind} {h}x{w}: worst {np.max(err / bound):.2f} of the bound"
        assert (tail == SENT).all()
        normal = ref >= 2.0 ** -126
        if normal.any():
            worst = max(worst, float(np.max(err[normal] / (bound - 2.0 ** -126)[normal])))
        if kind == "equal":
            assert np.allclose(got, 1.0 / 65, rtol=SM_REL * 2, atol=0)
        if kind == "dustbin":
            assert (got < 2.0 ** -126).all()
    print(f"softmax {kind}: largest |gpu - ref| / relative bound over normal results {worst:.3f}")


def ref_describe(sel_idx, counts, dense, h, w, fix):
    """oracle sample_descriptors in float64 on the float64-normalised dense map: per image (kpts [n][2], desc [256][n])."""
    from oracle import superpoint as o_sp
    import torch.nn.functional as F
    out = []
    for b in range(len(counts)):
        n = counts[b]
        p = sel_idx[b, :n].astype(np.int64)
        k = np.stack([p % (8 * w), p // (8 * w)], 1).astype(np.float64)
        d = torch.from_numpy(dense[b].astype(np.float64).T.reshape(1, 256, h, w).copy())
        d = F.normalize(d, p=2, dim=1)
        desc = o_sp.sample_descriptors(torch.from_numpy(k), d, fix).numpy() if n else np.zeros((256, 0))
        out.append((k, desc))
    return out


def dense_map(B, h, w, rng, zero_cell=False, scaled=False):
    d = rng.normal(0.0, 1.0, (B, h * w, 256))
    if scaled:
        d *= 10.0 ** rng.uniform(-3, 3, (B, h * w, 1))
    if zero_cell:
        d[:, (h // 2) * w + w // 2] = 0.0
    return d.astype(np.float32)


def check_describe(st, sel_idx, counts, dense, h, w, fix, what):
    B, cap = sel_idx.shape
    rng = np.random.default_rng(cap)
    sel_score = rng.uniform(0.0, 1.0, (B, cap)).astype(np.float32)
    out = st.sp_describe(sel_idx, sel_score, counts, dense, h, w, fix, sentinel=SENT)
    bound = DESC_ABS + DESC_COORD * max(h, w)
    worst = 0.0
    for b, (k, desc) in enumerate(ref_describe(sel_idx, counts, dense, h, w, fix)):
        n = min(counts[b], cap)
        assert np.array_equal(out["kpts"][b, :n], k.astype(np.float32)), f"{what}: image {b} keypoints"
        assert np.array_equal(_bits(out["scores"][b, :n]), _bits(sel_score[b, :n])), f"{what}: image {b} scores"
        err = np.abs(out["desc"][b, :, :n].astype(np.float64) - desc)
        worst = max(worst, float(err.max()) if n else 0.0)
        assert (err <= bound).all(), f"{what}: image {b} descriptor error {err.max():.2e} > {bound:.2e}"
        assert (out["kpts"][b, n:] == SENT).all() and (out["scores"][b, n:] == SENT).all() and (out["desc"][b, :, n:] == SENT).all(), \
            f"{what}: image {b} rows >= {n} written"
    for k in ("kpts", "scores", "desc"):
        assert (out[k + "_tail"] == SENT).all(), f"{what}: write past {k}"
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("fix", [False, True], ids=["align_corners", "fix_sampling"])
def test_sp_describe_every_pixel(st, fix):
    """A keypoint at every pixel of 2 x 2 and 3 x 5 cell grids: every bilinear phase and every border corner (zero padding), with one
    all-zero cell (the 1e-12 clamp) and cells scaled across 1e-3 .. 1e3."""
    worst = 0.0
    for h, w in [(2, 2), (3, 5)]:
        for zero_cell, scaled in [(False, False), (True, False), (False, True)]:
            n = 64 * h * w
            sel = np.tile(np.arange(n, dtype=np.int32), (2, 1))
            dense = dense_map(2, h, w, np.random.default_rng(h * w), zero_cell, scaled)
            worst = max(worst, check_describe(st, sel, [n, n], dense, h, w, fix, f"{h}x{w} zero {zero_cell} scaled {scaled}"))
    print(f"describe every pixel fix {fix}: largest |gpu - ref| {worst:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("fix", [False, True], ids=["align_corners", "fix_sampling"])
def test_sp_describe_counts(st, fix):
    """192 x 256 cells with random keypoints; counts below cap leave the remaining rows as they were, count 0 writes nothing, and two
    images with different counts stay apart."""
    h, w, cap = 192, 256, 2048
    rng = np.random.default_rng(7)
    sel = rng.integers(0, 64 * h * w, (2, cap)).astype(np.int32)
    dense = dense_map(2, h, w, rng)
    worst = 0.0
    for counts in ([cap, 1500], [0, 37], [5, 0]):
        worst = max(worst, check_describe(st, sel, counts, dense, h, w, fix, f"counts {counts}"))
    print(f"describe 192x256 fix {fix}: largest |gpu - ref| {worst:.2e}")
