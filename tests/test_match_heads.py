"""The matching heads on their own: LightGlue's assignment and per-layer tail (csrc/lg_assign.cuh), the shape-generic LightGlue
assignment with its filter (csrc/lgx_assign.cuh) and SuperGlue's Sinkhorn and mutual-max matching
(csrc/sg_assign.cuh), through the self-test entries that run the production launch helpers on host fp32 inputs.  Every output buffer
starts as a sentinel and is followed by a tail, and padded score cells hold a finite poison (1e6), so unwritten slots, stray writes and
reads of padding all show.

Each head turns float scores into discrete decisions, and every decision is a pure fp32 expression of values the kernel returns itself:
  LightGlue  la = ((x - rmax) - rlog) + ((x - cmax) - clog), then + (lz0 + lz1)       (lg_assign.cuh la_value)
  generic    la = ((s - rlse) + (s - clse)) + (ls0 + ls1)                            (generic_kernels.cuh gx_argmax_one)
  SuperGlue  la = ((Z + u) + v) - norm                                               (sg_assign.cuh sg_row_max_kernel)
  stop test  1 - float(counter) / float(n0 + n1) > depth_conf                        (lg_assign.cuh lg_decide_kernel)
None holds a multiply, so nothing contracts into an FMA and numpy float32 reproduces them exactly.  The statistics (rlog, clog, rlse,
clse, u, v, tok, mat) are compared with float64 references under the bounds derived below; argmaxes (torch.max order: the first NaN,
else the first maximum), the mutual check, compaction, the indf mapping, stop and prune decisions, the tables and the counts are compared
bitwise with a float32 emulation built from the kernel's own statistics.  Only expf stands between a kernel's best and its threshold
decision: mscores are held to 2 ulp of float64 exp(best), and the decision exp(best) > th is judged against float64 only where the two
are more than 4 ulp apart.  The float64 references are the inner block of oracle.lightglue.log_assignment / filter_matches,
oracle.superglue.log_optimal_transport, and the adaptive rules check_if_stop / get_pruning_mask (oracle.lightglue.match).

Designs, each for what it forces:
  random     production-like scores: few ties, some mutual matches.
  ties       duplicated columns at j + 1 and j + 32 (adjacent lanes, the same lane one wrap later) and duplicated rows at i + 1 and i + 32
             (other / same ty stride of the column kernels) and i + 1024 (another compaction chunk), with equal matchability: exact fp32
             ties where the maxima are, so only first-index-wins gives the reference's argmax.
  constant   one value everywhere: every argmax is index 0, only (0, 0) is mutual.
  diag       a strong diagonal under a permutation: many mutual matches, compaction across 1024-row chunks and cap below the count.
  chains     row i prefers column i, column i prefers row i + 1: mutual checks that fail.
  wide       scores in +-80: most expf terms underflow.
  nan        a NaN score in a few rows and columns: those rows and columns are NaN throughout (after the fix only).
  neginf     rows and columns whose log assignment is -inf throughout (matchability logsigmoid -inf) (after the fix only).
SuperGlue runs with alpha small, typical and large (everything goes to the dustbin: no match), m < n and m > n, and P = 5 in waves of 1,
2 and 5.  The CPU tests show the designs are sharp: last-index-wins ties, >= in the match filter, a row-only filter, tables from
positions instead of indf, a compaction rank restarting every 1024 rows, Sinkhorn without the dustbin, with log m and log n swapped, or a
row pass skipping the dustbin column, >= for keep, < for confidence, pruning at n >= prune_min, and the first-cut argmax that returned
0x7fffffff on a NaN row all differ from the references."""
import math
import zlib

import numpy as np
import pytest
import torch

SENT = -777.0                                  # every output buffer before the call
ISENT = int(np.float32(SENT).view(np.int32))   # ... its int buffers hold the sentinel's bits
POISON = 1e6                                   # padded score cells: wins any max a kernel wrongly takes over padding
U = 2.0 ** -24                                 # unit roundoff of fp32
INT_MAX = 0x7fffffff
# Bounds, against float64 references of the same fp32 inputs.
#   rlog / clog / rlse / clse: |gpu - ref| <= 2^-24 (max|x - max| + len / 32 + K) + ulp(ref).  The max is exact.  x - max rounds by at most
#   2^-24 |x - max|, which exp turns into that relative error of the term; expf adds 2 ulp (4 units of 2^-24).  Each lane adds len / 32
#   positive terms in sequence, then the row kernels combine 5 shuffle levels (K_ROW = 12 = 4 + 5 + 3 for logf and the final addition of
#   the generic path) and the column kernel 31 partial sums in shared memory (K_COL = 38 = 4 + 31 + 3).  A relative error of the sum is
#   the absolute error of its log; logf adds 1 ulp of the result.
#   Largest measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: 0.19 of the bound (rows), 0.19 (columns), 0.32 (generic).
K_ROW, K_COL = 12.0, 38.0
#   logsigmoid of the generic path: |gpu - ref| <= 2^-21 |ref| + 2^-140: fminf is exact, log1pf(expf(-|z|)) is within 3 ulp of a value
#   below |ref|, the subtraction rounds once.  Largest measured: 0.36 of the bound.
LS_REL = 2.0 ** -21
#   tok / mat: sigmoid(w . x + b) with a 256-term fp32 dot product (8 fmaf per lane, then 5 shuffle levels: 13 roundings of partial sums
#   bounded by sum |w x|), plus the bias: |dy| <= 14 2^-24 (sum |w x| + |b|); the sigmoid's slope is at most 1/4; expf (2 ulp of
#   exp(-y), which moves 1 / (1 + e) by at most 2 ulp of a value below 1), the addition and the division add 4 units of 2^-24:
#   |gpu - ref| <= 2^-24 (3.5 (sum |w x| + |b|) + 4).  Largest measured: 0.035 of the bound.
TOK_DOT, TOK_ABS = 3.5, 4.0
#   One Sinkhorn half step from given u / v (the sharp test): x = fl(Z + v) rounds by 2^-24 |x|, and the exponent arguments x - max are
#   off by at most 3 max|x| 2^-24; expf adds 4 units per term; the online sum takes per element one rescale (expf, multiply) and one
#   addition (6 units), the 5 shuffle levels two expf, two multiplies and an addition each (~30 units); logf 2 ulp of log s, then two
#   subtractions round by 2^-24 |result| each:
#   |gpu - ref| <= 2^-24 (3 max|x| + 6 (len + 1) / 32 + 40 + 2 |log s| + 2 |ref|).  Largest measured: 0.11 of the bound.
#   100 iterations: each half step maps its input through a logsumexp, which is 1-Lipschitz in the max norm, so errors add at most
#   linearly: the bound is derived as the sum of the 200 per-step bounds along the float64 trajectory.  Largest measured: 0.067 of it.
SK_XS, SK_LEN, SK_ABS = 3.0, 6.0, 40.0
DESIGNS = ["random", "ties", "constant", "diag", "chains", "wide"]
NONFINITE = ["nan", "neginf"]


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def _np_rng(*key):
    return np.random.default_rng([zlib.crc32(k.encode()) if isinstance(k, str) else int(k) for k in key])


# ------------------------------------------------------------------ designs
def design(name, m, n, rng):
    """(sim [m][n], lz0 [m], lz1 [n]) float32; lz = logsigmoid(matchability), as lg_final_gather_kernel leaves z."""
    lz0 = np.log(1.0 / (1.0 + np.exp(-rng.normal(1.0, 2.0, m))))
    lz1 = np.log(1.0 / (1.0 + np.exp(-rng.normal(1.0, 2.0, n))))
    if name == "random":
        sim = rng.normal(0.0, 3.0, (m, n))
    elif name == "constant":
        sim = np.full((m, n), 0.75)
        lz0[:], lz1[:] = -0.25, -0.25
    elif name in ("diag", "ties"):
        sim = rng.normal(0.0, 1.0, (m, n))
        k = min(m, n)
        rows, cols = rng.permutation(m)[:k], rng.permutation(n)[:k]
        sim[rows, cols] += 12.0
        if name == "ties":
            sim, lz0, lz1 = _ties(sim, lz0, lz1, rows, cols)
    elif name == "chains":
        sim = rng.normal(0.0, 0.5, (m, n))
        k = min(m, n)
        sim[np.arange(k), np.arange(k)] += 8.0
        i = np.arange(min(m - 1, n))
        sim[i + 1, i] += 9.0
    elif name == "wide":
        sim = rng.uniform(-80.0, 80.0, (m, n))
    elif name in NONFINITE:
        sim = rng.normal(0.0, 1.0, (m, n))
        k = min(m, n)
        sim[rng.permutation(m)[:k], rng.permutation(n)[:k]] += 12.0
        r = sorted({0, m // 2, m - 1})
        c = sorted({0, n // 3, n - 1})
        if name == "nan":
            sim[r, [min(x, n - 1) for x in (n // 2, 0, n - 1)][:len(r)]] = np.nan
            sim[[min(x, m - 1) for x in (1, m // 3, m - 1)][:len(c)], c] = np.nan
        else:
            lz0[r] = -np.inf
            lz1[c] = -np.inf
    else:
        raise ValueError(name)
    return sim.astype(np.float32), lz0.astype(np.float32), lz1.astype(np.float32)


def _ties(sim, lz0, lz1, rows, cols):
    """Copy the preferred column of some rows to j + 1 and j + 32 and some rows to i + 1, i + 32 and i + 1024 (whole columns / rows and
    their matchability), so the maxima sit on exact ties across lanes, lane wraps, ty strides and compaction chunks."""
    m, n = sim.shape
    order = np.argsort(rows)
    for a, b in ((1, 0), (32, 3), (1, 7), (32, 11)):
        if len(order) > b:
            j = cols[order[b]]
            if j + a < n:
                sim[:, j + a] = sim[:, j]
                lz1[j + a] = lz1[j]
    for a, start in ((1, 6), (32, 20), (1024, 50)):  # starts apart, so no copy is copied again
        for i in range(start, m - a, max(m // 4, 64)):
            sim[i + a] = sim[i]
            lz0[i + a] = lz0[i]
    return sim, lz0, lz1


# ------------------------------------------------------------------ float32 emulations (the kernels' own arithmetic)
def la_lg(sim, rmax, rlog, cmax, clog, lz0, lz1):
    """lg_assign.cuh la_value over the block, float32."""
    with np.errstate(invalid="ignore", over="ignore"):
        s0 = (sim - rmax[:, None]) - rlog[:, None]
        s1 = (sim - cmax[None, :]) - clog[None, :]
        return (s0 + s1) + (lz0[:, None] + lz1[None, :])


def la_gx(sim, rlse, clse, ls0, ls1):
    with np.errstate(invalid="ignore", over="ignore"):
        return ((sim - rlse[:, None]) + (sim - clse[None, :])) + (ls0[:, None] + ls1[None, :])


def la_sg(Z, u, v, norm):
    with np.errstate(invalid="ignore", over="ignore"):
        return ((Z + u[:, None]) + v[None, :]) - np.float32(norm)


def first_argmax(a, axis):
    """torch.max order: the first NaN, else the first maximum (numpy's argmax is exactly that)."""
    return np.argmax(a, axis)


def last_argmax(a, axis):
    """Mutant: the last maximum wins ties."""
    b = np.flip(a, axis)
    return a.shape[axis] - 1 - np.argmax(b, axis)


def old_warp_argmax(row):
    """numpy model of the parent's lane and warp reduction: bv = -inf, bi = 0x7fffffff, take v > bv per lane, then the shuffle tree with
    (ov > bv || (ov == bv && oi < bi))."""
    bv, bi = np.full(32, -np.inf, np.float32), np.full(32, INT_MAX, np.int64)
    for j, v in enumerate(row):
        if v > bv[j % 32]:
            bv[j % 32], bi[j % 32] = v, j
    o = 16
    while o:
        ov, oi = bv[np.arange(32) ^ o], bi[np.arange(32) ^ o]
        take = (ov > bv) | ((ov == bv) & (oi < bi))
        bv, bi = np.where(take, ov, bv), np.where(take, oi, bi)
        o >>= 1
    return int(bi[0])


def exp_decision(best, th):
    """(clear, above): float64 exp(best) > th wherever the two are more than 4 ulp of th apart."""
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.exp(best.astype(np.float64))
        d = np.abs(e - th)
    clear = ~(d <= 4 * ulp(th)) | np.isnan(e)
    return clear, e > th


def expected_table(best, a0, a1, ind0, ind1, th, got_pairs, ge=False, mutual=True, rank_block=None):
    """Rows that match in row order: a0[i] in range, a1[a0[i]] == i (unless mutual=False), exp(best) > th (>= with ge).  Rows whose
    threshold decision is within 4 ulp take the kernel's own (whether (ind0[i], ind1[a0[i]]) is in got_pairs).  rank_block: mutant
    whose compaction rank restarts every rank_block rows.  Returns (list of (ind0, ind1, row)) in table order."""
    m = len(best)
    clear, above = exp_decision(best, th)
    if ge:  # mutant: every decision taken as exp(best) >= th, exact ones included
        with np.errstate(invalid="ignore", over="ignore"):
            clear, above = np.ones(m, bool), np.exp(best.astype(np.float64)) >= th
    out = []
    for i in range(m):
        j = int(a0[i])
        if not (0 <= j < len(a1)) or (mutual and a1[j] != i):
            continue
        pair = (int(ind0[i]), int(ind1[j]))
        if above[i] if clear[i] else pair in got_pairs:
            out.append((pair[0], pair[1], i))
    if rank_block:
        slots = {}
        for k, (a, b, i) in enumerate(out):
            before = sum(1 for (_, _, r) in out[:k] if r // rank_block == i // rank_block)
            slots[before] = (a, b, i)
        out = [slots[k] for k in sorted(slots)]
    return out


# ------------------------------------------------------------------ float64 references
def ref_lg_stats(sim):
    """float64 (rmax, rlog, cmax, clog) of the fp32 block; the maxima start from -inf and skip NaN, as the fmaxf reductions do."""
    s = sim.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        rm, cm = np.fmax.reduce(s, 1, initial=-np.inf), np.fmax.reduce(s, 0, initial=-np.inf)
        return rm, np.log(np.exp(s - rm[:, None]).sum(1)), cm, np.log(np.exp(s - cm[None]).sum(0))


def ref_lg_scores(sim, lz0, lz1):
    """The inner block of oracle.lightglue.log_assignment in float64, padded to (m + 1) x (n + 1) for filter_matches."""
    s = torch.from_numpy(sim.astype(np.float64))
    inner = torch.log_softmax(s, 1) + torch.log_softmax(s, 0) + torch.from_numpy(lz0.astype(np.float64))[:, None] + \
        torch.from_numpy(lz1.astype(np.float64))[None]
    sc = torch.zeros(sim.shape[0] + 1, sim.shape[1] + 1, dtype=torch.float64)
    sc[:-1, :-1] = inner
    return sc


def stat_bound(x, mx, ref, k):
    """2^-24 (max|x - max| + len / 32 + k) + ulp(ref) per row of x (reduced over axis 1)."""
    with np.errstate(invalid="ignore"):
        spread = np.nanmax(np.abs(x.astype(np.float64) - mx[:, None]), 1)
    return U * (spread + x.shape[1] / 32.0 + k) + ulp(ref)


def ref_sinkhorn(Z, alpha, steps, u0=None, v0=None):
    """log_optimal_transport in float64 (oracle.superglue), one half step at a time: u / v after `steps` half steps and, per step, the
    half-step bound along the trajectory (the right-hand sides of the bound above, from the float64 values)."""
    m, n = Z.shape
    c = np.full((m + 1, n + 1), float(alpha))
    c[:m, :n] = Z
    norm = -math.log(m + n)
    log_mu = np.r_[np.full(m, norm), math.log(n) + norm]
    log_nu = np.r_[np.full(n, norm), math.log(m) + norm]
    u = np.zeros(m + 1) if u0 is None else u0.astype(np.float64)
    v = np.zeros(n + 1) if v0 is None else v0.astype(np.float64)
    bounds = []
    for h in range(steps):
        if h % 2 == 0:
            x = c + v[None]
            mx = x.max(1)
            ls = np.log(np.exp(x - mx[:, None]).sum(1))
            u = log_mu - (mx + ls)
            bounds.append(U * (SK_XS * np.abs(x).max() + SK_LEN * (n + 1) / 32 + SK_ABS + 2 * np.abs(ls).max() + 2 * np.abs(u).max()))
        else:
            x = c + u[:, None]
            mx = x.max(0)
            ls = np.log(np.exp(x - mx[None]).sum(0))
            v = log_nu - (mx + ls)
            bounds.append(U * (SK_XS * np.abs(x).max() + SK_LEN * (m + 1) / 32 + SK_ABS + 2 * np.abs(ls).max() + 2 * np.abs(v).max()))
    return u, v, bounds


def decide_ref(n_act, n_orig, stopped, counter, tok, mat, NP, layer, thr, depth_conf, keep_thr, do_stop, do_prune, prune_min,
               keep_ge=False, conf_lt=False, prune_ge=False, isent=ISENT):
    """check_if_stop / get_pruning_mask as lg_decide_kernel evaluates them, float32: (counter, stopped, map [2P][NP], n_next [2P])."""
    P = len(stopped)
    counter, stopped = np.array(counter, np.int32), np.array(stopped, np.int32)
    mp, nn = np.full((2 * P, NP), isent, np.int32), np.full(2 * P, isent, np.int32)
    for p in range(P):
        if stopped[p]:
            continue
        stop = False
        if do_stop:
            ratio = np.float32(1.0) - np.float32(counter[p]) / np.float32(n_orig[2 * p] + n_orig[2 * p + 1])
            stop = bool(ratio > np.float32(depth_conf))
        counter[p] = 0
        if stop:
            stopped[p] = layer + 1
        for s in (2 * p, 2 * p + 1):
            n = int(n_act[s])
            prune = not stop and do_prune and (n >= prune_min if prune_ge else n > prune_min)
            if not prune:
                mp[s, :n] = np.arange(n)
                nn[s] = n
                continue
            t, a = tok[s, :n], mat[s, :n]
            keep = (a >= np.float32(keep_thr)) if keep_ge else (a > np.float32(keep_thr))
            if do_stop:
                keep |= (t < np.float32(thr)) if conf_lt else (t <= np.float32(thr))
            k = np.flatnonzero(keep)
            mp[s, :len(k)] = k
            nn[s] = len(k)
    return counter, stopped, mp, nn


# ------------------------------------------------------------------ CPU: references agree, designs are sharp
def _emulated_lg(sim, lz0, lz1):
    """Decisions of the LightGlue head from float32 statistics computed in numpy (stand-ins for the kernel's)."""
    rm, rl, cm, cl = (a.astype(np.float32) for a in ref_lg_stats(sim))
    la = la_lg(sim, rm, rl, cm, cl, lz0, lz1)
    return la


def test_emulation_matches_the_float64_reference():
    """On random and diagonal designs the float32 emulation (argmaxes, mutual filter, threshold) gives filter_matches' matches."""
    from oracle import lightglue as o_lg
    for name in ("random", "diag", "chains"):
        for m, n in [(33, 255), (256, 31), (300, 300)]:
            sim, lz0, lz1 = design(name, m, n, _np_rng(name, m, n))
            la = _emulated_lg(sim, lz0, lz1)
            a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
            best = la[np.arange(m), a0]
            got = expected_table(best, a0, a1, np.arange(m), np.arange(n), 0.1, set())
            m0 = o_lg.filter_matches(ref_lg_scores(sim, lz0, lz1), 0.1)[0].numpy()
            want = [(i, int(m0[i])) for i in range(m) if m0[i] >= 0]
            assert [(a, b) for a, b, _ in got] == want, (name, m, n)


def test_reference_sinkhorn_is_the_oracle():
    """The half-step float64 Sinkhorn equals oracle.superglue.log_optimal_transport run on float64 scores.  The oracle builds m, n and
    their logs as float32 tensors (as the reference model does), so the two differ by the rounding of those constants, below 1e-6."""
    from oracle import superglue as o_sg
    Z = _np_rng("sk", 1).normal(0.0, 2.0, (37, 70)).astype(np.float32)
    u, v, _ = ref_sinkhorn(Z, 1.3, 200)
    full = o_sg.log_optimal_transport(torch.from_numpy(Z.astype(np.float64)), torch.tensor(1.3, dtype=torch.float64), 100).numpy()
    c = np.full((38, 71), 1.3)
    c[:37, :70] = Z
    assert np.allclose(c + u[:, None] + v[None] + math.log(107), full, atol=1e-6, rtol=0)


def test_tie_mutant_differs():
    """On ties, last-index-wins changes row and column argmaxes (across j + 1 and j + 32, i + 1, i + 32 and i + 1024)."""
    sim, lz0, lz1 = design("ties", 2048, 1025, _np_rng("ties", 0))
    la = _emulated_lg(sim, lz0, lz1)
    assert not np.array_equal(first_argmax(la, 1), last_argmax(la, 1))
    assert not np.array_equal(first_argmax(la, 0), last_argmax(la, 0))
    a1 = first_argmax(la, 0)
    diff_rows = np.flatnonzero(first_argmax(la, 0) != last_argmax(la, 0))
    gaps = {int(last_argmax(la, 0)[c] - a1[c]) for c in diff_rows}
    assert {1, 32, 1024} <= gaps, gaps
    diff_cols = np.flatnonzero(first_argmax(la, 1) != last_argmax(la, 1))
    assert {1, 32} <= {int(last_argmax(la, 1)[r] - first_argmax(la, 1)[r]) for r in diff_cols}


def test_filter_mutants_differ():
    """>= in the threshold, a row-only filter, tables of positions and a compaction rank restarting every 1024 rows each change the
    tables on some design."""
    # exactly on the threshold: m = n = 1, lz = 0 -> best = 0, exp(best) = 1 = th
    best, a0, a1 = np.zeros(1, np.float32), np.zeros(1, np.int64), np.zeros(1, np.int64)
    assert expected_table(best, a0, a1, [0], [0], 1.0, set()) == []
    assert expected_table(best, a0, a1, [0], [0], 1.0, set(), ge=True) != []
    sim, lz0, lz1 = design("chains", 300, 300, _np_rng("chains", 1))
    la = _emulated_lg(sim, lz0, lz1)
    a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
    best = la[np.arange(300), a0]
    ref = expected_table(best, a0, a1, np.arange(300), np.arange(300), 0.0, set())
    assert expected_table(best, a0, a1, np.arange(300), np.arange(300), 0.0, set(), mutual=False) != ref
    indf0, indf1 = _np_rng("indf", 0).permutation(5000)[:300], _np_rng("indf", 1).permutation(5000)[:300]
    assert [t[:2] for t in expected_table(best, a0, a1, indf0, indf1, 0.0, set())] != [t[:2] for t in ref]  # positions, not indf
    sim, lz0, lz1 = design("diag", 2048, 2048, _np_rng("diag", 2))
    la = _emulated_lg(sim, lz0, lz1)
    a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
    best = la[np.arange(2048), a0]
    ref = expected_table(best, a0, a1, np.arange(2048), np.arange(2048), 0.1, set())
    assert len(ref) > 1500
    assert expected_table(best, a0, a1, np.arange(2048), np.arange(2048), 0.1, set(), rank_block=1024)[:len(ref)] != ref


def test_parent_argmax_leaves_the_row_on_nonfinite_rows():
    """The first-cut reduction returns 0x7fffffff on an all-NaN and an all--inf row (an index the consumers then read with), where
    torch.max returns 0; on finite rows, ties included, both give the first maximum."""
    for row in (np.full(70, np.nan, np.float32), np.full(70, -np.inf, np.float32)):
        assert old_warp_argmax(row) == INT_MAX
        assert int(torch.from_numpy(row).max(0).indices) == 0 == first_argmax(row, 0)
    row = np.array([1, np.nan, 3, np.nan], np.float32)
    assert int(torch.from_numpy(row).max(0).indices) == 1 == first_argmax(row, 0)
    rng = _np_rng("fin", 0)
    for n in (1, 31, 33, 100):
        row = rng.integers(0, 4, n).astype(np.float32)
        assert old_warp_argmax(row) == first_argmax(row, 0)


def test_sinkhorn_mutants_differ():
    """Sinkhorn without the dustbin, with log m and log n swapped, or with a row pass that skips the dustbin column lands further from
    the reference than the 100-iteration bound, for m != n."""
    Z = _np_rng("skm", 0).normal(0.0, 2.0, (40, 90)).astype(np.float32)
    alpha = 1.0
    u, v, b = ref_sinkhorn(Z, alpha, 200)
    bound = sum(b)
    m, n = Z.shape

    def run(dustbin=True, swap=False, skip_col=False):
        c = np.full((m + 1, n + 1), alpha)
        c[:m, :n] = Z
        norm = -math.log(m + n)
        lm, ln = (math.log(n), math.log(m)) if swap else (math.log(m), math.log(n))
        mu, nu = np.r_[np.full(m, norm), ln + norm], np.r_[np.full(n, norm), lm + norm]
        if not dustbin:
            c, mu, nu = c[:m, :n], mu[:m], nu[:n]
        uu, vv = np.zeros(len(mu)), np.zeros(len(nu))
        for _ in range(100):
            x = c + vv[None]
            if skip_col:
                x = x[:, :-1]
            uu = mu - np.log(np.exp(x - x.max(1, keepdims=True)).sum(1)) - x.max(1)
            x = c + uu[:, None]
            vv = nu - np.log(np.exp(x - x.max(0, keepdims=True)).sum(0)) - x.max(0)
        return uu, vv

    for kw in (dict(swap=True), dict(skip_col=True)):
        uu, vv = run(**kw)
        assert max(np.abs(uu - u).max(), np.abs(vv - v).max()) > bound, kw
    uu, vv = run(dustbin=False)
    assert max(np.abs(uu - u[:m]).max(), np.abs(vv - v[:n]).max()) > bound


def _decide_designs():
    """(name, dict of decide inputs) designed to sit on every boundary of the tail."""
    cases = []
    NP, thr, keep_thr, prune_min = 2176, np.float32(0.9), np.float32(0.95), 64
    ns = [(1023, 1024), (1025, 2049), (prune_min, prune_min + 1), (2049, 1), (300, 400)]
    P = len(ns)
    n_act = np.array([x for pr in ns for x in pr], np.int32)
    n_orig = n_act + np.array([0, 7, 3, 0, 0, 0, 11, 0, 0, 5], np.int32)
    rng = _np_rng("decide", 0)
    tok = rng.uniform(0.5, 1.0, (2 * P, NP)).astype(np.float32)
    mat = rng.uniform(0.5, 1.0, (2 * P, NP)).astype(np.float32)
    tok[:, ::7] = thr                      # == thr: kept (<=)
    mat[:, ::5] = keep_thr                 # == keep_thr: pruned unless tok <= thr (>)
    tok[:, ::5] = np.nextafter(thr, np.float32(2))
    tot = (n_orig[0::2] + n_orig[1::2]).astype(np.float32)
    counter = (tot * np.float32(0.125)).astype(np.int32)
    counter[2:] = (tot[2:] * np.float32(0.25)).astype(np.int32)      # the other pairs well below the boundary: they run and prune
    depth_conf = np.float32(1.0) - np.float32(counter[0]) / tot[0]   # pair 0 exactly on the boundary: runs on (>)
    counter[1] -= 1                                                      # pair 1 just above: stops
    stopped = np.array([0, 0, 0, 3, 0], np.int32)                        # pair 3 stopped at an earlier layer
    base = dict(n_act=n_act, n_orig=n_orig, stopped=stopped, counter=counter, tok=tok, mat=mat, NP=NP, layer=4, thr=thr,
                depth_conf=depth_conf, keep_thr=keep_thr, do_stop=True, do_prune=True, prune_min=prune_min)
    cases.append(("stop_and_prune", base))
    cases.append(("prune_only", {**base, "do_stop": False}))
    cases.append(("stop_only", {**base, "do_prune": False}))
    return cases


def test_decide_mutants_differ():
    """>= for keep, < for confidence, pruning at n >= prune_min, > replaced by >= in the stop test all change the tail's output."""
    name, c = _decide_designs()[0]
    ref = decide_ref(**c)
    for kw in (dict(keep_ge=True), dict(conf_lt=True), dict(prune_ge=True)):
        got = decide_ref(**c, **kw)
        assert not all(np.array_equal(a, b) for a, b in zip(got, ref)), kw
    # the depth boundary: stop on ratio >= depth_conf would stop pair 0
    assert ref[1][0] == 0 and ref[1][1] == 5
    tot = np.float32(c["n_orig"][0] + c["n_orig"][1])
    assert np.float32(1.0) - np.float32(c["counter"][0]) / tot == c["depth_conf"]


def test_entries_refuse_bad_arguments_without_a_context():
    """Every matching-head entry checks its arguments before any CUDA call: a null context is refused."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    buf = np.zeros(1 << 16, np.float32)
    p = _native._ptr(buf)
    ib = np.full(8, 4, np.int32)
    q = _native._ptr(ib)
    assert lib.dimb_selftest_lg_assign(None, 1, 128, p, q, q, q, q, p, 0.1, 4, SENT, *([p] * 8)) == -3
    assert lib.dimb_selftest_lg_tail(None, 1, 128, p, p, 0.0, p, 0.0, None, None, q, q, q, q, 0, 0.9, 0.95, 0.99, 1, 1, 64, SENT,
                                     *([p] * 6)) == -3
    assert lib.dimb_selftest_lgx_assign(None, 4, 4, 4, p, p, p, q, q, 0.1, 4, SENT, *([p] * 11)) == -3
    assert lib.dimb_selftest_sg_sinkhorn(None, 1, q, q, p, 1.0, POISON, None, None, 1, 2, 0.2, 4, SENT, *([p] * 9)) == -3


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def st():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the GPU tests of this module run on an H100")
    from dim_b200 import _native
    return _native.SelfTest(0)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    """bitwise equality of float32 arrays, NaN payloads aside"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(_bits(np.where(np.isnan(a), 0, a)), _bits(np.where(np.isnan(b), 0, b)))


WORST = {}


def _worst(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


def check_table(what, got_m, got_s, got_n, best, a0, a1, ind0, ind1, th, cap):
    """Tables bitwise against the emulation (threshold decisions within 4 ulp taken from the kernel), mscores within 2 ulp of float64
    exp(best), slots past min(count, cap) untouched.  Returns the count."""
    pairs = {tuple(int(x) for x in r) for r in got_m[:min(int(got_n), cap)]}
    want = expected_table(best, a0, a1, ind0, ind1, th, pairs)
    assert int(got_n) == len(want), f"{what}: n_matches {got_n} != {len(want)}"
    k = min(len(want), cap)
    assert np.array_equal(got_m[:k], np.array([(a, b) for a, b, _ in want[:k]], np.int64).reshape(k, 2)), f"{what}: match table"
    rows = np.array([r for _, _, r in want[:k]], np.int64)
    e = np.exp(best[rows].astype(np.float64))
    assert (np.abs(got_s[:k].astype(np.float64) - e) <= 2 * ulp(e)).all(), f"{what}: mscores"
    assert (got_m[k:] == ISENT).all() and (got_s[k:] == SENT).all(), f"{what}: slots past the count written"
    return len(want)


# ---- LightGlue assignment
def _lg_batch(pairs, names, seed, NP=None, empty=()):
    """P pairs (m_p, n_p) with designs names[p] in the production layout: sim [P][NP][NP] with POISON padding, nf / n_orig, layer,
    indf (a random injection into [0, n_orig)), z (POISON padding)."""
    P = len(pairs)
    NP = NP or -(-max(max(pr) for pr in pairs) // 128) * 128
    sim = np.full((P, NP, NP), POISON, np.float32)
    z = np.full((2 * P, NP), POISON, np.float32)
    indf = np.full((2 * P, NP), -5, np.int32)
    nf = np.array([x for pr in pairs for x in pr], np.int32)
    n_orig = nf + np.array([(7 * s) % 50 for s in range(2 * P)], np.int32)
    for p in empty:
        n_orig[2 * p] = 0
    layer = np.array([(3 * p + 1) % 9 for p in range(P)], np.int32)
    blocks = []
    for p, (m, n) in enumerate(pairs):
        rng = _np_rng(names[p], m, n, seed)
        s, l0, l1 = design(names[p], m, n, rng)
        sim[p, :m, :n] = s
        z[2 * p, :m], z[2 * p + 1, :n] = l0, l1
        for sd, k in ((0, m), (1, n)):
            indf[2 * p + sd, :k] = rng.permutation(max(int(n_orig[2 * p + sd]), k))[:k]
        blocks.append((s, l0, l1))
    return sim, nf, n_orig, layer, indf, z, blocks


def run_lg_assign(st, pairs, names, seed, cap, th=0.1, empty=()):
    sim, nf, n_orig, layer, indf, z, blocks = _lg_batch(pairs, names, seed, empty=empty)
    out = st.lg_assign(sim, nf, n_orig, layer, indf, z, th, cap, sentinel=SENT)
    P, NP = sim.shape[:2]
    for p, ((m, n), (s, l0, l1)) in enumerate(zip(pairs, blocks)):
        what = f"{names[p]} pair {p} ({m} x {n})"
        assert out["stop_layer"][p] == (1 if p in empty else layer[p] + 1), what
        for k, live in (("rmax", m), ("rlog", m), ("best", m), ("arg0", m), ("cmax", n), ("clog", n), ("arg1", n)):
            rest = out[k][p, live:]
            assert (rest == (ISENT if k.startswith("arg") else SENT)).all(), f"{what}: {k} written past the live count"
        assert (out["best_other"][p] == SENT).all(), f"{what}: best written on the column side"
        rm, rl, cm, cl = ref_lg_stats(s)
        assert _same(out["rmax"][p, :m], rm.astype(np.float32)) and _same(out["cmax"][p, :n], cm.astype(np.float32)), f"{what}: max"
        if names[p] not in NONFINITE:
            for key, got, ref, mx, x, k in (("rlog", out["rlog"][p, :m], rl, rm, s, K_ROW), ("clog", out["clog"][p, :n], cl, cm, s.T, K_COL)):
                bound = stat_bound(x, mx, ref, k)
                err = np.abs(got.astype(np.float64) - ref)
                assert (err <= bound).all(), f"{what}: {key} {err.max():.3g} > bound at {np.argmax(err - bound)}"
                _worst(key, (err / bound).max())
        la = la_lg(s, out["rmax"][p, :m], out["rlog"][p, :m], out["cmax"][p, :n], out["clog"][p, :n], l0, l1)
        a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
        assert np.array_equal(out["arg0"][p, :m], a0), f"{what}: row argmax at {np.flatnonzero(out['arg0'][p, :m] != a0)[:5]}"
        assert np.array_equal(out["arg1"][p, :n], a1), f"{what}: column argmax at {np.flatnonzero(out['arg1'][p, :n] != a1)[:5]}"
        best = la[np.arange(m), a0]
        assert _same(out["best"][p, :m], best), f"{what}: row maxima"
        if p in empty:
            assert out["n_matches"][p] == 0 and (out["matches"][p] == ISENT).all(), what
            continue
        cnt = check_table(what, out["matches"][p], out["mscores"][p], out["n_matches"][p], best, a0, a1, indf[2 * p], indf[2 * p + 1], th,
                          cap)
        if names[p] in NONFINITE:  # such rows exist, and none of them matched
            bad = set(np.flatnonzero(np.isnan(best) | np.isneginf(best)).tolist())
            assert bad and not bad & {int(np.flatnonzero(indf[2 * p, :m] == a)[0]) for a in out["matches"][p, :min(cnt, cap), 0]}, what
        if names[p] == "constant":
            assert cnt == (1 if math.exp(float(best[0])) > th else 0) and (a0 == 0).all() and (a1 == 0).all()
    for k in ("smax", "slog", "best", "mscores"):
        assert (out[k + "_tail"] == SENT).all(), f"write past {k}"
    for k in ("arg", "n_matches", "stop_layer", "matches"):
        assert (out[k + "_tail"] == ISENT).all(), f"write past {k}"
    return out


# pair shapes per batch: m, n in {1, 2, 31, 32, 33, 255, 256, 1023, 1024, 1025, 2048}, unequal; each batch runs one design on every pair
LG_BATCHES = [[(1, 2), (31, 33), (33, 255), (2, 1)], [(256, 1023), (1024, 1025), (255, 32)], [(2048, 1023), (1025, 2048), (32, 31)]]


@pytest.mark.gpu
@pytest.mark.parametrize("name", DESIGNS + NONFINITE)
def test_lg_assign(st, name):
    """One design on every pair of three batches (P = 3, 4; a different nf per pair, non-identity indf, cap below the count on the
    largest batch), statistics within bounds, everything discrete bitwise."""
    for b, pairs in enumerate(LG_BATCHES):
        cap = 700 if b == 2 else 2048
        run_lg_assign(st, pairs, [name] * len(pairs), b, cap)
    print(f"lg_assign {name}: worst of bound {WORST}")


@pytest.mark.gpu
def test_lg_assign_mixed_batch_empty_pair_and_cap(st):
    """Designs mixed within one batch, a pair with an empty side (stop_layer 1, no match, nothing written) and cap below the count on a
    2048 x 2048 diagonal (compaction across 1024-row chunks)."""
    pairs = [(2048, 2048), (5, 7), (1023, 256), (300, 301)]
    out = run_lg_assign(st, pairs, ["diag", "random", "ties", "chains"], 9, cap=1500, empty=(1,))
    assert out["n_matches"][0] > 1500


@pytest.mark.gpu
def test_lg_assign_exact_threshold(st):
    """m = n = 1 with lz = 0: best = 0 and expf(best) = 1 exactly; th = 1 gives no match (>), th just below 1 gives one."""
    for th, want in ((1.0, 0), (float(np.nextafter(np.float32(1), np.float32(0))), 1)):
        sim = np.full((1, 128, 128), POISON, np.float32)
        sim[0, 0, 0] = 0.3
        z = np.full((2, 128), POISON, np.float32)
        z[:, 0] = 0.0
        out = st.lg_assign(sim, [1, 1], [1, 1], [2], np.zeros((2, 128), np.int32), z, th, 4, sentinel=SENT)
        assert out["best"][0, 0] == 0.0 and out["n_matches"][0] == want
        if want:
            assert out["mscores"][0, 0] == 1.0 and (out["matches"][0, 0] == 0).all()


# ---- generic path
@pytest.mark.gpu
@pytest.mark.parametrize("name", DESIGNS + NONFINITE)
def test_lgx_assign(st, name):
    """The shape-generic assignment and device filter (launch_lgx_assign at P = 1) on one pair at a time: unequal sizes, padding columns
    of POISON in sim's rows, compaction across 1024-row chunks (m = 1025 and 2048)."""
    for m, n in [(1, 2), (33, 31), (255, 1024), (1025, 256), (2048, 1023)]:
        rng = _np_rng("gx", name, m, n)
        s, l0, l1 = design(name, m, n, rng)
        z0, z1 = (rng.normal(0.0, 3.0, k).astype(np.float32) for k in (m, n))
        if name == "neginf":
            z0[l0 == -np.inf], z1[l1 == -np.inf] = -np.inf, -np.inf
        ld = -(-n // 128) * 128 + 64
        sim = np.full((m, ld), POISON, np.float32)
        sim[:, :n] = s
        ind0, ind1 = rng.permutation(m + 40)[:m], rng.permutation(n + 40)[:n]
        cap = max(1, min(m, n) // 2)
        o = st.lgx_assign(sim, z0, z1, ind0, ind1, 0.1, cap, sentinel=SENT)
        what = f"{name} {m} x {n}"
        for key, ls, z in (("ls0", o["ls0"], z0), ("ls1", o["ls1"], z1)):
            ref = -np.logaddexp(0.0, -z.astype(np.float64))
            with np.errstate(invalid="ignore"):
                err = np.abs(ls.astype(np.float64) - ref)
            fin = np.isfinite(ref)
            assert (err[fin] <= LS_REL * np.abs(ref[fin]) + 2.0 ** -140).all(), f"{what}: {key}"
            assert np.array_equal(ls[~fin], ref[~fin].astype(np.float32))
            _worst(key, (err[fin] / (LS_REL * np.abs(ref[fin]) + 2.0 ** -140)).max(initial=0))
        if name not in NONFINITE:
            rm, rl, cm, cl = ref_lg_stats(s)
            for key, got, ref, mx, x in (("rlse", o["rlse"], rm + rl, rm, s), ("clse", o["clse"], cm + cl, cm, s.T)):
                bound = stat_bound(x, mx, ref, K_ROW)
                err = np.abs(got.astype(np.float64) - ref)
                assert (err <= bound).all(), f"{what}: {key} {err.max():.3g}"
                _worst("gx_" + key, (err / bound).max())
        la = la_gx(s, o["rlse"], o["clse"], o["ls0"], o["ls1"])
        a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
        assert np.array_equal(o["arg0"], a0) and np.array_equal(o["arg1"], a1), f"{what}: argmax"
        assert _same(o["best0"], la[np.arange(m), a0]) and _same(o["best1"], la[a1, np.arange(n)]), f"{what}: maxima"
        check_table(what, o["matches"], o["mscores"], o["n_matches"], o["best0"], a0, a1, ind0, ind1, 0.1, cap)
        for k, v in o.items():
            if k.endswith("_tail"):
                assert (v == (ISENT if k.startswith(("arg", "matches")) else SENT)).all(), f"{what}: write past {k}"
    print(f"lgx_assign {name}: worst of bound {WORST}")


# ---- tail
@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in _decide_designs()])
def test_lg_decide(st, case):
    """lg_decide_kernel alone on designed confidences: the depth boundary, tok == thr, mat == keep_thr, n == prune_min and + 1,
    multi-chunk compaction (1023 .. 2049 rows), a stopped pair left alone, counters reset for pairs that ran."""
    c = dict(_decide_designs())[case]
    P, NP = len(c["stopped"]), c["NP"]
    out = st.lg_tail(P, NP, c["n_act"], c["n_orig"], c["stopped"], c["counter"], c["layer"], c["thr"], c["depth_conf"], c["keep_thr"],
                     c["do_stop"], c["do_prune"], c["prune_min"], tok=c["tok"].reshape(-1), mat=c["mat"].reshape(-1), sentinel=SENT)
    counter, stopped, mp, nn = decide_ref(**c)
    assert np.array_equal(out["stopped"], stopped) and np.array_equal(out["counter"], counter)
    assert np.array_equal(out["n_next"], nn), (out["n_next"], nn)
    assert np.array_equal(out["map"], mp)
    assert np.array_equal(_bits(out["tok"]), _bits(c["tok"])) and np.array_equal(_bits(out["mat"]), _bits(c["mat"]))
    for k in ("counter", "stopped", "map", "n_next"):
        assert (out[k + "_tail"] == ISENT).all(), f"write past {k}"
    if case == "stop_and_prune":
        assert stopped[0] == 0 and stopped[1] == c["layer"] + 1 and stopped[3] == 3
        assert nn[4] == c["prune_min"] and nn[5] < c["prune_min"] + 1


@pytest.mark.gpu
def test_lg_tail_from_tokens(st):
    """lg_conf_kernel then lg_decide_kernel from token rows: tok / mat within bounds of float64 sigmoids; the low-confidence count,
    the stop decision (depth_conf placed exactly on pair 0's ratio, from a first call), the prune maps and counts bitwise."""
    P, NP = 4, 1152
    n_act = np.array([1025, 1100, 64, 65, 700, 3, 900, 1024], np.int32)
    n_orig = n_act + 10
    stopped = np.array([0, 0, 2, 0], np.int32)
    rng = _np_rng("tail", 0)
    x32 = rng.normal(0.0, 1.0, (2 * P * NP, 256)).astype(np.float32)
    wt, wm = (rng.normal(0.0, 0.08, 256).astype(np.float32) for _ in range(2))
    bt, bm, thr, keep_thr = np.float32(2.0), np.float32(2.5), np.float32(0.9), np.float32(0.95)
    args = dict(x32=x32, wt=wt, bt=bt, wm=wm, bm=bm, sentinel=SENT)
    zero = np.zeros(P, np.int32)
    first = st.lg_tail(P, NP, n_act, n_orig, stopped, zero, 3, thr, 2.0, keep_thr, True, True, 64, **args)
    live = np.zeros((2 * P, NP), bool)
    for s in range(2 * P):
        live[s, :n_act[s]] = stopped[s // 2] == 0
    x = x32.reshape(2 * P, NP, 256).astype(np.float64)
    for key, w, b in (("tok", wt, bt), ("mat", wm, bm)):
        y = x @ w.astype(np.float64) + float(b)
        ref = 1.0 / (1.0 + np.exp(-y))
        bound = U * (TOK_DOT * (np.abs(x * w.astype(np.float64)).sum(2) + abs(float(b))) + TOK_ABS)
        err = np.abs(first[key].astype(np.float64) - ref)
        assert (err[live] <= bound[live]).all(), f"{key}: {err[live].max():.3g}"
        assert (first[key][~live] == SENT).all(), f"{key} written for a stopped pair or past n_act"
        _worst(key, (err[live] / bound[live]).max())
    cnt = np.array([int((first["tok"][2 * p:2 * p + 2][live[2 * p:2 * p + 2]] < thr).sum()) for p in range(P)], np.int32)
    tot = (n_orig[0::2] + n_orig[1::2]).astype(np.float32)
    ratio = np.float32(1.0) - cnt.astype(np.float32) / tot
    assert len(set(ratio[[0, 1, 3]].tolist())) == 3
    depth_conf = ratio[0]
    out = st.lg_tail(P, NP, n_act, n_orig, stopped, zero, 3, thr, depth_conf, keep_thr, True, True, 64, **args)
    assert np.array_equal(_bits(out["tok"]), _bits(first["tok"])) and np.array_equal(_bits(out["mat"]), _bits(first["mat"]))
    counter, st_ref, mp, nn = decide_ref(n_act, n_orig, stopped, cnt, out["tok"], out["mat"], NP, 3, thr, depth_conf, keep_thr, True, True, 64)
    assert np.array_equal(out["stopped"], st_ref) and st_ref[0] == 0
    assert np.array_equal(out["counter"], np.where(stopped != 0, 0, counter))
    assert np.array_equal(out["n_next"], nn) and np.array_equal(out["map"], mp)
    print(f"lg_tail: worst of bound {WORST}")


# ---- SuperGlue
def _sg_pairs(kind, rng):
    if kind == "random":
        shapes = [(33, 255), (255, 33), (1, 2), (1025, 256), (256, 1024)]
    else:
        shapes = [(31, 32), (256, 255), (2, 1), (1024, 1023), (32, 33)]
    return [rng.normal(0.0, 2.0, s).astype(np.float32) for s in shapes]


def sg_check_matches(what, out, scores, th, cap):
    """Argmaxes, maxima and tables bitwise from the kernel's own u, v and pc."""
    for p, Z in enumerate(scores):
        m, n = Z.shape
        la = la_sg(Z, out["u"][p, :m], out["v"][p, :n], out["pc"][p, 0])
        a0, a1 = first_argmax(la, 1), first_argmax(la, 0)
        w = f"{what} pair {p} ({m} x {n})"
        assert np.array_equal(out["arg0"][p, :m], a0), f"{w}: row argmax at {np.flatnonzero(out['arg0'][p, :m] != a0)[:5]}"
        assert np.array_equal(out["arg1"][p, :n], a1), f"{w}: column argmax"
        best = la[np.arange(m), a0]
        assert _same(out["best0"][p, :m], best), f"{w}: maxima"
        assert (out["arg0"][p, m:] == ISENT).all() and (out["arg1"][p, n:] == ISENT).all() and (out["best0"][p, m:] == SENT).all()
        check_table(w, out["matches"][p], out["mscores"][p], out["n_matches"][p], best, a0, a1, np.arange(m), np.arange(n), th, cap)
    for k in ("u", "v", "best0", "mscores", "pc"):
        assert (out[k + "_tail"] == SENT).all(), f"{what}: write past {k}"
    for k in ("arg0", "arg1", "matches", "n_matches"):
        assert (out[k + "_tail"] == ISENT).all(), f"{what}: write past {k}"


@pytest.mark.gpu
def test_sg_half_step(st):
    """One row pass and one column pass from given u / v against float64, under the per-step bound; pc bitwise."""
    rng = _np_rng("sgh", 0)
    scores = [rng.normal(0.0, 3.0, s).astype(np.float32) for s in [(1, 2), (33, 31), (255, 1024), (2048, 1025), (1023, 256)]]
    NPt = 2048
    u0 = np.zeros((5, NPt + 1), np.float32)
    v0 = rng.normal(-7.0, 2.0, (5, NPt + 1)).astype(np.float32)
    for alpha in (-2.0, 1.0, 6.0):
        out = st.sg_sinkhorn(scores, alpha, wave=2, half_steps=2, u=u0, v=v0, th=0.2, sentinel=SENT)
        assert out["NPt"] == NPt
        for p, Z in enumerate(scores):
            m, n = Z.shape
            assert np.array_equal(out["pc"][p, :3], np.array([-math.log(m + n), math.log(n), math.log(m)], np.float32))
            u, _, bu = ref_sinkhorn(Z, np.float32(alpha), 1, v0=v0[p, :n + 1])
            v, bv = _col_pass(Z, np.float32(alpha), out["u"][p, :m + 1])  # the column pass from the kernel's own u
            eu, ev = np.abs(out["u"][p, :m + 1] - u).max(), np.abs(out["v"][p, :n + 1] - v).max()
            assert eu <= bu[0] and ev <= bv, f"alpha {alpha} pair {p}: {eu:.3g} / {bu[0]:.3g}, {ev:.3g} / {bv:.3g}"
            assert (out["u"][p, m + 1:] == 0).all() and (out["v"][p, n + 1:] == v0[p, n + 1:]).all()
            _worst("sk_half", max(eu / bu[0], ev / bv))
        sg_check_matches(f"half step alpha {alpha}", out, scores, 0.2, out["matches"].shape[1])
    print(f"sg half step: worst of bound {WORST}")


def _col_pass(Z, alpha, u):
    """The column half step in float64 from the given u, and its bound."""
    m, n = Z.shape
    c = np.full((m + 1, n + 1), float(alpha))
    c[:m, :n] = Z
    x = c + u.astype(np.float64)[:, None]
    mx = x.max(0)
    ls = np.log(np.exp(x - mx[None]).sum(0))
    v = np.r_[np.full(n, -math.log(m + n)), math.log(m) - math.log(m + n)] - (mx + ls)
    return v, U * (SK_XS * np.abs(x).max() + SK_LEN * (m + 1) / 32 + SK_ABS + 2 * np.abs(ls).max() + 2 * np.abs(v).max())


@pytest.mark.gpu
@pytest.mark.parametrize("alpha", [-3.0, 1.0, 40.0], ids=["alpha_small", "alpha_typical", "alpha_large"])
@pytest.mark.parametrize("kind", ["random", "shapes2"])
def test_sg_sinkhorn_100_iterations(st, alpha, kind):
    """100 iterations against log_optimal_transport in float64 under the summed per-step bound, in waves of 1, 2 and P = 5 with
    identical results; matches bitwise from the kernel's u / v.  At alpha 40 everything goes to the dustbin: no match."""
    scores = _sg_pairs(kind, _np_rng("sg", kind))
    outs = [st.sg_sinkhorn(scores, alpha, wave=w, half_steps=200, th=0.2, cap=600, sentinel=SENT) for w in (1, 2, 5)]
    for o in outs[1:]:
        for k in ("u", "v", "arg0", "arg1", "matches", "mscores", "n_matches"):
            assert np.array_equal(np.asarray(o[k]).view(np.uint8), np.asarray(outs[0][k]).view(np.uint8)), f"wave changes {k}"
    out = outs[0]
    for p, Z in enumerate(scores):
        m, n = Z.shape
        u, v, b = ref_sinkhorn(Z, np.float32(alpha), 200)
        err = max(np.abs(out["u"][p, :m + 1] - u).max(), np.abs(out["v"][p, :n + 1] - v).max())
        assert err <= sum(b), f"pair {p} ({m} x {n}): {err:.3g} > {sum(b):.3g}"
        _worst("sk_100", err / sum(b))
    sg_check_matches(f"{kind} alpha {alpha}", out, scores, 0.2, 600)
    if alpha == 40.0:
        assert (out["n_matches"] == 0).all()
    print(f"sg 100 iterations: worst of bound {WORST}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ties", "constant", "diag", "chains", "wide"] + NONFINITE)
def test_sg_matches(st, name):
    """The match kernels on designed scores with given u / v (no Sinkhorn step): ties across lanes, lane wraps, ty strides and
    compaction chunks, a constant block, many matches with cap below the count, non-mutual chains, a wide range; NaN and -inf rows and
    columns (after the fix) never match and keep every index in range."""
    rng = _np_rng("sgm", name)
    scores, us, vs = [], [], []
    NPt = 2048
    for m, n in [(2048, 1025), (1023, 1024), (33, 32), (1, 1), (255, 256)]:
        s, l0, l1 = design(name if name != "neginf" else "random", m, n, rng)
        if name == "neginf":
            s[[0, m // 2, m - 1]] = -np.inf
            s[:, [0, n - 1]] = -np.inf
        scores.append(s)
        us.append(np.r_[l0, 0.0, np.zeros(NPt - m)].astype(np.float32))
        vs.append(np.r_[l1, 0.0, np.zeros(NPt - n)].astype(np.float32))
    out = st.sg_sinkhorn(scores, 1.0, wave=5, half_steps=0, u=np.stack(us), v=np.stack(vs), th=0.2, cap=900, sentinel=SENT)
    sg_check_matches(name, out, scores, 0.2, 900)
    for p, Z in enumerate(scores):
        m, n = Z.shape
        assert (out["arg0"][p, :m] >= 0).all() and (out["arg0"][p, :m] < n).all() and (out["arg1"][p, :n] < m).all()
        if name in NONFINITE:  # rows whose maximum is NaN or -inf
            bad = ~np.isfinite(out["best0"][p, :m])
            assert bad.any()
            rows = {int(r) for r in out["matches"][p, :min(int(out["n_matches"][p]), 900), 0]}
            assert not rows & set(np.flatnonzero(bad).tolist()), f"{name}: a non-finite row matched"
