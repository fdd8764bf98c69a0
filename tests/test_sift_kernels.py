"""The SIFT kernels (csrc/sift_kernels.cuh) stage by stage, against float64 references on the same inputs.

tests/test_sift.py compares whole extractions with cv2, with slack for differences between OpenCV builds; a kernel bug that touches a
rare class of keypoints fits inside that slack.  Here the self-test library runs each stage through the launch helper sift_run calls
(dimb_selftest_sift_extrema / _ori / _select / _desc), on levels, candidates and records given in the production layout, with every
output buffer starting as a sentinel and followed by a tail, so missing and stray writes both show.

The references follow oracle.sift's recipe in float64, with OpenCV's float32 fastAtan2, and report the margin of every decision they
take: the distance of the deciding quantity from its threshold.  The device may disagree with a reference only where that margin is
below the bound stated for the stage:
  extrema      the 26-neighbour test reads the same floats on both sides, so it is exact.  Survivors agree with the float64
               refinement unless a decision's relative margin is below REFINE_MARGIN; kept offsets within OFFSET_TOL, contr within
               CONTR_REL relative.
  orientation  the angle set equals the float64 set, each angle within ANGLE_TOL degrees; an angle may be missing on one side only when
               its bin is within HIST_REL relative of 0.8 of the maximum or of a neighbour.  x, y, response and the packed octave are
               bitwise the formulas' float32 values; size within 2 ulp (powf).
  selection    bitwise numpy: lexsort on (x asc, y asc, size desc, angle asc, response desc, octave desc), stable; duplicates in (x, y,
               size, angle) dropped, the first kept; retainBest keeps every row at or above the n-th response.
  descriptors  every byte is rint of the float64 value unless that value is within HALF_TIE of a half-integer, and within DESC_ABS of
               the float64 value always.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import sift as O

SENT = -777.0
ISENT = int(np.float32(SENT).view(np.int32))
ERR_ARG, ERR_UNSUPPORTED = -3, -4
REFINE_MARGIN = 1e-4
OFFSET_TOL = 1e-4
CONTR_REL = 1e-5
ANGLE_TOL = 1e-3
HIST_REL = 1e-5
HALF_TIE = 0.01
DESC_ABS = 0.51
K_CHUNK, K_SORT_TILE = 4096, 2048
# (n_octave_layers, contrast_threshold, edge_threshold, sigma) that the sift+kornia_matcher pipeline never runs: cv2's defaults (integer
# extremum threshold 1 instead of 0), other layer counts, a tighter edge ratio, and sigma on both sides of the first blur's branch
SETTINGS = [(3, 0.04, 10.0, 1.6), (2, 0.0004, 10.0, 1.6), (5, 0.04, 10.0, 1.6), (3, 0.04, 5.0, 1.6), (3, 0.04, 10.0, 1.0),
            (3, 0.04, 10.0, 2.5)]


# ------------------------------------------------------------------ references
def refine(dog, o, layer, r, c, L, contrast, edge):
    """adjustLocalExtrema in float64 on float32 DoG levels dog[o][level] ([h][w]).  Returns (result, margin, reason, path): result (layer,
    r, c, xc, xr, xi, contr) or None, reason the outcome ('ok', 'steps', 'outside', 'contrast', 'edge', 'det'), margin the smallest
    relative distance of a deciding quantity from its threshold along the way (offsets against 0.5 and half-integers, the determinants
    against 0, contrast and edge ratios against theirs), path the (layer, r, c) positions visited, the last one where it stopped.
    A determinant that is 0 because a row of its matrix is exactly 0 (equal levels, a plateau) is 0 in float32 too: an exact decision,
    not a margin of 0."""
    ds, ss, cs = 0.5 / 255, 1.0 / 255, 0.25 / 255
    h, w = dog[o][0].shape
    margin = np.inf
    X = np.zeros(3)
    rr, cc = r, c
    path = [(layer, rr, cc)]
    for step in range(6):
        if step == 5:
            return None, margin, "steps", path
        I, P, N = _nbhd(dog, o, layer, rr, cc)
        r, c = 1, 1  # centre of the 3 x 3 neighbourhoods (the position is kept in rr, cc)
        g = np.array([(I[r, c + 1] - I[r, c - 1]) * ds, (I[r + 1, c] - I[r - 1, c]) * ds, (N[r, c] - P[r, c]) * ds])
        v2 = I[r, c] * 2
        dxx, dyy, dss = (I[r, c + 1] + I[r, c - 1] - v2) * ss, (I[r + 1, c] + I[r - 1, c] - v2) * ss, (N[r, c] + P[r, c] - v2) * ss
        dxy = (I[r + 1, c + 1] - I[r + 1, c - 1] - I[r - 1, c + 1] + I[r - 1, c - 1]) * cs
        dxs = (N[r, c + 1] - N[r, c - 1] - P[r, c + 1] + P[r, c - 1]) * cs
        dys = (N[r + 1, c] - N[r - 1, c] - P[r + 1, c] + P[r - 1, c]) * cs
        H = np.array([[dxx, dxy, dxs], [dxy, dyy, dys], [dxs, dys, dss]])
        if np.any(np.all(H == 0, axis=1)):
            X = np.zeros(3)  # Cramer's d is exactly 0 in float as well: X = 0
        else:
            det = np.linalg.det(H)
            margin = min(margin, abs(det) / (np.prod(np.abs(H).sum(1))))
            X = -np.linalg.solve(H, g) if det != 0 else np.zeros(3)
        xc, xr, xi = X
        margin = min(margin, np.min(np.abs(np.abs(X) - 0.5)) / 0.5)
        if np.all(np.abs(X) < 0.5):
            break
        margin = min(margin, np.min(np.abs(np.abs(X - np.floor(X)) - 0.5)) / 0.5)
        cc, rr, layer = cc + int(np.rint(xc)), rr + int(np.rint(xr)), layer + int(np.rint(xi))
        path.append((layer, rr, cc))
        if layer < 1 or layer > L or cc < O.BORDER or cc >= w - O.BORDER or rr < O.BORDER or rr >= h - O.BORDER:
            return None, margin, "outside", path
    I, P, N = _nbhd(dog, o, layer, rr, cc)
    r, c = 1, 1
    g = np.array([(I[r, c + 1] - I[r, c - 1]) * ds, (I[r + 1, c] - I[r - 1, c]) * ds, (N[r, c] - P[r, c]) * ds])
    contr = I[r, c] / 255 + 0.5 * float(g @ np.array([xc, xr, xi]))
    if contrast > 0:
        margin = min(margin, abs(abs(contr) * L - contrast) / contrast)
    if abs(contr) * L < contrast:
        return None, margin, "contrast", path
    v2 = I[r, c] * 2
    dxx, dyy = (I[r, c + 1] + I[r, c - 1] - v2) * ss, (I[r + 1, c] + I[r - 1, c] - v2) * ss
    dxy = (I[r + 1, c + 1] - I[r + 1, c - 1] - I[r - 1, c + 1] + I[r - 1, c - 1]) * cs
    tr, det = dxx + dyy, dxx * dyy - dxy * dxy
    if abs(dxx * dyy) + dxy * dxy > 0:  # else every term is exactly 0, in float32 too
        margin = min(margin, abs(det) / (abs(dxx * dyy) + dxy * dxy))
    if det <= 0:
        return None, margin, "det", path
    lhs, rhs = tr * tr * edge, (edge + 1) ** 2 * det
    margin = min(margin, abs(lhs - rhs) / max(lhs, rhs))
    if lhs >= rhs:
        return None, margin, "edge", path
    return (layer, rr, cc, xc, xr, xi, contr), margin, "ok", path


def _nbhd(dog, o, layer, r, c):
    """The 3 x 3 neighbourhoods of (r, c) in DoG levels layer, layer - 1 and layer + 1, in float64."""
    return [dog[o][layer + k][r - 1:r + 2, c - 1:c + 2].astype(np.float64) for k in (0, -1, 1)]


def initial_extrema(dog, o, layer, thr):
    """The 26-neighbour test of findScaleSpaceExtrema on float32 levels (>= / <= every neighbour, |value| > thr), outside the border."""
    stack = np.stack(dog[o][layer - 1:layer + 2])
    h, w = stack.shape[1:]
    B = O.BORDER
    core = stack[1, B:h - B, B:w - B]
    mx, mn = np.full(core.shape, -np.inf, np.float32), np.full(core.shape, np.inf, np.float32)
    for dl in range(3):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                s = stack[dl, B + dy:h - B + dy, B + dx:w - B + dx]
                mx, mn = np.maximum(mx, s), np.minimum(mn, s)
    rr, cc = np.nonzero((np.abs(core) > thr) & (((core > 0) & (core >= mx)) | ((core < 0) & (core <= mn))))
    return rr + B, cc + B


def ref_extrema(dog, L, contrast, edge):
    """Refinement of every initial extremum of one image: list of (o, result, margin, reason, path)."""
    thr = np.floor(0.5 * contrast / L * 255)
    out = []
    for o in range(len(dog)):
        h, w = dog[o][0].shape
        if h <= 2 * O.BORDER or w <= 2 * O.BORDER:
            continue
        for layer in range(1, L + 1):
            for r, c in zip(*initial_extrema(dog, o, layer, thr)):
                out.append((o,) + refine(dog, o, layer, int(r), int(c), L, contrast, edge))
    return out


def decode_cand(cand, n):
    """Cand records [n][6] int32 -> (o, layer, r, c) int array [n][4] and (xc, xr, xi, contr) float32 [n][4]."""
    u = cand[:n].view(np.uint32)
    ints = np.stack([u[:, 0] >> 8, u[:, 0] & 255, u[:, 1] >> 16, u[:, 1] & 0xffff], 1).astype(np.int64)
    return ints, cand[:n, 2:].view(np.float32)


def encode_cand(rows):
    """(o, layer, r, c, xc, xr, xi, contr) tuples -> Cand records [n][6] int32."""
    out = np.zeros((len(rows), 6), np.int32)
    for k, (o, ly, r, c, *f) in enumerate(rows):
        out[k, 0] = (o << 8) | ly
        out[k, 1] = np.uint32((r << 16) | c).view(np.int32)
        out[k, 2:] = np.array(f, np.float32).view(np.int32)
    return out


def ori_hist(img, r, c, radius, sig):
    """calcOrientationHist in float64 with the float32 fastAtan2 and bin rounding: the smoothed 36-bin histogram."""
    h, w = img.shape
    i, j = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    y, x = r + i, c + j
    ok = (y > 0) & (y < h - 1) & (x > 0) & (x < w - 1)
    i, j, y, x = i[ok], j[ok], y[ok], x[ok]
    dx = img[y, x + 1] - img[y, x - 1]
    dy = img[y - 1, x] - img[y + 1, x]
    wt = np.exp((i * i + j * j) * (-1.0 / (2.0 * sig * sig)))
    mag = np.sqrt(dx.astype(np.float64) ** 2 + dy.astype(np.float64) ** 2)
    b = np.rint(np.float32(O.ORI_BINS / 360.0) * O.fast_atan2(dy, dx)).astype(int) % O.ORI_BINS
    t = np.bincount(b, weights=wt * mag, minlength=O.ORI_BINS)
    tp = np.concatenate([t[-2:], t, t[:2]])
    return (tp[:-4] + tp[4:]) / 16 + (tp[1:-3] + tp[3:-1]) * 4 / 16 + tp[2:-2] * 6 / 16


def ref_ori(img, o, layer, r, c, xi, L, sigma):
    """One candidate: (angles [(angle, hist margin)], the float32 size formula's float64 value, every bin's margin).  The margin of a
    bin is its relative distance from 0.8 of the maximum and from its neighbours, the decisions of a peak."""
    size = sigma * 2.0 ** ((layer + float(xi)) / L) * (1 << o) * 2
    scl = np.float32(np.float32(size) * np.float32(0.5) / np.float32(1 << o))
    radius = int(np.rint(np.float32(4.5) * scl))
    hist = ori_hist(img, r, c, radius, float(np.float32(1.5) * scl))
    thr = hist.max() * 0.8
    out = []
    for j in range(O.ORI_BINS):
        lft, rgt = hist[j - 1], hist[(j + 1) % O.ORI_BINS]
        m = min(abs(hist[j] - thr), abs(hist[j] - lft), abs(hist[j] - rgt)) / max(hist.max(), 1e-300)
        if hist[j] > lft and hist[j] > rgt and hist[j] >= thr:
            b = j + 0.5 * (lft - rgt) / (lft - 2 * hist[j] + rgt)
            b = b + O.ORI_BINS if b < 0 else (b - O.ORI_BINS if b >= O.ORI_BINS else b)
            a = 360.0 - 360.0 / O.ORI_BINS * b
            out.append((0.0 if abs(a - 360.0) < O.FLT_EPS else a, m))
        elif m < HIST_REL:
            out.append((None, m, j))
    return out


def ori_fields(o, layer, r, c, xc, xr, xi, contr):
    """x, y, response and the packed octave of sift_ori_kernel's formulas, in float32."""
    f = np.float32
    kx, ky = f(f(c) + f(xc)) * f(1 << o), f(f(r) + f(xr)) * f(1 << o)
    oct_ = o + (layer << 8) + (int(np.rint((float(f(xi)) + 0.5) * 255)) << 16)
    return kx, ky, abs(f(contr)), oct_


def ref_select(rec, n, n_features, kcap):
    """sift.select of one image in numpy: (kept record indices, output rows kpts [k][2], frames [k][3], octave [k], count)."""
    if n > kcap:
        return np.zeros(0, int), None, None, None, -1
    f = rec[:, :n]
    octu = f[5].view(np.uint32)
    order = np.lexsort((np.arange(n), -octu.astype(np.int64), -f[4].astype(np.float64), f[3], -f[2].astype(np.float64), f[1], f[0]))
    keep = [i for k, i in enumerate(order) if k == 0 or not np.array_equal(f[:4, i], f[:4, order[k - 1]])]
    keep = np.array(keep, int)
    if n_features > 0 and len(keep) > n_features:
        t = np.sort(f[4, keep])[::-1][n_features - 1]
        keep = keep[f[4, keep] >= t]
    half = np.float32(0.5)
    oc = f[5, keep].view(np.int32)
    return keep, np.stack([f[0, keep] * half, f[1, keep] * half], 1), np.stack([f[2, keep] * half, f[3, keep], f[4, keep]], 1), \
        (oc & ~255) | ((oc - 1) & 255), len(keep)


def ref_descriptor(img, x, y, angle, size):
    """calcSIFTDescriptor(img, (x, y), 360 - angle, size / 2, 4, 8) in float64, before rounding: 128 values (OpenCV's float32 angle
    conversion 360 - angle, then oracle.sift.descriptor's arithmetic)."""
    d, nb = 4, 8
    ori = float(np.float32(360) - np.float32(angle))
    if abs(ori - 360.0) < O.FLT_EPS:
        ori = 0.0
    scl = size * 0.5
    px, py = int(np.rint(np.float32(x))), int(np.rint(np.float32(y)))
    hw = 3.0 * scl
    radius = int(np.rint(np.float32(hw) * np.float32(1.4142135623730951) * np.float32((d + 1) * 0.5)))
    h, w = img.shape
    radius = min(radius, int(np.sqrt(float(w) * w + float(h) * h)))
    ct = np.cos(np.float32(ori) * np.float32(np.pi / 180)) / hw
    st = np.sin(np.float32(ori) * np.float32(np.pi / 180)) / hw
    i, j = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    i, j = i.ravel(), j.ravel()
    c_rot, r_rot = j * ct - i * st, j * st + i * ct
    rbin, cbin = r_rot + d / 2 - 0.5, c_rot + d / 2 - 0.5
    yy, xx = py + i, px + j
    ok = (rbin > -1) & (rbin < d) & (cbin > -1) & (cbin < d) & (yy > 0) & (yy < h - 1) & (xx > 0) & (xx < w - 1)
    rbin, cbin, c_rot, r_rot, yy, xx = rbin[ok], cbin[ok], c_rot[ok], r_rot[ok], yy[ok], xx[ok]
    dx = img[yy, xx + 1] - img[yy, xx - 1]
    dy = img[yy - 1, xx] - img[yy + 1, xx]
    wt = np.exp((c_rot * c_rot + r_rot * r_rot) * (-1.0 / (d * d * 0.5)))
    obin = (O.fast_atan2(dy, dx).astype(np.float64) - ori) * (nb / 360.0)
    mag = np.sqrt(dx.astype(np.float64) ** 2 + dy.astype(np.float64) ** 2) * wt
    r0, c0, o0 = np.floor(rbin).astype(int), np.floor(cbin).astype(int), np.floor(obin).astype(int)
    rbin, cbin, obin = rbin - r0, cbin - c0, obin - o0
    o0 = np.where(o0 < 0, o0 + nb, o0)
    o0 = np.where(o0 >= nb, o0 - nb, o0)
    hist = np.zeros((d + 2) * (d + 2) * (nb + 2))
    for dr, wr in ((0, 1 - rbin), (1, rbin)):
        for dc, wc in ((0, 1 - cbin), (1, cbin)):
            for do, wo in ((0, 1 - obin), (1, obin)):
                np.add.at(hist, ((r0 + 1 + dr) * (d + 2) + c0 + 1 + dc) * (nb + 2) + o0 + do, mag * wr * wc * wo)
    hist = hist.reshape(d + 2, d + 2, nb + 2)[1:d + 1, 1:d + 1]
    hist[:, :, :2] += hist[:, :, nb:nb + 2]
    v = hist[:, :, :nb].ravel()
    v = np.minimum(v, np.sqrt(np.sum(v * v)) * 0.2)
    return v * (512.0 / max(np.sqrt(np.sum(v * v)), O.FLT_EPS))


def check_desc_bytes(got, ref, what):
    """The descriptor bars: bytes are rint of the float64 value off a half-integer tie, and within DESC_ABS of it always."""
    ref = np.clip(ref, 0, 255)
    assert np.abs(got - ref).max() <= DESC_ABS, (what, np.abs(got - ref).max())
    clear = np.abs(np.abs(ref - np.floor(ref)) - 0.5) > HALF_TIE
    bad = clear & (got != np.rint(ref))
    assert not bad.any(), (what, np.argwhere(bad)[:5], got[bad][:5], ref[bad][:5])


# ------------------------------------------------------------------ synthetic inputs
def planted_dog(seed, h, w, L, n_bumps=40, explicit=True):
    """One octave of L + 2 DoG levels [L + 2][h][w] with planted extrema: Gaussian bumps of both signs at sub-pixel centres, elongated
    and sheared (edge ratio on both sides, refinement over several steps), centred between layers (a step across a layer), at rows
    and columns 5 and w - 6 and beyond the border; explicit 3 x 3 x 3 patterns: a saddle, a singular Hessian (no change across
    layers), a flat plateau and a ridge (ties that must pass >=), a faint extremum (contrast test)."""
    rng = np.random.default_rng(seed)
    D = np.zeros((L + 2, h, w), np.float64)
    ll, yy, xx = np.meshgrid(np.arange(L + 2), np.arange(h), np.arange(w), indexing="ij")
    for k in range(n_bumps):
        edge_pos = k % 5 == 0
        y0 = rng.choice([5.0, h - 6.0, 4.6, h - 5.4]) if edge_pos else rng.uniform(3, h - 4)
        x0 = rng.choice([5.0, w - 6.0, 4.6, w - 5.4]) if k % 5 == 1 else rng.uniform(3, w - 4)
        y0, x0 = y0 + rng.uniform(-0.49, 0.49) * (not edge_pos), x0 + rng.uniform(-0.49, 0.49) * (k % 5 != 1)
        l0 = rng.uniform(0.5, L + 0.5)
        sx, sy, sl = rng.uniform(0.7, 3.0), rng.uniform(0.7, 3.0) * (rng.uniform(1, 6) if k % 3 == 0 else 1), rng.uniform(0.6, 1.5)
        sh = rng.uniform(-1.5, 1.5) if k % 4 == 0 else 0.0
        amp = rng.choice([-1, 1]) * rng.uniform(0.5, 12)
        u, v = xx - x0 + sh * (yy - y0), yy - y0
        D += amp * np.exp(-(u * u / (2 * sx * sx) + v * v / (2 * sy * sy) + (ll - l0) ** 2 / (2 * sl * sl)))
    D = D.astype(np.float32)
    if explicit and h >= 40 and w >= 40:
        def put(y, x, l, block):
            D[l - 1:l + 2, y - 1:y + 2, x - 1:x + 2] = block
        base = np.zeros((3, 3, 3), np.float32)
        saddle = base.copy()
        saddle[1] = [[9.9, 9.0, 5.0], [9.0, 10.0, 9.0], [5.0, 9.0, 9.9]]
        saddle[0] = saddle[2] = 4.0
        singular = np.stack([np.float32([[8, 9, 8], [9, 10, 9], [8, 9, 8]])] * 3)
        plateau = np.full((3, 3, 3), 6.0, np.float32)
        ridge = base.copy()
        ridge[1] = [[3, 3, 3], [7, 7, 7], [3, 3, 3]]
        faint = base.copy()
        faint[1, 1, 1] = 1.2
        for k, blk in enumerate([saddle, singular, plateau, ridge, faint]):
            put(12, 10 + 6 * k, 1 + k % L, blk)
    return D


# sheared bumps whose maximum lies between columns w - 6 and w - 5 of a 24 x 32 level: the extremum at column w - 6 = 26 steps to
# w - 5, the first column refinement must not keep (c >= w - 5 drops it; from there it would converge, clear of every threshold)
EDGE_COLUMN_BUMPS = [(27.3768, 12.362, 1.5555, 1.5534, 1.7267, 0.8216, 1.4396), (26.798, 9.2546, 1.9472, 1.8603, 1.5611, 0.9242, -1.2534),
                     (26.6241, 9.8388, 2.3365, 1.7775, 1.1809, 1.4333, 0.8668)]


def edge_column_dog(x0, y0, l0, sx, sy, sl, sh, h=24, w=32, L=3):
    ll, yy, xx = np.meshgrid(np.arange(L + 2), np.arange(h), np.arange(w), indexing="ij")
    u = xx - x0 + sh * (yy - y0)
    return (8 * np.exp(-(u * u / (2 * sx * sx) + (yy - y0) ** 2 / (2 * sy * sy) + (ll - l0) ** 2 / (2 * sl * sl)))).astype(np.float32)


def gauss_patch(kind, h=48, w=48, seed=0):
    """One Gaussian level [h][w] for the orientation and descriptor kernels: 'ramp<deg>' a linear ramp whose gradient points at deg
    (0 / 360 and bin edges included), 'peaks<k>' k sectors of different directions and near-equal weight, 'plateau' two directions
    of equal weight two bins apart (an equal-neighbour pair), 'flat' a constant, 'noise' random values."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    if kind.startswith("ramp"):
        t = np.deg2rad(float(kind[4:]))
        return (17.0 * (np.cos(t) * xx - np.sin(t) * yy)).astype(np.float32)
    if kind.startswith("peaks"):
        k = int(kind[5:])
        ang = np.arctan2(yy - h / 2 + 0.5, xx - w / 2 + 0.5)
        sector = np.floor((ang + np.pi) / (2 * np.pi) * k).astype(int) % k
        out = np.zeros((h, w))
        for s in range(k):
            t = np.deg2rad(37.0 + 360.0 / k * s + 11 * s)
            out += (sector == s) * (9.0 + s) * (np.cos(t) * xx - np.sin(t) * yy)
        return out.astype(np.float32)
    if kind == "plateau":
        return (np.where(xx + yy < h, 5.0 * xx, 5.0 * (np.cos(0.349) * xx - np.sin(0.349) * yy))).astype(np.float32)
    if kind == "flat":
        return np.full((h, w), 100.0, np.float32)
    return (rng.random((h, w)) * 255).astype(np.float32)


# ------------------------------------------------------------------ helpers
def _octave_levels(stack, B=None):
    """[n_levels][h][w] of one image, or a list of B of them -> [n_levels][B][h][w]."""
    if isinstance(stack, list):
        return np.stack(stack, 1)
    return stack[:, None]


def _device_pyramid(ctx, img, L=3, contrast=0.0004, edge=10.0, sigma=1.6):
    """Gaussian and DoG levels of the production pyramid of img, read back (SiftNet.debug_read)."""
    from dim_b200 import _native
    H, W = img.shape
    net = _native.SiftNet(ctx, 0, L, contrast, edge, sigma, 1, H, W)
    net.extract(img)
    n_oct = len(_native.sift_octaves(H, W))
    gauss = [[net.debug_read(0, 0, o, i, H, W) for i in range(L + 3)] for o in range(n_oct)]
    dog = [[net.debug_read(1, 0, o, i, H, W) for i in range(L + 2)] for o in range(n_oct)]
    return gauss, dog


def _compare_extrema(cand, count, tail, dogs, L, contrast, edge, what):
    """Device candidates of B images against ref_extrema; returns (number compared, reasons seen)."""
    assert np.all(tail["cand"] == ISENT) and np.all(tail["count"] == ISENT), what
    reasons, total = {}, 0
    for b, dog in enumerate(dogs):
        n = int(count[b])
        assert n <= cand.shape[1], (what, b, n)
        assert np.all(cand[b, n:] == ISENT), (what, b)
        ints, fl = decode_cand(cand[b], n)
        ref = ref_extrema(dog, L, contrast, edge)
        for _, _, _, why, _ in ref:
            reasons[why] = reasons.get(why, 0) + 1
        dev = {}
        for k in range(n):
            dev.setdefault(tuple(ints[k]), []).append(fl[k])
        # two initial extrema can refine to one position; sure survivors take their device entries first, so a low-margin one is
        # the one left over when the device took the other side of its decision
        for o, res, m, why, _ in sorted(ref, key=lambda t: -t[2]):
            if res is None:
                continue
            key = (o, res[0], res[1], res[2])
            got = dev.get(key)
            if not got:
                assert m < REFINE_MARGIN, (what, b, "missing on the device", key, res, m)
                continue
            err = [np.abs(np.array(g[:3], np.float64) - res[3:6]).max() for g in got]
            g = got.pop(int(np.argmin(err)))
            assert min(err) <= OFFSET_TOL or m < REFINE_MARGIN, (what, b, key, min(err), m)
            if not any(res[3:6]) and m >= REFINE_MARGIN:  # a singular Hessian: d == 0 in float too, so X = 0 exactly
                assert not np.any(g[:3]), (what, b, key, "singular Hessian with offsets", g)
            assert abs(g[3] - res[6]) <= CONTR_REL * abs(res[6]) or m < REFINE_MARGIN, (what, b, key, float(g[3]), res[6], m)
            total += 1
        # a device survivor the reference does not keep there is excused only by a reference candidate with a low-margin decision
        # whose refinement passed within one pixel and one layer of that position (the device took the other side of that decision)
        near = [(o, path) for o, res, m, why, path in ref if m < REFINE_MARGIN]
        for key, vals in dev.items():
            if not vals:
                continue
            ok = any(o == key[0] and max(abs(p[0] - key[1]), abs(p[1] - key[2]), abs(p[2] - key[3])) <= 1 for o, path in near for p in path)
            assert ok, (what, b, "extra on the device", key, vals)
    return total, reasons


# ------------------------------------------------------------------ no GPU needed
def test_references_agree_with_oracle_on_real_levels():
    """The margin-reporting references reduce to oracle.sift's detector and descriptor on the oracle's own pyramid of real240x320."""
    from test_sift import _golden
    img = _golden("real240x320")
    gauss, dog = O.pyramid(img, 3, 1.6)
    kps = O.detect(gauss, dog, 3, 0.0004, 10.0, 1.6)
    ref = [(o, res) for o, res, m, why, _ in ref_extrema(dog, 3, 0.0004, 10.0) if res is not None]
    assert len(ref) > 300
    # every oracle keypoint comes from a survivor at the same position (the two solvers round differently in the last bits)
    pos = np.array([((res[2] + res[3]) * (1 << o), (res[1] + res[4]) * (1 << o)) for o, res in ref])
    assert all(np.abs(pos - np.array([k[0], k[1]], np.float64)).max(1).min() < 1e-4 for k in kps)
    for q, k in enumerate(kps[:40]):
        o, ly = k[5] & 255, (k[5] >> 8) & 255
        scale = 2.0 if o == 0 else 1.0 / (1 << (o - 1))
        x, y, s = float(k[0]) * 0.5 * scale, float(k[1]) * 0.5 * scale, float(k[2]) * 0.5 * scale
        v = ref_descriptor(gauss[o][ly], np.float32(x), np.float32(y), k[3], s)
        assert np.array_equal(np.clip(np.rint(v), 0, 255), O.descriptor(gauss[o][ly], x, y, float(k[3]), s))


def test_synthetic_stacks_cover_every_refinement_outcome():
    """The planted DoG stacks reach every branch of adjustLocalExtrema in the reference: kept, not converged in 5 steps, stepped out of
    the border or the layer range, contrast, det <= 0 and the edge ratio.  Kept extrema converge after 1 to 4 interpolations (0 to 3
    moves), some after a move across a layer, and the planted singular Hessian (equal levels) is kept with X = 0 exactly."""
    seen, moves, across, singular = {}, set(), 0, 0
    for L in (1, 2, 3, 5):
        for seed in range(3):
            dog = [list(planted_dog(10 * L + seed, 48, 64, L))]
            for contrast in (0.0004, 0.04):
                for o, res, m, why, path in ref_extrema(dog, L, contrast, 10.0):
                    seen[why] = seen.get(why, 0) + 1
                    if why == "ok":
                        moves.add(len(path) - 1)
                        across += len({p[0] for p in path}) > 1
                        singular += res[1:3] == (12, 16) and not any(res[3:6]) and m >= REFINE_MARGIN
    assert set(seen) == {"ok", "steps", "outside", "contrast", "det", "edge"}, seen
    assert {0, 1, 2, 3} <= moves and across > 0, (moves, across)
    assert singular > 0


def test_edge_column_bumps_step_out_of_the_border():
    """Each EDGE_COLUMN_BUMPS extremum starts at column w - 6 and is dropped for stepping to w - 5, with a margin far above
    REFINE_MARGIN, so a device that kept column w - 5 would fail test_extrema_leaving_by_one_column."""
    for bump in EDGE_COLUMN_BUMPS:
        ref = ref_extrema([list(edge_column_dog(*bump))], 3, 0.0004, 10.0)
        out = [(m, why) for o, res, m, why, _ in ref if why == "outside"]
        assert len(out) == 1 and out[0][0] > 1e-2, ref


def test_selection_reference_is_oracle_select():
    """ref_select on records is oracle.sift.select (sorted order, dedup, retainBest ties) on the same keypoints."""
    rng = np.random.default_rng(1)
    n = 300
    rec = _records(rng, n, dup=0.3, ties=0.5)
    kps = [(rec[0, i], rec[1, i], rec[2, i], rec[3, i], rec[4, i], int(rec[5, i:i + 1].view(np.int32)[0])) for i in range(n)]
    for nf in (0, 1, 50, 299, 400):
        keep, kp, fr, oc, cnt = ref_select(rec, n, nf, n)
        exp = O.select(kps, nf)
        assert cnt == len(exp)
        assert np.array_equal(kp * 2, np.array([[k[0], k[1]] for k in exp], np.float32).reshape(-1, 2))
        assert np.array_equal(fr[:, 2], np.array([k[4] for k in exp], np.float32))


def test_sift_selftest_entries_reject_bad_arguments_without_touching_the_gpu():
    """DIMB_ERR_ARG (-3) before any CUDA call: null pointers, and inconsistent sizes with a context pointer never dereferenced."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    null, fake, buf = C.c_void_p(), C.c_void_p(16), C.c_void_p(16)
    hw = np.array([64, 32], np.int32)
    hp = hw.ctypes.data
    assert lib.dimb_selftest_sift_extrema(null, buf, 1, 3, 1, hp, hp, 0.04, 10.0, 1.6, 64, SENT, buf, buf) == ERR_ARG
    for B, L, n_oct, ccap, con, edge, sig in [(0, 3, 1, 64, 0.04, 10, 1.6), (1, 0, 1, 64, 0.04, 10, 1.6), (1, 33, 1, 64, 0.04, 10, 1.6),
                                              (1, 3, 0, 64, 0.04, 10, 1.6), (1, 3, 17, 64, 0.04, 10, 1.6), (1, 3, 1, 0, 0.04, 10, 1.6),
                                              (1, 3, 1, 64, -1, 10, 1.6), (1, 3, 1, 64, 0.04, 0, 1.6), (1, 3, 1, 64, 0.04, 10, 0),
                                              (4096, 32, 1, 64, 0.04, 10, 1.6)]:
        assert lib.dimb_selftest_sift_extrema(fake, buf, B, L, n_oct, hp, hp, con, edge, sig, ccap, SENT, buf, buf) == ERR_ARG
    assert lib.dimb_selftest_sift_extrema(fake, buf, 1, 3, 1, None, hp, 0.04, 10.0, 1.6, 64, SENT, buf, buf) == ERR_ARG
    zero = np.zeros(2, np.int32)
    assert lib.dimb_selftest_sift_extrema(fake, buf, 1, 3, 1, zero.ctypes.data, hp, 0.04, 10.0, 1.6, 64, SENT, buf, buf) == ERR_ARG
    # candidates outside the octaves, layers or level, or with offsets beyond 1
    good = (0, 1, 10, 10, 0.1, -0.2, 0.3, 0.05)
    for bad in [(1, 1, 10, 10, 0, 0, 0, 0.05), (0, 0, 10, 10, 0, 0, 0, 0.05), (0, 4, 10, 10, 0, 0, 0, 0.05), (0, 1, 64, 10, 0, 0, 0, 0.05),
                (0, 1, 10, 64, 0, 0, 0, 0.05), (0, 1, 10, 10, 1.5, 0, 0, 0.05), (0, 1, 10, 10, 0, 0, np.nan, 0.05)]:
        cand = encode_cand([good, bad])
        cc = np.array([2], np.int32)
        assert lib.dimb_selftest_sift_ori(fake, buf, 1, 3, 1, hw[:1].ctypes.data, hw[:1].ctypes.data, 1.6, cand.ctypes.data, cc.ctypes.data,
                                          2, 8, SENT, buf, buf) == ERR_ARG, bad
    neg = np.array([-1], np.int32)
    assert lib.dimb_selftest_sift_ori(fake, buf, 1, 3, 1, hp, hp, 1.6, buf, neg.ctypes.data, 2, 8, SENT, buf, buf) == ERR_ARG
    # a sigma beyond what the 127-tap blurs allow (the sample disc grows with it)
    cand, cc = encode_cand([good]), np.array([1], np.int32)
    assert lib.dimb_selftest_sift_ori(fake, buf, 1, 3, 1, hp, hp, 16.5, cand.ctypes.data, cc.ctypes.data, 1, 8, SENT, buf, buf) == ERR_ARG
    rec = np.zeros((1, 6, 4), np.float32)
    cnt = np.array([4], np.int32)
    for f, v in [(0, -1.0), (4, np.nan), (2, -0.0)]:
        r = rec.copy()
        r[0, f, 2] = v
        assert lib.dimb_selftest_sift_select(fake, r.ctypes.data, cnt.ctypes.data, 1, 4, 0, 4, SENT, buf, buf, buf, buf, buf) == ERR_ARG
    for B, kcap, nf, cap in [(0, 4, 0, 4), (1, 0, 0, 4), (1, 4, -1, 4), (1, 4, 0, 0)]:
        assert lib.dimb_selftest_sift_select(fake, rec.ctypes.data, cnt.ctypes.data, B, kcap, nf, cap, SENT, buf, buf, buf, buf,
                                             buf) == ERR_ARG
    assert lib.dimb_selftest_sift_select(fake, rec.ctypes.data, np.array([-1], np.int32).ctypes.data, 1, 4, 0, 4, SENT, buf, buf, buf, buf,
                                         buf) == ERR_ARG
    rows = np.array([[[10, 10, 3, 45]]], np.float32)
    octv = np.array([[255 | (1 << 8)]], np.int32)
    one = np.array([1], np.int32)
    for rr, oo, cc in [(rows, octv, np.array([2], np.int32)), (rows * [1, 1, 0, 1], octv, one), (rows * [1, 1, 1, 9], octv, one),
                       (rows, np.array([[1 | (1 << 8)]], np.int32), one), (rows, np.array([[255 | (6 << 8)]], np.int32), one)]:
        assert lib.dimb_selftest_sift_desc(fake, buf, 1, 3, 1, hp, hp, np.ascontiguousarray(rr, np.float32).ctypes.data, oo.ctypes.data,
                                           cc.ctypes.data, 1, 1, SENT, buf) == ERR_ARG


@pytest.mark.parametrize("setting", SETTINGS)
def test_oracle_against_cv2_at_other_settings(setting):
    """oracle.sift against cv2.SIFT on real240x320 at parameter settings the pipeline never runs, with test_sift's bars."""
    from test_sift import _check_against, _golden
    L, con, edge, sig = setting
    img = _golden("real240x320")
    conf = dict(n_layers=L, contrast=con, edge=edge, sigma=sig)
    ref = O.cv2_extract(img, 0, **conf)
    assert len(ref["keypoints"]) > 100
    _check_against(O.extract(img, 0, **conf), ref, setting)


# ------------------------------------------------------------------ on the GPU
@pytest.fixture(scope="module")
def st():
    from dim_b200 import _native
    return _native.SelfTest()


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 3, 5])
@pytest.mark.parametrize("contrast", [0.0004, 0.04, 0.0])
def test_extrema_on_planted_stacks(st, L, contrast):
    """Three images with different planted extrema in one call, two octaves (the second smaller than 2 x 5 + 1 rows is skipped when
    tiny), at integer thresholds 0 and 1."""
    dogs = [[list(planted_dog(100 * L + b, 48 + 8 * b, 64, L)), list(planted_dog(7 + b, 24, 32, L, n_bumps=8, explicit=False))]
            for b in range(3)]
    # batches take images of one size: crop to the smallest
    dogs = [[[lv[:48, :64] for lv in d[0]], [lv[:24, :32] for lv in d[1]]] for d in dogs]
    levels = [_octave_levels([np.stack(d[o]) for d in dogs]) for o in range(2)]
    cand, count, tail = st.sift_extrema(levels, L, contrast, 10.0, 1.6, ccap=2048)
    n, reasons = _compare_extrema(cand, count, tail, dogs, L, contrast, 10.0, ("planted", L, contrast))
    assert n > 5, (n, reasons)


@pytest.mark.gpu
def test_extrema_leaving_by_one_column(st):
    """Three images, one EDGE_COLUMN_BUMPS extremum each: the refinement that steps to column w - 5 is dropped on the device too."""
    dogs = [[list(edge_column_dog(*bump))] for bump in EDGE_COLUMN_BUMPS]
    cand, count, tail = st.sift_extrema([_octave_levels([np.stack(d[0]) for d in dogs])], 3, 0.0004, 10.0, 1.6, ccap=64)
    _compare_extrema(cand, count, tail, dogs, 3, 0.0004, 10.0, "edge column")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real240x320", "real_odd237x315", "upscale768x1024"])
def test_extrema_on_device_levels(ctx, st, name):
    """The device's own DoG levels of real images: survivors and their refinement against float64."""
    from test_sift import _golden, _upscale
    img = _upscale() if name.startswith("upscale") else _golden(name)
    for L, contrast in ([(3, 0.0004), (3, 0.04)] if name != "upscale768x1024" else [(3, 0.0004)]):
        gauss, dog = _device_pyramid(ctx, img, L, contrast)
        levels = [_octave_levels(np.stack(d)) for d in dog]
        cand, count, tail = st.sift_extrema(levels, L, contrast, 10.0, 1.6, ccap=200000)
        n, _ = _compare_extrema(cand, count, tail, [dog], L, contrast, 10.0, (name, L, contrast))
        assert n > 200


def _check_ori(rec, kp_count, tail, gauss, cands, L, sigma, what):
    """Device records against ref_ori for the candidates cands[b] (tuples (o, layer, r, c, xc, xr, xi, contr))."""
    assert np.all(tail["rec"] == SENT) and np.all(tail["kp_count"] == ISENT), what
    kcap = rec.shape[2]
    n_total = 0
    for b, cb in enumerate(cands):
        n = int(kp_count[b])
        assert n <= kcap, (what, b, n)
        assert np.all(rec[b, :, n:] == SENT), (what, b)
        r = rec[b, :, :n]
        octs = r[5].view(np.int32)
        rows, close_keys = {}, set()
        for k in range(n):
            rows.setdefault((r[0, k], r[1, k], octs[k]), []).append(k)
        for cd in cb:
            o, layer, rr, cc, xc, xr, xi, contr = cd
            kx, ky, resp, oct_ = ori_fields(o, layer, rr, cc, xc, xr, xi, contr)
            key = (kx, ky, oct_)
            ks = rows.get(key, [])
            angles = ref_ori(gauss[o][layer][b], o, layer, rr, cc, xi, L, sigma)
            exp = [a for a in angles if a[0] is not None]
            size64 = sigma * 2.0 ** ((layer + float(np.float32(xi))) / L) * (1 << o) * 2
            # two candidates that refined to one position share the key: each takes the records of its own angles
            for a, m in exp:
                d = [min(abs(float(r[3, k]) - a), 360 - abs(float(r[3, k]) - a)) for k in ks]
                hit = [i for i in range(len(ks)) if d[i] <= ANGLE_TOL]
                if hit:
                    k = ks.pop(hit[0])
                    assert r[4, k] == resp, (what, b, cd)
                    assert abs(float(r[2, k]) - size64) <= 2 * np.spacing(np.float32(size64)), (what, b, cd, float(r[2, k]), size64)
                    n_total += 1
                else:
                    assert m < HIST_REL, (what, b, cd, "angle missing on the device", a, m)
            if any(a[0] is None or a[1] < HIST_REL for a in angles):
                close_keys.add(key)
        extra = {k: v for k, v in rows.items() if v and k not in close_keys}
        assert not extra, (what, b, "records no candidate's angles explain", [(k, [float(r[3, i]) for i in v]) for k, v in extra.items()][:3])
    return n_total


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real240x320", "real_odd237x315"])
def test_orientation_at_device_candidates(ctx, st, name):
    from test_sift import _golden
    img = _golden(name)
    L, sigma = 3, 1.6
    gauss, dog = _device_pyramid(ctx, img, L)
    cand, count, _ = st.sift_extrema([_octave_levels(np.stack(d)) for d in dog], L, 0.0004, 10.0, sigma, ccap=200000)
    n = int(count[0])
    ints, fl = decode_cand(cand[0], n)
    cds = [tuple(int(v) for v in ints[k]) + tuple(fl[k]) for k in range(n)]
    rec, kc, tail = st.sift_ori([_octave_levels(np.stack(g)) for g in gauss], L, sigma, cand[:, :n], [n], kcap=4 * n)
    g1 = [[lv[None] for lv in g] for g in gauss]
    assert _check_ori(rec, kc, tail, g1, [cds], L, sigma, name) >= n


@pytest.mark.gpu
def test_orientation_on_designed_patches(st):
    """Dominant directions at bin centres and edges, 0 / 360 included (bins 35 and 0), two and three peaks, an equal-neighbour pair, a
    flat patch, candidates whose sample disc is cut by the level's border, and a radius larger than a 12 x 12 level; B = 2 images with
    different counts, and more keypoints than kcap (the counter keeps counting)."""
    L, sigma = 3, 1.6
    kinds = ["ramp0", "ramp5", "ramp10", "ramp355", "ramp356", "ramp359.9", "ramp175", "ramp185", "ramp270", "peaks2", "peaks3",
             "plateau", "flat", "noise"]
    imgs = [np.stack([gauss_patch(k, seed=s) for k in kinds]) for s in (0, 1)]  # [kinds][h][w] per image
    # one octave with L + 3 levels per image: level `layer` of candidate k holds patch k (levels are the patches, cycled)
    cands = [[], []]
    for b in range(2):
        for k in range(len(kinds)):
            for (r, c) in [(24, 24), (5, 24), (24, 42), (1, 1)][: 4 if b == 0 else 2]:
                cands[b].append((0, 1 + k % L, r, c, 0.1 * (k % 3) - 0.1, 0.05, 0.3 * ((k % 5) - 2) / 2, 0.02))
    # every octave is a 48 x 48 level stack of one patch (scl is per octave, so the octave changes only x, y and size)
    n_oct = len(kinds)
    gauss = []
    for o in range(n_oct):
        lv = np.zeros((L + 3, 2, 48, 48), np.float32)
        for b in range(2):
            lv[:, b] = imgs[b][o]
        gauss.append(lv)
    cands = [[(o,) + c[1:] for o in range(n_oct) for c in cands[b] if c[1] == 1 + o % L] for b in range(2)]
    ccap = max(len(c) for c in cands)
    cand = np.full((2, ccap, 6), 0, np.int32)
    for b in range(2):
        cand[b, :len(cands[b])] = encode_cand(cands[b])
    rec, kc, tail = st.sift_ori(gauss, L, sigma, cand, [len(c) for c in cands], kcap=512)
    g1 = [[gauss[o][i] for i in range(L + 3)] for o in range(n_oct)]
    assert _check_ori(rec, kc, tail, g1, cands, L, sigma, "designed") > 20
    # the flat patch gives no keypoint; ramps give one; the two- and three-sector patches several
    per = {}
    octs = rec[0, 5, :kc[0]].view(np.int32)
    for o in octs & 255:
        per[kinds[o]] = per.get(kinds[o], 0) + 1
    assert "flat" not in per and per["peaks3"] > per["ramp10"], per
    # a radius larger than a 12 x 12 level, at its corner and centre, with an xi that makes the scale large
    small = [np.stack([gauss_patch("noise", 12, 12, s)[None] for s in range(L + 3)])]
    cs = [(0, 2, 6, 6, 0.0, 0.0, 0.9, 0.1), (0, 1, 0, 11, 0.2, -0.2, -0.9, 0.1), (0, 3, 11, 0, 0.0, 0.0, 0.5, 0.1)]
    rec, kc, tail = st.sift_ori(small, L, 6.0, encode_cand(cs)[None], [3], kcap=64)
    assert _check_ori(rec, kc, tail, [[small[0][i] for i in range(L + 3)]], [cs], L, 6.0, "small level") >= 3
    # kcap below the keypoint count: the count keeps counting, only kcap records are written
    rec, kc, tail = st.sift_ori(gauss, L, sigma, cand, [len(c) for c in cands], kcap=4)
    assert kc[0] > 4 and np.all(tail["rec"] == SENT)


def _records(rng, n, dup=0.2, ties=0.3, zero_resp=0.05):
    """Keypoint records [6][n] with exact duplicates, duplicates differing only in response or octave, repeated responses and zero
    responses; octave fields are packed ints >= 0 stored as float bits."""
    rec = np.zeros((6, n), np.float32)
    rec[0] = rng.integers(0, 400, n).astype(np.float32) + rng.choice([0, 0.25, 0.5], n)
    rec[1] = rng.integers(0, 300, n).astype(np.float32)
    rec[2] = rng.choice(np.float32([3.2, 4.0, 5.04, 6.4]), n)
    rec[3] = rng.choice(np.float32([0, 10.5, 90, 359.9]), n)
    rec[4] = rng.random(n).astype(np.float32) * 0.1
    octv = (rng.integers(0, 5, n) + (rng.integers(1, 4, n) << 8) + (rng.integers(0, 256, n) << 16)).astype(np.int32)
    rec[5] = octv.view(np.float32)
    k = int(n * dup)
    if n > 1 and k:
        src, dst = rng.integers(0, n, k), rng.integers(0, n, k)
        rec[:, dst] = rec[:, src]
        third = dst[: k // 3]
        rec[4, third] = rng.random(len(third)).astype(np.float32)       # duplicates differing in response only
        rec[5, dst[k // 3: 2 * k // 3]] = np.int32(7).view(np.float32)  # ... in octave only
    t = rng.random(n) < ties
    rec[4, t] = np.float32(0.0625)
    rec[4, rng.random(n) < zero_resp] = 0
    return rec


@pytest.mark.gpu
def test_selection_bitwise(st):
    """Counts 0, 1 and around the compaction chunk (4096) and sort tile (2048) edges and above 3 x 4096, B = 8 images of different
    counts in one call, n_features 0, 1, count - 1, count, count + 1 and a cut inside a run of equal responses, cap below the kept
    count, the overflow path, and a permuted input."""
    rng = np.random.default_rng(5)
    counts = [0, 1, 2047, 2049, 4095, 4096, 4097, 3 * 4096 + 5]
    kcap = max(counts) + 3
    rec = np.zeros((8, 6, kcap), np.float32)
    for b, n in enumerate(counts):
        rec[b, :, :n] = _records(rng, n)
    full = [ref_select(rec[b], counts[b], 0, kcap) for b in range(8)]
    uniq = [f[4] for f in full]
    # a limit 3 rows into the run of responses equal to 0.0625: the cut falls inside a tie
    tie = [max(1, int(np.sum(f[2][:, 2] > np.float32(0.0625))) + 3) for f in full]
    for cap in [kcap, 100]:
        # one limit for the whole batch: one call, every image checked
        for nf in [0, 1]:
            out = st.sift_select(rec, counts, nf, cap)
            for b in range(8):
                _check_select(out, rec, counts, b, nf, cap, kcap, (nf, cap, b))
        # limits of each image's own count: one call per image, that image checked
        for name, lim in [("c-1", [u - 1 for u in uniq]), ("c", uniq), ("c+1", [u + 1 for u in uniq]), ("tie", tie)]:
            for b in range(8):
                if lim[b] < 0:
                    continue
                _check_select(st.sift_select(rec, counts, lim[b], cap), rec, counts, b, lim[b], cap, kcap, (name, lim[b], cap, b))
    # a permuted input gives bitwise the same rows (and numpy's, on the permuted records)
    perm = rng.permutation(counts[6])
    rp = rec.copy()
    rp[6, :, :counts[6]] = rec[6][:, perm]
    a, p = st.sift_select(rec, counts, 100, kcap), st.sift_select(rp, counts, 100, kcap)
    for k in ("kpts", "frames", "octave", "counts"):
        assert np.array_equal(a[k], p[k]), k
    for b in range(8):
        _check_select(p, rp, counts, b, 100, kcap, kcap, ("permuted", b))
    # a count above kcap: the overflow path reports -1 and writes no row; the other image of the call is unaffected
    ro = np.ascontiguousarray(rec[[2, 3], :, :3000])
    over = st.sift_select(ro, [2047, 3001], 0, 64)
    assert over["counts"][1] == -1 and np.all(over["sel"][1] == ISENT) and np.all(over["kpts"][1] == SENT)
    _check_select(over, ro, [2047, 3001], 0, 0, 64, 3000, "overflow neighbour")


def _check_select(out, rec, counts, b, nf, cap, kcap, what):
    """Image b of a sift_select call against ref_select: count, the first min(count, cap) rows bitwise, sentinels after them."""
    keep, kp, fr, oc, cnt = ref_select(rec[b], counts[b], nf, kcap)
    m = min(cnt, cap)
    assert out["counts"][b] == cnt, (what, out["counts"][b], cnt)
    assert np.array_equal(out["sel"][b, :m], keep[:m]), what
    assert np.array_equal(out["kpts"][b, :m], kp[:m]) and np.array_equal(out["frames"][b, :m], fr[:m]), what
    assert np.array_equal(out["octave"][b, :m], oc[:m]), what
    assert np.all(out["sel"][b, m:] == ISENT) and np.all(out["kpts"][b, m:] == SENT) and np.all(out["frames"][b, m:] == SENT), what
    assert np.all(out["octave"][b, m:] == ISENT), what
    for k in ("sel", "kpts", "frames", "octave", "counts"):
        assert np.all(out[k + "_tail"].view(np.int32) == ISENT), (what, k)


def _check_desc(st, gauss, L, rows, octv, counts, cap, what):
    desc, tail = st.sift_desc(gauss, L, rows, octv, counts, cap)
    assert np.all(tail == SENT), what
    for b in range(len(counts)):
        m = min(counts[b], cap)
        assert np.all(desc[b, :, m:] == SENT), (what, b)
        for k in range(m):
            oc = int(octv[b, k])
            o, ly = ((oc & 255) + 1) & 255, (oc >> 8) & 255
            scale = 2.0 if o == 0 else 1.0 / (1 << (o - 1))
            x, y, s, a = rows[b, k]
            f = np.float32
            ref = ref_descriptor(gauss[o][ly, b], f(x) * f(scale), f(y) * f(scale), a, float(f(s) * f(scale)))
            check_desc_bytes(desc[b, :, k], ref, (what, b, k, tuple(rows[b, k])))
    return desc


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real240x320", "real_odd237x315"])
def test_descriptors_at_device_keypoints(ctx, st, name):
    from test_sift import _golden
    from dim_b200 import _native
    img = _golden(name)
    L = 3
    gauss, _ = _device_pyramid(ctx, img, L)
    f = _native.SiftNet(ctx, 0, L, 0.0004, 10.0, 1.6, 1, *img.shape).extract(img)
    n = len(f["keypoints"])
    rows = np.concatenate([f["keypoints"], f["size"][:, None], f["angle"][:, None]], 1)[None]
    desc = _check_desc(st, [_octave_levels(np.stack(g)) for g in gauss], L, rows, f["octave"][None], [n], n, name)
    assert np.array_equal(desc[0], f["descriptors"])  # the same kernel on the same levels as the extraction


@pytest.mark.gpu
def test_descriptors_on_designed_keypoints(st):
    """Angles 0, 1e-5, 359.99997 and multiples of 45, positions within the descriptor radius of every border and corner, a radius
    clamped by sqrt(w^2 + h^2) on a 12 x 12 level, a flat patch (all bytes 0), one gradient direction (the 0.2 clamp binds), more rows
    than the grid's warps (warps stride), B = 8 with different counts, and cap below the count."""
    L = 3
    rng = np.random.default_rng(3)
    h = w = 64
    lv = np.zeros((L + 3, 8, h, w), np.float32)
    for b in range(8):
        lv[:, b] = [gauss_patch("noise", h, w, 10 * b + i) for i in range(L + 3)]
    lv[2, 1] = gauss_patch("flat", h, w)
    lv[3, 2] = gauss_patch("ramp30", h, w)
    # octave -1 (o = 0, output octave byte 255) level 64 x 64 and octave 0 (o = 1) a 12 x 12 level
    small = np.stack([[gauss_patch("noise", 12, 12, 100 + i + 7 * b) for b in range(8)] for i in range(L + 3)])
    gauss = [lv, small]
    angles = [0.0, 1e-5, 359.99997] + [45.0 * k for k in range(8)]
    edge_xy = [0, 0.4, 3, 31.6, 60, 63, 63.4]
    counts = [5, 0, 40, 2500, 2200, 700, 2600, 12]
    n = max(counts)
    rows = np.zeros((8, n, 4), np.float32)
    octv = np.zeros((8, n), np.int32)
    for b in range(8):
        for k in range(counts[b]):
            o = 1 if (b == 7 or k % 11 == 10) else 0
            lim = (12 if o else 64) * (1 if o else 0.5)  # output coordinates: half the octave -1 level, the octave 0 level as is
            ly = 1 + k % L if b not in (1, 2) else (2 if b == 1 else 3)
            x = rng.choice(edge_xy) * lim / 64 if k % 2 else rng.uniform(0, lim)
            y = rng.choice(edge_xy) * lim / 64 if k % 3 else rng.uniform(0, lim)
            size = rng.choice([1.6, 3.2, 7.0]) if k % 13 else 40.0  # 40 at octave 0: a radius beyond sqrt(12^2 + 12^2)
            rows[b, k] = (x, y, size, angles[k % len(angles)])
            octv[b, k] = ((o - 1) & 255) | (ly << 8) | (int(rng.integers(0, 256)) << 16)
    for cap in (n, 30):
        desc = _check_desc(st, gauss, L, rows, octv, counts, cap, ("designed", cap))
    assert np.all(desc[1] == SENT)  # count 0
    flat_oct = np.full((1, 3), 255 | (2 << 8), np.int32)  # level 2 of image 1 is the flat patch
    flat = _check_desc(st, [g[:, 1:2] for g in gauss], L, rows[0:1, :3], flat_oct, [3], 3, "flat")
    ramp = _check_desc(st, [g[:, 2:3] for g in gauss], L, rows[2:3, :40], octv[2:3, :40], [40], 40, "ramp")
    assert np.all(flat == 0)
    # one direction: the 0.2 clamp binds, so the largest bytes of a descriptor are equal
    top = np.sort(ramp[0, :, 0])[::-1]
    assert top[0] == top[1] and top[0] < 255


@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS)
def test_device_against_cv2_at_other_settings(ctx, setting):
    """The device against cv2 with test_sift's bars, and its pyramid levels against oracle.sift.pyramid within 2.5e-4, at settings the
    pipeline never runs.  cv2's defaults run as a batch of 3 odd-sized images."""
    from test_sift import _as_oracle, _check_against, _golden, _dev_extract, _upscale
    from dim_b200 import _native
    L, con, edge, sig = setting
    conf = dict(n_layers=L, contrast=con, edge=edge, sigma=sig)
    img = _golden("real240x320")
    net = _native.SiftNet(ctx, 0, L, con, edge, sig, 1, *img.shape)
    _check_against(_as_oracle(net.extract(img)), O.cv2_extract(img, 0, **conf), setting)
    gauss, dog = O.pyramid(img, L, sig)
    for o in range(len(gauss)):
        for i, g in enumerate(gauss[o]):
            assert np.abs(net.debug_read(0, 0, o, i, *img.shape) - g).max() <= 2.5e-4, (setting, "gauss", o, i)
        for i, d in enumerate(dog[o]):
            assert np.abs(net.debug_read(1, 0, o, i, *img.shape) - d).max() <= 2.5e-4, (setting, "dog", o, i)
    if setting == SETTINGS[0]:
        up = _upscale()
        imgs = np.stack([_golden("real_odd237x315"), up[100:337, 200:515], up[400:637, 601:916]])
        bnet = _native.SiftNet(ctx, 0, L, con, edge, sig, 3, 237, 315)
        kp, de, fr, oc, cnt = _dev_extract(bnet, imgs, 4000)
        for b in range(3):
            n = int(cnt[b])
            got = {"keypoints": kp[b, :n], "size": fr[b, :n, 0], "angle": fr[b, :n, 1], "response": fr[b, :n, 2], "octave": oc[b, :n],
                   "descriptors": de[b, :, :n]}
            _check_against(got, O.cv2_extract(imgs[b], 0, **conf), (setting, "batch", b))


@pytest.mark.gpu
def test_float_input_conversion_and_wide_sigma(ctx):
    """Float images with negative values, values above 255 and x.5 values give bitwise the features of to_u8(image) (saturation, half
    to even); a sigma that needs more than 127 taps is DIMB_ERR_UNSUPPORTED."""
    from test_sift import _dev_extract, _golden
    from dim_b200 import _native
    img = _golden("real240x320").astype(np.float32)
    rng = np.random.default_rng(2)
    f = img + rng.choice(np.float32([0, 0.5, -0.5, 0.25]), img.shape)
    f[:40] = f[:40] * 3 - 200
    f[100:110, :50] = 254.5
    f[120:130, :50] = 1.5
    net = _native.SiftNet(ctx, 0, 3, 0.0004, 10.0, 1.6, 2, *img.shape)
    a = _dev_extract(net, np.stack([f, f]), 3000)
    b = _dev_extract(net, np.stack([O.to_u8(f)] * 2).astype(np.float32), 3000)
    assert a[4][0] > 300
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    wide = _native.SiftNet(ctx, 0, 3, 0.04, 10.0, 15.9, 1, 64, 64)
    image, kpts, desc, frames, count = (np.zeros((64, 64), np.uint8), np.zeros((64, 2), np.float32), np.zeros((128, 64), np.float32),
                                        np.zeros((64, 3), np.float32), np.zeros(1, np.int32))
    assert ctx.lib.dimb_sift_extract(wide.h, image.ctypes.data, 64, 64, kpts.ctypes.data, desc.ctypes.data, frames.ctypes.data, None,
                                     count.ctypes.data, 64) == ERR_UNSUPPORTED


@pytest.mark.gpu
def test_one_row_or_column_images_have_no_keypoints(ctx):
    """An image of one row or column has no octave: count 0, as cv2 finds none, through the plugin and the batch entry, next to a
    normal image on the same handle."""
    import torch
    from test_sift import _dev_extract, _golden, _plugin
    from dim_b200 import _native
    ext = _plugin(256)
    for shape in [(1, 64), (64, 1), (2, 64)]:
        img = np.full(shape, 9, np.uint8)
        img[..., ::3] = 200
        assert len(O.cv2_extract(img, 256)["keypoints"]) == 0
        f = ext._extract(img)
        assert f["keypoints"].shape == (0, 2) and f["descriptors"].shape == (128, 0)
    real = _golden("real240x320")
    assert len(ext._extract(real)["keypoints"]) > 100
    net = _native.SiftNet(ctx, 0, 3, 0.0004, 10.0, 1.6, 2, 240, 320)
    one = _dev_extract(net, np.stack([real[:1], real[1:2]]), 64)
    assert list(one[4]) == [0, 0]
    full = _dev_extract(net, np.stack([real, real]), 3000)
    ref = net.extract(real)
    assert full[4][0] == len(ref["keypoints"]) and np.array_equal(full[0][0, :full[4][0]], ref["keypoints"])
    torch.cuda.synchronize()
