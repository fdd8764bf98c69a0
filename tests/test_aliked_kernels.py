"""The ALIKED kernels (csrc/aliked_kernels.cuh) stage by stage, against float64 references on the same inputs.

tests/test_gpu_parity.py compares whole extractions with oracle.aliked at three image sizes, with slack for keypoints near the threshold;
a kernel bug on a rare path (a map edge, a clamp, a CTA tail, a plan that those sizes never pick) fits inside that slack.  Here the
self-test library runs each stage through the launch helper dimb_aliked_extract_dev calls (dimb_selftest_aliked_*), on inputs staged in
the production layout with NaN after them, into output buffers that start as a sentinel and are followed by a tail, so reads past the
end, missing writes and stray writes all show.

The references restate oracle.aliked's operations in float64.  Where the kernel's specification rounds a coordinate to float32 (the
deformable sample position, the align_corners source index, SDDH's keypoint and sample coordinates), the reference forms it in float32 in
the same order, so both sides take the same integer decisions (floor indices, patch corners, in or out of the map).
Bars:
  sums          |dev - ref| <= 2 * 2^-24 * (n + 8) * M * L_act + 4 ulp(ref): n terms, M = |alpha| sum|w x| + |beta| + |resid| in float64,
                L_act the activation's largest slope (1, SELU 1.7581, sigmoid 0.25).  Input errors of a stage that sums over an earlier
                stage's output are carried into M.
  bitwise       pad, crop, avgpool (numpy float32 in the kernel's order), kpts_px, saturated offset clamps, thr when a candidate passed.
  DKD           kxy within 2^-20 (1 + r), disp within DISP_REL relative; kscore within 2^-20 of the bilinear sample at the device's
                own kxy.
  descriptors   EXACT within DESC_EXACT, FAST within DESC_FAST (unit vectors).
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

SENT = -777.0
ERR_ARG, ERR_UNSUPPORTED = -3, -4
EPS = 2.0 ** -24
L_ACT = {0: 1.0, 1: 1.7581, 2: 0.25}
DISP_REL = 1e-5
DESC_EXACT = 1e-5
DESC_FAST = 5e-3
F32 = np.float32


# ------------------------------------------------------------------ references
def act64(x, act):
    x = torch.as_tensor(x, dtype=torch.float64)
    return (torch.selu(x) if act == 1 else torch.sigmoid(x) if act == 2 else x).numpy()


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F32)).astype(np.float64)


def fma_bar(ref, M, n, act=0):
    return 2 * EPS * (n + 8) * M * L_ACT[act] + 4 * ulp(ref)


def check_bar(dev, ref, bar, what):
    """Every element within its bar; returns the largest error and its ratio to the bar."""
    dev = np.asarray(dev, np.float64)
    assert np.isfinite(dev).all(), f"{what}: non-finite output"
    err = np.abs(dev - ref)
    bad = err > bar
    assert not bad.any(), f"{what}: {int(bad.sum())} elements beyond the bar, worst {err.max():.3e} (bar there {bar.flat[err.argmax()]:.3e})"
    return float(err.max()), float((err / bar).max())


def conv3x3_ref(x, w, alpha=None, beta=None, resid=None, act=0):
    """(out, M) of act(alpha * conv3x3(x, w, pad 1) + beta + resid) in float64."""
    x64, w64 = torch.from_numpy(np.asarray(x, np.float64))[None], torch.from_numpy(np.asarray(w, np.float64))
    s = F.conv2d(x64, w64, padding=1)[0].numpy()
    a = F.conv2d(x64.abs(), w64.abs(), padding=1)[0].numpy()
    al = np.ones(len(w)) if alpha is None else np.asarray(alpha, np.float64)
    be = np.zeros(len(w)) if beta is None else np.asarray(beta, np.float64)
    y = s * al[:, None, None] + be[:, None, None]
    M = a * np.abs(al)[:, None, None] + np.abs(be)[:, None, None]
    if resid is not None:
        y = y + resid
        M = M + np.abs(resid)
    return act64(y, act), M


def bn_fold32(bn):
    """dimb_aliked_create's fold of eval BatchNorm, in float32: alpha = 1/sqrt(var + 1e-5) * gamma, beta = bias - mean * alpha."""
    g, b, m, v = (np.asarray(t, F32) for t in bn)
    al = (F32(1) / np.sqrt(v + F32(1e-5))).astype(F32) * g
    return al.astype(F32), (b - m * al).astype(F32)


def bilinear_tv(plane, h, w):
    """torchvision deform_conv2d's bilinear_interpolate on one plane at float32 positions h, w (arrays), in float64.  Returns (value,
    the same with |plane|)."""
    H, W = plane.shape
    h, w = np.asarray(h, np.float64), np.asarray(w, np.float64)
    inside = ~((h <= -1) | (h >= H) | (w <= -1) | (w >= W))
    hl, wl = np.floor(h).astype(np.int64), np.floor(w).astype(np.int64)
    lh, lw = h - hl, w - wl
    val, aval = np.zeros(h.shape), np.zeros(h.shape)
    for dy, dx, wt in [(0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)]:
        yy, xx = hl + dy, wl + dx
        ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        v = np.where(ok, plane[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0.0)
        val += wt * v
        aval += np.abs(wt * v)
    return val, aval


def deform_positions(offs, max_off, H, W):
    """The kernel's sample positions [9][H][W] (rows, columns) in float32: float(y - 1 + ky) + clamp(oy, +-max_off)."""
    o = np.clip(np.asarray(offs, F32).reshape(18, H, W), -F32(max_off), F32(max_off))
    ys, xs = np.mgrid[0:H, 0:W]
    py = np.stack([(ys - 1 + t // 3).astype(F32) + o[2 * t] for t in range(9)]).astype(F32)
    px = np.stack([(xs - 1 + t % 3).astype(F32) + o[2 * t + 1] for t in range(9)]).astype(F32)
    return py, px


def deform_ref(x, offs, max_off, w):
    """(conv, sum|w sample|) of the deformable 3x3 conv, torchvision semantics, in float64 from the float32 positions."""
    cin, H, W = x.shape
    py, px = deform_positions(offs, max_off, H, W)
    x64 = np.asarray(x, np.float64)
    vals, avals = np.zeros((cin, 9, H, W)), np.zeros((cin, 9, H, W))
    for c in range(cin):
        vals[c], avals[c] = bilinear_tv(x64[c], py, px)
    w9 = np.asarray(w, np.float64).reshape(len(w), cin, 9)
    return np.einsum("oct,cthw->ohw", w9, vals), np.einsum("oct,cthw->ohw", np.abs(w9), avals)


def deform_bn_ref(x, offs, max_off, w, bn, resid, act):
    """(out, M): act(batch_norm(deform conv) + resid), batch_norm in float64 from the raw parameters as oracle.aliked._bn."""
    conv, a = deform_ref(x, offs, max_off, w)
    g, b, m, v = (np.asarray(t, np.float64)[:, None, None] for t in bn)
    al = g / np.sqrt(v + 1e-5)
    y = (conv - m) * al + b
    M = a * np.abs(al) + np.abs(b) + np.abs(m * al)
    if resid is not None:
        y, M = y + resid, M + np.abs(resid)
    return act64(y, act), M


def up_ref(src, Hp, Wp, f):
    """upsample_bilinear2d(align_corners=True) x f of src [C][h][w] to [C][Hp][Wp] with the source index scale * dst in float32 (ATen's
    area_pixel_compute_source_index), lambdas in float32.  Returns (value, sum of |corner terms|)."""
    C_, h, w = src.shape

    def axis(n_in, n_out):
        s = F32(n_in - 1) / F32(n_out - 1) if n_in > 1 else F32(0)
        fi = (s * np.arange(n_out, dtype=F32)).astype(F32)
        i0 = fi.astype(np.int64)
        step = (i0 < n_in - 1).astype(np.int64)
        l1 = (fi - i0.astype(F32)).astype(F32)
        return i0, step, (F32(1) - l1).astype(np.float64), l1.astype(np.float64)

    y0, yp, l0y, l1y = axis(h, Hp)
    x0, xp, l0x, l1x = axis(w, Wp)
    s = np.asarray(src, np.float64)
    q = lambda dy, dx: s[:, (y0 + dy * yp)[:, None], (x0 + dx * xp)[None, :]]
    terms = [l0y[:, None] * l0x[None] * q(0, 0), l0y[:, None] * l1x[None] * q(0, 1), l1y[:, None] * l0x[None] * q(1, 0),
             l1y[:, None] * l1x[None] * q(1, 1)]
    return sum(terms), sum(np.abs(t) for t in terms)


def selu64(x):
    return torch.selu(torch.as_tensor(x, dtype=torch.float64)).numpy()


def fuse_ref(x1, l2o, l3o, l4o, l1, s0, top, left, H, W):
    """(sh0, bar of sh0, feat [H][W][128], bar of feat) of al_fuse_kernel in float64."""
    _, Hp, Wp = x1.shape
    x1_64, l1_64, s0_64 = (np.asarray(t, np.float64) for t in (x1, l1, s0))
    pre = np.einsum("oc,chw->ohw", l1_64, x1_64)
    amag = np.einsum("oc,chw->ohw", np.abs(l1_64), np.abs(x1_64)) * L_ACT[1] * (1 + 2 * EPS * 24)  # |v| bound of the lateral-1 channels
    vs, mags = [selu64(pre)], [amag]
    for src, f in ((l2o, 2), (l3o, 8), (l4o, 32)):
        v, a = up_ref(src, Hp, Wp, f)
        vs.append(v)
        mags.append(a)
    v, mag = np.concatenate(vs), np.concatenate(mags)
    # the upsampled channels carry the 3 rounded products and sums of the bilinear blend: 8 ulp of their corner sum
    err_v = np.concatenate([2 * EPS * (16 + 8) * amag, 8 * EPS * np.concatenate(mags[1:])])
    s = np.einsum("jc,chw->jhw", s0_64, v)
    M = np.einsum("jc,chw->jhw", np.abs(s0_64), mag)
    sh0 = selu64(s)
    bar_sh0 = L_ACT[1] * (2 * EPS * (128 + 8) * M + np.einsum("jc,chw->jhw", np.abs(s0_64), err_v)) + 4 * ulp(sh0)
    nrm = np.maximum(np.sqrt((v * v).sum(0)), 1e-12)
    feat = v / nrm
    bar_f = (err_v + 2 * EPS * (128 + 8) * np.abs(v) + 2 * EPS * (128 + 8) * (err_v * np.abs(v)).sum(0) / nrm) / nrm + 4 * ulp(feat)
    crop = lambda t: t[:, top:top + H, left:left + W].transpose(1, 2, 0)
    return sh0, bar_sh0, crop(feat), crop(bar_f)


def dkd_ref(score, idx, r):
    """oracle.aliked.dkd's refinement at given pixel indices (Unfold zero padding, soft-argmax T = 0.1, dispersity, grid_sample) in
    float64.  Returns (kxy [n][2], disp [n], kscore [n])."""
    H, W = score.shape
    s = torch.from_numpy(np.asarray(score, np.float64))[None, None]
    idx = torch.as_tensor(np.asarray(idx, np.int64))
    ks = 2 * r + 1
    xs = torch.linspace(-r, r, ks, dtype=torch.float64)
    grid = torch.stack(torch.meshgrid([xs, xs], indexing="ij")).view(2, -1).t()[:, [1, 0]]
    patch = F.unfold(s, kernel_size=ks, padding=r)[0].t()[idx]
    xy = torch.stack([idx % W, torch.div(idx, W, rounding_mode="trunc")], 1).to(torch.float64)
    e = ((patch - patch.max(1).values[:, None]) / 0.1).exp()
    res = e @ grid / e.sum(1)[:, None]
    d2 = torch.norm((grid[None] - res[:, None]) / r, dim=-1) ** 2
    disp = (e * d2).sum(1) / e.sum(1)
    kxy = (xy + res) / torch.tensor([W - 1, H - 1], dtype=torch.float64) * 2 - 1
    ksc = F.grid_sample(s, kxy.view(1, 1, -1, 2), mode="bilinear", align_corners=True)[0, 0, 0]
    return kxy.numpy(), disp.numpy(), ksc.numpy()


def kscore_at(score, kxy):
    """DKD's kscore: grid_sample(bilinear, align_corners, zero padding) of score at the device's kxy [n][2], with ix = ((kx + 1) / 2)
    (W - 1) formed in float32 as the kernel does, in float64.  The device's kxy carries its rounding (within the kxy bar); sampled at the
    float64 kxy instead, that rounding times the score's slope would dominate the comparison."""
    H, W = score.shape
    k = np.asarray(kxy, F32)
    ix, iy = ((k[:, 0] + F32(1)) / F32(2) * F32(W - 1)).astype(F32), ((k[:, 1] + F32(1)) / F32(2) * F32(H - 1)).astype(F32)
    fx, fy = np.floor(ix).astype(np.float64), np.floor(iy).astype(np.float64)
    acc = np.zeros(len(k))
    for dy in (0, 1):
        for dx in (0, 1):
            cx, cy = fx.astype(np.int64) + dx, fy.astype(np.int64) + dy
            wt = (ix - fx if dx else fx + 1 - ix) * (iy - fy if dy else fy + 1 - iy)
            ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
            acc += np.where(ok, wt * score[np.clip(cy, 0, H - 1), np.clip(cx, 0, W - 1)], 0.0)
    return acc


def sddh_kw(kxy, H, W):
    """SDDH's keypoint position in pixels, float32 as the kernels form it: (k / 2 + 0.5) * (size - 1)."""
    wh = np.array([W - 1, H - 1], F32)
    return ((np.asarray(kxy, F32) / F32(2) + F32(0.5)) * wh).astype(F32)


def sddh_offsets_ref(feat, kxy, w):
    """(off [n][32] clamped, pre-clamp value, bar, max_off) of al_sddh_offsets_kernel: get_patches (corner clamp), offset_conv.0 + SELU,
    offset_conv.2, clamp to +-max(H, W) / 4, in float64 on the float32 patch corners."""
    H, W = feat.shape[:2]
    kw = sddh_kw(kxy, H, W)
    corner = (kw.astype(np.int64).astype(F32) - F32(1.5) + F32(1)).astype(np.int64)
    cx, cy = np.clip(corner[:, 0], 0, W - 4), np.clip(corner[:, 1], 0, H - 4)
    f64 = np.asarray(feat, np.float64)
    patch = np.stack([f64[cy[i]:cy[i] + 3, cx[i]:cx[i] + 3].transpose(2, 0, 1) for i in range(len(kw))]).reshape(len(kw), 1152)
    w0 = np.asarray(w["desc_head.offset_conv.0.weight"], np.float64).reshape(32, 1152)
    b0, b2 = (np.asarray(w["desc_head." + k], np.float64) for k in ("offset_conv.0.bias", "offset_conv.2.bias"))
    w2 = np.asarray(w["desc_head.offset_conv.2.weight"], np.float64).reshape(32, 32)
    pre0 = patch @ w0.T + b0
    hid = selu64(pre0)
    err_hid = L_ACT[1] * (2 * EPS * (1152 + 8) * (np.abs(patch) @ np.abs(w0).T + np.abs(b0)) + 4 * ulp(hid))
    a = hid @ w2.T + b2
    bar = 2 * EPS * (32 + 8) * (np.abs(hid) @ np.abs(w2).T + np.abs(b2)) + err_hid @ np.abs(w2).T + 4 * ulp(a)
    mo = F32(max(H, W)) / F32(4)
    return np.clip(a, -float(mo), float(mo)), a, bar, mo


def sddh_desc_ref(feat, kxy, off, w):
    """Descriptors [128][n] of SDDH on given offsets off [n][32] (16 x, then 16 y): grid_sample (align_corners, zero padding) at the
    float32 sample coordinates, sf_conv + SELU, the aggregation einsum and F.normalize, in float64."""
    H, W = feat.shape[:2]
    kw = sddh_kw(kxy, H, W)
    whx, why = F32(W - 1), F32(H - 1)
    off = np.asarray(off, F32)
    posx, posy = (kw[:, :1] + off[:, :16]).astype(F32), (kw[:, 1:] + off[:, 16:]).astype(F32)
    gx, gy = (F32(2) * posx / whx - F32(1)).astype(F32), (F32(2) * posy / why - F32(1)).astype(F32)
    ix, iy = (((gx + F32(1)) / F32(2)) * whx).astype(F32), (((gy + F32(1)) / F32(2)) * why).astype(F32)
    fx, fy = np.floor(ix), np.floor(iy)
    f64 = np.asarray(feat, np.float64)
    samp = np.zeros(ix.shape + (128,))
    for dy in (0, 1):
        for dx in (0, 1):
            qx, qy = fx.astype(np.int64) + dx, fy.astype(np.int64) + dy
            wt = (ix.astype(np.float64) - fx if dx else fx + 1 - ix.astype(np.float64)) * \
                 (iy.astype(np.float64) - fy if dy else fy + 1 - iy.astype(np.float64))
            ok = (qx >= 0) & (qx < W) & (qy >= 0) & (qy < H)
            v = f64[np.clip(qy, 0, H - 1), np.clip(qx, 0, W - 1)] * ok[..., None]
            samp += wt[..., None] * v
    sf = np.asarray(w["desc_head.sf_conv.weight"], np.float64).reshape(128, 128)
    f2 = selu64(samp @ sf.T)  # [n][16][128]
    d = np.einsum("npc,pcd->nd", f2, np.asarray(w["desc_head.agg_weights"], np.float64))
    return (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12)).T


def rand(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(F32)


def bn_of(w, p):
    return np.stack([w[p + s] for s in (".weight", ".bias", ".running_mean", ".running_var")])


# ------------------------------------------------------------------ without a GPU
def test_conv_plan_rule():
    """conv3's instantiation: <8,1> (1) for maps of at most 64 x 64 pixels, else <16,4> (2) when cout >= 16, else <8,4> (3)."""
    from dim_b200 import _native
    for H, W in [(1, 1), (64, 64), (1, 4096), (4096, 1), (65, 64), (64, 65), (17, 66), (16, 68), (512, 512)]:
        for cout in (1, 4, 15, 16, 18, 32, 128):
            exp = 1 if H * W <= 4096 else (2 if cout >= 16 else 3)
            assert _native.aliked_conv_plan(H, W, cout) == exp, (H, W, cout)


def test_deform_reference_against_torchvision():
    """The float64 deformable reference equals torchvision.ops.deform_conv2d on offsets that are integers or multiples of 1/64 (every
    sample position exact in float32), on maps down to 1 x 1, and the zero-offset case equals F.conv2d."""
    import torchvision
    rng = np.random.default_rng(3)
    for H, W in [(1, 1), (1, 5), (3, 1), (4, 5), (7, 9), (8, 8)]:
        cin, cout = 8, 4
        x, w = rand(rng, cin, H, W), rand(rng, cout, cin, 3, 3)
        for offs in (np.zeros((18, H, W), F32), rng.integers(-3, 4, (18, H, W)).astype(F32),
                     (rng.integers(-192, 193, (18, H, W)) / 64).astype(F32)):
            got, _ = deform_ref(x, offs, 1e9, w)
            exp = torchvision.ops.deform_conv2d(torch.from_numpy(x.astype(np.float64))[None], torch.from_numpy(offs.astype(np.float64))[None],
                                                torch.from_numpy(w.astype(np.float64)), padding=(1, 1))[0].numpy()
            assert np.abs(got - exp).max() < 1e-12, (H, W)
        z, _ = deform_ref(x, np.zeros((18, H, W), F32), 0.0, w)
        assert np.abs(z - conv3x3_ref(x, w)[0]).max() < 1e-12


def test_fuse_and_dkd_references_against_oracle_ops():
    """up_ref equals F.interpolate(align_corners=True) and dkd_ref equals oracle.aliked.dkd's refinement (float32 torch) at its own
    indices, within float32 noise."""
    from oracle import aliked as o_al
    rng = np.random.default_rng(4)
    for h, w, f in [(1, 1, 32), (1, 2, 32), (3, 5, 8), (16, 20, 2)]:
        src = rand(rng, 2, h, w)
        got, _ = up_ref(src, h * f, w * f, f)
        exp = F.interpolate(torch.from_numpy(src.astype(np.float64))[None], scale_factor=f, mode="bilinear", align_corners=True)[0].numpy()
        assert np.abs(got - exp).max() < 1e-5  # the float32 source index against float64
    score = rng.random((24, 28)).astype(F32)
    kxy, disp, ksc = o_al.dkd(torch.from_numpy(score)[None, None], 2, 0.5, 1000)
    nms = o_al.simple_nms(torch.from_numpy(score)[None, None], 2)[0, 0].numpy()
    nms[:2], nms[-2:], nms[:, :2], nms[:, -2:] = 0, 0, 0, 0
    idx = np.nonzero((nms > 0.5).reshape(-1))[0]
    k2, d2, s2 = dkd_ref(score, idx, 2)
    assert len(idx) == len(kxy) > 0
    assert np.abs(k2 - kxy.numpy()).max() < 1e-5 and np.abs(d2 - disp.numpy()).max() < 1e-5 and np.abs(s2 - ksc.numpy()).max() < 1e-5


def test_sddh_reference_against_oracle(al_weights):
    """sddh_offsets_ref + sddh_desc_ref equal oracle.aliked.sddh on a normalised random map, keypoints at corners and edges included."""
    from oracle import aliked as o_al
    rng = np.random.default_rng(5)
    H, W = 12, 17
    feat = rand(rng, 128, H, W)
    feat /= np.linalg.norm(feat, axis=0, keepdims=True)
    kxy = np.concatenate([np.array([[-1, -1], [1, 1], [-1, 1], [1, -1], [0, -1], [1, 0.3]], F32), rng.uniform(-1, 1, (10, 2)).astype(F32)])
    feat_hw = np.ascontiguousarray(feat.transpose(1, 2, 0))
    off, _, _, _ = sddh_offsets_ref(feat_hw, kxy, al_weights)
    got = sddh_desc_ref(feat_hw, kxy, off, al_weights)
    with torch.no_grad():
        exp = o_al.sddh(torch.from_numpy(feat)[None], torch.from_numpy(kxy), al_weights, 3, 16).numpy().T
    assert np.abs(got - exp).max() < 1e-5


def test_aliked_selftest_entries_reject_bad_arguments_without_touching_the_gpu():
    """DIMB_ERR_ARG (-3) / DIMB_ERR_UNSUPPORTED (-4) before any CUDA call: null pointers, sizes below 1, a deformable cin that is not a
    multiple of 8 or a cout other than 64 / 128, r outside 1..5, count < 0; the context pointer is never dereferenced."""
    from dim_b200 import _native
    lib = _native.load_selftest_library()
    null, fake, buf = C.c_void_p(), C.c_void_p(16), C.c_void_p(16)
    out = np.zeros(1, np.int32)
    assert lib.dimb_selftest_aliked_conv_plan(0, 8, 16, out.ctypes.data) == ERR_ARG
    assert lib.dimb_selftest_aliked_conv_plan(8, 8, 0, out.ctypes.data) == ERR_ARG
    assert lib.dimb_selftest_aliked_conv_plan(8, 8, 16, None) == ERR_ARG
    c3 = lambda ctx, variant, x, cin, H, W, cout, act: lib.dimb_selftest_aliked_conv3x3(ctx, variant, x, cin, H, W, buf, None, None, None,
                                                                                        cout, act, SENT, buf, None)
    assert c3(null, 0, buf, 8, 8, 8, 8, 0) == ERR_ARG
    assert c3(fake, 0, None, 8, 8, 8, 8, 0) == ERR_ARG
    for variant, cin, H, W, cout, act in [(4, 8, 8, 8, 8, 0), (-1, 8, 8, 8, 8, 0), (0, 0, 8, 8, 8, 0), (0, 8, 0, 8, 8, 0), (0, 8, 8, 0, 8, 0),
                                          (0, 8, 8, 8, 0, 0), (0, 8, 8, 8, 8, 3)]:
        assert c3(fake, variant, buf, cin, H, W, cout, act) == ERR_ARG
    assert lib.dimb_selftest_aliked_conv1x1(fake, buf, 0, 16, buf, None, 16, 0, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_conv1x1(fake, buf, 16, 0, buf, None, 16, 0, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_conv1x1(fake, buf, 16, 16, None, None, 16, 0, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_avgpool(fake, buf, 4, 8, 8, 0, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_avgpool(fake, buf, 4, 8, 3, 4, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_pad(fake, buf, 8, 8, 2, SENT, buf, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_pad(fake, buf, 0, 8, 3, SENT, buf, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_crop(fake, buf, 32, 32, 1, 0, 32, 8, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_crop(fake, buf, 32, 32, -1, 0, 8, 8, SENT, buf) == ERR_ARG
    d = lambda cin, cout, offs=buf, r=None: lib.dimb_selftest_aliked_deform(fake, buf, cin, 4, 4, offs, 1.0, r, r, buf, buf, None, cout, 1,
                                                                            SENT, buf, None)
    assert d(12, 64) == ERR_UNSUPPORTED and d(136, 128) == ERR_UNSUPPORTED and d(32, 32) == ERR_UNSUPPORTED and d(32, 96) == ERR_UNSUPPORTED
    assert d(0, 64) == ERR_ARG and d(32, 64, offs=None) == ERR_ARG
    assert lib.dimb_selftest_aliked_deform(null, buf, 32, 4, 4, buf, 1.0, None, None, buf, buf, None, 64, 1, SENT, buf, None) == ERR_ARG
    assert lib.dimb_selftest_aliked_deform(fake, buf, 32, 4, 4, buf, -1.0, None, None, buf, buf, None, 64, 1, SENT, buf, None) == ERR_ARG
    fz = lambda Hp, Wp, top, left, H, W: lib.dimb_selftest_aliked_fuse(fake, buf, buf, buf, buf, buf, buf, Hp, Wp, top, left, H, W, SENT,
                                                                       buf, buf)
    for args in [(48, 32, 0, 0, 8, 8), (32, 32, 0, 0, 0, 8), (32, 32, 30, 0, 8, 8), (0, 32, 0, 0, 8, 8)]:
        assert fz(*args) == ERR_ARG, args
    idx = np.array([0, 5], np.int32)
    dk = lambda H, W, r, count, cap, ix=idx: lib.dimb_selftest_aliked_dkd(fake, buf, H, W, r, ix.ctypes.data, count, cap, SENT, buf, buf, buf)
    for args in [(8, 8, 0, 2, 4), (8, 8, 6, 2, 4), (8, 8, 2, -1, 4), (8, 8, 2, 2, 0), (1, 8, 2, 2, 4)]:
        assert dk(*args) == ERR_ARG, args
    assert dk(2, 2, 2, 2, 4) == ERR_ARG  # index 5 outside a 2 x 2 map
    kx = np.zeros(4, np.float32)
    sd = lambda H, W, count, cap, k=kx: lib.dimb_selftest_aliked_sddh(fake, buf, H, W, k.ctypes.data, count, cap, buf, buf, buf, buf, buf,
                                                                      buf, None, SENT, buf, buf, buf)
    for args in [(7, 8, 1, 4), (8, 7, 1, 4), (8, 8, -1, 4), (8, 8, 1, 0)]:
        assert sd(*args) == ERR_ARG, args
    assert sd(8, 8, 2, 4, np.array([0, 0, 1.5, 0], np.float32)) == ERR_ARG
    assert lib.dimb_selftest_aliked_threshold(fake, buf, 0, None, 0.2, SENT, buf) == ERR_ARG
    neg = np.array([-1], np.int32)
    assert lib.dimb_selftest_aliked_threshold(fake, buf, 16, neg.ctypes.data, 0.2, SENT, buf) == ERR_ARG
    assert lib.dimb_selftest_aliked_threshold(null, buf, 16, None, 0.2, SENT, buf) == ERR_ARG


def test_weight_layout_names(al_weights):
    """The production layers these tests take their weights from exist with the shapes the stages assume."""
    for p, shape in CONV3_LAYERS.values():
        assert al_weights[p + ".weight"].shape[:2] == shape, p
    for name, (cin, cout) in DEFORM_LAYERS.items():
        assert al_weights[name + ".regular_conv.weight"].shape == (cout, cin, 3, 3)


# ------------------------------------------------------------------ on the GPU
@pytest.fixture(scope="module")
def st():
    from dim_b200 import _native
    return _native.SelfTest()


# (cin, cout, act, bn prefix or None, resid) of every 3x3 conv dimb_aliked_extract_dev runs through conv3
CONV3_LAYERS = {
    "b1c1": ("block1.conv1", (16, 3)), "b1c2": ("block1.conv2", (16, 16)), "b2c1": ("block2.conv1", (32, 16)),
    "b2c2": ("block2.conv2", (32, 32)), "o31": ("block3.conv1.offset_conv", (18, 32)), "o32": ("block3.conv2.offset_conv", (18, 64)),
    "o42": ("block4.conv2.offset_conv", (18, 128)), "s2": ("score_head.2", (4, 8)), "s4": ("score_head.4", (4, 4)),
    "s6": ("score_head.6", (1, 4)),
}
CONV3_ROLE = {"b1c1": ("block1.bn1", False, 1), "b1c2": ("block1.bn2", False, 1), "b2c1": ("block2.bn1", False, 1),
              "b2c2": ("block2.bn2", True, 1), "o31": (None, False, 0), "o32": (None, False, 0), "o42": (None, False, 0),
              "s2": (None, False, 1), "s4": (None, False, 1), "s6": (None, False, 2)}
CONV3_SHAPES = [(1, 1), (1, 67), (9, 1), (7, 15), (8, 16), (9, 65), (17, 66), (16, 68), (64, 64), (65, 64)]
DEFORM_LAYERS = {"block3.conv1": (32, 64), "block3.conv2": (64, 64), "block4.conv1": (64, 128), "block4.conv2": (128, 128)}
DEFORM_SHAPES = [(1, 1), (1, 5), (3, 1), (4, 5), (7, 9), (8, 8), (28, 36)]
REPORT = {}


def report(stage, err, ratio):
    e, r = REPORT.get(stage, (0.0, 0.0))
    REPORT[stage] = (max(e, err), max(r, ratio))
    print(f"{stage}: max error {REPORT[stage][0]:.3e}, max error / bar {REPORT[stage][1]:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("layer", list(CONV3_LAYERS))
def test_conv3x3_every_plan(st, al_weights, layer):
    """Every production 3x3 conv (real weights, folded BN or bias only, SELU / none / sigmoid, resid) on every instantiation and the
    production rule, at shapes from 1 x 1 to past the 4096-pixel plan boundary, both epilogue paths of the 64-pixel tiles (W % 4 = 2 and
    0) and the 18-channel Cout tail."""
    from dim_b200 import _native
    p, (cout, cin) = CONV3_LAYERS[layer]
    bn, has_resid, act = CONV3_ROLE[layer]
    w = al_weights[p + ".weight"]
    if bn:
        alpha, beta = bn_fold32(bn_of(al_weights, bn))
    else:
        alpha, beta = None, al_weights.get(p + ".bias")
    rng = np.random.default_rng(sum(map(ord, layer)))
    for H, W in CONV3_SHAPES:
        x = rand(rng, cin, H, W)
        resid = rand(rng, cout, H, W) if has_resid else None
        ref, M = conv3x3_ref(x, w, alpha, beta, resid, act)
        bar = fma_bar(ref, M, cin * 9, act)
        for variant in (0, 1, 2, 3):
            out, tail, plan = st.aliked_conv3x3(x, w, alpha, beta, resid, act, variant, SENT)
            assert plan == (variant or _native.aliked_conv_plan(H, W, cout))
            assert np.all(tail == SENT), (H, W, variant)
            report("conv3x3", *check_bar(out, ref, bar, f"{layer} {H}x{W} variant {variant}"))


@pytest.mark.gpu
def test_conv3x3_alpha_beta_resid_combinations(st):
    """Seeded mixed-sign weights with alpha / beta / resid each null or set, SELU, on the 17 x 66 and 16 x 68 maps of the 64-pixel tiles."""
    rng = np.random.default_rng(11)
    for H, W in [(17, 66), (16, 68), (7, 15)]:
        cin, cout = 16, 20
        x, w = rand(rng, cin, H, W), rand(rng, cout, cin, 3, 3, scale=0.2)
        for use_a in (0, 1):
            for use_b in (0, 1):
                for use_r in (0, 1):
                    a = rand(rng, cout) if use_a else None
                    b = rand(rng, cout) if use_b else None
                    r = rand(rng, cout, H, W) if use_r else None
                    ref, M = conv3x3_ref(x, w, a, b, r, 1)
                    for variant in (1, 2, 3):
                        out, tail, _ = st.aliked_conv3x3(x, w, a, b, r, 1, variant, SENT)
                        assert np.all(tail == SENT)
                        report("conv3x3", *check_bar(out, ref, fma_bar(ref, M, cin * 9, 1), f"{H}x{W} a{use_a} b{use_b} r{use_r} v{variant}"))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 255, 256, 257, 4097])
def test_conv1x1_production_layers(st, al_weights, P):
    """The downsample shortcuts (bias, no activation) and the SELU laterals conv2..4 with their real weights."""
    rng = np.random.default_rng(P)
    layers = [("block2.downsample", 0), ("block3.downsample", 0), ("block4.downsample", 0), ("conv2", 1), ("conv3", 1), ("conv4", 1)]
    for p, act in layers:
        w = al_weights[p + ".weight"][:, :, 0, 0]
        b = al_weights.get(p + ".bias")
        x = rand(rng, w.shape[1], P)
        out, tail = st.aliked_conv1x1(x, w, b, act, SENT)
        w64, x64 = w.astype(np.float64), x.astype(np.float64)
        b64 = np.zeros((len(w), 1)) if b is None else b.astype(np.float64)[:, None]
        ref = act64(w64 @ x64 + b64, act)
        M = np.abs(w64) @ np.abs(x64) + np.abs(b64)
        assert np.all(tail == SENT)
        report("conv1x1", *check_bar(out, ref, fma_bar(ref, M, w.shape[1], act), f"{p} P={P}"))


@pytest.mark.gpu
def test_pad_crop_avgpool_bitwise(st):
    """InputPadder's split and replicate padding with x / 255 (1 and 3 channels), the crop, and the average pooling (sum over dy, then
    dx, divided by k k) bitwise against numpy float32 in the kernels' order."""
    rng = np.random.default_rng(7)
    for H, W in [(8, 8), (8, 40), (33, 31), (63, 65), (32, 64), (1, 1)]:
        for ch in (1, 3):
            img = (rng.random((H, W, ch) if ch == 3 else (H, W)) * 255).astype(F32)
            out, (Hp, Wp, top, left), tail = st.aliked_pad(img, SENT)
            ph, pw = (((H // 32) + 1) * 32 - H) % 32, (((W // 32) + 1) * 32 - W) % 32
            assert (Hp, Wp, top, left) == (H + ph, W + pw, ph // 2, pw // 2)
            src = img if ch == 3 else np.repeat(img[..., None], 3, 2)
            exp = np.pad(src / F32(255), ((top, Hp - H - top), (left, Wp - W - left), (0, 0)), mode="edge").transpose(2, 0, 1)
            assert np.array_equal(out, exp), (H, W, ch)
            assert np.all(tail == SENT)
            crop, ctail = st.aliked_crop(out[1], top, left, H, W, SENT)
            assert np.array_equal(crop, out[1, top:top + H, left:left + W]) and np.all(ctail == SENT)
    for C_, H, W, k in [(16, 64, 96, 2), (32, 32, 48, 4), (64, 8, 12, 4), (64, 4, 4, 4), (3, 9, 7, 2), (2, 5, 5, 5), (4, 30, 45, 3),
                          (3, 25, 35, 5)]:
        x = rand(rng, C_, H, W)
        out, tail = st.aliked_avgpool(x, k, SENT)
        Ho, Wo = H // k, W // k
        s = np.zeros((C_, Ho, Wo), F32)
        for dy in range(k):
            for dx in range(k):
                s = (s + x[:, dy:Ho * k:k, dx:Wo * k:k]).astype(F32)
        assert np.array_equal(out, (s / F32(k * k)).astype(F32)), (C_, H, W, k)
        assert np.all(tail == SENT)


def _deform_check(st, x, w, bn, offs, max_off, resid, what, act=1):
    ref, M = deform_bn_ref(x, offs, max_off, w, bn, resid, act)
    out, tail, _ = st.aliked_deform(x, w, bn, offs=offs, max_off=max_off, resid=resid, act=act, sentinel=SENT)
    assert np.all(tail == SENT), what
    report("deform", *check_bar(out, ref, fma_bar(ref, M, x.shape[0] * 9, act), what))
    return out


def _edge_offsets(rng, H, W):
    """Offsets whose float32 sample positions sit exactly at -1, H (rows) / W (columns), one float32 step inside them, on the last
    row / column, or at a random place; dy and dx chosen independently."""
    ys, xs = np.mgrid[0:H, 0:W]
    offs = np.zeros((18, H, W), F32)
    for t in range(9):
        for comp, (base, n) in enumerate([((ys - 1 + t // 3).astype(F32), H), ((xs - 1 + t % 3).astype(F32), W)]):
            targets = np.array([-1, np.nextafter(F32(-1), F32(0)), n, np.nextafter(F32(n), F32(0)), n - 1, 0, -0.5, n - 0.5], F32)
            pick = targets[rng.integers(0, len(targets), (H, W))]
            rnd = rng.uniform(-2, n + 1, (H, W)).astype(F32)
            tgt = np.where(rng.random((H, W)) < 0.75, pick, rnd).astype(F32)
            offs[2 * t + comp] = (tgt - base).astype(F32)
    return offs


@pytest.mark.gpu
@pytest.mark.parametrize("layer", list(DEFORM_LAYERS))
def test_deform_mode_a_planted_offsets(st, al_weights, layer):
    """Deformable conv on planted offsets, real weights and BN through the create-time transforms, on maps from 1 x 1 (block 4 of images
    up to 32 px) to 28 x 36 (a tail CTA whenever H W % 16 != 0): zero offsets (also against the 3x3 reference), integers and multiples
    of 1/64, positions at and one step inside -1, H and W, offsets at and beyond +-max_off, resid on and off."""
    cin, cout = DEFORM_LAYERS[layer]
    idx = layer[-1]
    w, bn = al_weights[layer + ".regular_conv.weight"], bn_of(al_weights, layer.replace(f"conv{idx}", f"bn{idx}"))
    rng = np.random.default_rng(int(cin + cout))
    for H, W in DEFORM_SHAPES:
        mo = F32(max(H, W)) / F32(4)
        x = rand(rng, cin, H, W)
        for with_resid in (False, True):
            resid = rand(rng, cout, H, W) if with_resid else None
            zero = _deform_check(st, x, w, bn, np.zeros((18, H, W), F32), mo, resid, f"{layer} {H}x{W} zero")
            al, be = bn_fold32(bn)
            ref3, M3 = conv3x3_ref(x, w, al, be, resid, 1)
            report("deform vs conv3x3", *check_bar(zero, ref3, fma_bar(ref3, M3, cin * 9, 1) * 2, f"{layer} {H}x{W} zero vs conv3x3"))
        _deform_check(st, x, w, bn, rng.integers(-2, 3, (18, H, W)).astype(F32), 1e6, None, f"{layer} {H}x{W} integer")
        _deform_check(st, x, w, bn, (rng.integers(-160, 161, (18, H, W)) / 64).astype(F32), 1e6, resid, f"{layer} {H}x{W} 1/64")
        _deform_check(st, x, w, bn, _edge_offsets(rng, H, W), 1e6, None, f"{layer} {H}x{W} edges")
        clamp = (rng.choice([-2.0, -1.0, 1.0, 2.0, 0.5], (18, H, W)) * float(mo)).astype(F32)
        _deform_check(st, x, w, bn, clamp, mo, None, f"{layer} {H}x{W} clamp")
        asym = np.zeros((18, H, W), F32)
        asym[0::2], asym[1::2] = F32(0.75), F32(-0.25)
        _deform_check(st, x, w, bn, asym, 1e6, resid, f"{layer} {H}x{W} dy != dx")


@pytest.mark.gpu
@pytest.mark.parametrize("layer", list(DEFORM_LAYERS))
def test_deform_mode_b_dcn_helper(st, al_weights, layer):
    """The whole dcn helper (offset conv, clamp at max(H, W) / 4, deformable conv) on H != W maps: the offsets against the float64 3x3
    conv, and the output against the deformable reference on those offsets."""
    cin, cout = DEFORM_LAYERS[layer]
    idx = layer[-1]
    w, bn = al_weights[layer + ".regular_conv.weight"], bn_of(al_weights, layer.replace(f"conv{idx}", f"bn{idx}"))
    ow, ob = al_weights[layer + ".offset_conv.weight"], al_weights[layer + ".offset_conv.bias"]
    rng = np.random.default_rng(cin * 3 + cout)
    for H, W in [(1, 3), (4, 5), (7, 9), (9, 7), (28, 36)]:
        x = rand(rng, cin, H, W, scale=3.0)  # large enough that some offsets reach the clamp
        for resid in (None, rand(rng, cout, H, W)):
            out, tail, off = st.aliked_deform(x, w, bn, offw=ow, offb=ob, resid=resid, act=1, sentinel=SENT)
            oref, oM = conv3x3_ref(x, ow, None, ob)
            report("deform offsets", *check_bar(off, oref, fma_bar(oref, oM, cin * 9), f"{layer} {H}x{W} offsets"))
            mo = F32(max(H, W)) / F32(4)
            ref, M = deform_bn_ref(x, off, mo, w, bn, resid, 1)
            assert np.all(tail == SENT)
            report("deform", *check_bar(out, ref, fma_bar(ref, M, cin * 9, 1), f"{layer} {H}x{W} mode B"))


FUSE_SIZES = [(32, 32), (32, 64), (64, 32), (96, 160), (224, 288)]


@pytest.mark.gpu
@pytest.mark.parametrize("Hp, Wp", FUSE_SIZES)
def test_fuse(st, al_weights, Hp, Wp):
    """Fusion with the real conv1 and score_head.0 weights: lateral 1 + SELU, align_corners upsampling x2 / x8 / x32 (from 1 x 1 maps at
    32 x 32), score_head.0 + SELU over the whole padded map, and the normalised crop at (top, left) into [H][W][128]; the feat tail stays
    sentinel.  An all-zero input gives feat exactly 0."""
    rng = np.random.default_rng(Hp * 7 + Wp)
    l1, s0 = al_weights["conv1.weight"][:, :, 0, 0], al_weights["score_head.0.weight"][:, :, 0, 0]
    x1 = rand(rng, 16, Hp, Wp)
    lat = [selu64(rand(rng, 32, Hp // f, Wp // f)).astype(F32) for f in (2, 8, 32)]
    for top, left in [(0, 0), (1, 0), (0, 1), (15, 16)]:
        H = Hp - 2 * top - 1 if top else Hp
        W = max(1, Wp - 2 * left - 1) if left else Wp
        sh0, feat, tail = st.aliked_fuse(x1, *lat, l1, s0, top, left, H, W, SENT)
        rsh, bsh, rf, bf = fuse_ref(x1, *lat, l1, s0, top, left, H, W)
        report("fuse sh0", *check_bar(sh0, rsh, bsh, f"{Hp}x{Wp} sh0"))
        report("fuse feat", *check_bar(feat, rf, bf, f"{Hp}x{Wp} ({top},{left}) feat"))
        assert np.all(tail["feat"] == SENT) and np.all(tail["sh0"] == SENT)
    zeros = [np.zeros_like(t) for t in [x1] + lat]
    sh0, feat, tail = st.aliked_fuse(*zeros, l1, s0, 0, 0, Hp, Wp, SENT)
    assert np.all(feat == 0) and np.all(sh0 == 0) and np.all(tail["feat"] == SENT)


def _dkd_check(st, score, idx, r, count, cap, what):
    out, tail = st.aliked_dkd(score, r, idx, count, cap, SENT)
    n = min(count, cap)
    for k in ("kxy", "disp", "kscore"):
        assert np.all(tail[k] == SENT), what
    assert np.all(out["kxy"][n:] == SENT) and np.all(out["disp"][n:] == SENT) and np.all(out["kscore"][n:] == SENT), what
    if n == 0:
        return out
    kxy, disp, ksc = dkd_ref(score, idx[:n], r)
    report("dkd kxy", *check_bar(out["kxy"][:n], kxy, np.full(kxy.shape, 2.0 ** -20 * (1 + r)), what))
    report("dkd disp", *check_bar(out["disp"][:n], disp, DISP_REL * np.abs(disp) + 1e-30, what))
    report("dkd kscore", *check_bar(out["kscore"][:n], kscore_at(score, out["kxy"][:n]), np.full(ksc.shape, 2.0 ** -20), what))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 2, 3, 4, 5])
def test_dkd_refinement(st, r):
    """DKD at every radius on every border pixel (the top-k fill's zero pixels reach them) and random interior pixels, count 0, 1, below
    and above cap; planted windows: flat (residual exactly 0), a single spike, two equal maxima, and a zero window at x = W - 1 whose
    refined position is exactly kx = 1."""
    rng = np.random.default_rng(r)
    H, W = 20, 26
    score = rng.random((H, W)).astype(F32)
    border = [y * W + x for y in range(H) for x in range(W) if y in (0, H - 1) or x in (0, W - 1)]
    idx = np.array(border + list(rng.integers(0, H * W, 40)), np.int64)
    for count, cap in [(0, 8), (1, 8), (len(idx), len(idx) + 5), (len(idx), len(idx) - 7)]:
        _dkd_check(st, score, idx, r, count, cap, f"r={r} count={count} cap={cap}")
    # planted windows
    s = rng.random((H, W)).astype(F32) * F32(0.1)
    cy, cx = 10, 12
    s[cy - r:cy + r + 1, cx - r:cx + r + 1] = F32(0.5)                    # flat
    s[2, 3] = F32(1.0)                                                 # single spike
    s[17, 5] = s[17, 7] = F32(0.9)                                     # two equal maxima around (17, 6)
    s[4:4 + 2 * r + 1, W - 1 - r:W] = 0                                # zero window at the last column
    planted = np.array([cy * W + cx, 2 * W + 3, 17 * W + 6, (4 + r) * W + W - 1, 0, H * W - 1], np.int64)
    out = _dkd_check(st, s, planted, r, len(planted), 8, f"r={r} planted")
    exp = np.array([F32(cx) / F32(W - 1) * F32(2) - F32(1), F32(cy) / F32(H - 1) * F32(2) - F32(1)], F32)
    assert np.array_equal(out["kxy"][0], exp), (out["kxy"][0], exp)  # flat window: residual exactly 0
    assert out["kxy"][3, 0] == 1.0


def _sddh_w(al_weights, bias_scale=1.0):
    w = dict(al_weights)
    w["desc_head.offset_conv.2.bias"] = (al_weights["desc_head.offset_conv.2.bias"] * F32(bias_scale)).astype(F32)
    return w


def _feat_map(rng, H, W):
    f = rand(rng, H, W, 128)
    return (f / np.linalg.norm(f, axis=2, keepdims=True)).astype(F32)


def _edge_kxy(rng, H, W, n):
    """Keypoints at the four corners, along each edge, with kw in (0, 1) and at exact integers, then random."""
    kw = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (0.3, 0.6), (W - 1.2, 0.5), (0.7, H - 1.5), (1, 1), (W - 2, H - 2), (2, H - 1),
          (W - 1, 2), (W / 2, 0), (0, H / 2), (W - 1, H / 2), (W / 2, H - 1), (3, 4)]
    k = np.array(kw, np.float64) / np.array([W - 1, H - 1]) * 2 - 1
    k = np.concatenate([k, rng.uniform(-1, 1, (max(n - len(k), 0), 2))])[:n]
    return np.clip(k, -1, 1).astype(F32)


def _sddh_offsets_check(out, feat, kxy, n, w, what):
    off_ref, a, bar, mo = sddh_offsets_ref(feat, kxy[:n], w)
    H, W = feat.shape[:2]
    wh = np.array([W - 1, H - 1], F32)
    assert np.array_equal(out["kpts"][:n], (wh * (kxy[:n] + F32(1)) / F32(2)).astype(F32)), what
    sat = np.abs(a) - float(mo) > bar
    dev = out["off"][:n]
    assert np.array_equal(dev[sat], (np.sign(a[sat]) * mo).astype(F32)), what
    report("sddh offsets", *check_bar(dev, off_ref, bar, what))
    return int(sat.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("H, W", [(8, 8), (8, 40), (33, 8), (24, 31)])
def test_sddh_offsets(st, al_weights, H, W):
    """The offsets stage at keypoints on the corners and edges (both patch-corner clamps fire), kw in (0, 1) and at integers, on maps
    down to 8 pixels; count 1, 7, 8, 9, 300 (CTA tails) and above cap; biases scaled so that offsets saturate at exactly +-max_off."""
    rng = np.random.default_rng(H * W)
    feat = _feat_map(rng, H, W)
    saturated = 0
    for scale in (1.0, 400.0):
        w = _sddh_w(al_weights, scale)
        for count, cap in [(1, 4), (7, 8), (8, 8), (9, 16), (300, 310), (20, 13)]:
            kxy = _edge_kxy(rng, H, W, count)
            out, tail = st.aliked_sddh(feat, kxy, count, cap, w, sentinel=SENT)
            n = min(count, cap)
            saturated += _sddh_offsets_check(out, feat, kxy, n, w, f"{H}x{W} count={count} cap={cap} scale={scale}")
            assert np.all(out["off"][n:] == SENT) and np.all(out["kpts"][n:] == SENT)
            for k in tail:
                assert np.all(tail[k] == SENT)
    assert saturated > 0


def _desc_check(out, ref, n, cap, bar, what, stage):
    assert np.all(out["desc"][:, n:] == SENT), what
    err = np.abs(out["desc"][:, :n].astype(np.float64) - ref)
    assert np.isfinite(out["desc"][:, :n]).all() and err.max(initial=0) <= bar, (what, err.max(initial=0))
    report(stage, float(err.max(initial=0)), float(err.max(initial=0) / bar))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("count", [0, 1, 127, 128, 129, 300])
def test_sddh_descriptors(st, al_weights, precision, count):
    """Sampling, both GEMMs and the normalisation, EXACT and FAST, on the device's own offsets and on planted offsets that put samples
    fully and partly outside each side of the map and on its last row and column; desc columns from min(count, cap) on stay sentinel."""
    rng = np.random.default_rng(count + 17)
    H, W = 19, 27
    feat = _feat_map(rng, H, W)
    cap = count + 9
    kxy = _edge_kxy(rng, H, W, count)
    bar = DESC_EXACT if precision == "exact" else DESC_FAST
    st.set_precision(precision)
    try:
        out, tail = st.aliked_sddh(feat, kxy, count, cap, al_weights, sentinel=SENT)
        assert np.all(tail["desc"] == SENT)
        if count:
            _desc_check(out, sddh_desc_ref(feat, kxy, out["off"][:count], al_weights), count, cap, bar, f"{precision} count={count}",
                        f"sddh desc {precision}")
        else:
            assert np.all(out["desc"] == SENT)
        if count:
            kw = sddh_kw(kxy, H, W)
            tx = np.array([-1.5, -0.5, -1.0, 0.0, W - 1, W - 0.5, W, W + 1, 0.25, W - 1.25, -3.0, 2.5, W - 1, -0.99, W - 0.01, 5.0], F32)
            ty = np.array([-0.5, -1.5, H - 1, H - 0.5, H, -1.0, H + 1, 0.0, H - 1.25, 0.25, 2.5, -3.0, H - 1, H - 0.01, -0.99, 5.0], F32)
            roll = rng.integers(0, 16, count)
            off = np.zeros((count, 32), F32)
            for i in range(count):
                off[i, :16] = np.roll(tx, roll[i]) - kw[i, 0]
                off[i, 16:] = np.roll(ty, roll[i] + 3) - kw[i, 1]
            out, tail = st.aliked_sddh(feat, kxy, count, cap, al_weights, off=off, sentinel=SENT)
            _desc_check(out, sddh_desc_ref(feat, kxy, off, al_weights), count, cap, bar, f"{precision} count={count} planted",
                        f"sddh desc {precision}")
    finally:
        st.set_precision("exact")


@pytest.mark.gpu
def test_threshold(st):
    """thr is passed through bitwise when a candidate passed it; otherwise (and in mean mode) it is the mean of the score map within 1 ulp
    of float32."""
    rng = np.random.default_rng(9)
    for HW in (1, 1023, 1025, 100000):
        s = rng.random(HW).astype(F32)
        thr, tail = st.aliked_threshold(s, 3, 0.2, SENT)
        assert thr == F32(0.2) and np.all(tail == SENT)
        for cc in (0, None):
            thr, tail = st.aliked_threshold(s, cc, 0.2, SENT)
            m = s.astype(np.float64).mean()
            assert abs(float(thr) - m) <= float(np.spacing(F32(m))), (HW, cc, thr, m)
            assert np.all(tail == SENT)


# ------------------------------------------------------------------ end to end, at sizes the goldens do not reach
@pytest.mark.gpu
@pytest.mark.parametrize("H, W", [(8, 8), (8, 40), (33, 31), (63, 65)])
def test_small_and_odd_images(ctx, al_weights, H, W):
    """Small and odd images: every convolution on <8,1>, block 4 on 1 x 1 or 1 x 2 maps, most keypoints on the patch clamp; against
    oracle.aliked.extract, dense score and feature taps within 2e-5."""
    from dim_b200 import _native
    from oracle import aliked as o_al
    from oracle.compare import compare_aliked
    from test_keypoint_limits import rgb_image
    img = rgb_image(H * 100 + W, H, W)
    conf = {"model_name": "aliked-n16rot", "max_num_keypoints": 4000, "detection_threshold": 0.2, "nms_radius": 2}
    net = _native.AlikedNet(ctx, al_weights, 4000, 0.2, 2, max(H, 32), max(W, 32))
    out = net.extract(img)
    ref = o_al.extract(img, al_weights, conf, return_debug=True)
    thr = 0.2 if (ref["_score_map"] > 0.2).any() else float(ref["_score_map"].mean())
    rep = compare_aliked(out, ref, ref["_score_map"], thr, 2, tol=1e-4, tol_kpt=1e-3)
    print(H, W, rep["n"], rep["max_dkpt"], rep["max_dscore"], rep["max_ddesc"])
    assert np.abs(net.debug_read(0, (H, W)) - ref["_score_map"]).max() < 2e-5
    assert np.abs(net.debug_read(1, (128, H, W)) - ref["_feature_map"]).max() < 2e-5


@pytest.mark.gpu
def test_topk_fill_through_dkd_and_sddh(ctx, al_weights):
    """Top-k with K above the candidate count on a small image: the zero fill hands border pixels to DKD and SDDH; every keypoint
    against the index-given oracle refinement."""
    from dim_b200 import _native
    from test_keypoint_limits import al_maps, border_zeroed_nms, pair_aliked, refine_oracle, rgb_image, topk_oracle
    H, W, K = 40, 56, 600
    img = rgb_image(77, H, W)
    feat, score = al_maps(img, al_weights)
    net = _native.AlikedNet(ctx, al_weights, K, 0.0, 2, H, W)
    out = net.extract(img)
    assert len(out["keypoints"]) == K
    nms_dev = border_zeroed_nms(torch.from_numpy(net.debug_read(0, (H, W)))[None, None], 2).reshape(-1)
    cand = torch.nonzero(nms_dev > 0)[:, 0]
    C_ = len(cand)
    assert 0 < C_ < K
    head = refine_oracle(feat, score, topk_oracle(score, 2, C_), 2, al_weights)
    pair_aliked({k: (v[:C_] if k != "descriptors" else v[:, :C_]) for k, v in out.items()}, head, max_unpaired=4)
    zero = torch.nonzero(nms_dev == 0)[:, 0][:K - C_]
    tail = refine_oracle(feat, score, zero, 2, al_weights)
    got = {k: (v[C_:] if k != "descriptors" else v[:, C_:]) for k, v in out.items()}
    ys, xs = zero.numpy() // W, zero.numpy() % W
    assert ((ys == 0) | (ys == H - 1) | (xs == 0) | (xs == W - 1)).any()
    assert np.abs(got["keypoints"] - tail["keypoints"]).max() < 1e-3
    assert np.abs(got["scores"] - tail["scores"]).max() < 1e-4
    assert np.abs(got["descriptors"] - tail["descriptors"]).max() < 1e-4


@pytest.mark.gpu
def test_fast_precision_extraction(ctx, al_golden, al_weights):
    """FAST precision on a golden image: detection runs on the CUDA cores in fp32, so keypoints and scores equal EXACT's bitwise; the
    descriptors (plain fp16 GEMM operands in SDDH) stay within DESC_FAST of EXACT's and of the oracle's."""
    from dim_b200 import _native
    from conftest import al_case
    img, conf, ref = al_case(al_golden, "real224x288")
    H, W = img.shape[:2]
    args = (al_weights, conf["max_num_keypoints"], conf["detection_threshold"], conf["nms_radius"], H, W)
    ex = _native.AlikedNet(ctx, *args).extract(img)
    fctx = _native.Context(0, precision="fast")
    fa = _native.AlikedNet(fctx, *args).extract(img)
    assert np.array_equal(fa["keypoints"], ex["keypoints"]) and np.array_equal(fa["scores"], ex["scores"])
    d_ex = float(np.abs(fa["descriptors"] - ex["descriptors"]).max())
    d = np.linalg.norm(fa["keypoints"][:, None].astype(np.float64) - ref["keypoints"][None], axis=2)
    j, ok = d.argmin(1), d.min(1) < 1e-3
    overlap = float(ok.mean())
    d_ref = float(np.abs(fa["descriptors"][:, ok] - ref["descriptors"][:, j[ok]]).max())
    print(f"FAST: {len(fa['keypoints'])} keypoints, overlap with the oracle {overlap:.4f}, max descriptor delta vs EXACT {d_ex:.2e}, "
          f"vs oracle {d_ref:.2e}")
    assert overlap > 0.99 and d_ex < DESC_FAST and d_ref < DESC_FAST
