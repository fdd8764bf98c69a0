"""numpy restatement of OpenCV 4.x SIFT (cv2.SIFT_create(...).detectAndCompute(gray_uint8, None), enable_precise_upscale = false).

Test-only reference for csrc/sift.cu.  The blurs run in float64 and are rounded to float32 after each separable pass; the per-keypoint
arithmetic (interpolation, histograms, descriptors) runs in float64 with OpenCV's float32 constants and its fastAtan2 polynomial.
The output order is removeDuplicatedSorted's (x, y ascending; size descending; angle ascending; response descending; octave
descending), which is also the device's.
"""
from __future__ import annotations

import math

import numpy as np

BORDER = 5
MAX_INTERP = 5
ORI_BINS = 36
FLT_EPS = float(np.finfo(np.float32).eps)


def gaussian_taps(sigma: float) -> np.ndarray:
    """getGaussianKernel(cvRound(8 sigma + 1) | 1, sigma, CV_32F)."""
    n = int(np.rint(sigma * 8 + 1)) | 1
    x = np.arange(n) - (n - 1) * 0.5
    k = np.exp(-0.5 / (sigma * sigma) * x * x).astype(np.float32)
    return (k.astype(np.float64) * (1.0 / float(np.sum(k, dtype=np.float64)))).astype(np.float32)


def blur(img: np.ndarray, sigma: float) -> np.ndarray:
    """GaussianBlur(img, Size(), sigma, sigma) on float32 with BORDER_REFLECT_101: row pass, then column pass."""
    k = gaussian_taps(sigma).astype(np.float64)
    r = len(k) // 2
    out = img.astype(np.float64)
    for axis in (1, 0):
        pad = [(0, 0), (0, 0)]
        pad[axis] = (r, r)
        p = np.pad(out, pad, mode="reflect")
        n = out.shape[axis]
        acc = np.zeros_like(out)
        for j in range(len(k)):
            acc += k[j] * (p[:, j:j + n] if axis == 1 else p[j:j + n, :])
        out = acc.astype(np.float32).astype(np.float64)
    return out.astype(np.float32)


def to_u8(img: np.ndarray) -> np.ndarray:
    """convertTo(CV_8U): round half to even, saturate."""
    return np.clip(np.rint(np.asarray(img, np.float64)), 0, 255).astype(np.uint8)


def upsample2(img: np.ndarray) -> np.ndarray:
    """resize(img, (2W, 2H), INTER_LINEAR) of a uint8-valued image (exact in float32)."""
    def table(n):
        f = (np.arange(2 * n) + 0.5) * 0.5 - 0.5
        s = np.floor(f).astype(int)
        a = f - s
        a[s < 0] = 0
        s[s < 0] = 0
        hi = s >= n - 1
        a[hi] = 0
        s[hi] = n - 1
        return s, np.minimum(s + 1, n - 1), a
    H, W = img.shape
    x = img.astype(np.float64)
    sx0, sx1, ax = table(W)
    sy0, sy1, ay = table(H)
    rows = x[:, sx0] * (1 - ax) + x[:, sx1] * ax
    return (rows[sy0] * (1 - ay)[:, None] + rows[sy1] * ay[:, None]).astype(np.float32)


def n_octaves(H: int, W: int) -> int:
    return int(np.rint(math.log(min(2 * H, 2 * W)) / math.log(2.0) - 2)) + 1


def pyramid(img_u8: np.ndarray, n_layers: int = 3, sigma: float = 1.6):
    """Gaussian levels gauss[o][i] (i < n_layers + 3) and DoG levels dog[o][i] (i < n_layers + 2), octave 0 being OpenCV's -1."""
    sf = np.float32(sigma)
    sig_diff = float(np.sqrt(np.float32(max(sf * sf - np.float32(1), np.float32(0.01)))))
    base = blur(upsample2(img_u8), sig_diff)
    k = 2.0 ** (1.0 / n_layers)
    sig = [sigma] + [math.sqrt((k ** (i - 1) * sigma * k) ** 2 - (k ** (i - 1) * sigma) ** 2) for i in range(1, n_layers + 3)]
    gauss, dog = [], []
    for o in range(n_octaves(*img_u8.shape)):
        lv = [base if o == 0 else gauss[o - 1][n_layers][::2, ::2][: gauss[o - 1][n_layers].shape[0] // 2,
                                                                   : gauss[o - 1][n_layers].shape[1] // 2].copy()]
        for i in range(1, n_layers + 3):
            lv.append(blur(lv[-1], sig[i]))
        gauss.append(lv)
        dog.append([lv[i + 1] - lv[i] for i in range(n_layers + 2)])
    return gauss, dog


def fast_atan2(y, x):
    """cv::fastAtan2 in degrees (float32 arithmetic)."""
    y = np.asarray(y, np.float32)
    x = np.asarray(x, np.float32)
    c180 = np.float32(180 / np.pi)
    p1, p3 = np.float32(0.9997878412794807) * c180, np.float32(-0.3258083974640975) * c180
    p5, p7 = np.float32(0.1555786518463281) * c180, np.float32(-0.04432655554792128) * c180
    ax, ay = np.abs(x), np.abs(y)
    eps = np.float32(np.finfo(np.float64).eps)
    big = ax >= ay
    c = np.where(big, ay / (ax + eps), ax / (ay + eps)).astype(np.float32)
    c2 = c * c
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c
    a = np.where(big, a, np.float32(90) - a)
    a = np.where(x < 0, np.float32(180) - a, a)
    a = np.where(y < 0, np.float32(360) - a, a)
    return a.astype(np.float32)


def _refine(dog, o, layer, r, c, n_layers, contrast, edge, sigma):
    img_scale = 1.0 / 255
    ds, ss, cs = img_scale * 0.5, img_scale, img_scale * 0.25
    h, w = dog[o][0].shape
    xi = xr = xc = 0.0
    i = 0
    while i < MAX_INTERP:
        I, P, N = dog[o][layer], dog[o][layer - 1], dog[o][layer + 1]
        dD = np.array([(I[r, c + 1] - I[r, c - 1]) * ds, (I[r + 1, c] - I[r - 1, c]) * ds, (N[r, c] - P[r, c]) * ds], np.float64)
        v2 = float(I[r, c]) * 2
        dxx = (float(I[r, c + 1]) + I[r, c - 1] - v2) * ss
        dyy = (float(I[r + 1, c]) + I[r - 1, c] - v2) * ss
        dss = (float(N[r, c]) + P[r, c] - v2) * ss
        dxy = (float(I[r + 1, c + 1]) - I[r + 1, c - 1] - I[r - 1, c + 1] + I[r - 1, c - 1]) * cs
        dxs = (float(N[r, c + 1]) - N[r, c - 1] - P[r, c + 1] + P[r, c - 1]) * cs
        dys = (float(N[r + 1, c]) - N[r - 1, c] - P[r + 1, c] + P[r - 1, c]) * cs
        Hm = np.array([[dxx, dxy, dxs], [dxy, dyy, dys], [dxs, dys, dss]])
        det = np.linalg.det(Hm)
        X = np.linalg.solve(Hm, dD) if det != 0 else np.zeros(3)
        xi, xr, xc = -X[2], -X[1], -X[0]
        if abs(xi) < 0.5 and abs(xr) < 0.5 and abs(xc) < 0.5:
            break
        if max(abs(xi), abs(xr), abs(xc)) > 2 ** 31 / 3:
            return None
        c += int(np.rint(xc))
        r += int(np.rint(xr))
        layer += int(np.rint(xi))
        if layer < 1 or layer > n_layers or c < BORDER or c >= w - BORDER or r < BORDER or r >= h - BORDER:
            return None
        i += 1
    if i >= MAX_INTERP:
        return None
    I, P, N = dog[o][layer], dog[o][layer - 1], dog[o][layer + 1]
    dD = np.array([(I[r, c + 1] - I[r, c - 1]) * ds, (I[r + 1, c] - I[r - 1, c]) * ds, (N[r, c] - P[r, c]) * ds], np.float64)
    contr = float(I[r, c]) * img_scale + float(dD @ np.array([xc, xr, xi])) * 0.5
    if abs(contr) * n_layers < contrast:
        return None
    v2 = float(I[r, c]) * 2
    dxx = (float(I[r, c + 1]) + I[r, c - 1] - v2) * ss
    dyy = (float(I[r + 1, c]) + I[r - 1, c] - v2) * ss
    dxy = (float(I[r + 1, c + 1]) - I[r + 1, c - 1] - I[r - 1, c + 1] + I[r - 1, c - 1]) * cs
    tr, det = dxx + dyy, dxx * dyy - dxy * dxy
    if det <= 0 or tr * tr * edge >= (edge + 1) ** 2 * det:
        return None
    return layer, r, c, xc, xr, xi, contr


def _ori_hist(img, r, c, radius, sig):
    h, w = img.shape
    i, j = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    y, x = r + i, c + j
    ok = (y > 0) & (y < h - 1) & (x > 0) & (x < w - 1)
    i, j, y, x = i[ok], j[ok], y[ok], x[ok]
    dx = img[y, x + 1] - img[y, x - 1]
    dy = img[y - 1, x] - img[y + 1, x]
    wt = np.exp((i * i + j * j) * (-1.0 / (2.0 * sig * sig)))
    ori = fast_atan2(dy, dx)
    mag = np.sqrt(dx.astype(np.float64) ** 2 + dy.astype(np.float64) ** 2)
    b = np.rint(np.float32(ORI_BINS / 360.0) * ori).astype(int) % ORI_BINS
    t = np.bincount(b, weights=wt * mag, minlength=ORI_BINS)
    tp = np.concatenate([t[-2:], t, t[:2]])
    return (tp[:-4] + tp[4:]) / 16 + (tp[1:-3] + tp[3:-1]) * 4 / 16 + tp[2:-2] * 6 / 16


def detect(gauss, dog, n_layers=3, contrast=0.04, edge=10.0, sigma=1.6):
    """findScaleSpaceExtrema: list of (x, y, size, angle, response, octave) with octave packed as cv2 does before scaling."""
    thr = math.floor(0.5 * contrast / n_layers * 255)
    kps = []
    for o in range(len(dog)):
        h, w = dog[o][0].shape
        if h <= 2 * BORDER or w <= 2 * BORDER:
            continue
        for layer in range(1, n_layers + 1):
            stack = np.stack(dog[o][layer - 1: layer + 2])
            core = stack[1, BORDER:h - BORDER, BORDER:w - BORDER]
            mx = np.full(core.shape, -np.inf, np.float32)
            mn = np.full(core.shape, np.inf, np.float32)
            for dl in range(3):
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        s = stack[dl, BORDER + dy:h - BORDER + dy, BORDER + dx:w - BORDER + dx]
                        mx = np.maximum(mx, s)
                        mn = np.minimum(mn, s)
            cand = (np.abs(core) > thr) & (((core > 0) & (core >= mx)) | ((core < 0) & (core <= mn)))
            for rr, cc in zip(*np.nonzero(cand)):
                ref = _refine(dog, o, layer, int(rr) + BORDER, int(cc) + BORDER, n_layers, contrast, edge, sigma)
                if ref is None:
                    continue
                ly, r, c, xc, xr, xi, contr = ref
                size = sigma * 2.0 ** ((ly + xi) / n_layers) * (1 << o) * 2
                scl = size * 0.5 / (1 << o)
                hist = _ori_hist(gauss[o][ly], r, c, int(np.rint(4.5 * scl)), 1.5 * scl)
                thr_m = hist.max() * 0.8
                oct_packed = o + (ly << 8) + (int(np.rint((xi + 0.5) * 255)) << 16)
                for j in range(ORI_BINS):
                    lft, rgt = hist[j - 1], hist[(j + 1) % ORI_BINS]
                    if hist[j] > lft and hist[j] > rgt and hist[j] >= thr_m:
                        b = j + 0.5 * (lft - rgt) / (lft - 2 * hist[j] + rgt)
                        b = b + ORI_BINS if b < 0 else (b - ORI_BINS if b >= ORI_BINS else b)
                        ang = 360.0 - 360.0 / ORI_BINS * b
                        if abs(ang - 360.0) < FLT_EPS:
                            ang = 0.0
                        kps.append((np.float32((c + xc) * (1 << o)), np.float32((r + xr) * (1 << o)), np.float32(size),
                                    np.float32(ang), np.float32(abs(contr)), oct_packed))
    return kps


def select(kps, n_features):
    """removeDuplicatedSorted, then retainBest(n_features) keeping boundary ties, in the sorted order."""
    kps = sorted(kps, key=lambda k: (k[0], k[1], -k[2], k[3], -k[4], -k[5]))
    out = []
    for k in kps:
        if out and out[-1][:4] == k[:4]:
            continue
        out.append(k)
    if n_features > 0 and len(out) > n_features:
        t = sorted((k[4] for k in out), reverse=True)[n_features - 1]
        out = [k for k in out if k[4] >= t]
    return out


def descriptor(img, x, y, angle, size):
    """calcSIFTDescriptor(img, (x, y), 360 - angle, size / 2, 4, 8) -> 128 integral values."""
    d, n = 4, 8
    ori = 360.0 - angle
    if abs(ori - 360.0) < FLT_EPS:
        ori = 0.0
    scl = size * 0.5
    px, py = int(np.rint(x)), int(np.rint(y))
    hw = 3.0 * scl
    radius = int(np.rint(hw * 1.4142135623730951 * (d + 1) * 0.5))
    h, w = img.shape
    radius = min(radius, int(math.sqrt(float(w) * w + float(h) * h)))
    ct = math.cos(np.float32(ori) * np.float32(np.pi / 180)) / hw
    st = math.sin(np.float32(ori) * np.float32(np.pi / 180)) / hw
    i, j = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    i, j = i.ravel(), j.ravel()
    c_rot = j * ct - i * st
    r_rot = j * st + i * ct
    rbin = r_rot + d / 2 - 0.5
    cbin = c_rot + d / 2 - 0.5
    yy, xx = py + i, px + j
    ok = (rbin > -1) & (rbin < d) & (cbin > -1) & (cbin < d) & (yy > 0) & (yy < h - 1) & (xx > 0) & (xx < w - 1)
    rbin, cbin, c_rot, r_rot, yy, xx = rbin[ok], cbin[ok], c_rot[ok], r_rot[ok], yy[ok], xx[ok]
    dx = img[yy, xx + 1] - img[yy, xx - 1]
    dy = img[yy - 1, xx] - img[yy + 1, xx]
    wt = np.exp((c_rot * c_rot + r_rot * r_rot) * (-1.0 / (d * d * 0.5)))
    obin = (fast_atan2(dy, dx).astype(np.float64) - ori) * (n / 360.0)
    mag = np.sqrt(dx.astype(np.float64) ** 2 + dy.astype(np.float64) ** 2) * wt
    r0, c0, o0 = np.floor(rbin).astype(int), np.floor(cbin).astype(int), np.floor(obin).astype(int)
    rbin, cbin, obin = rbin - r0, cbin - c0, obin - o0
    o0 = np.where(o0 < 0, o0 + n, o0)
    o0 = np.where(o0 >= n, o0 - n, o0)
    hist = np.zeros((d + 2) * (d + 2) * (n + 2))
    for dr, wr in ((0, 1 - rbin), (1, rbin)):
        for dc, wc in ((0, 1 - cbin), (1, cbin)):
            for do, wo in ((0, 1 - obin), (1, obin)):
                idx = ((r0 + 1 + dr) * (d + 2) + c0 + 1 + dc) * (n + 2) + o0 + do
                np.add.at(hist, idx, mag * wr * wc * wo)
    hist = hist.reshape(d + 2, d + 2, n + 2)[1:d + 1, 1:d + 1]
    hist[:, :, :2] += hist[:, :, n:n + 2]
    v = hist[:, :, :n].ravel()
    v = np.minimum(v, np.sqrt(np.sum(v * v)) * 0.2)
    v = v * (512.0 / max(np.sqrt(np.sum(v * v)), FLT_EPS))
    return np.clip(np.rint(v), 0, 255)


def extract(img, n_features=0, n_layers=3, contrast=0.04, edge=10.0, sigma=1.6, return_pyramid=False):
    """img uint8 (H,W) (other dtypes go through convertTo(CV_8U)) -> keypoints (N,2), size, angle, response, octave (N,) and
    descriptors (128,N) float32, in removeDuplicatedSorted order."""
    img = np.asarray(img)
    if img.dtype != np.uint8:
        img = to_u8(img)
    gauss, dog = pyramid(img, n_layers, sigma)
    kps = select(detect(gauss, dog, n_layers, contrast, edge, sigma), n_features)
    N = len(kps)
    kp = np.array([[k[0], k[1]] for k in kps], np.float32).reshape(N, 2) * np.float32(0.5)
    size = np.array([k[2] for k in kps], np.float32) * np.float32(0.5)
    ang = np.array([k[3] for k in kps], np.float32)
    resp = np.array([k[4] for k in kps], np.float32)
    octv = np.array([(k[5] & ~255) | ((k[5] - 1) & 255) for k in kps], np.int64).astype(np.int32)
    desc = np.zeros((128, N), np.float32)
    for q, k in enumerate(kps):
        o, ly = k[5] & 255, (k[5] >> 8) & 255
        scale = 2.0 if o == 0 else 1.0 / (1 << (o - 1))
        desc[:, q] = descriptor(gauss[o][ly], float(kp[q, 0]) * scale, float(kp[q, 1]) * scale, float(ang[q]),
                                float(size[q]) * scale)
    out = {"keypoints": kp, "size": size, "angle": ang, "response": resp, "octave": octv, "descriptors": desc}
    if return_pyramid:
        out["gauss"], out["dog"] = gauss, dog
    return out


def cv2_extract(img_u8, n_features=0, n_layers=3, contrast=0.04, edge=10.0, sigma=1.6):
    """cv2's SIFT in the same dict layout (its own keypoint order)."""
    import cv2

    sift = cv2.SIFT_create(nfeatures=n_features, nOctaveLayers=n_layers, contrastThreshold=contrast, edgeThreshold=edge, sigma=sigma)
    kps, des = sift.detectAndCompute(img_u8, None)
    N = len(kps)
    return {"keypoints": np.array([k.pt for k in kps], np.float32).reshape(N, 2),
            "size": np.array([k.size for k in kps], np.float32), "angle": np.array([k.angle for k in kps], np.float32),
            "response": np.array([k.response for k in kps], np.float32), "octave": np.array([k.octave for k in kps], np.int32),
            "descriptors": (des.T.astype(np.float32) if des is not None else np.zeros((128, 0), np.float32))}


def agreement(a: dict, b: dict, px=0.01, deg=0.1, rel_size=0.01):
    """Keypoints of a with a partner in b within px pixels, deg degrees (circular) and rel_size of size.  Returns (fraction of a
    matched, index pairs (ia, ib))."""
    ka, kb = a["keypoints"], b["keypoints"]
    if len(ka) == 0:
        return 1.0, np.zeros((0, 2), int)
    if len(kb) == 0:
        return 0.0, np.zeros((0, 2), int)
    order = np.argsort(kb[:, 0], kind="stable")
    xs = kb[order, 0]
    pairs = []
    for i, (x, y) in enumerate(ka):
        lo, hi = np.searchsorted(xs, x - px, "left"), np.searchsorted(xs, x + px, "right")
        best = None
        for j in order[lo:hi]:
            if abs(kb[j, 1] - y) > px:
                continue
            da = abs(float(a["angle"][i]) - float(b["angle"][j])) % 360.0
            if min(da, 360.0 - da) > deg or abs(a["size"][i] - b["size"][j]) > rel_size * b["size"][j]:
                continue
            best = j
            break
        if best is not None:
            pairs.append((i, best))
    pairs = np.array(pairs, int).reshape(-1, 2)
    return len(pairs) / len(ka), pairs
