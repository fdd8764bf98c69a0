"""Keypoint limits and ALIKED detection modes on one GPU.

Configurations (one JSON line each):
  SuperPoint on 8 gray 2048 x 1536 images (nms_radius 3, keypoint_threshold 0.0005, fix_sampling) at max_keypoints 4096 / 16384
  (sp_select_kernel) and 16385 / 32768 (the grid-wide top-k), batches of 4 through SuperPointNet.extract_dev;
  ALIKED n16rot on 8 RGB 1024 x 1024 images (nms_radius 2) in threshold mode (0.2, 4096), top-k 4096, top-k 32768 and mean mode,
  one image per AlikedNet.extract_dev call.
For each: images/s (host clock around the timed runs, ended by a device synchronise, after a warm-up run), the selection's device time
(`sp.select+describe` / `al.detect` from dimb_ctx_profile, in a separate profiled run), the mean keypoint count, and whether the outputs
equal the plugin's (SuperPointExtractor / AlikedExtractor._extract per image).
A last line times the selection alone through dimb_selftest_select at K = 16384 on a 2048 x 1536 SuperPoint-like map with every pixel
a candidate: sp_select_kernel (one CTA per image) against the grid-wide path, batches of 1 and 8.
The card's name and power limit are read in the same process.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "clocks_max_sm": clock}


def images(n, H, W, gray):
    from dim_b200 import synthetic
    out = []
    for k in range(n):
        a = synthetic.blocks_image(100 + k, max(H, W), 8)[:H, :W]
        out.append(synthetic.to_gray_like_reference(np.ascontiguousarray(a)) if gray else a)
    return np.stack(out).astype(np.float32)


def timed(run, repeats):
    import torch
    run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        t = time.perf_counter()
        run()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return ts


def profiled(ctx, run, tag):
    import torch
    ctx.profile(True)
    run()
    torch.cuda.synchronize()
    prof = ctx.profile_read()
    ctx.profile(False)
    return prof.get(tag, [0.0, 0])[0]


def same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("keypoints", "scores", "descriptors"))


def bench_superpoint(ctx, K, imgs, repeats, batch):
    import torch

    from dim_b200 import _native, weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    n, H, W = imgs.shape
    w = weights.superpoint_v1()
    conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "remove_borders": 4, "fix_sampling": True, "max_keypoints": K}
    net = _native.SuperPointNet(ctx, w, max_batch=batch, max_height=H, max_width=W, **conf)
    dev = torch.device("cuda", ctx.device)
    d_img = torch.from_numpy(imgs).to(dev)
    kp, sc = torch.zeros(n, K, 2, device=dev), torch.zeros(n, K, device=dev)
    de, cnt = torch.zeros(n, 256, K, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)

    def run():
        for b0 in range(0, n, batch):
            net.extract_dev(d_img[b0].data_ptr(), batch, H, W, kp[b0].data_ptr(), sc[b0].data_ptr(), de[b0].data_ptr(), cnt[b0:].data_ptr(), K)

    ts = timed(run, repeats)
    sel_ms = profiled(ctx, run, "sp.select+describe")
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={"name": "superpoint", **conf, "weights_dict": w}))
    c = cnt.cpu().numpy()
    kpn, scn, den = kp.cpu().numpy(), sc.cpu().numpy(), de.cpu().numpy()
    identical = all(same({"keypoints": kpn[i, :c[i]], "scores": scn[i, :c[i]], "descriptors": den[i, :, :c[i]]}, ext._extract(imgs[i]))
                    for i in range(n))
    return {"config": f"superpoint max_keypoints {K}", "images": n, "batch": batch, "images_per_s": round(n / min(ts), 2),
            "seconds": [round(t, 4) for t in ts], "sp_select_describe_ms_per_run": round(sel_ms, 3),
            "mean_keypoints": float(c.mean()), "identical_to_plugin": bool(identical)}


def bench_aliked(ctx, name, K, thr, imgs, repeats):
    import torch

    from dim_b200 import _native, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    n, H, W, _ = imgs.shape
    w = weights.aliked_n16rot()
    net = _native.AlikedNet(ctx, w, K, thr, 2, H, W)
    cap = K if K > 0 else _native.ALIKED_N_LIMIT
    dev = torch.device("cuda", ctx.device)
    d_img = torch.from_numpy(imgs).to(dev)
    kp, sc = torch.zeros(n, cap, 2, device=dev), torch.zeros(n, cap, device=dev)
    de, cnt = torch.zeros(n, 128, cap, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)

    def run():
        for i in range(n):
            net.extract_dev(d_img[i].data_ptr(), H, W, 3, kp[i].data_ptr(), sc[i].data_ptr(), de[i].data_ptr(), cnt[i:].data_ptr(), cap)

    ts = timed(run, repeats)
    det_ms = profiled(ctx, run, "al.detect")
    ext = AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", "max_num_keypoints": K,
                                                                         "detection_threshold": thr, "nms_radius": 2, "weights_dict": w}))
    c = cnt.cpu().numpy()
    kpn, scn, den = kp.cpu().numpy(), sc.cpu().numpy(), de.cpu().numpy()
    identical = all(same({"keypoints": kpn[i, :c[i]], "scores": scn[i, :c[i]], "descriptors": den[i, :, :c[i]]}, ext._extract(imgs[i]))
                    for i in range(n))
    return {"config": f"aliked {name}", "max_num_keypoints": K, "detection_threshold": thr, "images": n,
            "images_per_s": round(n / min(ts), 2), "seconds": [round(t, 4) for t in ts], "al_detect_ms_per_run": round(det_ms, 3),
            "mean_keypoints": float(c.mean()), "identical_to_plugin": bool(identical)}


def bench_select_paths(iters):
    from dim_b200 import _native
    st = _native.SelfTest(0)
    rng = np.random.default_rng(0)
    out = {"config": "selection alone, K 16384, 2048 x 1536, every pixel a candidate (r 0)"}
    for B in (1, 8):
        s = rng.uniform(2.0 ** -24, 1.0, (B, 1536, 2048)).astype(np.float32)
        res = {}
        for path, grid in (("sp_select_kernel", False), ("grid_wide", True)):
            o = st.select(s, 0, 16384, grid=grid, iters=iters)
            res[path] = o
        same_out = all(np.array_equal(res["sp_select_kernel"][k], res["grid_wide"][k]) for k in ("sel_idx", "sel_score", "sel_count"))
        out[f"batch_{B}"] = {"ms_per_run": {p: round(res[p]["ms"], 4) for p in res}, "identical": bool(same_out)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    args = ap.parse_args()
    import torch

    from dim_b200 import _native
    if not torch.cuda.is_available():
        raise SystemExit("bench_keypoint_limits.py needs a GPU")
    info = card()
    ctx = _native.Context.get(0)
    lines = []
    gray = images(args.images, 1536, 2048, True)
    for K in (4096, 16384, 16385, 32768):
        lines.append(bench_superpoint(ctx, K, gray, args.repeats, 4))
    rgb = images(args.images, 1024, 1024, False)
    for name, K, thr in (("threshold 0.2", 4096, 0.2), ("top-k 4096", 4096, -1.0), ("top-k 32768", 32768, -1.0), ("mean", -1, -1.0)):
        lines.append(bench_aliked(ctx, name, K, thr, rgb, args.repeats))
    lines.append(bench_select_paths(args.iters))
    for line in lines:
        s = json.dumps({"bench": "keypoint_limits", **info, **line})
        print(s, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(s + "\n")


if __name__ == "__main__":
    main()
