"""SIFT on the device against cv2.SIFT on the host: extraction of 16 gray 2048 x 1536 images, and the sift+kornia_matcher pipeline over
an image set of those 16 images (all 120 pairs).

Images: the three SuperPoint golden test images resized to 2048 x 1536 (INTER_CUBIC) and warped by seeded homographies, 16 in all.
Extraction, at n_features 2048 and 8000 (contrastThreshold 0.0004 and the other keys of config.py's sift+kornia_matcher):
  device  SiftNet.extract_dev on the 16 images in one call, timed with CUDA events after a warm-up; per-group device times
          (sift.pyr / extrema / ori / select / desc) from a separate profiled call;
  host    cv2.SIFT_create(...).detectAndCompute per image with cv2.setNumThreads(all host cores);
  agreement of device and cv2 keypoints (within 0.01 px, 0.1 degree, 1 % of size, both ways) and of their descriptor bytes (within 1),
  next to the agreement of cv2's SSE2 baseline (cv2.setUseOptimized(False)) with its optimised build on the same images.
Set: ImageSetMatcher(extractor="sift", matcher="kornia_matcher") run() on the 16 images (extract, exchange, match, tables on the
host) against the host flow: cv2 SIFT per image, the float16 round trip of features.h5, then KorniaMatcher._match_pairs per pair.
The card's name and power limit are read in the same process.  Prints one JSON line per measurement; --out appends them to a file.
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

H, W, N = 1536, 2048, 16
CONF = {"n_layers": 3, "contrast": 0.0004, "edge": 10.0, "sigma": 1.6}
NET = {"n_octave_layers": 3, "contrast_threshold": 0.0004, "edge_threshold": 10.0, "sigma": 1.6}


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "clocks_max_sm": clock}


def images():
    import cv2

    from dim_b200 import synthetic
    g = np.load(os.path.join(ROOT, "tests", "golden", "superpoint_golden.npz"))
    base = [cv2.resize(g[k + ".image"], (W, H), interpolation=cv2.INTER_CUBIC) for k in ("real240x320", "real_odd237x315",
                                                                                            "blocks384x512_top512")]
    return np.stack([base[k % 3] if k < 3 else synthetic.warp_pair(base[k % 3], k, jitter=120.0) for k in range(N)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--features", type=int, nargs="+", default=[2048, 8000])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    import cv2
    import torch

    from dim_b200 import _native
    from dim_b200.config import Config
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    from oracle import sift as O

    cores = os.cpu_count()
    cv2.setNumThreads(cores)
    info = card()
    imgs = images()
    ctx = _native.Context.get(0)
    d_imgs = torch.from_numpy(imgs.astype(np.float32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    lines = []

    def emit(rec):
        rec = {**rec, **info, "host_cores": cores}
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for nf in args.features:
        net = _native.SiftNet(ctx, n_features=nf, max_batch=N, max_height=H, max_width=W, **NET)
        cap = nf + 64
        kp = torch.zeros(N, cap, 2, device="cuda")
        de = torch.zeros(N, 128, cap, device="cuda")
        fr = torch.zeros(N, cap, 3, device="cuda")
        cnt = torch.zeros(N, dtype=torch.int32, device="cuda")

        def run():
            net.extract_dev(d_imgs.data_ptr(), N, H, W, kp.data_ptr(), de.data_ptr(), cnt.data_ptr(), cap, fr.data_ptr(), 0, st)

        run()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            run()
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.steps
        ctx.profile(True)
        run()
        torch.cuda.synchronize()
        prof = {k: round(v[0], 3) for k, v in sorted(ctx.profile_read().items()) if k.startswith("sift.")}
        ctx.profile(False)
        counts = cnt.cpu().numpy()
        assert counts.min() >= 0 and counts.max() <= cap, counts
        k_h, d_h, f_h = kp.cpu().numpy(), de.cpu().numpy(), fr.cpu().numpy()
        dev = [{"keypoints": k_h[b, :counts[b]], "size": f_h[b, :counts[b], 0], "angle": f_h[b, :counts[b], 1],
                "descriptors": d_h[b, :, :counts[b]]} for b in range(N)]
        t0 = time.perf_counter()
        ref = [O.cv2_extract(im, nf, **CONF) for im in imgs]
        host_s = time.perf_counter() - t0
        cv2.setUseOptimized(False)  # calibration: cv2's SSE2 baseline against its optimised build, image by image
        base = [O.cv2_extract(im, nf, **CONF) for im in imgs]
        cv2.setUseOptimized(True)
        agree_d, agree_r, agree_cv2, desc_ok, n_d, n_r = [], [], [], [], 0, 0
        for a, r, c in zip(dev, ref, base):
            fa, pairs = O.agreement(a, r)
            fb, _ = O.agreement(r, a)
            agree_d.append(fa)
            agree_r.append(fb)
            agree_cv2.append(min(O.agreement(c, r)[0], O.agreement(r, c)[0]))
            if len(pairs):
                desc_ok.append(np.mean(np.abs(a["descriptors"][:, pairs[:, 0]] - r["descriptors"][:, pairs[:, 1]]).max(0) <= 1))
            n_d += len(a["keypoints"])
            n_r += len(r["keypoints"])
        emit({"metric": f"SIFT extraction images/s, {N} gray {W}x{H} images, n_features {nf}", "n_features": nf,
              "device_images_per_s": round(N / (ms / 1e3), 2), "device_ms_per_batch": round(ms, 2),
              "cv2_images_per_s": round(N / host_s, 3), "speedup": round((N / (ms / 1e3)) / (N / host_s), 1),
              "device_profile_ms": prof, "keypoints_device": int(n_d), "keypoints_cv2": int(n_r),
              "agree_device_in_cv2_min": round(float(min(agree_d)), 5), "agree_cv2_in_device_min": round(float(min(agree_r)), 5),
              "agree_device_in_cv2_mean": round(float(np.mean(agree_d)), 5),
              "agree_device_cv2_per_image": [round(float(min(x, y)), 4) for x, y in zip(agree_d, agree_r)],
              "agree_cv2_baseline_vs_optimised_per_image": [round(float(x), 4) for x in agree_cv2],
              "desc_bytes_within_1_min": round(float(min(desc_ok)), 5), "data": "golden test images resized and warped"})
        del net, kp, de, fr
        torch.cuda.empty_cache()

    # the sift+kornia_matcher pipeline over the set
    nf = 2048
    pairs = pairs_from_bruteforce(list(range(N)))
    eng = ImageSetMatcher(ctx, None, None, N, H, W, {"n_features": nf}, {"match_mode": "smnn", "th": 0.85}, batch_images=N,
                          batch_pairs=32, extractor="sift", matcher="kornia_matcher")
    eng.run(d_imgs, list(range(N)), pairs)  # warm-up of every shape
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tables = eng.run(d_imgs, list(range(N)), pairs)
    set_s = time.perf_counter() - t0
    plugin = KorniaMatcher(Config(pipeline="sift+kornia_matcher"))
    sift = cv2.SIFT_create(nfeatures=nf, nOctaveLayers=3, contrastThreshold=0.0004, edgeThreshold=10, sigma=1.6)
    plugin._match_pairs(*[as_half_roundtrip({"keypoints": np.zeros((4, 2), np.float32),
                                             "descriptors": np.random.default_rng(0).random((128, 4)).astype(np.float32)})] * 2)
    t0 = time.perf_counter()
    feats = []
    for im in imgs:
        k, d = sift.detectAndCompute(im, None)
        feats.append(as_half_roundtrip({"keypoints": cv2.KeyPoint_convert(k), "descriptors": d.astype(float).T}))
    ext_s = time.perf_counter() - t0
    host_tables = [plugin._match_pairs(feats[i], feats[j]) for i, j in pairs]
    host_s = time.perf_counter() - t0
    emit({"metric": f"sift+kornia_matcher image set pairs/s, {N} gray {W}x{H} images, {len(pairs)} pairs, n_features {nf}",
          "set_pairs_per_s": round(len(pairs) / set_s, 2), "set_s": round(set_s, 3), "host_flow_pairs_per_s": round(len(pairs) / host_s, 2),
          "host_flow_s": round(host_s, 3), "host_flow_cv2_extract_s": round(ext_s, 3), "speedup": round(host_s / set_s, 1),
          "matches_set": int(sum(len(t) for t in tables)), "matches_host_flow": int(sum(len(t) for t in host_tables)),
          "data": "golden test images resized and warped"})
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
