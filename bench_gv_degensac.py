"""The three geometric-verification estimators on dominant-plane scenes, on one GPU: ransac8, lo-ransac and degensac (lo-ransac's waves
plus DEGENSAC's plane test and plane-and-parallax recovery), with OpenCV USAC_ACCURATE and USAC_MAGSAC on the host for reference.

Synthetic scenes (tests/test_gv_lo.scene: two cameras, a fraction of the points on one tilted plane, each match replaced by a random
point with the outlier probability) at 2048 matches, 256 pairs per scene in batches of 32 through dimb_gv_verify_dev (float32
keypoints, 1 px, max_iters 10000, confidence 0.9999): plane fractions 0.97 / 0.98 / 0.99 / 0.995 x 20 / 50 % outliers.  Per
estimator: pairs/s from CUDA events (median of alternating repetitions), mean 7-point hypotheses, overall recall, off-plane recall
(mean, min, pairs below 0.9) and the fraction of outliers kept.  The plane scenes are where the off-plane matches, the parallax that
SfM needs, are few: the recall of those is the number this benchmark exists for.  Then bench_verify.py's image set through
ImageSetMatcher.run_verified with each estimator.  One JSON line per scene and one for the set, with the card and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_verify import SIZE, SP_CONF, card  # noqa: E402

PLANES, OUTLIERS = (0.97, 0.98, 0.99, 0.995), (0.2, 0.5)
ESTIMATORS = ("ransac8", "lo-ransac", "degensac")
THR, ITERS, CONF = 1.0, 10000, 0.9999


def quality(masks, gts, onps):
    rec = [(m & g).sum() / g.sum() for m, g in zip(masks, gts)]
    out = [(m & ~g).sum() / max(1, (~g).sum()) for m, g in zip(masks, gts)]
    off = np.array([(m & g & ~o).sum() / max(1, (g & ~o).sum()) for m, g, o in zip(masks, gts, onps)])
    return {"recall_mean": round(float(np.mean(rec)), 4), "off_plane_recall_mean": round(float(off.mean()), 4),
            "off_plane_recall_min": round(float(off.min()), 4), "pairs_off_plane_below_0.9": int((off < 0.9).sum()),
            "outliers_kept_mean": round(float(np.mean(out)), 4)}


def plane_scenes(ctx, args):
    import cv2
    import torch

    from dim_b200 import _native
    from dim_b200.geometric_verification import gv_seed
    from test_gv_lo import scene

    N, B, P = args.n, args.batch, args.pairs
    for pl in PLANES:
        for of in OUTLIERS:
            data = [scene(2000 + k, n=N, plane=pl, out_frac=of) for k in range(P)]
            seeds = [gv_seed(0, k) for k in range(P)]
            k0 = torch.from_numpy(np.stack([d[0] for d in data])).cuda()
            k1 = torch.from_numpy(np.stack([d[1] for d in data])).cuda()
            f0 = [_native.FeatsDev(k0[k].data_ptr(), 0, 0, N, 0, 0, 0.0, 0.0, 0, 0, None) for k in range(P)]
            f1 = [_native.FeatsDev(k1[k].data_ptr(), 0, 0, N, 0, 0, 0.0, 0.0, 0, 0, None) for k in range(P)]
            m = torch.arange(N, device="cuda").view(1, N, 1).expand(B, N, 2).contiguous()
            nm = torch.full((B,), N, dtype=torch.int32, device="cuda")
            v = torch.zeros(P, N, 2, dtype=torch.int64, device="cuda")
            nv, ninl = torch.zeros(P, dtype=torch.int32, device="cuda"), torch.zeros(P, dtype=torch.int32, device="cuda")
            F, mask = torch.zeros(P, 9, device="cuda"), torch.zeros(P, N, dtype=torch.uint8, device="cuda")

            def run(est):
                for s in range(0, P, B):
                    ctx.gv_verify_dev(f0[s:s + B], f1[s:s + B], m.data_ptr(), nm.data_ptr(), N, seeds[s:s + B], THR, ITERS, 15, 0.2,
                                      v[s].data_ptr(), nv[s:].data_ptr(), F[s].data_ptr(), mask[s].data_ptr(), ninl[s:].data_ptr(),
                                      torch.cuda.current_stream().cuda_stream, est, CONF)

            for est in ESTIMATORS:  # warm-up: grows the scratch, loads the modules
                run(est)
            torch.cuda.synchronize()
            ms, res = {est: [] for est in ESTIMATORS}, {}
            for _ in range(args.reps):
                for est in ESTIMATORS:
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    ev[0].record()
                    run(est)
                    ev[1].record()
                    torch.cuda.synchronize()
                    ms[est].append(ev[0].elapsed_time(ev[1]))
                    res[est] = mask.cpu().numpy().astype(bool)
            gts, onps = [d[2] for d in data], [d[3] for d in data]
            line = {"bench": "gv_degensac", "scene": f"plane {pl}, {int(of * 100)}% out", **card(), "pairs": P, "n": N, "batch": B,
                    "reps": args.reps}
            for est in ESTIMATORS:
                med = float(np.median(ms[est]))
                hyp = [8192] * P if est == "ransac8" else \
                    [ctx.gv_estimate(d[0], d[1], THR, ITERS, seeds[k], est, CONF)[2] for k, d in enumerate(data)]
                line[est] = {"ms": [round(t, 3) for t in ms[est]], "pairs_per_s": round(P / (med / 1e3), 1),
                             "mean_hypotheses": round(float(np.mean(hyp)), 1), **quality(list(res[est]), gts, onps)}
            C = min(args.cv_pairs, P)
            for meth in ("USAC_ACCURATE", "USAC_MAGSAC"):
                t0 = time.perf_counter()
                cvm = []
                for d in data[:C]:
                    _, inl = cv2.findFundamentalMat(d[0], d[1], getattr(cv2, meth), THR, CONF, ITERS)
                    cvm.append(inl.ravel() > 0 if inl is not None else np.zeros(N, bool))
                line["cv2." + meth] = {"pairs": C, "pairs_per_s": round(C / (time.perf_counter() - t0), 1), **quality(cvm, gts[:C], onps[:C])}
            line["cv2_threads"] = cv2.getNumThreads()
            yield line


def image_set(ctx, args):
    import torch

    from dim_b200 import synthetic, weights
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher

    n = args.images
    imgs = []
    for k in range((n + 1) // 2):
        imgs += list(synthetic.synthetic_pair(7000 + k, SIZE))
    d_imgs = torch.from_numpy(np.stack(imgs[:n]).astype(np.float32)).cuda()
    ids, pairs = list(range(n)), pairs_from_bruteforce(list(range(n)))
    engs = {est: ImageSetMatcher(ctx, weights.superpoint_v1(), weights.lightglue_seeded(seed=0), n, SIZE, SIZE, SP_CONF, {}, batch_images=8,
                                 batch_pairs=32, verification={"threshold": THR, "max_iters": ITERS, "seed": 0, "estimator": est,
                                                               "confidence": CONF}) for est in ESTIMATORS}
    for eng in engs.values():
        eng.run_verified(d_imgs, ids, pairs)
    ms, out = {est: [] for est in ESTIMATORS}, {}
    for _ in range(args.reps):
        for est, eng in engs.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            torch.cuda.synchronize()
            ev[0].record()
            out[est] = eng.run_verified(d_imgs, ids, pairs)
            ev[1].record()
            torch.cuda.synchronize()
            ms[est].append(ev[0].elapsed_time(ev[1]))
    ninl = {est: np.array([r[3] for r in out[est]]) for est in ESTIMATORS}
    nver = {est: np.array([len(r[1]) for r in out[est]]) for est in ESTIMATORS}
    return {"bench": "gv_degensac", "workload": "bench_verify image set (SuperPoint 2048 kpts + seeded LightGlue, 1024x1024)", **card(),
            "images": n, "pairs": len(pairs), "batch_pairs": 32, "reps": args.reps,
            "run_verified_ms": {est: [round(t, 2) for t in ms[est]] for est in ESTIMATORS},
            "run_verified_ms_median": {est: round(float(np.median(ms[est])), 2) for est in ESTIMATORS},
            "mean_n_inliers": {est: float(ninl[est].mean()) for est in ESTIMATORS},
            "pairs_kept_by_gate": {est: int((nver[est] > 0).sum()) for est in ESTIMATORS}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256, help="pairs per plane scene")
    ap.add_argument("--n", type=int, default=2048, help="matches per pair")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each estimator")
    ap.add_argument("--cv-pairs", type=int, default=64, help="pairs per scene of the OpenCV arms")
    ap.add_argument("--images", type=int, default=24)
    ap.add_argument("--skip-image-set", action="store_true")
    ap.add_argument("--out", help="also append the JSON lines to this file")
    args = ap.parse_args()
    from dim_b200 import _native
    ctx = _native.Context.get(0)
    lines = plane_scenes(ctx, args)
    for line in (*lines, *([] if args.skip_image_set else [image_set(ctx, args)])):
        print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
