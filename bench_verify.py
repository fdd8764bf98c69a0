"""Verified matching of an image set on one GPU: ImageSetMatcher.run against run_verified, and the device verification against
OpenCV on the host.

n synthetic 1024 x 1024 images (default 24 -> 276 pairs) go through SuperPoint with cfg2's configuration (2048 keypoints) into the
device feature store and every pair is matched with seeded LightGlue out of it.  Timed, with CUDA events after a warm-up and in
alternating repetitions:
  run           extract -> match -> tables to the host (no verification),
  run_verified  the same plus dimb_gv_verify_dev on every pair batch (fundamental-matrix RANSAC, ordered inlier compaction, gate).
A profiled run_verified gives the per-group device times (``gv.*`` is the verification alone).  The host arm runs
cv2.findFundamentalMat(RANSAC) per pair on the same raw tables and keypoints, which is what the reference does per pair.
synthetic_pair warps by a homography, so the scenes are planar: the numbers are timings, not a test of the estimator (the tests
check correctness).  Prints one JSON line.
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

SIZE, KPTS = 1024, 2048
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": KPTS}  # cfg2 (config.py:93-99)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "clocks_max_sm": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=24)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--host-pairs", type=int, default=0, help="pairs of the OpenCV arm (0: all)")
    args = ap.parse_args()
    import torch

    from dim_b200 import _native, synthetic, weights
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, store_slot

    n = args.images
    ctx = _native.Context.get(0)
    verification = {"method": "pydegensac", "threshold": 1.0, "max_iters": 10000, "seed": 0}
    eng = ImageSetMatcher(ctx, weights.superpoint_v1(), weights.lightglue_seeded(seed=0), n, SIZE, SIZE, SP_CONF, {}, batch_images=8,
                          batch_pairs=args.batch_pairs, verification=verification)
    imgs = []
    for k in range((n + 1) // 2):
        imgs += list(synthetic.synthetic_pair(7000 + k, SIZE))
    d_imgs = torch.from_numpy(np.stack(imgs[:n]).astype(np.float32)).cuda()
    ids = list(range(n))
    pairs = pairs_from_bruteforce(ids)

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        l0 = ctx.launches
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1]), ctx.launches - l0

    arms = {"run": lambda: eng.run(d_imgs, ids, pairs), "run_verified": lambda: eng.run_verified(d_imgs, ids, pairs)}
    for fn in arms.values():  # warm-up: every batch shape of both arms
        fn()
    ms = {k: [] for k in arms}
    launches, out = {}, {}
    for _ in range(args.reps):
        for k, fn in arms.items():
            out[k], t, launches[k] = timed(fn)
            ms[k].append(t)
    raw_same = sum(np.array_equal(a, r[0]) for a, r in zip(out["run"], out["run_verified"]))

    ctx.profile(True)
    arms["run_verified"]()
    torch.cuda.synchronize()
    prof = {k: [round(v[0], 3), int(v[1])] for k, v in sorted(ctx.profile_read().items())}
    ctx.profile(False)
    gv_ms = sum(v[0] for k, v in prof.items() if k.startswith("gv."))

    res = out["run_verified"]
    n_raw = np.array([len(r[0]) for r in res])
    n_inl = np.array([r[3] for r in res])
    kept = sum(len(r[1]) > 0 for r in res)

    # host arm: OpenCV RANSAC per pair on the same matches (features.h5 values of the store)
    import cv2
    feats = [eng.store.get(store_slot(i, n, 1))["keypoints"] for i in range(n)]
    sel = [k for k in range(len(pairs)) if n_raw[k] >= 8][:args.host_pairs or None]
    t0 = time.perf_counter()
    cv_inl, cv_err = [], 0
    for k in sel:
        (i, j), m = pairs[k], res[k][0]
        try:
            _, inl = cv2.findFundamentalMat(feats[i][m[:, 0]], feats[j][m[:, 1]], cv2.RANSAC, 1.0, 0.9999, 10000)
        except cv2.error:  # OpenCV rejects some degenerate (e.g. all-coincident) point sets by raising
            cv_err += 1
            inl = None
        cv_inl.append(int(inl.sum()) if inl is not None else 0)
    host_s = time.perf_counter() - t0

    med = {k: float(np.median(v)) for k, v in ms.items()}
    print(json.dumps({
        "metric": "verified image-set matching (SuperPoint 2048 kpts + seeded LightGlue, 1024x1024, F-RANSAC 8192 hypotheses/pair)",
        **card(), "images": n, "pairs": len(pairs), "batch_pairs": args.batch_pairs, "reps": args.reps,
        "run_ms": [round(t, 2) for t in ms["run"]], "run_verified_ms": [round(t, 2) for t in ms["run_verified"]],
        "run_ms_median": round(med["run"], 2), "run_verified_ms_median": round(med["run_verified"], 2),
        "verification_overhead_ms": round(med["run_verified"] - med["run"], 2),
        "gpu_launches": {"run": launches["run"], "run_verified": launches["run_verified"]},
        "profile_run_verified_ms_launches": prof,
        "gv_device_ms": round(gv_ms, 3), "gv_verified_pairs_per_s": len(pairs) / (gv_ms / 1e3) if gv_ms > 0 else None,
        "mean_raw_matches": float(n_raw.mean()), "mean_inliers": float(n_inl.mean()), "pairs_kept_by_gate": int(kept),
        "raw_tables_equal_run": f"{raw_same}/{len(pairs)}",
        "host_opencv_ransac": {"pairs": len(sel), "s": round(host_s, 3), "pairs_per_s": len(sel) / host_s if host_s > 0 else None,
                               "mean_inliers": float(np.mean(cv_inl)) if cv_inl else None, "cv2_errors": cv_err,
                               "cv2_threads": cv2.getNumThreads(),
                               "host_cpus": os.cpu_count()},
        "data": "synthetic, homography-warped (planar scenes): timing only; correctness rests on tests/test_verify_sets.py"}))


if __name__ == "__main__":
    main()
