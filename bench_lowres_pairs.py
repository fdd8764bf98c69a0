"""Low-resolution pair generation ("matching_lowres", the reference's default pair strategy) on one GPU: the host
pairs_generator.pairs_from_lowres against ImageSetMatcher(pair_generation=...).lowres_pairs().

Two sets of 16 synthetic gray images (120 brute-force pairs each), resize_max 1000 and min_matches 20 as the reference's defaults:
  downsample  2048 x 1536, down-sampled to 1000 x 750 (dimb_resize_area_dev);
  enlarge     800 x 533, enlarged to 1000 x 666 (dimb_resize_area_linear_dev), as the reference does with its own test photos.
Each set is four scenes of a 16 px blocks image and three seeded homography warps of it, so that related and unrelated pairs mix.
Networks: SuperPoint (superpoint_v1, pairs_generator.SP_LOWRES_CONF) and seeded LightGlue weights (pairs_generator.LG_LOWRES_CONF).
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    cv2.resize(INTER_AREA) of every image on the host, then pairs_from_lowres(images=...): one batched SuperPoint call per
          image size, LightGlue over the pairs in batches of 16 through the host API (copies in and out around every call);
  device  the low-resolution pass of ImageSetMatcher.extract (device resize, batched SuperPoint into the float32 slot buffers) and
          lowres_pairs(): LightGlue per batch of batch_pairs on the device, one counts copy at the end.
A profiled device run gives the device times by kernel group.  Prints one JSON line per set.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_verify import card  # noqa: E402

SETS = {"downsample": (1536, 2048), "enlarge": (533, 800)}
RESIZE_MAX, MIN_MATCHES = 1000, 20
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 1024, "fix_sampling": True}


def scene(H, W, n):
    from dim_b200 import synthetic
    rgb = []
    for s in range(n // 4):
        a = synthetic.blocks_image(60 + s, max(H, W))[:H, :W]
        rgb += [a] + [synthetic.warp_pair(a, 60 + 4 * s + k, jitter=0.02 * max(H, W)) for k in range(1, 4)]
    return np.stack([synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in rgb]).astype(np.float32)


def run_set(ctx, name, H, W, n, batch_pairs, reps):
    import cv2
    import torch
    from pathlib import Path

    from dim_b200 import weights
    from dim_b200.pairs_generator import pairs_from_lowres
    from dim_b200.sharded import ImageSetMatcher
    w_sp, w_lg = weights.superpoint_v1(), weights.lightglue_seeded(seed=0)
    imgs = scene(H, W, n)
    ids = list(range(n))
    names = [Path(f"{k}.png") for k in ids]
    eng = ImageSetMatcher(ctx, w_sp, w_lg, n, H, W, SP_CONF, {}, batch_images=16, batch_pairs=batch_pairs,
                          pair_generation={"strategy": "matching_lowres", "resize_max": RESIZE_MAX, "min_matches": MIN_MATCHES})
    low = eng.lowres
    d_imgs = torch.from_numpy(imgs).cuda()

    def host():
        small = {p.name: cv2.resize(im, (low.w, low.h), interpolation=cv2.INTER_AREA) for p, im in zip(names, imgs)}
        pairs, counts = pairs_from_lowres(names, RESIZE_MAX, MIN_MATCHES, lightglue_weights=w_lg, superpoint_weights=w_sp, images=small,
                                          return_counts=True, device=ctx.device)
        return [(int(a.stem), int(b.stem)) for a, b in pairs], counts

    def device():
        st = torch.cuda.current_stream().cuda_stream
        for b0 in range(0, n, eng.B):  # the low-resolution pass of extract: one resize and its SuperPoint calls per batch
            batch = ids[b0:b0 + eng.B]
            low.extract(d_imgs[b0:b0 + len(batch)], batch, [eng.slots[i] for i in batch], st)
        return eng.lowres_pairs()

    arms = {"host": host, "device": device}
    out = {k: fn() for k, fn in arms.items()}  # warm-up
    secs = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out[k] = fn()
            torch.cuda.synchronize()
            secs[k].append(time.perf_counter() - t0)
    ctx.profile(True)
    launches = ctx.launches
    device()
    torch.cuda.synchronize()
    launches = ctx.launches - launches
    prof = ctx.profile_read()
    ctx.profile(False)
    med = {k: float(np.median(v)) for k, v in secs.items()}
    n_pairs = len(out["host"][1])
    group = lambda p: round(sum(v[0] for k, v in prof.items() if k.startswith(p)), 3)
    return {
        "metric": f"low-resolution pair generation (matching_lowres), {n} images {W}x{H} -> {low.w}x{low.h}: host cv2.resize + "
                  "pairs_from_lowres vs ImageSetMatcher(pair_generation=...) low-resolution extraction + lowres_pairs()",
        "set": name, **card(), "images": n, "pairs": n_pairs, "lowres_size": [low.w, low.h], "batch_pairs": batch_pairs, "reps": reps,
        "host_s": [round(s, 4) for s in secs["host"]], "device_s": [round(s, 4) for s in secs["device"]],
        "host_pairs_per_s": n_pairs / med["host"], "device_pairs_per_s": n_pairs / med["device"], "speedup": med["host"] / med["device"],
        "counts_identical": out["host"][1] == out["device"][1], "kept_identical": out["host"][0] == out["device"][0],
        "kept_pairs": len(out["device"][0]), "mean_count": float(np.mean(out["device"][1])), "launches_per_run": launches,
        "device_ms": {"tile.resize": group("tile.resize"), "lightglue": group("lg."), "superpoint": group("sp.")},
        "device_ms_by_group": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
        "data": "synthetic scenes under homography warps (planar), seeded LightGlue weights: timing only; correctness rests on "
                "tests/test_lowres_pairs.py"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--sets", default=",".join(SETS))
    args = ap.parse_args()
    from dim_b200 import _native
    ctx = _native.Context.get(0)
    for name in args.sets.split(","):
        print(json.dumps(run_set(ctx, name, *SETS[name], args.images, args.batch_pairs, args.reps)), flush=True)


if __name__ == "__main__":
    main()
