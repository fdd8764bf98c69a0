"""SuperGlue over an image set on one GPU: the per-pair plugin path against the batched device engine.

n synthetic 1024 x 1024 images (default 24 -> 276 pairs) go through SuperPoint with cfg2's configuration (2048 keypoints) into the
device feature store; then every pair is matched with SuperGlue twice:
  (a) SuperGlueMatcher._match_pairs per pair on store.get features (one host round trip per pair),
  (b) sharded.ImageSetMatcher(matcher="superglue"): dimb_sg_match_dev on batches of store slots.
Both arms are timed with CUDA events after a warm-up of every shape; the per-group device times of dimb_ctx_profile come from a
separate run.  Weights: seeded (oracle.superglue.seeded_weights), or the trained checkpoint named by DIMB_SUPERGLUE_WEIGHTS; SuperGlue
has no early exit, so its cost does not depend on the weights.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--batch-pairs", type=int, default=32, help="pairs per dimb_sg_match_dev call in arm (b)")
    ap.add_argument("--profile-pairs", type=int, default=32, help="pairs of arm (a) in the profiled run")
    args = ap.parse_args()
    import torch

    from dim_b200 import _native, synthetic, weights
    from dim_b200.config import Config
    from dim_b200.matchers.superglue import SuperGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    from oracle import superglue as o_sg

    path = os.environ.get("DIMB_SUPERGLUE_WEIGHTS")
    if path:
        w = weights.load_npz(path) if path.endswith(".npz") else weights.from_torch_checkpoint(path)
    else:
        w = o_sg.seeded_weights(0)
    n = args.images
    ctx = _native.Context.get(0)
    sg_conf = {"sinkhorn_iterations": 100, "match_threshold": 0.2, "gnn_layers": ("self", "cross") * 9}
    eng = ImageSetMatcher(ctx, weights.superpoint_v1(), w, n, SIZE, SIZE, SP_CONF, sg_conf, batch_images=8, batch_pairs=args.batch_pairs,
                          matcher="superglue")
    imgs = []
    for k in range((n + 1) // 2):
        imgs += list(synthetic.synthetic_pair(7000 + k, SIZE))
    eng.extract(torch.from_numpy(np.stack(imgs[:n]).astype(np.float32)).cuda(), list(range(n)))
    torch.cuda.synchronize()
    pairs = pairs_from_bruteforce(list(range(n)))
    ids = list(range(len(pairs)))
    feats = [eng.store.get(i) for i in range(n)]  # what get_features hands the plugin (features.h5 values)
    plugin = SuperGlueMatcher(Config(matcher={"name": "superglue", "weights_dict": w}))

    def arm_a(sel):
        return {k: plugin._match_pairs(feats[pairs[k][0]], feats[pairs[k][1]]) for k in sel}

    def arm_b():
        return eng.match(pairs, ids)

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1])

    # warm-up of every shape: one plugin pair (its handle is sized at the first call), a full and the last partial batch of (b)
    arm_a([0])
    tail = len(pairs) % args.batch_pairs or args.batch_pairs
    eng.match(pairs[:args.batch_pairs], ids[:args.batch_pairs])
    eng.match(pairs[-tail:], ids[-tail:])
    torch.cuda.synchronize()

    l0 = ctx.launches
    res_b, ms_b = timed(arm_b)
    launches_b = ctx.launches - l0
    l0 = ctx.launches
    res_a, ms_a = timed(lambda: arm_a(ids))
    launches_a = ctx.launches - l0
    same = sum(np.array_equal(res_a[k], res_b[k]) for k in ids)

    def profiled(fn):
        ctx.profile(True)
        fn()
        torch.cuda.synchronize()
        prof = ctx.profile_read()
        ctx.profile(False)
        return {k: [round(v[0], 3), int(v[1])] for k, v in sorted(prof.items())}

    prof_b = profiled(arm_b)
    prof_a = profiled(lambda: arm_a(ids[:args.profile_pairs]))
    print(json.dumps({
        "metric": "SuperGlue image-pairs/sec over an image set (SuperPoint 2048 kpts, 1024x1024, 100 Sinkhorn iterations)",
        **card(), "images": n, "pairs": len(pairs), "batch_pairs": args.batch_pairs,
        "weights": "checkpoint" if path else "seeded",
        "arm_a_plugin_per_pair": {"pairs_per_s": len(pairs) / (ms_a / 1e3), "ms": round(ms_a, 2), "gpu_launches": launches_a},
        "arm_b_batched_device": {"pairs_per_s": len(pairs) / (ms_b / 1e3), "ms": round(ms_b, 2), "gpu_launches": launches_b},
        "speedup_b_over_a": ms_a / ms_b,
        "tables_identical": f"{same}/{len(pairs)}", "total_matches": int(sum(len(res_b[k]) for k in ids)),
        "profile_arm_b_all_pairs_ms_launches": prof_b,
        f"profile_arm_a_first_{min(args.profile_pairs, len(pairs))}_pairs_ms_launches": prof_a,
        "data": "synthetic", "dtype": "f16 hi/lo split x3 MMA, f32 accumulate"}))


if __name__ == "__main__":
    main()
