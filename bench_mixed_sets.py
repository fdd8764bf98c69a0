"""Image sets of mixed sizes on one GPU: the reference's host flow against ImageSetMatcher on a set of landscape and portrait images.

Sizes are height x width throughout.  The set: 16 gray images, 8 landscape 1536 x 2048 and 8 portrait 2048 x 1536, crops of one larger blocks scene at different offsets,
each under a seeded homography warp (synthetic.warp_pair), so that every pair shares content.  All 120 pairs, SuperPoint (2048
keypoints) + LightGlue with seeded weights.  ``--tiled``: grid tiling, tile 1024 / overlap 128 (4 tiles per image of either shape).
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host     per image the plugin's _extract (_extract_by_tile), the float16 round trip of features.h5, then per pair the plugin's
           _match_pairs (_match_by_tile with tiling.tile_selection's grid list);
  mixed    ImageSetMatcher(height=[...], width=[...]).run on the mixed set (a list of per-image device tensors);
  uniform  ImageSetMatcher.run on 16 landscape 1536 x 2048 images (the same pixel count): the cost of mixing.
Reports pairs/s of every arm, whether the host and mixed tables are identical, launches per run and the sp.* / lg.* device times of
one profiled run of each device arm.  Prints one JSON line per configuration.
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

SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048}
LAND, PORT = (1536, 2048), (2048, 1536)


def scene(sizes, seed=120):
    """Crops of one blocks scene at offsets of 32 px per image, each warped, as gray float32 arrays."""
    from dim_b200 import synthetic
    big = synthetic.blocks_image(seed, max(max(s) for s in sizes) + 32 * len(sizes))
    out = []
    for k, (H, W) in enumerate(sizes):
        crop = np.ascontiguousarray(big[32 * k:32 * k + H, 32 * k:32 * k + W])
        warped = synthetic.warp_pair(crop, seed + k, jitter=0.02 * max(H, W))
        out.append(synthetic.to_gray_like_reference(np.ascontiguousarray(warped)).astype(np.float32))
    return out


def run_config(ctx, tiled, n, batch_images, batch_pairs, reps):
    import torch

    from dim_b200 import tiling, weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    w_sp, w_lg = weights.superpoint_v1(), weights.lightglue_seeded(seed=0)
    sizes = [LAND] * (n // 2) + [PORT] * (n - n // 2)
    sizes = [sizes[k // 2 + (k % 2) * (n // 2)] for k in range(n)]  # alternate landscape and portrait
    imgs = scene(sizes)
    flat = scene([LAND] * n, 121)
    pairs = pairs_from_bruteforce(list(range(n)))
    ids = list(range(n))
    sp_conf = {**SP_CONF, "fix_sampling": True} if tiled else SP_CONF
    tconf = {"tile_size": 1024, "tile_overlap": 128, "tile_selection": "grid"} if tiled else None
    general = {"general": {"tile_size": 1024, "tile_overlap": 128}} if tiled else {}
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={**sp_conf, "weights_dict": w_sp}, **general))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w_lg}), local_features="superpoint")
    kw = {"batch_images": batch_images, "batch_pairs": batch_pairs, "tiling": tconf}
    mixed = ImageSetMatcher(ctx, w_sp, w_lg, n, [h for h, _ in sizes], [w for _, w in sizes], sp_conf, {}, **kw)
    uniform = ImageSetMatcher(ctx, w_sp, w_lg, n, *LAND, sp_conf, {}, **kw)
    d_mixed = [torch.from_numpy(x).cuda() for x in imgs]
    d_flat = torch.from_numpy(np.stack(flat)).cuda()
    lists = [tiling.tile_selection(imgs[i], imgs[j], "grid", 1024, 128) for i, j in pairs] if tiled else None
    out = {}

    def host():
        feats = []
        for img in imgs:
            f = ext._extract_by_tile(img) if tiled else ext._extract(img)
            feats.append(as_half_roundtrip({**f, "image_size": np.array(img.shape[:2])}))
        if tiled:
            out["host"] = [plugin._match_by_tile(feats[i], feats[j], lst) for (i, j), lst in zip(pairs, lists)]
        else:
            out["host"] = [plugin._match_pairs(feats[i], feats[j]) for i, j in pairs]

    def run_mixed():
        out["mixed"] = mixed.run(d_mixed, ids, pairs)

    def run_uniform():
        out["uniform"] = uniform.run(d_flat, ids, pairs)

    arms = {"host": host, "mixed": run_mixed, "uniform": run_uniform}
    for fn in arms.values():  # warm-up
        fn()
    secs = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            secs[k].append(time.perf_counter() - t0)
    identical = len(out["host"]) == len(out["mixed"]) and all(np.array_equal(a, b) for a, b in zip(out["host"], out["mixed"]))
    prof, launches = {}, {}
    for k in ("mixed", "uniform"):
        ctx.profile(True)
        n0 = ctx.launches
        arms[k]()
        torch.cuda.synchronize()
        launches[k] = ctx.launches - n0
        prof[k] = ctx.profile_read()
        ctx.profile(False)
    med = {k: float(np.median(v)) for k, v in secs.items()}
    group = lambda p, k: round(sum(v[0] for g, v in prof[k].items() if g.startswith(p)), 3)
    return {
        "metric": f"{len(pairs)} pairs over {n} gray images (H x W: {n // 2} landscape {LAND[0]} x {LAND[1]}, {n - n // 2} portrait "
                  f"{PORT[0]} x {PORT[1]}), SuperPoint {SP_CONF['max_keypoints']} + LightGlue{', grid tiles 1024 / overlap 128' if tiled else ''}: "
                  "host plugin flow vs ImageSetMatcher on the mixed set vs on 16 landscape images",
        "config": "tiled" if tiled else "untiled", **card(), "images": n, "pairs": len(pairs), "batch_images": batch_images,
        "batch_pairs": batch_pairs, "reps": reps, **{f"{k}_s": [round(s, 4) for s in v] for k, v in secs.items()},
        **{f"{k}_pairs_per_s": len(pairs) / med[k] for k in arms}, "mixed_speedup_vs_host": med["host"] / med["mixed"],
        "mixing_cost": med["mixed"] / med["uniform"], "tables_identical": bool(identical),
        "matches_total": int(sum(len(t) for t in out["mixed"])), "launches_per_run": launches,
        "device_ms": {k: {"sp": group("sp.", k), "lg": group("lg.", k)} for k in prof},
        "data": "synthetic scenes under homography warps (planar): timing only; correctness rests on tests/test_mixed_sets.py"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-images", type=int, default=4)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--tiled", action="store_true", help="grid tiling, tile 1024 / overlap 128")
    args = ap.parse_args()
    from dim_b200 import _native
    ctx = _native.Context.get(0)
    print(json.dumps(run_config(ctx, args.tiled, args.images, args.batch_images, args.batch_pairs, args.reps)), flush=True)


if __name__ == "__main__":
    main()
