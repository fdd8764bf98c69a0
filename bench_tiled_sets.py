"""Tiled matching of an image set on one GPU: the reference's host tiling flow against ImageSetMatcher(tiling=...).

n synthetic 2048 x 1536 images of one scene (a blocks image and seeded homography warps of it; default 6 -> 15 pairs), tile 1024,
overlap 128 (4 tiles per image), grid selection (4 tile pairs per image pair), in two configurations:
  superpoint  SuperPoint 2048 keypoints per tile (nms 3, threshold 0.0005, fix_sampling) + seeded LightGlue,
  aliked      ALIKED-n16rot 4096 keypoints per tile (threshold 0.2, nms 3, BASELINE cfg3) + seeded LightGlue (input_dim 128).
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    ExtractorBase._extract_by_tile per image, as_half_roundtrip (the features.h5 round trip), MatcherBase._match_by_tile per
          pair - one batch-1 native call per tile and per tile pair, host np.vstack / np.unique - on the same native networks,
  device  ImageSetMatcher(tiling=...).run: device tile cut, batched extraction, tile merge, views, batched matching, match merge.
A profiled device run gives the tile.* device times.  Prints one JSON line.
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

H, W, TILE, OVERLAP = 1536, 2048, 1024, 128
CONFIGS = {
    "superpoint": {"K": 2048, "conf": {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048, "fix_sampling": True}},
    "aliked": {"K": 4096, "conf": {"max_num_keypoints": 4096, "detection_threshold": 0.2, "nms_radius": 3}},
}


def scene(n):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(300, W, 4)[:H]
    return [a] + [synthetic.warp_pair(a, 300 + k, jitter=48.0) for k in range(1, n)]


def run_config(name, rgb, args, ctx):
    import torch

    from dim_b200 import synthetic, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher, tile_pairs_for

    cfg = CONFIGS[name]
    n = len(rgb)
    ids = list(range(n))
    pairs = pairs_from_bruteforce(ids)
    general = {"tile_size": (TILE, TILE), "tile_overlap": OVERLAP}
    if name == "superpoint":
        imgs = np.stack([synthetic.to_gray_like_reference(x) for x in rgb]).astype(np.float32)
        w_ex, w_lg = weights.superpoint_v1(), weights.lightglue_seeded(seed=0)
        ext = SuperPointExtractor(Config(general=general, extractor={**cfg["conf"], "weights_dict": w_ex}))
        plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", general=general, matcher={"weights_dict": w_lg}), "superpoint")
    else:
        imgs = np.stack(rgb).astype(np.float32)
        w_ex, w_lg = weights.aliked_n16rot(), weights.lightglue_seeded(input_dim=128, seed=0)
        ext = AlikedExtractor(Config(general=general, extractor={"model_name": "aliked-n16rot", **cfg["conf"], "weights_dict": w_ex}))
        plugin = LightGlueMatcher(Config(pipeline="aliked+lightglue", general=general, matcher={"weights_dict": w_lg}), "aliked")
    eng = ImageSetMatcher(ctx, w_ex, w_lg, n, H, W, cfg["conf"], {}, batch_images=16, batch_pairs=args.batch_pairs, extractor=name,
                          tiling={**general, "tile_selection": "grid"})
    grid = tile_pairs_for("grid", eng.T)
    d_imgs = torch.from_numpy(imgs).cuda()

    def host():
        feats = [as_half_roundtrip({**ext._extract_by_tile(im), "image_size": np.array([H, W])}) for im in imgs]
        return [plugin._match_by_tile(feats[i], feats[j], grid) for i, j in pairs]

    def device():
        return eng.run(d_imgs, ids, pairs)

    arms = {"host": host, "device": device}
    out = {k: fn() for k, fn in arms.items()}  # warm-up
    secs = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out[k] = fn()
            torch.cuda.synchronize()
            secs[k].append(time.perf_counter() - t0)
    same = sum(np.array_equal(a, b) for a, b in zip(out["host"], out["device"]))

    ctx.profile(True)
    l0 = ctx.launches
    device()
    torch.cuda.synchronize()
    launches = ctx.launches - l0
    prof = ctx.profile_read()
    ctx.profile(False)
    merged = [eng.store.count(i)[0] for i in ids]
    concat = [len(ext._extract_by_tile(im, select_unique=False)["keypoints"]) for im in imgs]
    med = {k: float(np.median(v)) for k, v in secs.items()}
    return {
        "tiles_per_image": eng.T, "keypoints_per_tile": cfg["K"], "pairs": len(pairs), "tile_pairs": len(pairs) * len(grid),
        "host_s": [round(s, 4) for s in secs["host"]], "device_s": [round(s, 4) for s in secs["device"]],
        "host_pairs_per_s": len(pairs) / med["host"], "device_pairs_per_s": len(pairs) / med["device"],
        "speedup": med["host"] / med["device"], "tables_identical": f"{same}/{len(pairs)}",
        "mean_matches": float(np.mean([len(t) for t in out["device"]])),
        "merged_keypoints": merged, "duplicates_removed": [c - m for c, m in zip(concat, merged)],
        "tile_device_ms_launches": {k: [round(v[0], 3), int(v[1])] for k, v in sorted(prof.items()) if k.startswith("tile.")},
        "device_ms_by_group": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
        "gpu_launches_device_run": launches,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=6)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--configs", default="superpoint,aliked")
    args = ap.parse_args()
    from dim_b200 import _native

    ctx = _native.Context.get(0)
    rgb = scene(args.images)
    res = {name: run_config(name, rgb, args, ctx) for name in args.configs.split(",")}
    print(json.dumps({
        "metric": "tiled image-set matching, 2048x1536 images, tile 1024 / overlap 128, grid selection: host _extract_by_tile + "
                  "_match_by_tile vs ImageSetMatcher(tiling=...)",
        **card(), "images": args.images, "batch_pairs": args.batch_pairs, "reps": args.reps, **res,
        "data": "synthetic, one scene under homography warps (planar): timing only; correctness rests on tests/test_tiled_sets.py"}))


if __name__ == "__main__":
    main()
