"""Tile preselection on one GPU: the reference's host PRESELECTION flow against ImageSetMatcher(tiling={"tile_selection":
"preselection", ...}).

n synthetic 2048 x 1536 gray images of one scene (a 16 px blocks image and seeded homography warps of it; default 6 -> 15
pairs), tile 512, overlap 64 (12 tiles per image, 144 candidate tile pairs per image pair), tile_preselection_size 1024, min_matches_per_tile 5,
SuperPoint 1024 keypoints per tile (nms 3, threshold 0.0005, fix_sampling) + seeded LightGlue; the preselection networks are
SuperPoint with tiling.SP_PRESELECTION_CONF and LightGlue with tiling.LG_PRESELECTION_CONF (the same seeded weights).
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    per image ExtractorBase._extract_by_tile + as_half_roundtrip; per pair tiling.preselection_matches (cv2 INTER_AREA, one
          SuperPoint call per image of the pair, one LightGlue call) + tiling.tile_selection (the Python box loop) +
          MatcherBase._match_by_tile on the selected tile pairs - on the same native networks,
  device  ImageSetMatcher(tiling=...).run: device resize, batched low-resolution SuperPoint once per image, batched LightGlue and box
          count per pair batch, one flags copy, then the tiled path.
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

H, W, TILE, OVERLAP, PRE_SIZE, K = 1536, 2048, 512, 64, 1024, 1024
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": K, "fix_sampling": True}


def scene(n):
    from dim_b200 import synthetic
    a = synthetic.blocks_image(40, W)[:H]  # 16 px blocks: they survive the 2x down-sampling of the preselection pass
    rgb = [a] + [synthetic.warp_pair(a, 40 + k, jitter=24.0) for k in range(1, n)]
    return np.stack([synthetic.to_gray_like_reference(x) for x in rgb]).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=6)
    ap.add_argument("--batch-pairs", type=int, default=160)
    ap.add_argument("--reps", type=int, default=2, help="alternating timed repetitions of each arm")
    args = ap.parse_args()
    import torch

    from dim_b200 import _native, tiling, weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher

    ctx = _native.Context.get(0)
    imgs = scene(args.images)
    n = len(imgs)
    ids = list(range(n))
    pairs = pairs_from_bruteforce(ids)
    general = {"tile_size": (TILE, TILE), "tile_overlap": OVERLAP}
    w_sp, w_lg = weights.superpoint_v1(), weights.lightglue_seeded(seed=0)
    ext = SuperPointExtractor(Config(general=general, extractor={**SP_CONF, "weights_dict": w_sp}))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", general=general, matcher={"weights_dict": w_lg}), "superpoint")
    sp_nets = {}

    def sp_pre(h, w):  # the reference builds its preselection networks once (matcher_base.py:143-159)
        if (h, w) not in sp_nets:
            sp_nets[h, w] = _native.SuperPointNet(ctx, w_sp, max_height=h, max_width=w, **tiling.SP_PRESELECTION_CONF)
        return sp_nets[h, w]
    lg_pre = _native.LightGlueNet(ctx, w_lg, max_kpts=4000, **tiling.LG_PRESELECTION_CONF)
    eng = ImageSetMatcher(ctx, w_sp, w_lg, n, H, W, SP_CONF, {}, batch_images=16, batch_pairs=args.batch_pairs,
                          tiling={**general, "tile_selection": "preselection", "tile_preselection_size": PRE_SIZE})
    d_imgs = torch.from_numpy(imgs).cuda()
    host_lists = []

    def host():
        feats = [as_half_roundtrip({**ext._extract_by_tile(im), "image_size": np.array([H, W])}) for im in imgs]
        host_lists.clear()
        out = []
        for i, j in pairs:
            kp0, kp1 = tiling.preselection_matches(imgs[i], imgs[j], PRE_SIZE, sp_pre, lg_pre)
            lst = tiling.tile_selection(imgs[i], imgs[j], "preselection", (TILE, TILE), OVERLAP, kp0=kp0, kp1=kp1)
            host_lists.append(lst)
            out.append(plugin._match_by_tile(feats[i], feats[j], lst))
        return out

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
    dev_lists = eng._preselect(pairs)
    same_lists = sum(a == b for a, b in zip(host_lists, dev_lists))
    same_tables = sum(np.array_equal(a, b) for a, b in zip(out["host"], out["device"]))

    ctx.profile(True)
    device()
    torch.cuda.synchronize()
    prof = ctx.profile_read()
    ctx.profile(False)
    med = {k: float(np.median(v)) for k, v in secs.items()}
    print(json.dumps({
        "metric": "tiled image-set matching with PRESELECTION, 2048x1536 images, tile 512 / overlap 64, tile_preselection_size 1024: "
                  "host preselection_matches + tile_selection + _match_by_tile vs ImageSetMatcher(tiling={... preselection ...}).run",
        **card(), "images": n, "pairs": len(pairs), "tiles_per_image": eng.T, "batch_pairs": args.batch_pairs, "reps": args.reps,
        "host_s": [round(s, 4) for s in secs["host"]], "device_s": [round(s, 4) for s in secs["device"]],
        "host_pairs_per_s": len(pairs) / med["host"], "device_pairs_per_s": len(pairs) / med["device"],
        "speedup": med["host"] / med["device"], "lists_identical": f"{same_lists}/{len(pairs)}",
        "tables_identical": f"{same_tables}/{len(pairs)}", "mean_selected_tile_pairs": float(np.mean([len(lst) for lst in dev_lists])),
        "candidate_tile_pairs": eng.T * eng.T, "mean_matches": float(np.mean([len(t) for t in out["device"]])),
        "tile_device_ms_launches": {k: [round(v[0], 3), int(v[1])] for k, v in sorted(prof.items()) if k.startswith("tile.")},
        "device_ms_by_group": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
        "data": "synthetic, one scene under homography warps (planar): timing only; correctness rests on tests/test_preselection.py"}))


if __name__ == "__main__":
    main()
