"""upright over an image set on one GPU: the reference's host flow against ImageSetMatcher(upright=...).

Sizes are height x width throughout.  The set: 16 gray 2048 x 1536 images, 4 scenes of ``synthetic.blocks_image`` and 3
``synthetic.warp_pair`` warps of each, every image then turned by a seeded rotation in (0, 90, 180, 270), so the set mixes 2048 x 1536
and 1536 x 2048.  All 120 pairs, SuperPoint (2048 keypoints) + LightGlue with seeded weights; the search at resize_max 640 with 2048
keypoints.  With seeded LightGlue weights the rotations the search picks say nothing about accuracy: this measures equality and time
only (correctness against the host statement rests on tests/test_upright.py).

Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    upright.upright_rotations (plugin _extract / _match_pairs per decision and rotation), cv2.rotate of every full-size image,
          the plugin's _extract, the float16 round trip of features.h5, LightGlue through the host API per pair batch
          (LightGlueMatcher.match_many), upright.rotate_back_keypoints and FeatureStoreDev.put of every image;
  upright ImageSetMatcher(upright=...).run on the unrotated images (a list of per-image device tensors);
  turned  the same engine without upright, run on the images already turned by the rotations the search picked: the search's cost
          is the difference.
Reports pairs/s of every arm, whether rotations, per-decision counts, tables and stored features are identical between the host and
upright arms, launches per run, and from separate profiled runs the tile.rot device time of the upright run and the sp.* / lg.* device
time of the search alone.  Prints one JSON line.
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
UP = {"resize_max": 640, "max_keypoints": 2048}
SIZE = (2048, 1536)


def image_set(n, seed=130):
    """n // 4 scenes of one blocks image each, the scene and 3 warps of it, every image turned by a seeded rotation (gray float32)."""
    from dim_b200 import synthetic
    from dim_b200.upright import ROTATIONS, rotate_image
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n // 4):
        big = synthetic.blocks_image(seed + s, max(SIZE))
        base = np.ascontiguousarray(big[:SIZE[0], :SIZE[1]])
        for k in range(4):
            rgb = base if k == 0 else synthetic.warp_pair(base, seed + 10 * s + k, jitter=0.02 * max(SIZE))
            gray = synthetic.to_gray_like_reference(np.ascontiguousarray(rgb)).astype(np.float32)
            out.append(np.ascontiguousarray(rotate_image(gray, ROTATIONS[int(rng.integers(4))])))
    return out


def run(ctx, n, batch_images, batch_pairs, reps):
    import torch

    from dim_b200 import _native, weights
    from dim_b200.config import Config
    from dim_b200.extractors.superpoint import SuperPointExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher
    from dim_b200.upright import rotate_back_keypoints, rotate_image, search_plugins, upright_rotations
    w_sp, w_lg = weights.superpoint_v1(), weights.lightglue_seeded(seed=0)
    imgs = image_set(n)
    pairs, ids = pairs_from_bruteforce(list(range(n))), list(range(n))
    ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={**SP_CONF, "weights_dict": w_sp}))
    plugin = LightGlueMatcher(Config(pipeline="superpoint+lightglue", matcher={"weights_dict": w_lg}), local_features="superpoint")
    plugins = search_plugins(UP["max_keypoints"], False, w_lg, w_sp, ctx.device)
    host_store = _native.FeatureStoreDev(ctx, n, SP_CONF["max_keypoints"], 256)
    kw = {"batch_images": batch_images, "batch_pairs": batch_pairs}
    hs, ws = [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]
    up = ImageSetMatcher(ctx, w_sp, w_lg, n, hs, ws, SP_CONF, {}, upright=UP, **kw)
    d_imgs = [torch.from_numpy(x).cuda() for x in imgs]
    out = {}

    def host():
        rot, counts = upright_rotations(imgs, pairs, UP["resize_max"], UP["max_keypoints"], plugins=plugins)
        feats = []
        for im, r in zip(imgs, rot):
            turned = rotate_image(im, r)
            feats.append(as_half_roundtrip({**ext._extract(turned), "image_size": np.array(turned.shape[:2])}))
        tables = []
        for b0 in range(0, len(pairs), batch_pairs):
            tables += plugin.match_many([(feats[i], feats[j]) for i, j in pairs[b0:b0 + batch_pairs]])
        for i, (im, r) in enumerate(zip(imgs, rot)):
            host_store.put(i, {**feats[i], "keypoints": rotate_back_keypoints(feats[i]["keypoints"], r, *im.shape),
                               "image_size": np.array(im.shape[:2])})
        out["host"] = (rot, counts, tables)

    def run_up():
        out["upright"] = up.run(d_imgs, ids, pairs)

    host()  # the rotations fix the turned arm's sizes
    rot = out["host"][0]
    turned_imgs = [np.ascontiguousarray(rotate_image(im, r)) for im, r in zip(imgs, rot)]
    turned = ImageSetMatcher(ctx, w_sp, w_lg, n, [t.shape[0] for t in turned_imgs], [t.shape[1] for t in turned_imgs], SP_CONF, {}, **kw)
    d_turned = [torch.from_numpy(x).cuda() for x in turned_imgs]

    def run_turned():
        out["turned"] = turned.run(d_turned, ids, pairs)

    arms = {"host": host, "upright": run_up, "turned": run_turned}
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
    h_rot, h_counts, h_tables = out["host"]
    same = lambda a, b: len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))  # noqa: E731
    features_identical = all(all(np.array_equal(up.store.get(i)[k], host_store.get(i)[k]) for k in ("keypoints", "descriptors", "scores",
                                                                                                      "image_size")) for i in ids)
    u_rot, u_counts = up.upright(d_imgs, ids, pairs)  # the search alone, profiled below; then the run again for the launch count
    prof, launches = {}, {}
    for k, fn in (("search", lambda: up.upright(d_imgs, ids, pairs)), ("upright", run_up), ("turned", run_turned)):
        ctx.profile(True)
        n0 = ctx.launches
        fn()
        torch.cuda.synchronize()
        launches[k] = ctx.launches - n0
        prof[k] = ctx.profile_read()
        ctx.profile(False)
    med = {k: float(np.median(v)) for k, v in secs.items()}
    group = lambda p, k: round(sum(v[0] for g, v in prof[k].items() if g.startswith(p)), 3)  # noqa: E731
    px = sum(im.size for im in imgs)
    rot_ms = group("tile.rot", "upright")
    return {
        "metric": f"upright over {n} gray images ({SIZE[0]} x {SIZE[1]} turned by seeded rotations), {len(pairs)} pairs, SuperPoint "
                  f"{SP_CONF['max_keypoints']} + LightGlue, search resize_max {UP['resize_max']} / {UP['max_keypoints']} keypoints: host flow "
                  "vs ImageSetMatcher(upright=...) vs the engine on the already-turned images",
        **card(), "images": n, "pairs": len(pairs), "rotations": list(h_rot), "batch_images": batch_images, "batch_pairs": batch_pairs,
        "reps": reps, **{f"{k}_s": [round(s, 4) for s in v] for k, v in secs.items()},
        **{f"{k}_pairs_per_s": len(pairs) / med[k] for k in arms}, "upright_speedup_vs_host": med["host"] / med["upright"],
        "search_overhead_s": med["upright"] - med["turned"],
        "rotations_identical": list(u_rot) == list(h_rot) and up.rotations == list(h_rot),
        "counts_identical": {k: list(v) for k, v in u_counts.items()} == {k: list(v) for k, v in h_counts.items()},
        "tables_identical": same(out["upright"], h_tables), "turned_tables_identical": same(out["turned"], h_tables),
        "features_identical": bool(features_identical), "matches_total": int(sum(len(t) for t in out["upright"])),
        "launches_per_run": launches,
        "device_ms": {"tile_rot_upright_run": rot_ms, "search_sp": group("sp.", "search"), "search_lg": group("lg.", "search"),
                      "search_tile_rot": group("tile.rot", "search"), "upright_sp": group("sp.", "upright"), "upright_lg": group("lg.", "upright"),
                      "turned_sp": group("sp.", "turned"), "turned_lg": group("lg.", "turned")},
        # tile.rot of the run less that of the search alone: the full-size turns (2 * px * 4 bytes moved) and the one back-rotation
        # launch (a few hundred KB), so the rate below slightly understates the turn kernel's
        "full_size_turn_bytes": 2 * px * 4, "full_size_turn_ms": round(rot_ms - group("tile.rot", "search"), 4),
        "full_size_turn_TB_per_s": 2 * px * 4 / max(rot_ms - group("tile.rot", "search"), 1e-6) / 1e9,
        "data": "synthetic scenes under homography warps with seeded LightGlue weights: equality and time only, not accuracy"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-images", type=int, default=4)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    args = ap.parse_args()
    from dim_b200 import _native
    print(json.dumps(run(_native.Context.get(0), args.images, args.batch_images, args.batch_pairs, args.reps)), flush=True)


if __name__ == "__main__":
    main()
