"""The low-resolution passes of an ALIKED image set on one GPU: pair generation ("matching_lowres"), tile preselection and upright,
each as the host flow on gray_from_rgb images against ImageSetMatcher(extractor="aliked", ...).

Sizes are height x width.  The set is cfg3's geometry: 16 RGB 1536 x 2048 images (4 scenes of ``synthetic.blocks_image`` and 3
``synthetic.warp_pair`` warps of each), ALIKED n16rot with 4096 keypoints per tile, tiles 1024 / overlap 128 (4 tiles per image),
LightGlue input_dim 128, all 120 pairs.  The low-resolution passes run superpoint_v1 and seeded SuperPoint-LightGlue weights
(``weights.lightglue_seeded``, as bench_lowres_pairs.py uses), so what they pick says nothing about accuracy: this measures equality
and time.  Modes, one JSON line each:
  lowres        matching_lowres at resize_max 1000 (1536 x 2048 -> 750 x 1000), min_matches 20, then the grid tile pairs of the kept
                pairs;
  preselection  tile_selection "preselection" at tile_preselection_size 1024;
  upright       the search at resize_max 640 / 2048 keypoints on the images turned by seeded rotations, then the grid tile pairs.
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    gray_from_rgb and the host flow of the pass: cv2.resize + pairs_from_lowres(images=...), tiling.preselection_matches +
          tiling.tile_selection per pair, or upright.upright_rotations;
  device  the pass in the engine: the low-resolution part of extract (dimb_resize_area_rgb_dev, SuperPoint) + lowres_pairs(), + the
          preselection lists, or upright().
Then, once, the engine's full run against the host: the tiled ALIKED features (AlikedExtractor._extract_by_tile, float16) and
LightGlueMatcher._match_by_tile of the same tile pairs.  A profiled device run gives tile.resize (with its bytes per second: 12 B
read per RGB source pixel and 4 B written per gray output pixel) and the low-resolution SuperPoint and LightGlue device times.
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

SIZE = (1536, 2048)
AL_CONF = {"max_num_keypoints": 4096, "detection_threshold": 0.2, "nms_radius": 3}
TILING = {"tile_size": (1024, 1024), "tile_overlap": 128}  # (x, y), as the host tile selection takes it
PAIRGEN = {"strategy": "matching_lowres", "resize_max": 1000, "min_matches": 20}
PRE_SIZE = 1024
UP = {"resize_max": 640, "max_keypoints": 2048}


def image_set(n, turned, seed=160):
    """n // 4 scenes, the scene and 3 warps of it, RGB float32; with `turned` each image turned by a seeded rotation."""
    from dim_b200 import synthetic
    from dim_b200.upright import ROTATIONS, rotate_image
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n // 4):
        base = np.ascontiguousarray(synthetic.blocks_image(seed + s, max(SIZE))[:SIZE[0], :SIZE[1]])
        for k in range(4):
            rgb = (base if k == 0 else synthetic.warp_pair(base, seed + 10 * s + k, jitter=0.02 * max(SIZE))).astype(np.float32)
            out.append(np.ascontiguousarray(rotate_image(rgb, ROTATIONS[int(rng.integers(4))]) if turned else rgb))
    return out


def run_mode(ctx, mode, n, batch_images, batch_pairs, reps):
    import cv2
    import torch
    from pathlib import Path

    from dim_b200 import _native, tiling, weights
    from dim_b200.config import Config
    from dim_b200.extractors.aliked import AlikedExtractor
    from dim_b200.io_h5 import as_half_roundtrip
    from dim_b200.matchers.lightglue import LightGlueMatcher
    from dim_b200.pairs_generator import gray_from_rgb, pairs_from_bruteforce, pairs_from_lowres
    from dim_b200.sharded import ImageSetMatcher, tile_pairs_for
    from dim_b200.upright import rotate_image, search_plugins, upright_rotations
    w_sp, w_al = weights.superpoint_v1(), weights.aliked_n16rot()
    w128, w256 = weights.lightglue_seeded(input_dim=128, seed=0), weights.lightglue_seeded(seed=0)
    imgs = image_set(n, turned=mode == "upright")
    ids, pairs = list(range(n)), pairs_from_bruteforce(list(range(n)))
    hs, ws = [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]
    tiled = {**TILING, "tile_selection": "grid"}
    kw = {"lowres": {"pair_generation": PAIRGEN, "lowres_weights": w256},
          "preselection": {"preselection_weights": w256},
          "upright": {"upright": UP, "upright_weights": w256}}[mode]
    if mode == "preselection":
        tiled = {**TILING, "tile_selection": "preselection", "tile_preselection_size": PRE_SIZE}
    eng = ImageSetMatcher(ctx, w_al, w128, n, hs, ws, AL_CONF, {}, batch_images=batch_images, batch_pairs=batch_pairs, tiling=tiled,
                          extractor="aliked", **kw)
    d_imgs = [torch.from_numpy(x).cuda() for x in imgs]
    stacked = torch.stack(d_imgs) if mode != "upright" else None  # the unturned set has one size
    low = {"lowres": eng.lowres, "preselection": eng.pre, "upright": eng.search}[mode]
    names = [Path(f"{k}.png") for k in ids]
    sp_nets = {}
    lg_pre = _native.LightGlueNet(ctx, w256, max_kpts=tiling.SP_PRESELECTION_CONF["max_keypoints"], **tiling.LG_PRESELECTION_CONF)
    plugins = search_plugins(UP["max_keypoints"], True, w256, w_sp, ctx.device)  # tiling: fixed descriptor sampling (quirk A.6)

    def sp_pre(H, W):
        if (H, W) not in sp_nets:
            sp_nets[(H, W)] = _native.SuperPointNet(ctx, w_sp, max_height=H, max_width=W, **tiling.SP_PRESELECTION_CONF)
        return sp_nets[(H, W)]

    def host():
        grays = [gray_from_rgb(im) for im in imgs]
        if mode == "lowres":
            small = {p.name: cv2.resize(g, low.low_sizes[0][::-1], interpolation=cv2.INTER_AREA) for p, g in zip(names, grays)}
            kept, counts = pairs_from_lowres(names, PAIRGEN["resize_max"], PAIRGEN["min_matches"], lightglue_weights=w256,
                                             superpoint_weights=w_sp, images=small, return_counts=True, device=ctx.device)
            return [(int(a.stem), int(b.stem)) for a, b in kept], counts
        if mode == "preselection":
            lists = []
            for i, j in pairs:
                kp0, kp1 = tiling.preselection_matches(grays[i], grays[j], PRE_SIZE, sp_pre, lg_pre)
                lists.append(tiling.tile_selection(grays[i], grays[j], "preselection", TILING["tile_size"], TILING["tile_overlap"],
                                                   kp0=kp0, kp1=kp1))
            return lists
        return upright_rotations(grays, pairs, UP["resize_max"], UP["max_keypoints"], plugins=plugins)

    def device():
        st = torch.cuda.current_stream().cuda_stream
        if mode == "upright":
            return eng.upright(d_imgs, ids, pairs)
        for b0 in range(0, n, eng.B):  # the low-resolution part of extract: one fused resize and its SuperPoint calls per batch
            batch = ids[b0:b0 + eng.B]
            low.extract(stacked[b0:b0 + len(batch)], batch, [eng.slots[i] for i in batch], st)
        return eng.lowres_pairs() if mode == "lowres" else eng._preselect(pairs)

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

    # the engine's full run against the host's tiled ALIKED features and tile-pair matching
    if mode == "lowres":
        kept, _, tables = eng.run_lowres(d_imgs, ids)
    else:
        kept = pairs
        tables = eng.run(d_imgs, ids, pairs)
    turned = imgs if mode != "upright" else [rotate_image(im, r) for im, r in zip(imgs, out["host"][0])]
    ext = AlikedExtractor(Config(general={"tile_size": TILING["tile_size"], "tile_overlap": TILING["tile_overlap"]},
                                 extractor={"model_name": "aliked-n16rot", **AL_CONF, "weights_dict": w_al}))
    plugin = LightGlueMatcher(Config(pipeline="aliked+lightglue", matcher={"weights_dict": w128}), local_features="aliked")
    feats = [as_half_roundtrip({**ext._extract_by_tile(im), "image_size": np.array(im.shape[:2])}) for im in turned]
    T = eng.tile_counts
    lists = out["host"] if mode == "preselection" else [tile_pairs_for("grid", T[i], T[j]) for i, j in kept]
    host_tables = [plugin._match_by_tile(feats[i], feats[j], lst) for (i, j), lst in zip(kept, lists)]
    tables_identical = len(tables) == len(host_tables) and all(np.array_equal(a, b) for a, b in zip(tables, host_tables))

    med = {k: float(np.median(v)) for k, v in secs.items()}
    group = lambda p: round(sum(v[0] for k, v in prof.items() if k.startswith(p)), 4)  # noqa: E731
    src_px, low_px = sum(im.shape[0] * im.shape[1] for im in imgs), sum(h * w for h, w in low.low_sizes)
    resize_bytes = 12 * src_px + 4 * low_px
    same = {"lowres": lambda: {"pairs_identical": out["host"][0] == out["device"][0], "counts_identical": out["host"][1] == out["device"][1],
                               "kept_pairs": len(out["device"][0])},
            "preselection": lambda: {"lists_identical": out["host"] == out["device"],
                                     "tile_pairs_selected": sum(len(lst) for lst in out["device"])},
            "upright": lambda: {"rotations_identical": list(out["host"][0]) == list(out["device"][0]),
                                "counts_identical": {k: list(v) for k, v in out["host"][1].items()} ==
                                                    {k: list(v) for k, v in out["device"][1].items()},
                                "rotations": list(out["device"][0])}}[mode]()
    return {
        "metric": f"ALIKED image set, {mode}: {n} RGB {SIZE[0]} x {SIZE[1]} images, ALIKED n16rot {AL_CONF['max_num_keypoints']} keypoints "
                  f"per tile, tiles {TILING['tile_size']} / overlap {TILING['tile_overlap']}: host flow on gray_from_rgb images vs "
                  "ImageSetMatcher(extractor=\"aliked\") on the device",
        "mode": mode, **card(), "images": n, "pairs": len(pairs), "low_sizes": sorted({tuple(s) for s in low.low_sizes}),
        "batch_images": batch_images, "batch_pairs": batch_pairs, "reps": reps,
        "host_s": [round(s, 4) for s in secs["host"]], "device_s": [round(s, 4) for s in secs["device"]],
        "speedup": med["host"] / med["device"], **same, "tables_identical": bool(tables_identical),
        "matches_total": int(sum(len(t) for t in tables)), "launches_per_run": launches,
        "device_ms": {"tile.resize": group("tile.resize"), "superpoint": group("sp."), "lightglue": group("lg.")},
        "tile_resize_bytes": resize_bytes, "tile_resize_TB_per_s": resize_bytes / max(group("tile.resize"), 1e-6) / 1e9,
        "data": "synthetic scenes under homography warps with seeded LightGlue weights: equality and time only, not accuracy"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-images", type=int, default=16)
    ap.add_argument("--batch-pairs", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--modes", default="lowres,preselection,upright")
    args = ap.parse_args()
    from dim_b200 import _native
    ctx = _native.Context.get(0)
    for mode in args.modes.split(","):
        print(json.dumps(run_mode(ctx, mode, args.images, args.batch_images, args.batch_pairs, args.reps)), flush=True)


if __name__ == "__main__":
    main()
