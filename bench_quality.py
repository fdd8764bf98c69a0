"""Extraction quality on one GPU: the reference's host flow per image against ImageSetMatcher(quality=...).extract.

Configurations (synthetic scenes: four blocks images and three seeded homography warps of each):
  sp_medium      16 gray 4000 x 3000 images, SuperPoint (2048 keypoints), quality "medium" (one pyrDown: 2000 x 1500);
  sp_low         the same images at "low" (two pyrDown: 1000 x 750);
  aliked_medium  16 RGB 2048 x 1536 images, ALIKED (aliked-n16rot, 4000 keypoints), "medium" (1024 x 768).
Arms, each timed with a host clock around work that ends in a device synchronise, after a warm-up, in alternating repetitions:
  host    per image: ExtractorBase._resize_image (cv2.pyrDown on the host), the plugin's _extract, _resize_features, then
          FeatureStoreDev.put (the float16 cast of features.h5);
  device  ImageSetMatcher(quality=...).extract on the full-size images already in device memory: dimb_pyr_dev per extraction batch,
          batched SuperPoint (ALIKED one image per call) on the resized images, put_dev and one dimb_fstore_rescale_dev.
Reports images/s of both arms, whether every stored feature is identical, the device time of the pyramid (tile.pyr) against the
extractor's kernel groups (sp.* / al.*) from one profiled device run, and its launches.  Prints one JSON line per configuration.
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

CONFIGS = {"sp_medium": ("superpoint", 3000, 4000, "medium"), "sp_low": ("superpoint", 3000, 4000, "low"),
           "aliked_medium": ("aliked", 1536, 2048, "medium")}
SP_CONF = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": 2048}
AL_CONF = {"max_num_keypoints": 4000, "detection_threshold": 0.2, "nms_radius": 3}


def scene(H, W, n, rgb):
    from dim_b200 import synthetic
    out = []
    for s in range(n // 4):
        a = synthetic.blocks_image(70 + s, max(H, W))[:H, :W]
        out += [a] + [synthetic.warp_pair(a, 70 + 4 * s + k, jitter=0.02 * max(H, W)) for k in range(1, 4)]
    if not rgb:
        out = [synthetic.to_gray_like_reference(np.ascontiguousarray(x)) for x in out]
    return np.stack(out).astype(np.float32)


def run_config(ctx, name, extractor, H, W, quality, n, batch_images, reps):
    import torch

    from dim_b200 import _native, weights
    from dim_b200.config import Config
    from dim_b200.sharded import ImageSetMatcher
    if extractor == "superpoint":
        from dim_b200.extractors.superpoint import SuperPointExtractor
        w_ex, conf, D = weights.superpoint_v1(), SP_CONF, 256
        ext = SuperPointExtractor(Config(pipeline="superpoint+lightglue", extractor={**SP_CONF, "weights_dict": w_ex}))
        w_lg = weights.lightglue_seeded(seed=0)
    else:
        from dim_b200.extractors.aliked import AlikedExtractor
        w_ex, conf, D = weights.aliked_n16rot(), AL_CONF, 128
        ext = AlikedExtractor(Config(pipeline="aliked+lightglue", extractor={"model_name": "aliked-n16rot", **AL_CONF, "weights_dict": w_ex}))
        w_lg = weights.lightglue_seeded(input_dim=128, seed=0)
    imgs = scene(H, W, n, extractor == "aliked")
    ids = list(range(n))
    eng = ImageSetMatcher(ctx, w_ex, w_lg, n, H, W, conf, {}, batch_images=batch_images, extractor=extractor, quality=quality)
    host_store = _native.FeatureStoreDev(ctx, n, eng.store.cap, D)
    d_imgs = torch.from_numpy(imgs).cuda()

    def host():
        for i, img in enumerate(imgs):
            f = ext._resize_features(quality, ext._extract(ext._resize_image(quality, img)))
            host_store.put(eng.slots[i], {**f, "image_size": np.array(img.shape[:2])})

    def device():
        eng.extract(d_imgs, ids)

    arms = {"host": host, "device": device}
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
    identical = True
    n_kpts = []
    for i in ids:
        a, b = host_store.get(eng.slots[i]), eng.store.get(eng.slots[i])
        identical &= all(a[k].shape == b[k].shape and np.array_equal(a[k], b[k]) for k in ("keypoints", "descriptors", "scores", "image_size"))
        n_kpts.append(len(b["keypoints"]))
    ctx.profile(True)
    launches = ctx.launches
    device()
    torch.cuda.synchronize()
    launches = ctx.launches - launches
    prof = ctx.profile_read()
    ctx.profile(False)
    med = {k: float(np.median(v)) for k, v in secs.items()}
    group = lambda p: round(sum(v[0] for k, v in prof.items() if k.startswith(p)), 3)
    ex_prefix = "sp." if extractor == "superpoint" else "al."
    return {
        "metric": f"extraction at quality {quality!r}, {n} {'gray' if extractor == 'superpoint' else 'RGB'} images {W}x{H} -> "
                  f"{eng.w2}x{eng.h2}, {extractor}: host cv2 pyramid + plugin _extract + scale + store.put vs ImageSetMatcher(quality=...).extract",
        "config": name, **card(), "images": n, "quality": quality, "resized": [eng.w2, eng.h2], "batch_images": batch_images, "reps": reps,
        "host_s": [round(s, 4) for s in secs["host"]], "device_s": [round(s, 4) for s in secs["device"]],
        "host_images_per_s": n / med["host"], "device_images_per_s": n / med["device"], "speedup": med["host"] / med["device"],
        "features_identical": bool(identical), "mean_keypoints": float(np.mean(n_kpts)), "launches_per_run": launches,
        "device_ms": {"tile.pyr": group("tile.pyr"), "extractor": group(ex_prefix)},
        "device_ms_by_group": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
        "data": "synthetic scenes under homography warps (planar): timing only; correctness rests on tests/test_quality.py"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-images", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed repetitions of each arm")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    args = ap.parse_args()
    from dim_b200 import _native
    ctx = _native.Context.get(0)
    for name in args.configs.split(","):
        print(json.dumps(run_config(ctx, name, *CONFIGS[name], args.images, args.batch_images, args.reps)), flush=True)


if __name__ == "__main__":
    main()
