"""LighterGlue over an image set of given XFeat features on one GPU: the plugin one pair at a time against image-set batches.

n "images" (default 24 -> 276 pairs) are built from the golden XFeat features of the reference's two photos (tests/golden/
lighterglue_golden.npz): the photos, then seeded subsets and permutations of their keypoints, up to 2048 each.  Every pair is matched
  (a) by LighterGlueMatcher._match_pairs per pair on store.get features (dimb_lg_match: each pair staged from the host into the
      batched engine at P = 1, synchronising),
  (b) by sharded.ImageSetMatcher(extractor=None, matcher="lighterglue").match at batch_pairs 8 and 32 (dimb_lg_match_dev on the store).
The tables of (a) and (b) are compared.  Each arm is timed after a warm-up run with a device synchronise at the end; the lgx.* device
times (dimb_ctx_profile) and launch counts come from a separate profiled run.  The card's name and power limit are read in the same
process.  Prints one JSON line.
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


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "clocks_max_sm": clock}


def image_set(n):
    g = np.load(os.path.join(ROOT, "tests", "golden", "lighterglue_golden.npz"))
    base = [{"keypoints": g[f"kpts{i}"].astype(np.float32), "descriptors": g[f"desc{i}"].astype(np.float32),
             "image_size": g[f"size{i}"].astype(np.int32)} for i in (0, 1)]
    out = list(base)
    rng = np.random.default_rng(0)
    for k in range(2, n):
        f = base[k % 2]
        N = len(f["keypoints"])
        m = int(rng.integers(N // 2, N + 1))
        idx = rng.permutation(N)[:m] if k % 3 == 0 else np.sort(rng.choice(N, m, replace=False))
        out.append({**f, "keypoints": f["keypoints"][idx], "descriptors": f["descriptors"][:, idx]})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=24)
    ap.add_argument("--batch-pairs", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch

    from dim_b200 import _native
    from dim_b200.config import Config
    from dim_b200.matchers.lighterglue import LighterGlueMatcher, lighterglue_weights
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher

    if not torch.cuda.is_available():
        raise SystemExit("bench_lighterglue_sets.py measures on the GPU; none is available")
    ctx = _native.Context.get(0)
    w = lighterglue_weights()
    n = args.images
    feats = image_set(n)
    pairs = pairs_from_bruteforce(list(range(n)))
    H, W = [int(f["image_size"][0]) for f in feats], [int(f["image_size"][1]) for f in feats]
    sp = {"max_keypoints": 2048, "descriptor_dim": 64}
    engines = {bp: ImageSetMatcher(ctx, None, w, n, H, W, sp, {}, batch_pairs=bp, matcher="lighterglue", extractor=None)
               for bp in args.batch_pairs}
    for eng in engines.values():
        eng.put_features(feats, list(range(n)))
        eng.exchange()
    ids = list(range(len(pairs)))
    store = next(iter(engines.values())).store
    got = [store.get(eng_slot) for eng_slot in next(iter(engines.values())).slots]
    plugin = LighterGlueMatcher(Config(matcher={"name": "lighterglue", "weights_dict": w}), local_features="xfeat")

    def per_pair():
        return [plugin._match_pairs(got[i], got[j]) for i, j in pairs]

    def batched(bp):
        res = engines[bp].match(pairs, ids)
        return [res[k] for k in ids]

    arms = {"per_pair": per_pair, **{f"batched_{bp}": (lambda bp=bp: batched(bp)) for bp in args.batch_pairs}}
    tables, times, launches = {}, {}, {}
    for name, fn in arms.items():
        tables[name] = fn()  # warm-up of every shape
        torch.cuda.synchronize()
        best = []
        for _ in range(args.repeats):
            l0 = ctx.launches
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            best.append(time.perf_counter() - t0)
            launches[name] = ctx.launches - l0
        times[name] = best
    identical = {name: all(np.array_equal(a, b) for a, b in zip(tables[name], tables["per_pair"])) for name in arms}
    prof = {}
    for name, fn in arms.items():
        ctx.profile(True)
        fn()
        torch.cuda.synchronize()
        prof[name] = {k: [round(v[0], 3), v[1]] for k, v in ctx.profile_read().items() if k.startswith("lgx")}
        ctx.profile(False)
    out = {"bench": "lighterglue_sets", **card(), "images": n, "pairs": len(pairs), "matches_total": int(sum(len(t) for t in tables["per_pair"])),
           "tables_identical": identical,
           "pairs_per_s": {k: round(len(pairs) / min(v), 1) for k, v in times.items()},
           "seconds": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "launches": launches, "lgx_device_ms_and_launches": prof}
    print(json.dumps(out))
    return 0 if all(identical.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
