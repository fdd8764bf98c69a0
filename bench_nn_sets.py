"""Brute-force NN matching (kornia_matcher) over an image set on one GPU: the per-pair paths against the batched device engine.

n synthetic 1024 x 1024 images (default 24 -> 276 pairs) go through SuperPoint (2048 keypoints by default, --kpts 8192 for cfg5's size)
into the device feature store; then every pair is matched in modes smnn 0.85 and mnn three ways:
  (a) KorniaMatcher._match_pairs per pair on store.get features (host descriptors, one synchronising call per pair),
  (b) dimb_nn_match_dev per pair on the store's slots (counts read to the host once, before the timed loop),
  (c) sharded.ImageSetMatcher(matcher="kornia_matcher").match: dimb_nn_match_batch_dev on batches of 32 (and 8) store slots, counts
      on the device.
Every arm is timed with CUDA events after a warm-up of every shape; the per-group device times of dimb_ctx_profile come from a separate
run.  The card's name and power limit are read in the same process.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SIZE = 1024
MODES = (("smnn", 0.85), ("mnn", 0.0))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "clocks_max_sm": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=24)
    ap.add_argument("--kpts", type=int, default=2048, help="SuperPoint max_keypoints (8192: cfg5's size)")
    ap.add_argument("--batch-pairs", type=int, nargs="+", default=[32, 8], help="pairs per dimb_nn_match_batch_dev call in arm (c)")
    args = ap.parse_args()
    import torch

    from dim_b200 import _native, synthetic, weights
    from dim_b200.config import Config
    from dim_b200.matchers.kornia_matcher import KorniaMatcher
    from dim_b200.pairs_generator import pairs_from_bruteforce
    from dim_b200.sharded import ImageSetMatcher

    n, K = args.images, args.kpts
    ctx = _native.Context.get(0)
    sp_conf = {"nms_radius": 3, "keypoint_threshold": 0.0005, "max_keypoints": K}
    imgs = []
    for k in range((n + 1) // 2):
        imgs += list(synthetic.synthetic_pair(7000 + k, SIZE))
    d_imgs = torch.from_numpy(np.stack(imgs[:n]).astype(np.float32)).cuda()
    w_sp = weights.superpoint_v1()

    def make_engines(conf):
        engines = {}
        for bp in args.batch_pairs:
            engines[bp] = ImageSetMatcher(ctx, w_sp, None, n, SIZE, SIZE, sp_conf, conf, batch_images=8, batch_pairs=bp, matcher="kornia_matcher")
            engines[bp].extract(d_imgs, list(range(n)))
        torch.cuda.synchronize()
        return engines

    store = make_engines({})[args.batch_pairs[0]].store  # single process: slot i = image i; every engine extracts the same features
    pairs = pairs_from_bruteforce(list(range(n)))
    ids = list(range(len(pairs)))
    feats = [store.get(i) for i in range(n)]  # what get_features hands the plugin (features.h5 values)
    counts = [max(store.count(i)[0], 0) for i in range(n)]
    fd = [store.feats_dev(i) for i in range(n)]
    cap = store.cap
    st = torch.cuda.current_stream().cuda_stream
    b_idx = torch.zeros(len(pairs), cap, 2, dtype=torch.int64, device="cuda")
    b_dst = torch.zeros(len(pairs), cap, device="cuda")
    b_n = torch.zeros(len(pairs), dtype=torch.int32, device="cuda")

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1])

    def profiled(fn):
        ctx.profile(True)
        fn()
        torch.cuda.synchronize()
        prof = ctx.profile_read()
        ctx.profile(False)
        return {k: [round(v[0], 3), int(v[1])] for k, v in sorted(prof.items())}

    def counted(fn):
        l0 = ctx.launches
        out, ms = timed(fn)
        return out, ms, ctx.launches - l0

    out = {}
    for mode, th in MODES:
        plugin = KorniaMatcher(Config(matcher={"name": "kornia_matcher", "match_mode": mode, "th": th}))
        engines = make_engines({"match_mode": mode, "th": th})

        def arm_a(sel=ids):
            return {k: plugin._match_pairs(feats[pairs[k][0]], feats[pairs[k][1]]) for k in sel}

        def arm_b_enqueue():
            for k, (i, j) in enumerate(pairs):
                ctx.nn_match_dev(fd[i].descriptors, counts[i], fd[j].descriptors, counts[j], store.desc_dim, mode, th, b_idx[k].data_ptr(),
                                 b_dst[k].data_ptr(), b_n[k:k + 1].data_ptr(), cap, f16=True, ld0=fd[i].desc_ld, ld1=fd[j].desc_ld, stream=st)

        def arm_b_tables():
            nb = np.minimum(b_n.cpu().numpy(), cap)
            h = b_idx.cpu().numpy()
            return {k: h[k, :nb[k]].copy() for k in ids}

        # warm-up of every shape: one plugin pair, the per-pair loop, a full and the last partial batch of every engine
        arm_a([0])
        arm_b_enqueue()
        for bp, eng in engines.items():
            tail = len(pairs) % bp or bp
            eng.match(pairs[:bp], ids[:bp])
            eng.match(pairs[-tail:], ids[-tail:])
        torch.cuda.synchronize()
        res = {}
        _, ms_b, l_b = counted(arm_b_enqueue)
        res["b_per_pair_dev"] = {"pairs_per_s": len(pairs) / (ms_b / 1e3), "ms": round(ms_b, 2), "gpu_launches": l_b}
        tab_b = arm_b_tables()
        tabs_c = {}
        for bp, eng in engines.items():
            tab, ms_c, l_c = counted(lambda: eng.match(pairs, ids))
            tabs_c[bp] = tab
            res[f"c_batched_{bp}"] = {"pairs_per_s": len(pairs) / (ms_c / 1e3), "ms": round(ms_c, 2), "gpu_launches": l_c}
        tab_a, ms_a, l_a = counted(arm_a)
        res["a_plugin_per_pair"] = {"pairs_per_s": len(pairs) / (ms_a / 1e3), "ms": round(ms_a, 2), "gpu_launches": l_a}
        same = sum(np.array_equal(tab_a[k], tab_b[k]) and all(np.array_equal(tab_a[k], t[k]) for t in tabs_c.values()) for k in ids)
        res["tables_identical_all_arms"] = f"{same}/{len(pairs)}"
        res["total_matches"] = int(sum(len(tab_a[k]) for k in ids))
        res["profile_b_ms_launches"] = profiled(arm_b_enqueue)
        bp0 = args.batch_pairs[0]
        res[f"profile_c_{bp0}_ms_launches"] = profiled(lambda: engines[bp0].match(pairs, ids))
        res["speedup_c_over_b"] = res["b_per_pair_dev"]["ms"] / res[f"c_batched_{bp0}"]["ms"]
        out[f"{mode}_{th}"] = res
    print(json.dumps({
        "metric": f"kornia_matcher image-pairs/sec over an image set (SuperPoint {K} kpts, {SIZE}x{SIZE}, 256-d)", **card(), "images": n,
        "pairs": len(pairs), "mean_keypoints": float(np.mean(counts)), "batch_pairs": args.batch_pairs, **out,
        "data": "synthetic", "dtype": "f16 operands (the store's values: one MMA is exact), f32 accumulate"}))


if __name__ == "__main__":
    main()
