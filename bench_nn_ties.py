"""Device time of the brute-force NN engine on descriptor sets with and without exact ties.

The top-2 GEMM's epilogue scans a 32-column chunk a second time when the chunk's two best squared distances nearly tie (the first
column with the best's float32 distance wins, as in torch.cdist + min), so its cost depends on how often ties occur.  Three sets of
--images feature sets of --kpts descriptors each, stored as fp16 like the device feature store keeps them:
  superpoint  D = 256 unit float descriptors (noisy views of one pool): ties almost never occur;
  orb         D = 32 bytes with a quarter of every set copied from other rows of it (repeated texture);
  tie_heavy   D = 32 bytes drawn from a pool of 256 vectors: nearly every chunk of every row holds a tie for its best.
Each set is matched over all pairs of its images in mode smnn 0.95, (b) dimb_nn_match_dev per pair and (c) dimb_nn_match_batch_dev
in batches of 32 pairs, timed with CUDA events over --windows windows after a warm-up (median, min, max in ms).  The card's name and
power limit are read in the same process.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip()
    name, power = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power}


def descriptor_sets(name, n, K, rng):
    if name == "superpoint":
        pool = rng.standard_normal((4 * K, 256))
        out = []
        for _ in range(n):
            x = pool[rng.integers(0, len(pool), K)] + 0.4 * rng.standard_normal((K, 256))
            out.append(x / np.linalg.norm(x, axis=1, keepdims=True))
        return out
    if name == "orb":
        out = []
        for _ in range(n):
            x = rng.integers(0, 256, (K, 32)).astype(np.float64)
            dup = rng.choice(K, K // 4, replace=False)
            x[dup] = x[rng.integers(0, K, len(dup))]
            out.append(x)
        return out
    pool = rng.integers(0, 256, (256, 32)).astype(np.float64)
    return [pool[rng.integers(0, 256, K)] for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--kpts", type=int, default=2048)
    ap.add_argument("--windows", type=int, default=15)
    args = ap.parse_args()
    import torch

    from dim_b200 import _native

    ctx = _native.Context.get(0)
    n, K = args.images, args.kpts
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
    st = torch.cuda.current_stream().cuda_stream
    out = {}
    for name in ("superpoint", "orb", "tie_heavy"):
        sets = descriptor_sets(name, n, K, np.random.default_rng(7))
        D = sets[0].shape[1]
        desc = [torch.from_numpy(x.T.astype(np.float16).copy()).cuda() for x in sets]
        cnt = [torch.tensor([K], dtype=torch.int32, device="cuda") for _ in sets]
        fd = []
        for d, c in zip(desc, cnt):
            f = _native.FeatsDev()
            f.descriptors, f.n, f.n_cap, f.desc_layout, f.desc_ld, f.f16 = d.data_ptr(), c.data_ptr(), K, 0, K, 1
            fd.append(f)
        P = len(pairs)
        idx = torch.zeros(P, K, 2, dtype=torch.int64, device="cuda")
        dist = torch.zeros(P, K, device="cuda")
        nm = torch.zeros(P, dtype=torch.int32, device="cuda")

        def per_pair():
            for k, (i, j) in enumerate(pairs):
                ctx.nn_match_dev(desc[i].data_ptr(), K, desc[j].data_ptr(), K, D, "smnn", 0.95, idx[k].data_ptr(), dist[k].data_ptr(),
                                 nm[k:k + 1].data_ptr(), K, f16=True, stream=st)

        def batched():
            for b in range(0, P, 32):
                sel = pairs[b:b + 32]
                ctx.nn_match_batch_dev([fd[i] for i, _ in sel], [fd[j] for _, j in sel], D, "smnn", 0.95, idx[b].data_ptr(),
                                       dist[b].data_ptr(), nm[b:b + 32].data_ptr(), K, stream=st)

        res = {}
        for arm, fn in (("b_per_pair_dev", per_pair), ("c_batched_32", batched)):
            fn()
            torch.cuda.synchronize()
            ms = []
            for _ in range(args.windows):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                fn()
                ev[1].record()
                torch.cuda.synchronize()
                ms.append(ev[0].elapsed_time(ev[1]))
            res[arm] = {"ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3)}
        res["matches"] = int(nm.sum().item())
        out[name] = res
    print(json.dumps({"metric": f"brute-force NN device ms, smnn 0.95, {len(pairs)} pairs of {K} descriptors (fp16 store layout)", **card(),
                      **out}))


if __name__ == "__main__":
    main()
