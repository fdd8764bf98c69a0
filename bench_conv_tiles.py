"""The SuperPoint 64 -> 64 channel 3x3 convolutions on 8 x 16 and on 16 x 16 pixel tiles, on one GPU.

Layers at the shapes of the bench.py step (66 images of 1024 x 1024): conv1b (1024 x 1024, 2x2 max pool), conv2a (512 x 512) and conv2b
(512 x 512, pool).  Each runs through the self-test library's timing entry (dimb_selftest_conv3x3_time: the production launch of one
tile shape on device-generated activations, CUDA events around `iters` calls after `warm` untimed ones), the two tile shapes
alternating within every repetition.  Besides the median device time per call it prints the bytes per output pixel one tile fetches
(the three dx boxes of every channel block, plus the nine weight tiles unless the plan keeps them resident) and the executed tensor
rate (EXACT issues three MMAs per product).  One JSON line per (layer, precision).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_verify import card  # noqa: E402

LAYERS = {"conv1b": (1024, 1024, True), "conv2a": (512, 512, False), "conv2b": (512, 512, True)}
TILE_H = {8: 8, 16: 16}


def bytes_per_pixel(tile, precision, resb):
    """(A bytes, B bytes, bytes per output pixel) one tile of a 64 -> 64 conv fetches; resident weights are loaded once per CTA."""
    planes = 2 if precision == "exact" else 1
    a = 3 * (TILE_H[tile] + 2) * 16 * 128 * planes
    b = 0 if resb else 9 * 64 * 128 * planes
    return a, b, (a + b) / (TILE_H[tile] * 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=66)
    ap.add_argument("--reps", type=int, default=3, help="alternating repetitions of the two tile shapes")
    ap.add_argument("--iters", type=int, default=10, help="timed calls per repetition")
    ap.add_argument("--precision", default="exact,fast")
    ap.add_argument("--layers", default=",".join(LAYERS))
    args = ap.parse_args()
    from dim_b200 import _native
    st = _native.SelfTest(0)
    info = card()
    for precision in args.precision.split(","):
        st.set_precision(precision)
        for layer in args.layers.split(","):
            H, W, pool = LAYERS[layer]
            ms = {8: [], 16: []}
            plans = {}
            for _ in range(args.reps):
                for tile in (8, 16):
                    t, plan, mode = st.conv3x3_time(args.images, H, W, 64, 64, pool, tile, warm=2, iters=args.iters)
                    ms[tile].append(round(t, 4))
                    plans[tile] = (plan, mode)
            flop = 2.0 * args.images * H * W * 64 * 576 * (3 if precision == "exact" else 1)
            line = {"source": "bench_conv_tiles.py", "layer": layer, "precision": precision, "images": args.images, "H": H, "W": W,
                    "pool": pool, **info}
            for tile in (8, 16):
                plan, mode = plans[tile]
                a, b, bpp = bytes_per_pixel(tile, precision, bool(plan[0]))
                med = statistics.median(ms[tile])
                line[f"tile{tile}"] = {"mode": mode, "plan": {"resb": plan[0], "sa": plan[1], "sb": plan[2], "smem": plan[3], "grid": plan[4]},
                                       "ms": ms[tile], "median_ms": med, "tile_bytes_a": a, "tile_bytes_b": b, "bytes_per_pixel": bpp,
                                       "executed_tflops": round(flop / med * 1e-9, 1)}
            line["speedup_16_over_8"] = round(line["tile8"]["median_ms"] / line["tile16"]["median_ms"], 3)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
