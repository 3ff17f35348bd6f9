"""multi_regions_bench.py -- w2x_multi_convert_chain_regions against the one-context w2x_convert_chain_regions, host to host:

    python tools/multi_regions_bench.py [--devices 0,0] [--rounds 5] [--out DIR]

Workloads: the three of tools/regions_bench.py (uniform [0,1) noise planes from a seed, default precision, tensor-core engine):
  A  tiled scan: a 4096 x 4096 plane through noise1 + scale2.0x, its 8192 x 8192 output cut into 1024 tiles of 256 x 256
  B  viewer: 12 windows of 512 x 512 at fixed, scattered positions of that output
  C  dataset patches: 256 windows of 128 x 128, 16 at seeded positions on each of 16 planes of 1024 x 768, scale2.0x only
The source rectangles are views of the whole host planes and the windows go to host arrays of their own, as a tiling application
passes them.  Arms (every context with the same scratch limit, --scratch-gib): "one" = Context(first device).convert_chain_regions,
"multi" = Multi(--devices).convert_chain_regions, each with pinned host buffers and with pageable ones (which the multi call pins
for the call).  Every window of every arm is compared bit for bit with the pinned one-context call's.  Each arm is warmed up; every
round runs all arms in turn (the order rotates), timed by the wall clock around the synchronous call.  Reported per arm: the median,
the range and the rounds in ms, and the launches of one call per context.  With --devices 0,0 both "GPUs" are contexts of one device
and share its SMs: the figures then measure the driver's overhead and how evenly it spreads the work, not scaling.  The card's name
and power limit are read in the same run.  Prints one JSON line (and writes it to DIR/multi_regions_bench.json).
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import w2x_loader  # noqa: E402
from precision_bench import gpu_info  # noqa: E402
from regions_bench import workloads  # noqa: E402


def host(shape, pinned):
    return torch.empty(shape, dtype=torch.float32).pin_memory().numpy() if pinned else np.empty(shape, np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gib", type=float, default=4.0,
                    help="scratch limit of every context of both arms (several contexts of one device must share its memory)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("multi_regions_bench.py needs a CUDA device")
    devices = [int(v) for v in args.devices.split(",")]
    w2x = w2x_loader.load()
    one = w2x.Context(devices[0], engine=w2x.ENGINE_TC)
    multi = w2x.Multi(devices)
    w2x.lib().w2x_ctx_set_engine(w2x.lib().w2x_multi_ctx(multi._h, 0), w2x.ENGINE_TC)   # every context the call uses takes it
    scratch = int(args.scratch_gib * (1 << 30))
    one.set_scratch_limit(scratch)
    for i in range(len(devices)):
        w2x.lib().w2x_ctx_set_scratch_limit(w2x.lib().w2x_multi_ctx(multi._h, i), scratch)
    result = {"gpu": gpu_info(), "devices": devices, "precision": "f16+f8x2 (default)", "engine": "tensor-core", "rounds": args.rounds,
              "scratch_gib": args.scratch_gib,
              "note": ("all contexts on one device: overhead and spread of work, not scaling" if len(set(devices)) == 1 else
                       f"{len(set(devices))} distinct devices"), "workloads": {}}
    for name, (steps, planes, wins) in workloads(w2x, 2026).items():
        sizes = [(planes[p].shape[1], planes[p].shape[0]) for p, _ in wins]
        windows = [win for _, win in wins]
        rects = [w2x.chain_region_source(steps, size, win) for size, win in zip(sizes, windows)]
        arms, outs = {}, {}
        for pinned in (True, False):
            hp = [host(x.shape, pinned) for x in planes]
            for a, x in zip(hp, planes):
                a[:] = x
            srcs = [hp[p][sy0:sy0 + sh, sx0:sx0 + sw] for (p, _), (sx0, sy0, sw, sh) in zip(wins, rects)]
            tag = "pinned" if pinned else "pageable"
            for arm, runner, count in (("one", one, lambda: [one.launch_count()]), ("multi", multi, multi.launch_counts)):
                ys = [host((win[3], win[2]), pinned) for win in windows]
                outs[f"{arm}_{tag}"] = ys
                arms[f"{arm}_{tag}"] = (lambda r=runner, s=srcs, y=ys: r.convert_chain_regions(steps, s, sizes, windows, out=y), count)
        launches = {}
        for arm, (fn, count) in arms.items():
            for _ in range(args.warmup):
                fn()
            n0 = count()
            fn()
            launches[arm] = [a - b for a, b in zip(count(), n0)]
        want = outs["one_pinned"]
        equal = {arm: all(np.array_equal(a, b) for a, b in zip(outs[arm], want)) for arm in arms}
        secs = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                t0 = time.perf_counter()
                arms[arm][0]()
                secs[arm].append(time.perf_counter() - t0)
        w = result["workloads"][name] = {"steps": ", ".join(("scale2.0x" if up else "noise1") for _, up in steps), "n_planes": len(planes),
                                         "n_windows": len(wins), "window": list(windows[0][2:]), "arms": {}}
        for arm in arms:
            med = statistics.median(secs[arm])
            w["arms"][arm] = {"ms": round(med * 1e3, 2), "range_ms": [round(min(secs[arm]) * 1e3, 2), round(max(secs[arm]) * 1e3, 2)],
                              "ms_rounds": [round(s * 1e3, 2) for s in secs[arm]], "launches_per_call": launches[arm],
                              "bit_identical_to_one_context": equal[arm]}
        for tag in ("pinned", "pageable"):
            w[f"one_over_multi_{tag}"] = round(w["arms"][f"one_{tag}"]["ms"] / w["arms"][f"multi_{tag}"]["ms"], 3)
        del arms, outs, want
    multi.close()
    one.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "multi_regions_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
