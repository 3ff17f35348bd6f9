"""multi_planes_bench.py -- w2x_multi_convert_planes_chain against the one-context w2x_convert_planes_chain, host to host:

    python tools/multi_planes_bench.py [--devices 0,0] [--rounds 5] [--out DIR]

Workloads (uniform [0,1) noise planes from a seed, default precision, tensor-core engine, pinned host planes):
  A_scale         tools/planes_bench.py's collection A (2000 planes, sides in [16, 128]), scale2.0x
  A_noise_scale   A through noise1 + scale2.0x with W2X_STEP_TTA on both steps
  tta_1080p       one 1920 x 1080 plane through noise1 with W2X_STEP_TTA (its 8 variants spread over the GPUs)
Arms (every context with the same scratch limit, --scratch-gib): "one" = Context(first device).convert_planes_chain, "multi" = Multi(--devices).convert_planes_chain.  Every output of every arm
is compared bit for bit with the one-context call's.  Each arm is warmed up; every round runs both arms in turn (the order alternates),
timed by the wall clock around the synchronous call.  Reported per arm: the median, the range and the rounds in ms, output Mpix/s,
and the summed launches of one call.  With --devices 0,0 both "GPUs" are contexts of one device and share its SMs: the figures then
measure the driver's overhead and how evenly it spreads the work, not scaling.  The card's name and power limit are read in the same
run.  Prints one JSON line (and writes it to DIR/multi_planes_bench.json).
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
from planes_bench import workload  # noqa: E402
from precision_bench import gpu_info, load_model  # noqa: E402


def pinned_planes(sizes, seed, ups):
    rng = np.random.default_rng(seed)
    xs = [torch.from_numpy(rng.random((h, w), dtype=np.float32)).pin_memory().numpy() for w, h in sizes]
    ys = [torch.empty((h << ups, w << ups), dtype=torch.float32).pin_memory().numpy() for w, h in sizes]
    return xs, ys


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
        sys.exit("multi_planes_bench.py needs a CUDA device")
    devices = [int(v) for v in args.devices.split(",")]
    w2x = w2x_loader.load()
    one = w2x.Context(devices[0], engine=w2x.ENGINE_TC)
    multi = w2x.Multi(devices)
    scratch = int(args.scratch_gib * (1 << 30))
    one.set_scratch_limit(scratch)
    for i in range(len(devices)):
        w2x.lib().w2x_ctx_set_scratch_limit(w2x.lib().w2x_multi_ctx(multi._h, i), scratch)
    noise, scale = load_model(w2x, "noise1"), load_model(w2x, "scale2.0x")
    result = {"gpu": gpu_info(), "devices": devices, "precision": "f16+f8x2 (default)", "rounds": args.rounds, "scratch_gib": args.scratch_gib,
              "note": ("all contexts on one device: overhead and spread of work, not scaling" if len(set(devices)) == 1 else
                       f"{len(set(devices))} distinct devices"), "workloads": {}}
    for name, sizes, steps in (("A_scale", workload("A", 1), [(scale, True)]),
                               ("A_noise_scale", workload("A", 1), [(noise, False, True), (scale, True, True)]),
                               ("tta_1080p", [(1920, 1080)], [(noise, False, True)])):
        ups = sum(1 for s in steps if s[1])
        xs, ys_one = pinned_planes(sizes, 7, ups)
        _, ys_multi = pinned_planes(sizes, 7, ups)
        arms = {"one": (lambda: one.convert_planes_chain(steps, xs, out=ys_one), ys_one, lambda: [one.launch_count()]),
                "multi": (lambda: multi.convert_planes_chain(steps, xs, out=ys_multi), ys_multi, multi.launch_counts)}
        launches = {}
        for arm, (fn, _, count) in arms.items():
            for _ in range(args.warmup):
                fn()
            n0 = count()
            fn()
            launches[arm] = [a - b for a, b in zip(count(), n0)]
        equal = all(np.array_equal(a, b) for a, b in zip(ys_one, ys_multi))
        secs = {arm: [] for arm in arms}
        for r in range(args.rounds):
            for arm in (("one", "multi") if r % 2 == 0 else ("multi", "one")):
                t0 = time.perf_counter()
                arms[arm][0]()
                secs[arm].append(time.perf_counter() - t0)
        pix = sum((w << ups) * (h << ups) for w, h in sizes)
        w = result["workloads"][name] = {"planes": len(sizes), "output_megapixels": round(pix / 1e6, 3), "bit_identical": equal,
                                         "steps": [("scale2.0x (2x)" if s[1] else "noise1") + (" +tta" if len(s) > 2 and s[2] else "") for s in steps],
                                         "arms": {}}
        for arm in arms:
            med = statistics.median(secs[arm])
            w["arms"][arm] = {"ms": round(med * 1e3, 2), "range_ms": [round(min(secs[arm]) * 1e3, 2), round(max(secs[arm]) * 1e3, 2)],
                              "ms_rounds": [round(s * 1e3, 2) for s in secs[arm]], "mpix_s": round(pix / med / 1e6, 1),
                              "launches_per_call": launches[arm]}
        w["one_over_multi"] = round(w["arms"]["one"]["ms"] / w["arms"]["multi"]["ms"], 3)
        del xs, ys_one, ys_multi
    multi.close()
    one.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "multi_planes_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
