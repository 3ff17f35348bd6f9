"""multi_chain_bench.py -- the Y plane's noise pass and 2x scale steps (src/main.cpp:82-156) on several GPUs, host to host: one
w2x_multi_convert_chain call against the per-step multi-GPU path it replaces and against the one-GPU chain, in one process:

    python tools/multi_chain_bench.py [--devices 0,1] [--rounds 9] [--reps 4] [--out DIR]

Seeded workloads (uniform [0,1) noise planes, default precision, pinned host planes, block_splitting = 1 as the CLI uses):
  A   1920 x 1080, noise1 then scale2.0x           (the CLI's default mode on a full-HD image)
  B   960 x 540, noise1 then scale2.0x twice       (x4)
Arms per workload:
  one_gpu_chain   Context.convert_chain on one context of the first device
  multi_loop      Multi.convert_plane per step, the nearest 2x resize by numpy into a pinned plane (what `--gpus n` ran before)
  multi_chain     one Multi.convert_chain call
Every arm's output is compared bit for bit with one_gpu_chain's before anything is timed.  Then every round runs all arms in turn
(the order rotates from round to round), each arm `reps` calls back to back, timed by the wall clock (every call is synchronous).
Reported per arm: the median and the range of the rounds' milliseconds per call, the library's kernel launches per call, and the
bytes a call copies over PCIe, computed from the shapes (multi_loop moves every intermediate plane down and up again, its resized
plane at 4x the size; the chains move the input and the output).  The card's name and power limit are read in the same run.

--devices 0,0 runs the multi arms on two contexts of ONE GPU: they share its SMs, so the comparison measures the copies and host
resizes the chain removes, not multi-GPU scaling.  That needs CUDA_DEVICE_MAX_CONNECTIONS (set here when absent) for the two
contexts' streams to run side by side.  Prints one JSON line (and writes it to DIR/multi_chain_bench.json).
"""
import argparse
import json
import os
import statistics
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import w2x_loader  # noqa: E402
from precision_bench import gpu_info, load_model  # noqa: E402

WORKLOADS = (("A", 1920, 1080, "SU"), ("B", 960, 540, "SUU"))


def pcie_bytes(w, h, pattern, loop):
    """host <-> device bytes of one call: the loop uploads every step's (resized) input and downloads every step's output"""
    total, first = 0, True
    for c in pattern:
        if c == "U":
            w, h = 2 * w, 2 * h
        if loop:
            total += 2 * w * h * 4
        elif first:
            total += (w * h // 4 if c == "U" else w * h) * 4
        first = False
    return total if loop else total + w * h * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0")
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("multi_chain_bench.py needs a CUDA device")
    devices = [int(v) for v in args.devices.split(",")]
    w2x = w2x_loader.load()
    ctx = w2x.Context(devices[0], engine=w2x.ENGINE_TC)
    multi = w2x.Multi(devices)
    models = {"S": load_model(w2x, "noise1"), "U": load_model(w2x, "scale2.0x")}
    multi.convert_tiles(models["S"], np.zeros((len(devices), 8, 8), np.float32))      # every context's first launch, no exchange
    result = {"gpu": gpu_info(), "devices": devices, "shared_gpu": len(set(devices)) < len(devices), "precision": "f16+f8x2 (default)",
              "rounds": args.rounds, "reps": args.reps, "workloads": {}}
    for name, w, h, pattern in WORKLOADS:
        steps = [(models[c], c == "U") for c in pattern]
        ups = pattern.count("U")
        W, H = w << ups, h << ups
        x = np.random.default_rng(len(name) + w).random((h, w), dtype=np.float32)
        h_in = torch.from_numpy(x.copy()).pin_memory().numpy()
        bufs = [torch.empty(W * H).pin_memory().numpy() for _ in range(3)]             # two ping-pong planes and the 2x resize
        h_out = torch.empty((H, W)).pin_memory().numpy()

        def one_gpu_chain():
            ctx.convert_chain(steps, h_in, out=h_out)

        def multi_loop():
            cur, where = h_in, -1
            for k, (model, up) in enumerate(steps):
                ch, cw = cur.shape
                if up:
                    big = bufs[2][:4 * cw * ch].reshape(ch, 2, cw, 2)
                    big[...] = cur[:, None, :, None]
                    cur, where, ch, cw = big.reshape(2 * ch, 2 * cw), -1, 2 * ch, 2 * cw
                j = 1 if where == 0 else 0
                dst = h_out if k + 1 == len(steps) else bufs[j][:cw * ch].reshape(ch, cw)
                multi.convert_plane(model, cur, block_splitting=True, out=dst)
                cur, where = dst, j

        def multi_chain():
            multi.convert_chain(steps, h_in, out=h_out)

        arms = {"one_gpu_chain": one_gpu_chain, "multi_loop": multi_loop, "multi_chain": multi_chain}
        outputs, launches = {}, {}
        for arm, fn in arms.items():
            h_out[:] = 0
            fn()                                                                       # warm-up: models, plans, buffers
            before = ctx.launch_count() + sum(multi.launch_counts())
            fn()
            launches[arm] = ctx.launch_count() + sum(multi.launch_counts()) - before
            outputs[arm] = h_out.copy()
        same = {arm: bool(np.array_equal(outputs[arm], outputs["one_gpu_chain"])) for arm in arms}
        if not all(same.values()):
            sys.exit(f"workload {name}: outputs differ from the one-GPU chain's: {same}")
        ms = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    arms[arm]()
                ms[arm].append((time.perf_counter() - t0) * 1e3 / args.reps)
        res = result["workloads"][name] = {"input": [w, h], "output": [W, H], "steps": pattern, "arms": {}}
        for arm in arms:
            med = statistics.median(ms[arm])
            res["arms"][arm] = {"ms": round(med, 2), "ms_min": round(min(ms[arm]), 2), "ms_max": round(max(ms[arm]), 2),
                                "out_mpix_s": round(W * H / med / 1e3, 1), "launches_per_call": launches[arm],
                                "pcie_bytes_per_call": pcie_bytes(w, h, pattern, arm == "multi_loop"),
                                "bit_identical_to_one_gpu_chain": same[arm]}
    multi.close()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "multi_chain_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
