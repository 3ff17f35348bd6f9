"""chain_bench.py -- the Y plane's noise pass and 2x scale steps (src/main.cpp:82-156): one w2x_convert_chain call against the loop
of one conversion per step with the nearest 2x resize in between, in one process:

    python tools/chain_bench.py [--rounds 9] [--reps 4] [--out DIR]

Seeded workloads (uniform [0,1) noise planes, default precision, tensor-core engine, block_splitting = 1 as the CLI uses):
  A   1920 x 1080, noise1 then scale2.0x           (the CLI's default mode on a full-HD image)
  B   960 x 540, noise1 then scale2.0x twice       (x4)
  C   2048 x 2048, scale2.0x once
Arms per workload:
  device_loop    convert_plane_device per step, the nearest 2x resize by torch into a device buffer (same stream)
  device_chain   one convert_chain_device call
  host_loop      convert_plane per step on pinned host planes, the nearest 2x resize by numpy into a pinned plane
  host_chain     one convert_chain call on the same pinned planes
Each arm is warmed up; then every round runs all arms in turn (the order rotates from round to round), each arm `reps` calls back
to back, timed by the wall clock from a synchronised stream to a synchronised stream.  Reported per arm: milliseconds and output Mpix/s of every round, their
median, and whether the output is bit-identical to the loop's.  The card's name, power limit and maximum SM clock are read in the
same run.  Prints one JSON line (and writes it to DIR/chain_bench.json).
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
from precision_bench import gpu_info, load_model  # noqa: E402

WORKLOADS = (("A", 1920, 1080, "SU"), ("B", 960, 540, "SUU"), ("C", 2048, 2048, "U"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("chain_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    stream = torch.cuda.Stream()                        # torch's resize and the library's layers queue on one (non-default) stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    models = {"S": load_model(w2x, "noise1"), "U": load_model(w2x, "scale2.0x")}
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "rounds": args.rounds, "reps": args.reps, "workloads": {}}
    for name, w, h, pattern in WORKLOADS:
        steps = [(models[c], c == "U") for c in pattern]
        ups = pattern.count("U")
        W, H = w << ups, h << ups
        x = np.random.default_rng(len(name) + w).random((h, w), dtype=np.float32)
        # every plane a step may read or write, at the largest size: pinned host and device
        cap = W * H
        h_in = torch.from_numpy(x.copy()).pin_memory()
        h_bufs = [torch.empty(cap).pin_memory() for _ in range(3)]   # two ping-pong planes and the 2x resize
        h_out = torch.empty((H, W)).pin_memory()
        d_in = torch.from_numpy(x).cuda()
        d_bufs = [torch.empty(cap, device="cuda") for _ in range(3)]
        d_out = torch.empty((H, W), device="cuda")

        def dev_loop():
            cur, where, cw, ch = d_in, -1, w, h      # where: the buffer holding cur (-1: none of the two ping-pong buffers)
            for k, (model, up) in enumerate(steps):
                if up:
                    big = d_bufs[2][:4 * cw * ch].view(ch, 2, cw, 2)
                    big.copy_(cur.reshape(ch, 1, cw, 1).expand(ch, 2, cw, 2))
                    cur, where, cw, ch = big.view(2 * ch, 2 * cw), -1, 2 * cw, 2 * ch
                j = 1 if where == 0 else 0
                dst = d_out if k + 1 == len(steps) else d_bufs[j][:cw * ch].view(ch, cw)
                ctx.convert_plane_device(model, cur.data_ptr(), cw, ch, cw * 4, dst.data_ptr(), cw * 4, True)
                cur, where = dst, j

        def dev_chain():
            ctx.convert_chain_device(steps, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), W * 4)

        def host_loop():
            cur, where = h_in.numpy(), -1
            bufs = [b.numpy() for b in h_bufs]
            for k, (model, up) in enumerate(steps):
                ch, cw = cur.shape
                if up:
                    big = bufs[2][:4 * cw * ch].reshape(ch, 2, cw, 2)
                    big[...] = cur[:, None, :, None]
                    cur, where, ch, cw = big.reshape(2 * ch, 2 * cw), -1, 2 * ch, 2 * cw
                j = 1 if where == 0 else 0
                dst = h_out.numpy() if k + 1 == len(steps) else bufs[j][:cw * ch].reshape(ch, cw)
                ctx.convert_plane(model, cur, block_splitting=True, out=dst)
                cur, where = dst, j

        def host_chain():
            ctx.convert_chain(steps, h_in.numpy(), out=h_out.numpy())

        arms = {"device_loop": (dev_loop, lambda: d_out.cpu().numpy()), "device_chain": (dev_chain, lambda: d_out.cpu().numpy()),
                "host_loop": (host_loop, lambda: h_out.numpy().copy()), "host_chain": (host_chain, lambda: h_out.numpy().copy())}
        outputs = {}
        for arm, (fn, fetch) in arms.items():
            d_out.zero_()
            h_out.zero_()
            torch.cuda.synchronize()
            for _ in range(args.warmup + 1):
                fn()
            stream.synchronize()
            outputs[arm] = fetch()
        ms = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                stream.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    arms[arm][0]()
                stream.synchronize()
                ms[arm].append((time.perf_counter() - t0) * 1e3 / args.reps)
        res = result["workloads"][name] = {"input": [w, h], "output": [W, H], "steps": pattern, "arms": {}}
        for arm in arms:
            ref = "device_loop" if arm.startswith("device") else "host_loop"
            med = statistics.median(ms[arm])
            res["arms"][arm] = {"ms": round(med, 2), "ms_rounds": [round(v, 2) for v in ms[arm]], "out_mpix_s": round(W * H / med / 1e3, 1),
                                "bit_identical_to_loop": bool(np.array_equal(outputs[arm], outputs[ref]))}
        res["device_and_host_identical"] = bool(np.array_equal(outputs["device_loop"], outputs["host_loop"]))
        del d_in, d_bufs, d_out, h_in, h_bufs, h_out
        torch.cuda.empty_cache()
    ctx.set_stream(0)
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "chain_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
