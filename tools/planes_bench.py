"""planes_bench.py -- many independent planes: one w2x_convert_planes call against a loop of w2x_convert_plane, in one process:

    python tools/planes_bench.py [--rounds 3] [--out DIR]

Seeded workloads (uniform [0,1) noise planes, default precision, tensor-core engine):
  A   2000 planes, width and height uniform in [16, 128], scale2.0x
  B   500 planes, width and height uniform in [64, 512], scale2.0x
  C   config 5: 64 planes of 512 x 512, noise2 -- also through w2x_convert_tiles, the same-shape batch
Arms per workload, each device-resident (dense device buffers, *_device entry points) and host-to-host (pinned host planes):
  loop     one convert_plane call per plane (block_splitting = 0)
  planes   one convert_planes call for the whole collection
  tiles    (C only) one convert_tiles call
Each arm is warmed up; then every round runs all arms in turn (the order rotates from round to round), timed by the wall clock
from a synchronised context to a synchronised context.  Reported per arm: output Mpix/s of every round, their median and
spread, launches per call, and whether every output plane is bit-identical to the loop's.  The card's name, power limit and
maximum SM clock are read in the same run.  Prints one JSON line (and writes it to DIR/planes_bench.json).
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


def workload(name, seed):
    rng = np.random.default_rng(seed)
    if name == "A":
        sizes = rng.integers(16, 129, size=(2000, 2))
    elif name == "B":
        sizes = rng.integers(64, 513, size=(500, 2))
    else:
        sizes = np.full((64, 2), 512)
    return [(int(w), int(h)) for w, h in sizes]


class Collection:
    """The planes of one workload: dense on the device (input and output buffers) and in pinned host memory."""

    def __init__(self, sizes, seed):
        self.sizes = sizes
        self.off = np.concatenate([[0], np.cumsum([w * h for w, h in sizes])])
        total = int(self.off[-1])
        flat = np.random.default_rng(seed).random(total, dtype=np.float32)
        self.d_in = torch.from_numpy(flat).cuda()
        self.d_out = torch.zeros(total, device="cuda")
        self.h_in = torch.from_numpy(flat).pin_memory()
        self.h_out = torch.zeros(total).pin_memory()
        self.ws = [w for w, _ in sizes]
        self.hs = [h for _, h in sizes]
        self.pix = total

    def ptr(self, t, i):
        return t.data_ptr() + int(self.off[i]) * 4

    def host_planes(self, t):
        a = t.numpy()
        return [a[self.off[i]:self.off[i + 1]].reshape(h, w) for i, (w, h) in enumerate(self.sizes)]

    def device_result(self):
        return self.d_out.cpu().numpy().copy()

    def host_result(self):
        return self.h_out.numpy().copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("planes_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    models = {"scale2.0x": load_model(w2x, "scale2.0x"), "noise2": load_model(w2x, "noise2")}
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "rounds": args.rounds, "workloads": {}}
    for name, seed, mname in (("A", 1, "scale2.0x"), ("B", 2, "scale2.0x"), ("C", 3, "noise2")):
        model = models[mname]
        c = Collection(workload(name, seed), 100 + seed)
        n = len(c.sizes)
        hin, hout = c.host_planes(c.h_in), c.host_planes(c.h_out)
        strides = [w * 4 for w in c.ws]

        def dev_loop():
            for i, (w, h) in enumerate(c.sizes):
                ctx.convert_plane_device(model, c.ptr(c.d_in, i), w, h, w * 4, c.ptr(c.d_out, i), w * 4, False)

        def dev_planes():
            ctx.convert_planes_device(model, [c.ptr(c.d_in, i) for i in range(n)], c.ws, c.hs, strides,
                                      [c.ptr(c.d_out, i) for i in range(n)], strides)

        def host_loop():
            for i in range(n):
                ctx.convert_plane(model, hin[i], block_splitting=False, out=hout[i])

        def host_planes():
            ctx.convert_planes(model, hin, out=hout)

        arms = {"device_loop": (dev_loop, c.device_result), "device_planes": (dev_planes, c.device_result),
                "host_loop": (host_loop, c.host_result), "host_planes": (host_planes, c.host_result)}
        if name == "C":
            T = c.sizes[0][0]
            arms["device_tiles"] = (lambda: ctx.convert_tiles_device(model, c.d_in.data_ptr(), c.d_out.data_ptr(), n, T, T), c.device_result)
            arms["host_tiles"] = (lambda: ctx.convert_tiles(model, c.h_in.numpy().reshape(n, T, T), out=c.h_out.numpy().reshape(n, T, T)),
                                  c.host_result)
        outputs, launches = {}, {}
        for arm, (fn, fetch) in arms.items():   # warm-up, launch count and outputs of every arm
            c.d_out.zero_()
            c.h_out.zero_()
            torch.cuda.synchronize()
            for _ in range(args.warmup):
                fn()
            ctx.synchronize()
            n0 = ctx.launch_count()
            fn()
            ctx.synchronize()
            launches[arm] = ctx.launch_count() - n0
            outputs[arm] = fetch()
        mpix = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                ctx.synchronize()
                t0 = time.perf_counter()
                arms[arm][0]()
                ctx.synchronize()
                mpix[arm].append(c.pix / (time.perf_counter() - t0) / 1e6)
        w = result["workloads"][name] = {"planes": n, "megapixels": round(c.pix / 1e6, 3), "model": mname, "arms": {}}
        for arm in arms:
            ref = "device_loop" if arm.startswith("device") else "host_loop"
            w["arms"][arm] = {"mpix_s": round(statistics.median(mpix[arm]), 1), "mpix_s_rounds": [round(v, 1) for v in mpix[arm]],
                              "spread": round(max(mpix[arm]) - min(mpix[arm]), 1), "launches_per_call": launches[arm],
                              "bit_identical_to_loop": bool(np.array_equal(outputs[arm], outputs[ref]))}
        w["device_and_host_identical"] = bool(np.array_equal(outputs["device_loop"], outputs["host_loop"]))
        del c
        torch.cuda.empty_cache()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "planes_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
