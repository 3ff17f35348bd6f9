"""planes_chain_bench.py -- a collection of planes through noise reduction and 2x scaling: one w2x_convert_planes_chain call against
a loop of w2x_convert_chain and against the per-step loop of w2x_convert_planes, in one process:

    python tools/planes_chain_bench.py [--rounds 3] [--out DIR]

Seeded workloads (the planes of tools/planes_bench.py, same seeds; default precision, tensor-core engine):
  A_SU    workload A (2000 planes, sides 16-128) through noise1 then scale2.0x
  B_SU    workload B (500 planes, sides 64-512) through noise1 then scale2.0x
  A_SUU   workload A through noise1 then scale2.0x twice
Arms per workload, each device-resident (dense device buffers, *_device entry points, one torch stream shared with the context) and
host-to-host (pinned host planes):
  chain_loop   one convert_chain call per plane (block_splitting = 0)
  step_loop    per step one convert_planes call, the nearest 2x resize between steps in torch (repeat_interleave, device) or numpy
               (np.repeat, host)
  planes_chain one convert_planes_chain call for the whole collection
Each arm is warmed up; then every round runs all arms in turn (the order rotates from round to round), timed by the wall clock from
a synchronised context to a synchronised context.  Reported per arm: output Mpix/s of every round, their median and spread,
launches per call, and whether every output plane is bit-identical to the device chain loop's.  The card's name, power limit and
maximum SM clock are read in the same run.  Prints one JSON line (and writes it to DIR/planes_chain_bench.json).
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


class Collection:
    """The planes of one workload and their outputs (u 2x steps): dense on the device and in pinned host memory."""

    def __init__(self, sizes, seed, ups):
        self.sizes, self.ups = sizes, ups
        self.off = np.concatenate([[0], np.cumsum([w * h for w, h in sizes])])
        self.out_off = self.off << (2 * ups)
        flat = np.random.default_rng(seed).random(int(self.off[-1]), dtype=np.float32)
        self.d_in = torch.from_numpy(flat).cuda()
        self.d_out = torch.zeros(int(self.out_off[-1]), device="cuda")
        self.h_in = torch.from_numpy(flat).pin_memory()
        self.h_out = torch.zeros(int(self.out_off[-1])).pin_memory()
        self.ws = [w for w, _ in sizes]
        self.hs = [h for _, h in sizes]
        self.out_pix = int(self.out_off[-1])

    def d_planes(self, t, off, s):
        return [t[int(off[i]):int(off[i + 1])].view(h << s, w << s) for i, (w, h) in enumerate(self.sizes)]

    def h_planes(self, t, off, s):
        a = t.numpy()
        return [a[off[i]:off[i + 1]].reshape(h << s, w << s) for i, (w, h) in enumerate(self.sizes)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("planes_chain_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)      # torch's resizes and the library's kernels in one stream order
    noise, scale = load_model(w2x, "noise1"), load_model(w2x, "scale2.0x")
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "rounds": args.rounds, "workloads": {}}
    for name, wl, seed, pattern in (("A_SU", "A", 1, "SU"), ("B_SU", "B", 2, "SU"), ("A_SUU", "A", 1, "SUU")):
        steps = [(noise, False) if ch == "S" else (scale, True) for ch in pattern]
        ups = pattern.count("U")
        c = Collection(workload(wl, seed), 100 + seed, ups)
        n = len(c.sizes)
        d_in, d_out = c.d_planes(c.d_in, c.off, 0), c.d_planes(c.d_out, c.out_off, ups)
        h_in, h_out = c.h_planes(c.h_in, c.off, 0), c.h_planes(c.h_out, c.out_off, ups)
        in_strides, out_strides = [w * 4 for w in c.ws], [(w << ups) * 4 for w in c.ws]

        def dev_chain_loop():
            for i, (w, h) in enumerate(c.sizes):
                ctx.convert_chain_device(steps, d_in[i].data_ptr(), w, h, w * 4, d_out[i].data_ptr(), (w << ups) * 4, block_splitting=False)

        def dev_step_loop():
            with torch.cuda.stream(stream):
                ys = d_in
                for k, (model, up) in enumerate(steps):
                    xs = [y.repeat_interleave(2, 0).repeat_interleave(2, 1) if up else y for y in ys]
                    outs = d_out if k + 1 == len(steps) else [torch.empty_like(x) for x in xs]
                    ctx.convert_planes_device(model, [x.data_ptr() for x in xs], [x.shape[1] for x in xs], [x.shape[0] for x in xs],
                                              [x.shape[1] * 4 for x in xs], [o.data_ptr() for o in outs], [x.shape[1] * 4 for x in xs])
                    ys = outs

        def dev_planes_chain():
            ctx.convert_planes_chain_device(steps, [x.data_ptr() for x in d_in], c.ws, c.hs, in_strides, [o.data_ptr() for o in d_out],
                                            out_strides)

        def host_chain_loop():
            for i in range(n):
                ctx.convert_chain(steps, h_in[i], out=h_out[i], block_splitting=False)

        def host_step_loop():
            ys = h_in
            for k, (model, up) in enumerate(steps):
                xs = [np.repeat(np.repeat(y, 2, 0), 2, 1) if up else y for y in ys]
                ys = ctx.convert_planes(model, xs, out=h_out if k + 1 == len(steps) else None)

        def host_planes_chain():
            ctx.convert_planes_chain(steps, h_in, out=h_out)

        device_result = lambda: c.d_out.cpu().numpy().copy()
        host_result = lambda: c.h_out.numpy().copy()
        arms = {"device_chain_loop": (dev_chain_loop, device_result), "device_step_loop": (dev_step_loop, device_result),
                "device_planes_chain": (dev_planes_chain, device_result), "host_chain_loop": (host_chain_loop, host_result),
                "host_step_loop": (host_step_loop, host_result), "host_planes_chain": (host_planes_chain, host_result)}
        same, launches, ref = {}, {}, None
        for arm, (fn, fetch) in arms.items():   # warm-up, launch count and outputs of every arm (the device chain loop's first)
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
            got = fetch()
            ref = got if ref is None else ref
            same[arm] = bool(np.array_equal(got, ref))
            del got
        mpix = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                ctx.synchronize()
                t0 = time.perf_counter()
                arms[arm][0]()
                ctx.synchronize()
                mpix[arm].append(c.out_pix / (time.perf_counter() - t0) / 1e6)
        w = result["workloads"][name] = {"workload": wl, "steps": pattern, "planes": n, "output_megapixels": round(c.out_pix / 1e6, 3),
                                         "arms": {}}
        for arm in arms:
            w["arms"][arm] = {"mpix_s": round(statistics.median(mpix[arm]), 1), "mpix_s_rounds": [round(v, 1) for v in mpix[arm]],
                              "spread": round(max(mpix[arm]) - min(mpix[arm]), 1), "launches_per_call": launches[arm],
                              "bit_identical_to_chain_loop": same[arm]}
        del c, d_in, d_out, h_in, h_out, ref
        torch.cuda.empty_cache()
    ctx.set_stream(0)
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "planes_chain_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
