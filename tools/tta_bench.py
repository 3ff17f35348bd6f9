"""tta_bench.py -- test-time augmentation as a chain step flag against the loop a user writes without it, in one process:

    python tools/tta_bench.py [--rounds 3] [--out DIR]

Workloads (uniform [0,1) noise planes from a seed, default precision, tensor-core engine):
  noise1_1080p        one 1920 x 1080 plane, noise1
  noise_scale_1080p   the same plane through noise1 + scale2.0x, as a chain
  A                   tools/planes_bench.py's collection A (2000 planes, sides in [16, 128]), scale2.0x
Arms per workload, each device-resident (dense device buffers, *_device entry points) and host-to-host (pinned host planes):
  tta    one call with W2X_STEP_TTA on every step: convert_chain(_device) for one plane, convert_planes_chain(_device) for A
  loop   per plane and step: the 8 flipped / transposed planes (torch on the device, numpy on the host), 8 convert_plane(_device)
         calls, the outputs flipped back and summed in float32 in variant order, times 0.125 -- what a user writes today
Before timing, every arm's outputs are compared bit for bit with the device loop's.  Each arm is warmed up; every round runs all arms
in turn (the order rotates), timed by the wall clock from a synchronised context to a synchronised context.  Reported per arm: the
median and spread of the call time over the rounds, output Mpix/s, launches per call, and for the tta arms the share of the call's
kernel time spent in tta_variants_kernel and tta_mean_kernel (torch.profiler, in a separate pass after the timed rounds).  The card's
name, power limit and maximum SM clock are read in the same run.  Prints one JSON line (and writes it to DIR/tta_bench.json).
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

TTA_KERNELS = ("tta_variants_kernel", "tta_mean_kernel")


def variant_np(x, j):
    v = x.T if j & 4 else x
    if j & 2:
        v = v[::-1, :]
    if j & 1:
        v = v[:, ::-1]
    return np.array(v, order="C", copy=True)


def unvariant_np(o, j):
    if j & 1:
        o = o[:, ::-1]
    if j & 2:
        o = o[::-1, :]
    return o.T if j & 4 else o


def variant_t(x, j):
    v = x.t() if j & 4 else x
    if j & 2:
        v = v.flip(0)
    if j & 1:
        v = v.flip(1)
    return v.contiguous()


def unvariant_t(o, j):
    if j & 1:
        o = o.flip(1)
    if j & 2:
        o = o.flip(0)
    return o.t() if j & 4 else o


def mean8(outs):
    acc = outs[0]
    for o in outs[1:]:
        acc = acc + o
    return acc * 0.125


class Planes:
    """n planes (sizes (w, h)) through `steps` ((model, upscale) pairs): inputs and outputs dense on the device and pinned on the host"""

    def __init__(self, sizes, steps, seed):
        self.sizes, self.steps = sizes, steps
        self.u = sum(1 for _, up in steps if up)
        self.out_sizes = [(w << self.u, h << self.u) for w, h in sizes]
        self.ioff = np.concatenate([[0], np.cumsum([w * h for w, h in sizes])]).astype(int)
        self.ooff = np.concatenate([[0], np.cumsum([w * h for w, h in self.out_sizes])]).astype(int)
        flat = np.random.default_rng(seed).random(int(self.ioff[-1]), dtype=np.float32)
        self.d_in = torch.from_numpy(flat).cuda()
        self.d_out = torch.zeros(int(self.ooff[-1]), device="cuda")
        self.h_in = torch.from_numpy(flat).pin_memory()
        self.h_out = torch.zeros(int(self.ooff[-1])).pin_memory()
        self.pix = int(self.ooff[-1])

    def view(self, t, i, out):
        off, (w, h) = (self.ooff, self.out_sizes[i]) if out else (self.ioff, self.sizes[i])
        return t[int(off[i]):int(off[i + 1])].view(h, w)

    def ptr(self, t, i, out):
        return t.data_ptr() + int((self.ooff if out else self.ioff)[i]) * 4


def arms_for(ctx, p, stream):
    n = len(p.sizes)
    tta_steps = [(m, up, True) for m, up in p.steps]
    ws, hs = [w for w, _ in p.sizes], [h for _, h in p.sizes]
    h_in = [p.view(p.h_in, i, False).numpy() for i in range(n)]
    h_out = [p.view(p.h_out, i, True).numpy() for i in range(n)]

    def dev_tta():
        if n == 1:
            w, h = p.sizes[0]
            ctx.convert_chain_device(tta_steps, p.d_in.data_ptr(), w, h, w * 4, p.d_out.data_ptr(), (w << p.u) * 4, block_splitting=False)
        else:
            ctx.convert_planes_chain_device(tta_steps, [p.ptr(p.d_in, i, False) for i in range(n)], ws, hs, [w * 4 for w in ws],
                                            [p.ptr(p.d_out, i, True) for i in range(n)], [(w << p.u) * 4 for w in ws])

    def host_tta():
        if n == 1:
            ctx.convert_chain(tta_steps, h_in[0], out=h_out[0], block_splitting=False)
        else:
            ctx.convert_planes_chain(tta_steps, h_in, out=h_out)

    def dev_loop():
        with torch.cuda.stream(stream):
            for i in range(n):
                y = p.view(p.d_in, i, False)
                for model, up in p.steps:
                    src = y.repeat_interleave(2, 0).repeat_interleave(2, 1) if up else y
                    outs = []
                    for j in range(8):
                        v = variant_t(src, j)
                        o = torch.empty_like(v)
                        ctx.convert_plane_device(model, v.data_ptr(), v.shape[1], v.shape[0], v.shape[1] * 4, o.data_ptr(), v.shape[1] * 4, False)
                        outs.append(unvariant_t(o, j))
                    y = mean8(outs)
                p.view(p.d_out, i, True).copy_(y)

    def host_loop():
        for i in range(n):
            y = h_in[i]
            for model, up in p.steps:
                src = np.repeat(np.repeat(y, 2, 0), 2, 1) if up else y
                y = mean8([unvariant_np(ctx.convert_plane(model, variant_np(src, j), block_splitting=False), j) for j in range(8)])
            h_out[i][...] = y

    return {"device_tta": (dev_tta, lambda: p.d_out.cpu().numpy().copy(), p.d_out),
            "device_loop": (dev_loop, lambda: p.d_out.cpu().numpy().copy(), p.d_out),
            "host_tta": (host_tta, lambda: p.h_out.numpy().copy(), p.h_out),
            "host_loop": (host_loop, lambda: p.h_out.numpy().copy(), p.h_out)}


def tta_kernel_share(ctx, fn):
    """share of the call's kernel time spent in the two TTA kernels (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.synchronize()
    total, tta, seen = 0.0, 0.0, 0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if getattr(e, "device_type", None) is not None and "CUDA" not in str(e.device_type):
            continue
        total += t
        if any(k in e.key for k in TTA_KERNELS):
            tta += t
            seen += e.count
    return {"tta_kernels_us": round(tta, 1), "all_kernels_us": round(total, 1), "share": round(tta / total, 4) if total else None,
            "tta_kernel_launches_seen": seen}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tta_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)    # the device loop's torch transforms and the library's kernels share one stream
    noise, scale = load_model(w2x, "noise1"), load_model(w2x, "scale2.0x")
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "rounds": args.rounds, "workloads": {}}
    for name, sizes, steps in (("noise1_1080p", [(1920, 1080)], [(noise, False)]),
                               ("noise_scale_1080p", [(1920, 1080)], [(noise, False), (scale, True)]),
                               ("A", workload("A", 1), [(scale, True)])):
        p = Planes(sizes, steps, 7)
        arms = arms_for(ctx, p, stream)
        outputs, launches = {}, {}
        for arm, (fn, fetch, buf) in arms.items():   # warm-up, launch count and outputs of every arm
            buf.zero_()
            torch.cuda.synchronize()
            for _ in range(args.warmup):
                fn()
            ctx.synchronize()
            torch.cuda.synchronize()
            n0 = ctx.launch_count()
            fn()
            ctx.synchronize()
            torch.cuda.synchronize()
            launches[arm] = ctx.launch_count() - n0
            outputs[arm] = fetch()
        secs = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                ctx.synchronize()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                arms[arm][0]()
                ctx.synchronize()
                torch.cuda.synchronize()
                secs[arm].append(time.perf_counter() - t0)
        w = result["workloads"][name] = {"planes": len(sizes), "output_megapixels": round(p.pix / 1e6, 3),
                                         "steps": ["scale2.0x (2x)" if up else "noise1" for _, up in steps], "arms": {}}
        for arm in arms:
            med = statistics.median(secs[arm])
            w["arms"][arm] = {"ms": round(med * 1e3, 2), "ms_rounds": [round(s * 1e3, 2) for s in secs[arm]],
                              "spread_ms": round((max(secs[arm]) - min(secs[arm])) * 1e3, 2), "mpix_s": round(p.pix / med / 1e6, 1),
                              "launches_per_call": launches[arm], "bit_identical_to_device_loop": bool(np.array_equal(outputs[arm], outputs["device_loop"]))}
        for side in ("device", "host"):
            w[f"{side}_loop_over_tta"] = round(w["arms"][f"{side}_loop"]["ms"] / w["arms"][f"{side}_tta"]["ms"], 2)
            w["arms"][f"{side}_tta"]["tta_kernels"] = tta_kernel_share(ctx, arms[f"{side}_tta"][0])
        del p, arms
        torch.cuda.empty_cache()
    # the cost of TTA itself: a plain chain call on the 1080p plane, for the "about 8x" comparison
    p = Planes([(1920, 1080)], [(noise, False)], 7)
    plain = lambda: ctx.convert_chain_device([(noise, False)], p.d_in.data_ptr(), 1920, 1080, 1920 * 4, p.d_out.data_ptr(), 1920 * 4,  # noqa: E731
                                             block_splitting=False)
    plain()
    ctx.synchronize()
    ts = []
    for _ in range(max(3, args.rounds)):
        t0 = time.perf_counter()
        plain()
        ctx.synchronize()
        ts.append(time.perf_counter() - t0)
    result["plain_noise1_1080p_device_ms"] = round(statistics.median(ts) * 1e3, 2)
    result["tta_over_plain_noise1_1080p_device"] = round(result["workloads"]["noise1_1080p"]["arms"]["device_tta"]["ms"] / (statistics.median(ts) * 1e3), 2)
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tta_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
