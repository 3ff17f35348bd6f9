"""regions_bench.py -- many windows of chains' outputs: one w2x_convert_chain_regions call against a loop of w2x_convert_chain_region,
in one process:

    python tools/regions_bench.py [--rounds 5] [--out DIR]

Seeded workloads (uniform [0,1) noise planes, default precision, tensor-core engine):
  A  tiled scan: a 4096 x 4096 plane through noise1 + scale2.0x, its 8192 x 8192 output cut into 1024 tiles of 256 x 256
  B  viewer: 12 windows of 512 x 512 at fixed, scattered positions of that output, odd and even rows and columns
  C  dataset patches: 256 windows of 128 x 128, 16 at seeded positions on each of 16 planes of 1024 x 768, scale2.0x only
Arms per workload, each device-resident (the whole planes on the device, *_device entry points, windows into device buffers) and
host-to-host (pinned host planes, source rectangles passed as views of them, windows into pinned buffers):
  loop     one convert_chain_region call per window
  regions  one convert_chain_regions call for every window
  whole    (A only) one convert_chain call on the whole plane (block_splitting = 0), the tiles being views of its output
Each arm is warmed up; then every round runs all arms of a workload in turn (the order rotates from round to round), one call each,
timed by the wall clock from a synchronised stream to a synchronised stream.  Reported per arm: the median milliseconds per call and
every round's, launches per call, and whether every window is bit-identical to the whole chain's crop.  The card's name, power limit
and maximum SM clock are read in the same run.  Prints one JSON line (and writes it to DIR/regions_bench.json).
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

VIEWER = [(0, 0), (3001, 2047), (7680, 7680), (1234, 5677), (4095, 1), (6000, 3333), (512, 7001), (2222, 2223), (7001, 400),
          (5120, 6143), (99, 3500), (3999, 4001)]


def workloads(w2x, seed):
    """name -> (steps, planes, [(plane index, window)])"""
    noise1, scale = load_model(w2x, "noise1"), load_model(w2x, "scale2.0x")
    rng = np.random.default_rng(seed)
    scan = rng.random((4096, 4096), dtype=np.float32)
    tiles = [(0, (x, y, 256, 256)) for y in range(0, 8192, 256) for x in range(0, 8192, 256)]
    viewer = [(0, (x, y, 512, 512)) for x, y in VIEWER]
    pages = [rng.random((768, 1024), dtype=np.float32) for _ in range(16)]
    patches = [(p, (int(rng.integers(0, 2048 - 128 + 1)), int(rng.integers(0, 1536 - 128 + 1)), 128, 128)) for p in range(16) for _ in range(16)]
    two = [(noise1, False), (scale, True)]
    return {"A": (two, [scan], tiles), "B": (two, [scan], viewer), "C": ([(scale, True)], pages, patches)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("regions_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "engine": "tensor-core", "rounds": args.rounds, "workloads": {}}
    for name, (steps, planes, wins) in workloads(w2x, 2026).items():
        ups = sum(1 for _, up in steps if up)
        sizes = [(planes[p].shape[1], planes[p].shape[0]) for p, _ in wins]
        rects = [w2x.chain_region_source(steps, size, win) for size, (_, win) in zip(sizes, wins)]
        d_planes = [torch.from_numpy(x).cuda() for x in planes]
        h_planes = [torch.from_numpy(x).pin_memory() for x in planes]
        d_whole = [torch.empty((x.shape[0] << ups, x.shape[1] << ups), device="cuda") for x in planes]
        h_whole = [torch.empty((x.shape[0] << ups, x.shape[1] << ups)).pin_memory() for x in planes]
        d_win = [torch.empty((win[3], win[2]), device="cuda") for _, win in wins]
        h_win = [torch.empty((win[3], win[2])).pin_memory() for _, win in wins]
        h_src = [h_planes[p].numpy()[sy0:sy0 + sh, sx0:sx0 + sw] for (p, _), (sx0, sy0, sw, sh) in zip(wins, rects)]
        d_src = [d_planes[p].data_ptr() + (sy0 * d_planes[p].shape[1] + sx0) * 4 for (p, _), (sx0, sy0, _, _) in zip(wins, rects)]
        src_st = [d_planes[p].shape[1] * 4 for p, _ in wins]
        windows = [win for _, win in wins]

        def dev_loop():
            for s, size, win, st, o in zip(d_src, sizes, windows, src_st, d_win):
                ctx.convert_chain_region_device(steps, s, size, win, st, o.data_ptr(), win[2] * 4)

        def dev_regions():
            ctx.convert_chain_regions_device(steps, d_src, sizes, windows, src_st, [o.data_ptr() for o in d_win], [w[2] * 4 for w in windows])

        def dev_whole():
            for x, o in zip(d_planes, d_whole):
                ctx.convert_chain_device(steps, x.data_ptr(), x.shape[1], x.shape[0], x.shape[1] * 4, o.data_ptr(), o.shape[1] * 4,
                                         block_splitting=False)

        def host_loop():
            for s, size, win, o in zip(h_src, sizes, windows, h_win):
                ctx.convert_chain_region(steps, s, size, win, out=o.numpy())

        def host_regions():
            ctx.convert_chain_regions(steps, h_src, sizes, windows, out=[o.numpy() for o in h_win])

        def host_whole():
            for x, o in zip(h_planes, h_whole):
                ctx.convert_chain(steps, x.numpy(), out=o.numpy(), block_splitting=False)

        def crops(whole):
            return [whole[p][y0:y0 + h, x0:x0 + w] for p, (x0, y0, w, h) in wins]

        arms = {"device_loop": (dev_loop, lambda: [o.cpu().numpy() for o in d_win]),
                "device_regions": (dev_regions, lambda: [o.cpu().numpy() for o in d_win]),
                "host_loop": (host_loop, lambda: [o.numpy().copy() for o in h_win]),
                "host_regions": (host_regions, lambda: [o.numpy().copy() for o in h_win])}
        if name == "A":
            arms["device_whole"] = (dev_whole, lambda: crops([o.cpu().numpy() for o in d_whole]))
            arms["host_whole"] = (host_whole, lambda: crops([o.numpy() for o in h_whole]))
        dev_whole()                                         # the reference: the whole chain's crops
        stream.synchronize()
        want = crops([o.cpu().numpy() for o in d_whole])
        launches, same = {}, {}
        for arm, (fn, fetch) in arms.items():
            for o in d_win:
                o.fill_(np.nan)
            for o in h_win:
                o.fill_(np.nan)
            torch.cuda.synchronize()
            for _ in range(args.warmup):
                fn()
            stream.synchronize()
            n0 = ctx.launch_count()
            fn()
            stream.synchronize()
            launches[arm] = ctx.launch_count() - n0
            same[arm] = all(np.array_equal(g, e) for g, e in zip(fetch(), want))
        ms = {arm: [] for arm in arms}
        names = list(arms)
        for r in range(args.rounds):
            for arm in names[r % len(names):] + names[:r % len(names)]:
                stream.synchronize()
                t0 = time.perf_counter()
                arms[arm][0]()
                stream.synchronize()
                ms[arm].append((time.perf_counter() - t0) * 1e3)
        res = {"steps": ", ".join(("scale2.0x" if up else "noise1") for _, up in steps), "planes": [list(x.shape[::-1]) for x in planes[:1]],
               "n_planes": len(planes), "n_windows": len(wins), "window": list(windows[0][2:]), "arms": {}}
        for arm in arms:
            res["arms"][arm] = {"ms": round(statistics.median(ms[arm]), 2), "ms_rounds": [round(v, 2) for v in ms[arm]],
                                "launches": launches[arm], "bit_identical_to_whole_crop": same[arm]}
        result["workloads"][name] = res
        del d_planes, h_planes, d_whole, h_whole, d_win, h_win, h_src
        torch.cuda.empty_cache()
    ctx.set_stream(0)
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "regions_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
