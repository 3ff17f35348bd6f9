"""region_bench.py -- a window of a chain's output (w2x_convert_chain_region*) against the whole chain plus a crop, in one process:

    python tools/region_bench.py [--rounds 7] [--reps 3] [--out DIR]

Seeded workload (a uniform [0,1) noise plane, default precision, tensor-core engine): noise1 then scale2.0x on a 4096 x 4096 plane,
output 8192 x 8192; the window is 1024 x 1024 of that output at (3001, 2047), odd column and odd row.  Arms:
  device_whole    convert_chain_device on the whole plane (block_splitting = 0), then the window's crop copied out on the device
  device_window   convert_chain_region_device from the source rectangle inside the same device plane
  host_whole      convert_chain on a pinned host plane into a pinned 8192 x 8192 output (the crop is a view)
  host_window     convert_chain_region from the source rectangle (a view of the pinned plane) into a pinned window
Each arm is warmed up; then every round runs all arms in turn (the order rotates from round to round), each arm `reps` calls back to
back, timed by the wall clock from a synchronised stream to a synchronised stream.  Reported per arm: the median milliseconds and every
round's, and whether its window is bit-identical to the whole chain's crop.  The card's name, power limit and maximum SM clock are
read in the same run.  Prints one JSON line (and writes it to DIR/region_bench.json).
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

SIZE = 4096
WINDOW = (3001, 2047, 1024, 1024)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("region_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    stream = torch.cuda.Stream()                        # torch's crop copy and the library's work queue on one (non-default) stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    steps = [(load_model(w2x, "noise1"), False), (load_model(w2x, "scale2.0x"), True)]
    w = h = SIZE
    W, H = 2 * w, 2 * h
    x0, y0, ww, wh = WINDOW
    sx0, sy0, sw, sh = w2x.chain_region_source(steps, (w, h), WINDOW)
    x = np.random.default_rng(4096).random((h, w), dtype=np.float32)
    d_in = torch.from_numpy(x).cuda()
    d_whole = torch.empty((H, W), device="cuda")
    d_win = torch.empty((wh, ww), device="cuda")
    h_in = torch.from_numpy(x.copy()).pin_memory()
    h_whole = torch.empty((H, W)).pin_memory()
    h_win = torch.empty((wh, ww)).pin_memory()

    def dev_whole():
        ctx.convert_chain_device(steps, d_in.data_ptr(), w, h, w * 4, d_whole.data_ptr(), W * 4, block_splitting=False)
        d_win.copy_(d_whole[y0:y0 + wh, x0:x0 + ww])

    def dev_window():
        ctx.convert_chain_region_device(steps, d_in.data_ptr() + (sy0 * w + sx0) * 4, (w, h), WINDOW, w * 4, d_win.data_ptr(), ww * 4)

    def host_whole():
        ctx.convert_chain(steps, h_in.numpy(), out=h_whole.numpy(), block_splitting=False)

    def host_window():
        ctx.convert_chain_region(steps, h_in.numpy()[sy0:sy0 + sh, sx0:sx0 + sw], (w, h), WINDOW, out=h_win.numpy())

    arms = {"device_whole": (dev_whole, lambda: d_win.cpu().numpy()), "device_window": (dev_window, lambda: d_win.cpu().numpy()),
            "host_whole": (host_whole, lambda: h_whole.numpy()[y0:y0 + wh, x0:x0 + ww].copy()),
            "host_window": (host_window, lambda: h_win.numpy().copy())}
    outputs = {}
    for arm, (fn, fetch) in arms.items():
        d_win.zero_()
        h_win.zero_()
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
    result = {"gpu": gpu_info(), "precision": "f16+f8x2 (default)", "input": [w, h], "output": [W, H], "window": list(WINDOW),
              "source_rectangle": [sx0, sy0, sw, sh], "steps": "noise1, scale2.0x", "rounds": args.rounds, "reps": args.reps, "arms": {}}
    for arm in arms:
        result["arms"][arm] = {"ms": round(statistics.median(ms[arm]), 2), "ms_rounds": [round(v, 2) for v in ms[arm]],
                               "bit_identical_to_whole_crop": bool(np.array_equal(outputs[arm], outputs["device_whole"]))}
    ctx.set_stream(0)
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "region_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
