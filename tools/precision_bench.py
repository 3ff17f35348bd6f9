"""precision_bench.py -- the tensor-core engine's three precisions side by side, in one process:

    python tools/precision_bench.py [--size 4096] [--rounds 3] [--steps 5] [--out DIR]

Workloads, both on device-resident data:
  plane   one size x size fp32 Y plane, scale2.0x weights (w2x_convert_plane_device)
  cfg5    64 tiles of 512 x 512, noise2 weights, one batched pass (w2x_convert_tiles_device)
Every precision is warmed up first; then each round runs every precision in turn (the order rotates from round to round),
`steps` back-to-back passes timed with CUDA events.  Reported per precision: Mpix/s of every round and their median, and
per-layer ms (w2x_ctx_layer_times, from a separate pass with the layer timers on).  Accuracy against the fp32 engine on
the same plane, over a seeded sample of rows: max-abs, and the share of values that change after rint(255 y).  The card's
name, power limit and maximum SM clock are read in the same run.  Prints one JSON line (and writes it to DIR/precision_bench.json).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import w2x_loader  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                             # the figures then stand without the card's limits
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "max_sm_clock": None, "nvidia_smi": repr(e)}


def load_model(w2x, name):
    z = np.load(os.path.join(ROOT, "tests", "golden", "models", f"{name}_model.npz"))
    n = int(z["n_layers"])
    return w2x.Model.from_arrays([z[f"w{i}"] for i in range(n)], [z[f"b{i}"] for i in range(n)])


def timed_ms(fn, steps):
    """ms per call over `steps` back-to-back calls: CUDA events on the stream the contexts run on"""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample-rows", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("precision_bench.py needs a CUDA device")
    w2x = w2x_loader.load()
    precs = {"f16x3": w2x.PRECISION_F16X3, "f16+f8x2": w2x.PRECISION_F16_F8X2, "f16": w2x.PRECISION_F16}
    stream = torch.cuda.Stream()                                      # the contexts run on it, the CUDA events are recorded on it
    torch.cuda.set_stream(stream)
    ctxs = {}
    for name, p in precs.items():
        ctxs[name] = w2x.Context(0, engine=w2x.ENGINE_TC)
        ctxs[name].set_precision(p)
        ctxs[name].set_stream(stream.cuda_stream)
    scale, noise2 = load_model(w2x, "scale2.0x"), load_model(w2x, "noise2")

    S = args.size
    x = np.random.default_rng(1).random((S, S), dtype=np.float32)
    d_in = torch.from_numpy(x).cuda()
    d_out = torch.empty_like(d_in)
    n_tiles, T = 64, 512
    d5_in = torch.from_numpy(np.random.default_rng(3).random((n_tiles, T, T), dtype=np.float32)).cuda()
    d5_out = torch.empty_like(d5_in)

    def plane(ctx):
        return lambda: ctx.convert_plane_device(scale, d_in.data_ptr(), S, S, S * 4, d_out.data_ptr(), S * 4, True)

    def cfg5(ctx):
        return lambda: ctx.convert_tiles_device(noise2, d5_in.data_ptr(), d5_out.data_ptr(), n_tiles, T, T)

    # accuracy on the plane: every precision and the fp32 engine over the same seeded rows
    rows = np.sort(np.random.default_rng(7).choice(S, size=min(args.sample_rows, S), replace=False))
    fp32 = w2x.Context(0, engine=w2x.ENGINE_FP32)
    plane(fp32)()
    fp32.synchronize()
    ref = d_out[torch.from_numpy(rows).cuda()].cpu().numpy().astype(np.float64)
    fp32.close()
    accuracy = {}
    for name, ctx in ctxs.items():
        plane(ctx)()
        ctx.synchronize()
        y = d_out[torch.from_numpy(rows).cuda()].cpu().numpy().astype(np.float64)
        u8 = lambda a: np.clip(np.rint(a * 255.0), 0, 255)               # noqa: E731
        d8 = np.abs(u8(y) - u8(ref))
        accuracy[name] = {"max_abs_vs_fp32_engine": float(np.abs(y - ref).max()), "u8_max_diff": int(d8.max()),
                          "u8_changed_share": float((d8 > 0).mean())}

    for ctx in ctxs.values():                                           # warm-up: every shape of both workloads
        for _ in range(args.warmup):
            plane(ctx)()
            cfg5(ctx)()
        ctx.synchronize()
    names = list(precs)
    mpix = {n: {"plane": [], "cfg5": []} for n in names}
    for r in range(args.rounds):
        for name in names[r % len(names):] + names[:r % len(names)]:
            ctx = ctxs[name]
            ms = timed_ms(plane(ctx), args.steps)
            mpix[name]["plane"].append(S * S / (ms * 1e-3) / 1e6)
            ms5 = timed_ms(cfg5(ctx), args.steps)
            mpix[name]["cfg5"].append(n_tiles * T * T / (ms5 * 1e-3) / 1e6)
    result = {"gpu": gpu_info(), "workloads": {"plane": f"{S}x{S} fp32 Y plane, scale2.0x, device-resident",
                                                "cfg5": f"{n_tiles} tiles of {T}x{T}, noise2, one batched pass, device-resident"},
              "rounds": args.rounds, "steps": args.steps, "accuracy_rows": len(rows), "precisions": {}}
    for name, ctx in ctxs.items():
        ctx.set_timing(True)
        plane(ctx)()
        layers = [(round(ms, 3), kname) for ms, _, kname in ctx.layer_times()]
        ctx.set_timing(False)
        result["precisions"][name] = {
            "plane_mpix_s": round(statistics.median(mpix[name]["plane"]), 1), "plane_mpix_s_rounds": [round(v, 1) for v in mpix[name]["plane"]],
            "cfg5_mpix_s": round(statistics.median(mpix[name]["cfg5"]), 1), "cfg5_mpix_s_rounds": [round(v, 1) for v in mpix[name]["cfg5"]],
            "layer_times": layers, **accuracy[name]}
    for ctx in ctxs.values():
        ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "precision_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
