"""cli_batch_bench.py -- the drop-in CLI on a folder of images: one process per image against one --input_list run:

    python tools/cli_batch_bench.py [--rounds 3] [--workloads A,B] [--jobs 4] [--limit N] [--loop-limit N] [--out DIR]

Seeded workloads (PNG inputs, default precision, tensor-core engine):
  A   64 frames of 1920x1080 (the frame size of BASELINE config 2) through -m noise_scale (noise1 + scale2.0x)
  B   1000 images with sides in [16, 128] through -m scale (scale2.0x)
Arms, alternating within every round (the order swaps from round to round):
  loop    one `w2x-converter -i <image> -o <file>` process per image, one after another (what a shell loop over a folder does)
  batch   one `w2x-converter --input_list <list> -o <dir>` process, with W2X_CLI_TIMING=1 for its timing line
Both arms run with the same flags, including -j.  Before the first round each arm converts the first two images, untimed.  Reported
per arm: the images converted, the wall seconds and images per second of every round, their median and range; for the batch arm its
timing line per round.  Every output of every run of both arms, untimed ones included, must be byte-identical to the first run's file
for that input.  The host's core count and the card's name, power limit and maximum SM clock are read in the same run.  --limit N keeps
the first N images of each workload (a quick rehearsal); --loop-limit N times the loop arm on the first N images only, where a process
per image would take too long for the whole workload (compare images per second then).  Prints one JSON line (and writes it to
DIR/cli_batch_bench.json).
"""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import write_model_json  # noqa: E402

CLI = os.path.join(ROOT, "waifu2x-converter-cpp_b200", "w2x-converter")
WORKLOADS = {"A": ("64 frames of 1920x1080, -m noise_scale (noise1 + scale2.0x)", ["-m", "noise_scale"]),
             "B": ("1000 images with sides in [16, 128], -m scale (scale2.0x)", ["-m", "scale"])}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                             # the figures then stand without the card's limits
        return {"name": None, "power_limit": None, "max_sm_clock": None, "nvidia_smi": repr(e)}


def make_inputs(d, workload, seed=2024):
    import cv2
    rng = np.random.default_rng(seed)
    if workload == "A":
        sizes = [(1920, 1080)] * 64
    else:
        sizes = [tuple(int(v) for v in rng.integers(16, 129, 2)) for _ in range(1000)]
    names = []
    for i, (w, h) in enumerate(sizes):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        ph = rng.random(3) * 6.28
        img = np.stack([128 + 90 * np.sin(xx / (7 + 3 * c) + ph[c]) * np.cos(yy / (5 + 2 * c) - ph[c]) for c in range(3)], -1)
        img += rng.normal(0, 10, img.shape).astype(np.float32)
        names.append(os.path.join(d, f"{workload}_{i:04d}.png"))
        cv2.imwrite(names[-1], np.clip(img, 0, 255).astype(np.uint8))
    return names


def digests(paths):
    out = []
    for p in paths:
        with open(p, "rb") as f:
            out.append(hashlib.sha256(f.read()).hexdigest())
    return out


def run_loop(names, out_dir, flags, model_dir, jobs):
    outs = []
    for i, n in enumerate(names):
        outs.append(os.path.join(out_dir, f"{i:04d}.png"))
        r = subprocess.run([CLI, "-i", n, "-o", outs[-1], "--model_dir", model_dir, "-j", str(jobs), *flags], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"single-image run failed on {n}: {r.stdout}{r.stderr}")
    return outs


def run_batch(names, out_dir, flags, model_dir, jobs):
    lst = out_dir + ".txt"
    with open(lst, "w") as f:
        f.write("\n".join(names) + "\n")
    r = subprocess.run([CLI, "--input_list", lst, "-o", out_dir, "--model_dir", model_dir, "-j", str(jobs), *flags], capture_output=True,
                       text=True, env=dict(os.environ, W2X_CLI_TIMING="1"))
    if r.returncode != 0:
        raise RuntimeError(f"batch run failed: {r.stdout[-2000:]}{r.stderr[-2000:]}")
    timing = [json.loads(l)["w2x_cli_batch_timing_ms"] for l in r.stderr.splitlines() if "w2x_cli_batch_timing_ms" in l]
    lines = r.stdout.splitlines()
    outs = [l.split(" -> ", 1)[1] for l in lines[:-1]]
    assert len(outs) == len(names) and lines[-1] == "process successfully done!"
    return outs, timing[-1]


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "rounds": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="A,B")
    ap.add_argument("--jobs", type=int, default=4)
    ap.add_argument("--limit", type=int, default=None)
    ap.add_argument("--loop-limit", type=int, default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not os.path.exists(CLI):
        raise SystemExit(f"{CLI} is missing: build first")
    tmp = tempfile.mkdtemp(prefix="w2x_cli_batch_")
    try:
        measure(args, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def measure(args, tmp):
    model_dir = os.path.join(tmp, "models")
    os.makedirs(model_dir)
    for name in ("noise1", "scale2.0x"):
        write_model_json(os.path.join(ROOT, "tests", "golden", "models", f"{name}_model.npz"), os.path.join(model_dir, f"{name}_model.json"))
    result = {"host_cores": os.cpu_count(), "gpu": gpu_info(), "jobs": args.jobs, "rounds": args.rounds, "workloads": {}}
    for wl in args.workloads.split(","):
        text, flags = WORKLOADS[wl]
        src = os.path.join(tmp, "in_" + wl)
        os.makedirs(src)
        names = make_inputs(src, wl)[:args.limit]
        arms = {"loop": run_loop, "batch": run_batch}
        images = {"loop": names[:args.loop_limit], "batch": names}
        wall = {a: [] for a in arms}
        timing, ref, identical = [], {}, True
        for r in range(-1, args.rounds):                                # round -1: the first two images, untimed
            order = ["loop", "batch"] if r % 2 == 0 else ["batch", "loop"]
            for arm in order:
                d = os.path.join(tmp, f"{wl}_{arm}_{r + 1}")
                os.makedirs(d)
                subset = names[:2] if r < 0 else images[arm]
                t0 = time.perf_counter()
                res = arms[arm](subset, d, flags, model_dir, args.jobs)
                dt = time.perf_counter() - t0
                print(f"{wl} round {r} {arm}: {len(subset)} images in {dt:.2f} s", file=sys.stderr, flush=True)
                outs = res[0] if arm == "batch" else res
                for n, h in zip(subset, digests(outs)):
                    identical = identical and ref.setdefault(n, h) == h
                if r >= 0:
                    wall[arm].append(dt)
                    if arm == "batch":
                        timing.append(res[1])
                for p in outs:
                    os.remove(p)
        result["workloads"][wl] = {
            "workload": text,
            "images": {a: len(images[a]) for a in arms},
            "wall_s": {a: stats(wall[a]) for a in arms},
            "images_per_s": {a: stats([len(images[a]) / t for t in wall[a]]) for a in arms},
            "batch_timing_ms": timing,
            "outputs_byte_identical": identical,
        }
    line = json.dumps({"cli_batch_bench": result})
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cli_batch_bench.json"), "w") as f:
            f.write(line + "\n")
    if not all(w["outputs_byte_identical"] for w in result["workloads"].values()):
        raise SystemExit("outputs differ between the arms")


if __name__ == "__main__":
    main()
