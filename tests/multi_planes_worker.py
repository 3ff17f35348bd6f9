"""multi_planes_worker.py -- runs the cases of tests/test_multi_planes.py in a process of its own (not a test module):

    python tests/multi_planes_worker.py <dir>

Reads <dir>/cases.json, <dir>/models.npz and <dir>/inputs.npz (the files of tests/band_worker.py: plane i of collection c is the input
"c/i"), runs every case and writes the planes to <dir>/out0.npz and everything else to <dir>/log0.json.  It compares nothing: the test
does.  CUDA_DEVICE_MAX_CONNECTIONS is set before CUDA initialises, so that the streams of k contexts of one device do not share
hardware queues.

A case is {id, k, calls}: one w2x_multi of k contexts of device 0 (and, for the reference, one context), the calls in order.  Call ops:
  chain   steps [[model, upscale, tta]], coll, precision, engine (default auto), scratch (bytes, default 1 GiB, on every context and the
          reference: k contexts of one device must not each size frames for the 16 GiB default),
          pinned [input, output], in_pad / out_pad (extra floats per host row), passes (default 2), entry ("chain" or "planes": a
          one-step W2X_STEP_SAME call through Multi.convert_planes)
          -> "<id>.<call>.<pass>.<i>" output plane i (row padding included, which must stay NaN) and "<id>.<call>.ref.<i>" what
          Context.convert_planes_chain on one context made; log "<id>.<call>" = {"passes": [{"events", "launches"}], "ref": {"events",
          "launches"}, "ref_planes": Context.convert_planes' launches and outputs' equality for one-step SAME calls}
  raw     steps, coll, bad: one argument spoiled ("n_steps", "null_model", "kind", "n_planes", "stride", "width") -> log "<id>.<call>" =
          {"multi": [status, message], "one": [status, message], "events": [...], "launches": per-context counts before / after}
  nomem   steps, coll: the call with device 0 all but full, then again with the memory back -> log = {"error", "launches", "untouched",
          "after"}; output "<id>.<call>.after.<i>" and the reference "<id>.<call>.ref.<i>"
"""
import json
import os
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402  (pinned host memory, the NOMEM filler)
import w2x_loader  # noqa: E402

w2x = w2x_loader.load()
d = sys.argv[1]
cases = json.load(open(os.path.join(d, "cases.json")))
inputs = dict(np.load(os.path.join(d, "inputs.npz")))
_mz = np.load(os.path.join(d, "models.npz"))
models = {}
for key in _mz.files:
    name = key.rsplit("/", 1)[0]
    if name not in models:
        nl = sum(1 for k in _mz.files if k.startswith(name + "/w"))
        models[name] = w2x.Model.from_arrays([_mz[f"{name}/w{k}"] for k in range(nl)], [_mz[f"{name}/b{k}"] for k in range(nl)])
outs, log = {}, {}
SCRATCH = 1 << 30


def coll(name):
    n = sum(1 for k in inputs if k.startswith(name + "/"))
    return [inputs[f"{name}/{i}"] for i in range(n)]


def host(shape, pinned):
    if pinned:
        return torch.empty(shape, dtype=torch.float32).pin_memory().numpy()
    return np.empty(shape, np.float32)


def steps_of(call):
    return [(models[m] if m is not None else None, up, tta) for m, up, tta in call["steps"]]


def contexts(multi):
    L = w2x.lib()
    return [L.w2x_multi_ctx(multi._h, i) for i in range(L.w2x_multi_device_count(multi._h))]


def settings(multi, ref, call):
    multi.set_precision(call.get("precision", 1))
    ref.set_precision(call.get("precision", 1))
    L = w2x.lib()
    for c in contexts(multi):
        L.w2x_ctx_set_scratch_limit(c, call.get("scratch", SCRATCH))
    L.w2x_ctx_set_engine(contexts(multi)[0], call.get("engine", 0))
    ref.set_scratch_limit(call.get("scratch", SCRATCH))
    ref.set_engine(call.get("engine", 0))


def run_chain(multi, ref, key, call):
    xs = coll(call["coll"])
    steps = steps_of(call)
    ups = sum(1 for s in call["steps"] if s[1])
    pinned = call.get("pinned", [True, True])
    ip, op = call.get("in_pad", 0), call.get("out_pad", 0)
    h_in = [host((x.shape[0], x.shape[1] + ip), pinned[0]) for x in xs]
    h_out = [host((x.shape[0] << ups, (x.shape[1] << ups) + op), pinned[1]) for x in xs]
    for a, x in zip(h_in, xs):
        a[:] = np.nan
        a[:, :x.shape[1]] = x
    views_in = [a[:, :x.shape[1]] for a, x in zip(h_in, xs)]
    views_out = [a[:, :x.shape[1] << ups] for a, x in zip(h_out, xs)]
    settings(multi, ref, call)
    rec = {"passes": []}
    events = []
    multi.set_log(events.append)
    try:
        for p in range(call.get("passes", 2)):
            for a in h_out:
                a[:] = np.nan
            del events[:]
            before = multi.launch_counts()
            if call.get("entry") == "planes":
                multi.convert_planes(steps[0][0], views_in, out=views_out)
            else:
                multi.convert_planes_chain(steps, views_in, out=views_out, on_step=lambda k: events.append(f"step {k}"))
            rec["passes"].append({"events": list(events), "launches": [a - b for a, b in zip(multi.launch_counts(), before)]})
            for i, a in enumerate(h_out):
                outs[f"{key}.{p}.{i}"] = a.copy()
    finally:
        multi.set_log(None)
    # the one-context call (its second run: the models are on the device by then)
    ref.convert_planes_chain(steps, xs)
    ev = []
    ref.set_log(ev.append)
    n0 = ref.launch_count()
    try:
        ys = ref.convert_planes_chain(steps, xs, on_step=lambda k: ev.append(f"step {k}"))
    finally:
        ref.set_log(None)
    rec["ref"] = {"events": ev, "launches": ref.launch_count() - n0}
    for i, y in enumerate(ys):
        outs[f"{key}.ref.{i}"] = y
    if call.get("entry") == "planes":
        n0 = ref.launch_count()
        zs = ref.convert_planes(steps[0][0], xs)
        rec["ref_planes"] = {"launches": ref.launch_count() - n0, "equal": all(np.array_equal(y, z) for y, z in zip(ys, zs))}
    log[key] = rec


def run_raw(multi, ref, key, call):
    xs = coll(call["coll"])
    n, ms, ks, _, ups = w2x.Context._chain_args(steps_of(call), None)
    bad = call["bad"]
    ys = [np.full((x.shape[0] << ups, x.shape[1] << ups), -3.25, np.float32) for x in xs]
    k = len(xs)
    ip = (C.c_void_p * k)(*[x.ctypes.data for x in xs])
    op = (C.c_void_p * k)(*[y.ctypes.data for y in ys])
    ws = (C.c_int * k)(*[x.shape[1] for x in xs])
    hs = (C.c_int * k)(*[x.shape[0] for x in xs])
    ist = (C.c_size_t * k)(*[x.strides[0] for x in xs])
    ost = (C.c_size_t * k)(*[y.strides[0] for y in ys])
    if bad == "n_steps":
        n = 0
    elif bad == "null_model":
        ms[1] = None
    elif bad == "kind":
        ks[1] = 2
    elif bad == "n_planes":
        k = 0
    elif bad == "stride":
        ist[1] = ws[1] * 4 - 4
    elif bad == "width":
        ws[2] = 0
    events = []
    cb = w2x.capi.STEP_FN(lambda s, _u: events.append(f"step {s}"))
    multi.set_log(events.append)
    ref.set_log(events.append)
    before = multi.launch_counts() + [ref.launch_count()]
    L = w2x.lib()
    try:
        rc = L.w2x_multi_convert_planes_chain(multi._h, n, ms, ks, k, ip, ws, hs, ist, op, ost, cb, None)
        multi_err = [rc, L.w2x_last_error().decode()]
        rc = L.w2x_convert_planes_chain(ref._h, n, ms, ks, k, ip, ws, hs, ist, op, ost, cb, None)
        one_err = [rc, L.w2x_last_error().decode()]
    finally:
        multi.set_log(None)
        ref.set_log(None)
    log[key] = {"multi": multi_err, "one": one_err, "events": events, "launches": [before, multi.launch_counts() + [ref.launch_count()]],
                "untouched": all(bool((y == -3.25).all()) for y in ys)}


def run_nomem(multi, ref, key, call):
    xs = coll(call["coll"])
    steps = steps_of(call)
    settings(multi, ref, call)
    multi.convert_planes_chain(steps, [np.zeros((16, 16), np.float32)])      # the models' device copies and small buffers exist
    ys = [np.full(x.shape, -3.25, np.float32) for x in xs]
    rec = {}
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    try:
        before = multi.launch_counts()
        try:
            multi.convert_planes_chain(steps, xs, out=ys)
            rec["error"] = [0, ""]
        except w2x.W2xError as e:
            rec["error"] = [e.status, e.message]
        rec["launches"] = [before, multi.launch_counts()]
        rec["untouched"] = all(bool((y == -3.25).all()) for y in ys)
    finally:
        del filler
        torch.cuda.empty_cache()
    multi.convert_planes_chain(steps, xs, out=ys)
    rec["after"] = True
    for i, y in enumerate(ys):
        outs[f"{key}.after.{i}"] = y
    for i, y in enumerate(ref.convert_planes_chain(steps, xs)):
        outs[f"{key}.ref.{i}"] = y
    log[key] = rec


for c in cases:
    t0 = time.time()
    multi = w2x.Multi([0] * c["k"])
    ref = w2x.Context(0)
    try:
        for j, call in enumerate(c["calls"]):
            key = f"{c['id']}.{j}"
            {"chain": run_chain, "raw": run_raw, "nomem": run_nomem}[call["op"]](multi, ref, key, call)
    finally:
        multi.close()
        ref.close()
    log.setdefault("seconds", {})[c["id"]] = round(time.time() - t0, 3)
np.savez(os.path.join(d, "out0.npz"), **outs)
json.dump(log, open(os.path.join(d, "log0.json"), "w"))
print(f"multi planes worker: {len(cases)} cases ok", flush=True)
