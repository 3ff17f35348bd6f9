"""multi_chain_worker.py -- runs the cases of tests/test_multi_chain.py in a process of its own (not a test module):

    python tests/multi_chain_worker.py <dir>

Reads <dir>/cases.json, <dir>/models.npz and <dir>/inputs.npz (the files of tests/band_worker.py), runs every case and writes
the planes it made to <dir>/out0.npz and everything else to <dir>/log0.json.  It compares nothing: the test does.

w2x_multi_convert_chain's exchange needs every band of a step to run at the same time.  On one device the "GPUs" are k
contexts of device 0, so the process must have CUDA_DEVICE_MAX_CONNECTIONS >= their number of streams before CUDA initialises,
and CUDA_MODULE_LOADING=EAGER keeps a band from loading modules while its neighbours wait in the exchange kernel.  The library
queues every GPU's work before it waits for any; this worker only ever calls it from one thread.

A case is {id, k, calls}: one w2x_multi of k contexts, the calls in order.  Call ops (fields beyond "op"):
  chain   steps [[model, upscale, tta]], precision, input, block_splitting, pinned [input, output], in_pad / out_pad (extra
          floats per host row), passes (default 3)
          -> "<id>.<call>.<pass>" the output plane with its row padding (which must stay NaN); log "<id>.<call>" = per pass
          {"events": on_step calls ("step k") and progress lines in order, "launches": per-context launch counts of the pass},
          or {"error": [status, message], "events": [...]} when the call failed
  plane   model, precision, input, block_splitting: Multi.convert_plane -> the same keys (one pass per PASSES)
  raw     steps, input, in_stride / out_stride (bytes; default dense): w2x_multi_convert_chain called through ctypes with these
          strides on dense planes -> log "<id>.<call>" = {"error": [status, message], "events": [...]}
  forget  model -> log "<id>.<call>" = [status, message] of w2x_ctx_forget_model on every context
  reopen  destroys the w2x_multi and creates a new one of k contexts
"""
import json
import os
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402  (pinned host memory only)
import w2x_loader  # noqa: E402

PASSES = 3

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


def host_rows(shape, pinned):
    if pinned:
        return torch.empty(shape, dtype=torch.float32).pin_memory().numpy()
    return np.empty(shape, np.float32)


def new_multi(k):
    multi = w2x.Multi([0] * k)
    multi.convert_tiles(next(iter(models.values())), np.zeros((k, 8, 8), np.float32))   # warm-up of every context, no exchange
    return multi


def run_convert(multi, key, call):
    x = inputs[call["input"]]
    H, W = x.shape
    chain = call["op"] == "chain"
    steps = [(models[m] if m is not None else None, up, tta) for m, up, tta in call["steps"]] if chain else None
    ups = sum(1 for s in call["steps"] if s[1]) if chain else 0
    pinned = call.get("pinned", [True, True])
    h_in = host_rows((H, W + call.get("in_pad", 0)), pinned[0])
    h_in[:] = np.nan
    h_in[:, :W] = x
    h_out = host_rows((H << ups, (W << ups) + call.get("out_pad", 0)), pinned[1])
    multi.set_precision(call["precision"])
    events = []
    multi.set_log(events.append)
    passes = []
    try:
        for p in range(call.get("passes", PASSES)):
            h_out[:] = np.nan
            del events[:]
            before = multi.launch_counts()
            try:
                if chain:
                    multi.convert_chain(steps, h_in[:, :W], out=h_out[:, :W << ups], block_splitting=call.get("block_splitting", True),
                                        on_step=lambda k: events.append(f"step {k}"))
                else:
                    multi.convert_plane(models[call["model"]], h_in[:, :W], block_splitting=call.get("block_splitting", True), out=h_out[:, :W])
            except w2x.W2xError as e:
                log[key] = {"error": [e.status, e.message], "events": list(events)}
                return
            passes.append({"events": list(events), "launches": [a - b for a, b in zip(multi.launch_counts(), before)]})
            outs[f"{key}.{p}"] = h_out.copy()
    finally:
        multi.set_log(None)
    log[key] = passes


for c in cases:
    t0 = time.time()
    multi = new_multi(c["k"])
    try:
        for j, call in enumerate(c["calls"]):
            key = f"{c['id']}.{j}"
            if call["op"] == "reopen":
                multi.close()
                multi = new_multi(c["k"])
            elif call["op"] == "raw":
                x = inputs[call["input"]]
                H, W = x.shape
                n, ms, ks, cb, ups = w2x.Context._chain_args([(models[m], up, tta) for m, up, tta in call["steps"]], None)
                out = np.empty((H << ups, W << ups), np.float32)
                events = []
                multi.set_log(events.append)
                rc = w2x.lib().w2x_multi_convert_chain(multi._h, n, ms, ks, x.ctypes.data, W, H, call.get("in_stride", W * 4), out.ctypes.data,
                                                       call.get("out_stride", (W << ups) * 4), 1, cb, None)
                multi.set_log(None)
                log[key] = {"error": [rc, w2x.lib().w2x_last_error().decode()], "events": events}
            elif call["op"] == "forget":
                try:
                    multi.forget_model(models[call["model"]])
                    log[key] = [0, ""]
                except w2x.W2xError as e:
                    log[key] = [e.status, e.message]
            else:
                run_convert(multi, key, call)
    finally:
        multi.close()
    log.setdefault("seconds", {})[c["id"]] = round(time.time() - t0, 3)
np.savez(os.path.join(d, "out0.npz"), **outs)
json.dump(log, open(os.path.join(d, "log0.json"), "w"))
print(f"multi chain worker: {len(cases)} cases ok", flush=True)
