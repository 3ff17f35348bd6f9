"""multi_regions_worker.py -- runs the cases of tests/test_multi_regions.py in a process of its own (not a test module):

    python tests/multi_regions_worker.py <dir>

Reads <dir>/cases.json, <dir>/models.npz and <dir>/inputs.npz (the files of tests/band_worker.py: plane i of collection c is the input
"c/i"), runs every case and writes the arrays to <dir>/out0.npz and everything else to <dir>/log0.json.  It compares nothing: the test
does.  CUDA_DEVICE_MAX_CONNECTIONS is set before CUDA initialises, so that the streams of k contexts of one device do not share
hardware queues.

A case is {id, k, calls}: one w2x_multi of k contexts of device 0 (and, for the reference, one context), the calls in order.  Call ops:
  regions steps [[model, upscale]], coll, wins [[plane, [x0, y0, w, h]]], precision, engine (default auto), scratch (bytes, default
          1 GiB, on every context and the reference), pinned [sources, outputs], out_pad (extra floats per output row, NaN, default 3),
          layout: "views" (sources are views of whole host planes, each window its own output), "padded" (each source rectangle in a
          buffer of its own that is NaN around it), "tiles" (sources are views of whole host planes, outputs views of one NaN-filled
          host array per plane), sources: "f32" (default), "f64" (float64 copies of the rectangles) or "colstride" (views of every
          other column of a twice as wide array), which the binding copies to float32 rows before the call; probe (tiles layout):
          whether the first plane and the first output array are registered with CUDA before the call, at on_step(0) and after it
          -> "<id>.<call>.<pass>.<i>" window i with its row padding (views, padded) or "<id>.<call>.<pass>.plane<p>" the output array
          of plane p (tiles); "<id>.<call>.ref.<i>" what Context.convert_chain_regions made on one context from float32 rectangles;
          "<id>.<call>.refsrc.<i>" what it made from the call's own sources; "<id>.<call>.whole.<p>" what
          Context.convert_chain(..., block_splitting=False) made of plane p.  Log "<id>.<call>" = {"passes": [{"events", "launches"}],
          "ref": {"events", "launches"}, "owner": every window's GPU, "owner_launches": per GPU used, the launches of
          Context.convert_chain_regions on the windows it owns, "probe": {"plane", "out"}: [before, during, after] per pass, and
          "controls": [a pinned torch buffer, a fresh numpy array] as the probe sees them}
  raw     steps, coll, wins, bad: one argument spoiled -> log "<id>.<call>" = {"multi": [status, message], "one": [status, message],
          "events": [...], "launches": per-context counts before / after, "untouched"}
  nomem   steps, coll, wins: the call with device 0 all but full, then again with the memory back -> log = {"error", "launches",
          "untouched", "after"}; outputs "<id>.<call>.after.<i>" and the reference "<id>.<call>.ref.<i>"
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
_cu = C.CDLL("libcuda.so.1")
CU_POINTER_ATTRIBUTE_MEMORY_TYPE, CU_MEMORYTYPE_HOST = 2, 1


def registered(a):
    """whether the middle of host array a is pinned memory CUDA knows (cudaHostAlloc or cudaHostRegister)"""
    v = C.c_uint(0)
    rc = _cu.cuPointerGetAttribute(C.byref(v), CU_POINTER_ATTRIBUTE_MEMORY_TYPE, C.c_void_p(a.ctypes.data + a.nbytes // 2))
    return rc == 0 and v.value == CU_MEMORYTYPE_HOST


def coll(name):
    n = sum(1 for k in inputs if k.startswith(name + "/"))
    return [inputs[f"{name}/{i}"] for i in range(n)]


def host(shape, pinned, fill=np.nan):
    a = torch.empty(shape, dtype=torch.float32).pin_memory().numpy() if pinned else np.empty(shape, np.float32)
    a[:] = fill
    return a


def steps_of(call):
    return [(models[m], up) for m, up in call["steps"]]


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


def layout(call, steps):
    """-> (sources, sizes, windows, outputs, the arrays the outputs live in, reset, the whole planes): the call's host buffers"""
    xs = coll(call["coll"])
    ups = sum(1 for _, up in steps if up)
    pinned = call.get("pinned", [True, True])
    pad = call.get("out_pad", 3)
    wins = [(p, tuple(w)) for p, w in call["wins"]]
    sizes = [(xs[p].shape[1], xs[p].shape[0]) for p, _ in wins]
    windows = [w for _, w in wins]
    rects = [w2x.chain_region_source(steps, size, w) for size, w in zip(sizes, windows)]
    kind = call.get("layout", "views")
    planes = None
    if kind == "padded":
        srcs = []
        for (p, _), (sx0, sy0, sw, sh) in zip(wins, rects):
            buf = host((sh + 10, sw + 12), pinned[0])
            buf[5:5 + sh, 6:6 + sw] = xs[p][sy0:sy0 + sh, sx0:sx0 + sw]
            srcs.append(buf[5:5 + sh, 6:6 + sw])
    else:
        planes = [host(x.shape, pinned[0], 0.0) for x in xs]
        for a, x in zip(planes, xs):
            a[:] = x
        srcs = [planes[p][sy0:sy0 + sh, sx0:sx0 + sw] for (p, _), (sx0, sy0, sw, sh) in zip(wins, rects)]
    if call.get("sources") == "f64":
        srcs = [s.astype(np.float64) for s in srcs]
    elif call.get("sources") == "colstride":
        wide = [np.full((s.shape[0], 2 * s.shape[1]), np.nan, np.float32) for s in srcs]
        for w, s in zip(wide, srcs):
            w[:, ::2] = s
        srcs = [w[:, ::2] for w in wide]
    if kind == "tiles":
        arrays = [host((x.shape[0] << ups, (x.shape[1] << ups) + pad), pinned[1]) for x in xs]
        views = [arrays[p][y0:y0 + h, x0:x0 + w] for p, (x0, y0, w, h) in wins]
    else:
        arrays = [host((w[3], w[2] + pad), pinned[1]) for w in windows]
        views = [a[:, :w[2]] for a, w in zip(arrays, windows)]

    def reset():
        for a in arrays:
            a[:] = np.nan
    return srcs, sizes, windows, views, arrays, reset, planes


def run_regions(multi, ref, key, call):
    steps = steps_of(call)
    settings(multi, ref, call)
    srcs, sizes, windows, views, arrays, reset, planes = layout(call, steps)
    plain = [np.ascontiguousarray(s, np.float32) for s in srcs]
    tiles = call.get("layout") == "tiles"
    rec = {"passes": []}
    events = []
    probe = {"plane": [], "out": []}

    def on_step(k):
        events.append(f"step {k}")
        if call.get("probe") and k == 0:
            probe["plane"][-1].append(registered(planes[0]))
            probe["out"][-1].append(registered(arrays[0]))
    multi.set_log(events.append)
    try:
        for p in range(call.get("passes", 2)):
            reset()
            del events[:]
            if call.get("probe"):
                probe["plane"].append([registered(planes[0])])
                probe["out"].append([registered(arrays[0])])
            before = multi.launch_counts()
            multi.convert_chain_regions(steps, srcs, sizes, windows, out=views, on_step=on_step)
            if call.get("probe"):
                probe["plane"][-1].append(registered(planes[0]))
                probe["out"][-1].append(registered(arrays[0]))
            rec["passes"].append({"events": list(events), "launches": [a - b for a, b in zip(multi.launch_counts(), before)]})
            for i, a in enumerate(arrays):
                outs[f"{key}.{p}.{'plane' if tiles else ''}{i}"] = a.copy()
    finally:
        multi.set_log(None)
    if call.get("probe"):
        rec["probe"] = probe
        rec["controls"] = [registered(torch.empty(1 << 20).pin_memory().numpy()), registered(np.zeros(1 << 20, np.float32))]
    if call.get("sources"):
        for i, y in enumerate(ref.convert_chain_regions(steps, srcs, sizes, windows)):
            outs[f"{key}.refsrc.{i}"] = y
    # the one-context call (its second run: the models are on the device by then)
    ref.convert_chain_regions(steps, plain, sizes, windows)
    ev = []
    ref.set_log(ev.append)
    n0 = ref.launch_count()
    try:
        ys = ref.convert_chain_regions(steps, plain, sizes, windows, on_step=lambda k: ev.append(f"step {k}"))
    finally:
        ref.set_log(None)
    rec["ref"] = {"events": ev, "launches": ref.launch_count() - n0}
    for i, y in enumerate(ys):
        outs[f"{key}.ref.{i}"] = y
    for p, x in enumerate(coll(call["coll"])):
        if any(q == p for q, _ in call["wins"]):
            outs[f"{key}.whole.{p}"] = ref.convert_chain(steps, x, block_splitting=False)
    nd, owner, _ = w2x.debug_plan_multi_regions(len(contexts(multi)), steps, sizes, windows)
    rec["owner"] = owner.tolist()
    rec["owner_launches"] = []
    for g in range(nd):
        mine = [i for i in range(len(windows)) if owner[i] == g]
        n0 = ref.launch_count()
        ref.convert_chain_regions(steps, [plain[i] for i in mine], [sizes[i] for i in mine], [windows[i] for i in mine])
        rec["owner_launches"].append(ref.launch_count() - n0)
    log[key] = rec


def raw_args(call, steps):
    """the C arguments of a region call on pageable buffers, one of them spoiled as call["bad"] says, and the outputs"""
    xs = coll(call["coll"])
    n, ms, ks, _, _ = w2x.Context._chain_args(steps, None)
    wins = [(p, tuple(w)) for p, w in call["wins"]]
    sizes = [(xs[p].shape[1], xs[p].shape[0]) for p, _ in wins]
    rects = [w2x.chain_region_source(steps, size, w) for size, (_, w) in zip(sizes, wins)]
    srcs = [xs[p][sy0:sy0 + sh, sx0:sx0 + sw] for (p, _), (sx0, sy0, sw, sh) in zip(wins, rects)]
    ys = [np.full((w[3], w[2]), -3.25, np.float32) for _, w in wins]
    k = len(wins)
    ws = (C.c_int * k)(*[s[0] for s in sizes])
    hs = (C.c_int * k)(*[s[1] for s in sizes])
    wa = (C.c_int * (4 * k))(*[v for _, w in wins for v in w])
    sp = (C.c_void_p * k)(*[s.ctypes.data for s in srcs])
    sst = (C.c_size_t * k)(*[s.strides[0] for s in srcs])
    op = (C.c_void_p * k)(*[y.ctypes.data for y in ys])
    ost = (C.c_size_t * k)(*[y.strides[0] for y in ys])
    bad = call.get("bad")
    if bad == "n_windows":
        k = 0
    elif bad == "n_steps":
        n = 0
    elif bad == "tta":
        ks[1] |= w2x.capi.STEP_TTA
    elif bad == "kind":
        ks[1] = 2
    elif bad == "null_model":
        ms[1] = None
    elif bad == "empty":
        wa[4 * 1 + 2] = 0
    elif bad == "outside":
        wa[4 * 2] = 10 ** 6
    elif bad == "size":
        ws[1] = 0
    elif bad == "null_source":
        sp[1] = None
    elif bad == "null_output":
        op[2] = None
    elif bad == "src_stride":
        sst[1] = 4
    elif bad == "out_stride":
        ost[0] += 2
    elif bad == "null_windows":
        wa = None
    return [n, ms, ks, k, ws, hs, wa, sp, sst, op, ost], ys


def run_raw(multi, ref, key, call):
    steps = steps_of(call)
    settings(multi, ref, call)
    args, ys = raw_args(call, steps)
    events = []
    cb = w2x.capi.STEP_FN(lambda s, _u: events.append(f"step {s}"))
    multi.set_log(events.append)
    ref.set_log(events.append)
    before = multi.launch_counts() + [ref.launch_count()]
    L = w2x.lib()
    try:
        rc = L.w2x_multi_convert_chain_regions(multi._h, *args, cb, None)
        multi_err = [rc, L.w2x_last_error().decode()]
        rc = L.w2x_convert_chain_regions(ref._h, *args, cb, None)
        one_err = [rc, L.w2x_last_error().decode()]
    finally:
        multi.set_log(None)
        ref.set_log(None)
    torch.cuda.synchronize()
    log[key] = {"multi": multi_err, "one": one_err, "events": events, "launches": [before, multi.launch_counts() + [ref.launch_count()]],
                "untouched": all(bool((y == -3.25).all()) for y in ys)}


def run_nomem(multi, ref, key, call):
    steps = steps_of(call)
    settings(multi, ref, call)
    xs = coll(call["coll"])
    small = np.zeros((16, 16), np.float32)
    multi.convert_chain_regions(steps, [small] * 2, [(16, 16)] * 2, [(0, 0, 32, 32)] * 2)   # the models' device copies exist
    wins = [tuple(w) for _, w in call["wins"]]
    sizes = [(xs[p].shape[1], xs[p].shape[0]) for p, _ in call["wins"]]
    srcs = []
    for (p, _), size, w in zip(call["wins"], sizes, wins):
        sx0, sy0, sw, sh = w2x.chain_region_source(steps, size, w)
        srcs.append(xs[p][sy0:sy0 + sh, sx0:sx0 + sw])
    ys = [np.full((w[3], w[2]), -3.25, np.float32) for w in wins]
    rec = {}
    events = []
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    try:
        before = multi.launch_counts()
        multi.set_log(events.append)
        try:
            multi.convert_chain_regions(steps, srcs, sizes, wins, out=ys, on_step=lambda k: events.append(f"step {k}"))
            rec["error"] = [0, ""]
        except w2x.W2xError as e:
            rec["error"] = [e.status, e.message]
        finally:
            multi.set_log(None)
        torch.cuda.synchronize()
        rec["launches"] = [before, multi.launch_counts()]
        rec["events"] = events
        rec["untouched"] = all(bool((y == -3.25).all()) for y in ys)
    finally:
        del filler
        torch.cuda.empty_cache()
    multi.convert_chain_regions(steps, srcs, sizes, wins, out=ys)
    rec["after"] = True
    for i, y in enumerate(ys):
        outs[f"{key}.after.{i}"] = y
    for i, y in enumerate(ref.convert_chain_regions(steps, srcs, sizes, wins)):
        outs[f"{key}.ref.{i}"] = y
    log[key] = rec


for c in cases:
    t0 = time.time()
    multi = w2x.Multi([0] * c["k"])
    ref = w2x.Context(0)
    try:
        for j, call in enumerate(c["calls"]):
            key = f"{c['id']}.{j}"
            {"regions": run_regions, "raw": run_raw, "nomem": run_nomem}[call["op"]](multi, ref, key, call)
    finally:
        multi.close()
        ref.close()
    log.setdefault("seconds", {})[c["id"]] = round(time.time() - t0, 3)
np.savez(os.path.join(d, "out0.npz"), **outs)
json.dump(log, open(os.path.join(d, "log0.json"), "w"))
print(f"multi regions worker: {len(cases)} cases ok", flush=True)
