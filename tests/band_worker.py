"""band_worker.py -- runs the multi-GPU cases of tests/test_band_exchange.py in a process of its own (not a test module):

    python tests/band_worker.py <dir> [rank]

Reads <dir>/cases.json (a list of cases), <dir>/models.npz (weights "<model>/w<k>", biases "<model>/b<k>") and
<dir>/inputs.npz (one plane per input key), runs every case and writes the planes it made to <dir>/out<rank>.npz and its
status lines, progress lines and errors to <dir>/log<rank>.json.  It compares nothing: the test does.

The in-library exchange needs every band of a group to run at the same time, so on one device every band has its own
context (three streams each) and the process must have CUDA_DEVICE_MAX_CONNECTIONS >= the number of streams before CUDA
initialises; CUDA_MODULE_LOADING=EAGER keeps a band from loading modules while its neighbours wait in the exchange kernel.
Every band or slab of a group is queued before the process waits for any of them, and every group runs PASSES passes.

Case kinds (fields beyond "id", "kind", "model", "width"):
  band      precision, rows [owned rows per band], in_pad / out_pad (extra floats per device row)
            -> "<id>.<pass>" the stitched plane
  slab      precision, rows, n_sub, order [per slab], in_pad / out_pad (host rows), pinned [input, output]
            -> "<id>.<pass>"  (a download into pageable memory blocks the host until the slab's layers are done, so only a
            slab without neighbours may have a pageable output: its neighbours would not be queued yet)
  slab_ipc  precision [per rank], rows [per rank], n_sub, run (default true); one slab per rank process, CUDA IPC
            (w2x_slab_export / _connect) -> "<id>.<rank>.<pass>" this rank's rows when every rank connected and run is
            set, log "<id>.connect" = the connect error
  multi     k, calls [{op: plane | tiles, model, precision, input, block_splitting, log}] on one w2x_multi of k contexts
            -> "<id>.<call>" the output, log "<id>.<call>" its progress lines
  forget    precision, rows (a band group), model2: w2x_ctx_forget_model while a band group, a slab and a w2x_multi plan
            hold the model -> log "<id>" the status of every forget, "<id>.<pass>" the band group's plane, run after the
            refused forgets
  plans     precision, models [m1, m2, m3]: on one w2x_multi of 2 contexts, convert_plane(m1), convert_chain([m2, m3^]), a forget
            of m1 and of m2, convert_plane(m1) again -> "<id>.plane", "<id>.chain", "<id>.plane again"; log "<id>" the status of
            each forget and the per-context launches of each call
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
import torch  # noqa: E402  (device buffers and pinned host memory only)
import w2x_loader  # noqa: E402

PASSES = 3
MAX_CONTEXTS = 8

w2x = w2x_loader.load()
d = sys.argv[1]
rank = int(sys.argv[2]) if len(sys.argv) > 2 else 0
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


class Pool:
    """up to MAX_CONTEXTS tensor-core contexts, each warmed up by one ordinary convert_plane"""

    def __init__(self):
        self.ctxs = []

    def take(self, k, precision):
        if k > MAX_CONTEXTS:
            raise SystemExit(f"a group of {k} needs more than {MAX_CONTEXTS} contexts")
        while len(self.ctxs) < k:
            c = w2x.Context(0, engine=w2x.ENGINE_TC)
            c.convert_plane(next(iter(models.values())), np.zeros((8, 8), np.float32))
            self.ctxs.append(c)
        for c in self.ctxs[:k]:
            c.set_precision(precision)
        return self.ctxs[:k]

    def close(self):
        for c in self.ctxs:
            c.close()
        self.ctxs = []


pool = Pool()


def cuts(rows):
    return np.concatenate([[0], np.cumsum(rows)]).astype(int).tolist()


def run_bands(key, ctxs, model, x, rows, in_pad, out_pad, before_passes=None):
    """one band per context, wired with connect_local; PASSES passes, each queued on every band before any wait"""
    H, W = x.shape
    r = cuts(rows)
    nb = len(rows)
    d_in = torch.full((H, W + in_pad), float("nan"), device="cuda")
    d_in[:, :W] = torch.from_numpy(x).cuda()
    d_out = torch.empty((H, W + out_pad), device="cuda")
    bands = []
    try:
        for b in range(nb):
            bands.append(w2x.Band(ctxs[b], model, W, rows[b], b > 0, b < nb - 1))
        for b in range(nb):
            bands[b].connect_local(bands[b - 1] if b > 0 else None, bands[b + 1] if b < nb - 1 else None)
        if before_passes:
            before_passes()
        sin, sout = (W + in_pad) * 4, (W + out_pad) * 4
        for p in range(PASSES):
            d_out.fill_(float("nan"))
            torch.cuda.synchronize()
            for b in range(nb):
                bands[b].run(d_in[r[b]].data_ptr(), sin, d_out[r[b]].data_ptr(), sout)
            for c in ctxs[:nb]:
                c.synchronize()
            outs[f"{key}.{p}"] = d_out.cpu().numpy()          # the pad columns too: they must stay NaN
    finally:
        for b in bands:
            b.close()


def host_rows(shape, pinned):
    if pinned:
        return torch.empty(shape, dtype=torch.float32).pin_memory().numpy()
    return np.empty(shape, np.float32)


def run_slabs(c):
    rows, ns = c["rows"], len(c["rows"])
    ctxs = pool.take(ns, c["precision"])
    x = inputs[c["id"]]
    H, W = x.shape
    r = cuts(rows)
    h_in = host_rows((H, W + c["in_pad"]), c["pinned"][0])
    h_in[:] = np.nan
    h_in[:, :W] = x
    h_out = host_rows((H, W + c["out_pad"]), c["pinned"][1])
    slabs = []
    try:
        for s in range(ns):
            slabs.append(w2x.Slab(ctxs[s], models[c["model"]], W, rows[s], s > 0, s < ns - 1, order=c["order"][s], n_sub=c["n_sub"][s]))
        for s in range(ns):
            slabs[s].connect_local(slabs[s - 1] if s > 0 else None, slabs[s + 1] if s < ns - 1 else None)
        for p in range(PASSES):
            h_out[:] = np.nan
            for s in range(ns):
                slabs[s].convert_async(h_in[r[s]:r[s + 1], :W], h_out[r[s]:r[s + 1], :W])
            for sl in slabs:
                sl.synchronize()
            outs[f"{c['id']}.{p}"] = h_out.copy()
    finally:
        for sl in slabs:
            sl.close()


def wait_for(path, what):
    t0 = time.time()
    while not os.path.exists(path):
        if time.time() - t0 > 120:
            raise SystemExit(f"rank {rank}: {what} never appeared")
        time.sleep(0.02)


def run_slab_ipc(c):
    """this rank's slab of a world of len(rows) processes; blobs travel through files in <dir>"""
    rows, world = c["rows"], len(c["rows"])
    ctx = pool.take(1, c["precision"][rank])[0]
    x = inputs[c["id"]]
    W = x.shape[1]
    r = cuts(rows)
    h_in = host_rows((rows[rank], W), True)
    h_in[:] = x[r[rank]:r[rank + 1]]
    h_out = host_rows((rows[rank], W), True)
    slab = w2x.Slab(ctx, models[c["model"]], W, rows[rank], rank > 0, rank < world - 1, order=rank & 1, n_sub=c["n_sub"])
    blob = os.path.join(d, f"{c['id']}.blob{{}}")
    try:
        open(blob.format(f"{rank}.tmp"), "wb").write(slab.export())
        os.replace(blob.format(f"{rank}.tmp"), blob.format(rank))

        def peer(q):
            wait_for(blob.format(q), f"the blob of rank {q}")
            return open(blob.format(q), "rb").read()

        try:
            slab.connect(peer(rank - 1) if rank > 0 else None, peer(rank + 1) if rank < world - 1 else None)
            connected = True
        except w2x.W2xError as e:
            log[f"{c['id']}.connect"] = [e.status, e.message]
            connected = False
        # every rank runs only if every rank connected, so no exchange waits for a rank that stopped
        open(os.path.join(d, f"{c['id']}.connected{rank}"), "w").write("1" if connected else "0")
        states = []
        for q in range(world):
            wait_for(os.path.join(d, f"{c['id']}.connected{q}"), f"the connect result of rank {q}")
            states.append(open(os.path.join(d, f"{c['id']}.connected{q}")).read() == "1")
        if all(states) and c.get("run", True):
            for p in range(PASSES):
                h_out[:] = np.nan
                slab.convert(h_in, h_out)
                outs[f"{c['id']}.{rank}.{p}"] = h_out.copy()
    finally:
        # the exported buffers stay alive until every neighbour is done with them
        open(os.path.join(d, f"{c['id']}.done{rank}"), "w").write("1")
        for q in range(world):
            wait_for(os.path.join(d, f"{c['id']}.done{q}"), f"the end of rank {q}")
        slab.close()


def run_multi(c):
    pool.close()                                    # the multi's contexts take the pool's place
    multi = w2x.Multi([0] * c["k"])
    try:
        first = c["calls"][0]
        multi.convert_tiles(models[first["model"]], np.zeros((c["k"], 8, 8), np.float32))   # warm-up, no exchange
        for j, call in enumerate(c["calls"]):
            multi.set_precision(call["precision"])
            lines = []
            multi.set_log(lines.append if call.get("log") else None)
            x = inputs[call["input"]]
            if call["op"] == "plane":
                outs[f"{c['id']}.{j}"] = multi.convert_plane(models[call["model"]], x, block_splitting=call.get("block_splitting", True))
            else:
                outs[f"{c['id']}.{j}"] = multi.convert_tiles(models[call["model"]], x)
            if call.get("log"):
                log[f"{c['id']}.{j}"] = lines
        multi.set_log(None)
    finally:
        multi.close()


def forget_status(ctx_or_multi, model):
    try:
        ctx_or_multi.forget_model(model)
        return [0, ""]
    except w2x.W2xError as e:
        return [e.status, e.message]


def run_forget(c):
    """w2x_ctx_forget_model against live band sessions, slabs and a w2x_multi plan"""
    m, m2 = models[c["model"]], models[c["model2"]]
    x = inputs[c["id"]]
    W = x.shape[1]
    st = {}
    ctxs = pool.take(len(c["rows"]), c["precision"])
    ctxs[0].convert_plane(m2, x)                     # m2's copies are on the context too, held by nothing

    def refuse():
        st["band open"] = forget_status(ctxs[0], m)
        st["band open, last context"] = forget_status(ctxs[-1], m)
        st["band open, other model"] = forget_status(ctxs[0], m2)

    # the group runs its passes after the refused forgets: its sessions' copies must still be there
    run_bands(c["id"], ctxs, m, x, c["rows"], 0, 0, before_passes=refuse)
    st["band closed"] = forget_status(ctxs[0], m)
    slab = w2x.Slab(ctxs[0], m, W, x.shape[0], False, False, n_sub=2)
    st["slab open"] = forget_status(ctxs[0], m)
    slab.close()
    st["slab closed"] = forget_status(ctxs[0], m)
    pool.close()
    multi = w2x.Multi([0, 0])
    try:
        multi.convert_plane(m, x)
        st["multi plan"] = forget_status(multi, m)
        multi.convert_plane(m2, x)
        st["multi plan of the other model"] = forget_status(multi, m)
        st["multi plan, its model"] = forget_status(multi, m2)
    finally:
        multi.close()
    log[c["id"]] = st


def run_plans(c):
    """a plane plan and a chain plan of one w2x_multi side by side: a plane, a chain, a forget of each plan's model, the plane again"""
    pool.close()
    m1, m2, m3 = (models[k] for k in c["models"])
    x = inputs[c["id"]]
    st = {}
    multi = w2x.Multi([0, 0])

    def counted(key, convert):
        before = multi.launch_counts()
        outs[f"{c['id']}.{key}"] = convert()
        st[f"{key} launches"] = [a - b for a, b in zip(multi.launch_counts(), before)]

    try:
        multi.set_precision(c["precision"])
        counted("plane", lambda: multi.convert_plane(m1, x))
        counted("chain", lambda: multi.convert_chain([(m2, False), (m3, True)], x))
        st["plane's model"] = forget_status(multi, m1)            # the first context refuses first
        st["chain's model"] = forget_status(multi, m2)
        counted("plane again", lambda: multi.convert_plane(m1, x))
    finally:
        multi.close()
    log[c["id"]] = st


RUN = {"slab": run_slabs, "slab_ipc": run_slab_ipc, "multi": run_multi, "forget": run_forget, "plans": run_plans}
for c in cases:
    t0 = time.time()
    if c["kind"] == "band":
        run_bands(c["id"], pool.take(len(c["rows"]), c["precision"]), models[c["model"]], inputs[c["id"]], c["rows"], c["in_pad"], c["out_pad"])
    else:
        RUN[c["kind"]](c)
    log.setdefault("seconds", {})[c["id"]] = round(time.time() - t0, 3)
pool.close()
np.savez(os.path.join(d, f"out{rank}.npz"), **outs)
json.dump(log, open(os.path.join(d, f"log{rank}.json"), "w"))
print(f"band worker rank {rank}: {len(cases)} cases ok", flush=True)
