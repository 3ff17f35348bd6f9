"""Band sessions, slabs and the one-process multi-GPU driver (csrc/engine_band.cu) on ONE device, bit for bit against the
selection-layer emulator of test_edge_exact.py and against convert_plane on one context in the same precision.

On one device the "neighbours" are other contexts (or processes) of the same GPU, so the in-library halo exchange runs
exactly as between GPUs, only through local pointers.  Its bands must run concurrently, which needs
CUDA_DEVICE_MAX_CONNECTIONS set before CUDA initialises: the cases run in tests/band_worker.py, a child process, and this
module builds the inputs and references and compares.

  * w2x_band_run + connect_local, 2 to 6 bands: owned rows 1, 2, n-1, n, n+1, 8, 16, 17 mixed within a plane and a 1-row
    band at each border; frame widths pw = w + 2n with pw % 16 in {0, 1, 15} and pw % 4 in {1, 2, 3} (the exchange kernel's
    16-byte and 4-byte paths for the padded input rows); row-strided input and output.
  * w2x_slab_* + connect_local, 1 to 4 slabs: n_sub 1, 2, 3, 8 and automatic, rows not divisible by n_sub, sub-bands of the
    4n-row minimum, a K = 1 slab beside a K > 1 one, both walk orders at every position, host rows with a stride larger
    than the row, pinned and pageable host memory.
  * w2x_slab_export / w2x_slab_connect between two processes (the path of bench.py's ranks), and their refusal of a
    neighbour in another precision.
  * w2x_multi_* on k = 2..4 contexts of one device: heights on both sides of the cut-or-not rule, automatic sub-bands, the
    plan cache across precision / model / width / height changes, convert_tiles with fewer, as many and more tiles than
    devices, and the progress lines.
  * w2x_ctx_forget_model while band sessions, slabs or a multi plan use the model; a w2x_multi's plane plan and chain plan kept
    side by side.

Every group runs three passes (flag values, events and buffers are reused); every pass must give the reference's bits.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_edge_exact import assert_selection, emulate_tc_model, plane_for, sel_model, selection_report

pytestmark = pytest.mark.gpu

WORKER = os.path.join(ROOT, "tests", "band_worker.py")
ENV = {"CUDA_DEVICE_MAX_CONNECTIONS": "32", "CUDA_MODULE_LOADING": "EAGER"}
PASSES = 3
F16X3, F16_F8X2, F16 = 0, 1, 2

# selection models (n = 4) for the emulator; the shipped models (n = 7) and a random 1 -> 128 -> 32 -> 64 -> 1 for convert_plane
SEL = {"sel32": ((32, 64, 32), 0, 4242), "sel128": ((64, 128, 32), 1, 7)}
RANDOM = {"rand128": ([(1, 128), (128, 32), (32, 64), (64, 1)], 5)}


@pytest.fixture(scope="module")
def layers(oracle_models, oracle_mod):
    out = {k: sel_model(*v) for k, v in SEL.items()}
    for name in ("noise1", "scale2.0x"):
        om = oracle_models[name]
        out[name] = list(zip(om.weights, om.biases))
    for k, (dims, seed) in RANDOM.items():
        om = oracle_mod.OracleModel.random(dims, seed=seed)
        out[k] = list(zip(om.weights, om.biases))
    return out


@pytest.fixture(scope="module")
def models(w2x, layers):
    return {k: w2x.Model.from_arrays([w for w, _ in v], [b for _, b in v]) for k, v in layers.items()}


class Reference:
    """the emulator for selection models in f16x3 / f16+f8x2, else convert_plane on one context in the precision"""

    def __init__(self, w2x, layers, models):
        self.layers, self.models = layers, models
        self.ctx = {}
        for p in (F16X3, F16_F8X2, F16):
            self.ctx[p] = w2x.Context(0, engine=w2x.ENGINE_TC)
            self.ctx[p].set_precision(p)

    def __call__(self, name, precision, x, block_splitting=True):
        if name in SEL and precision != F16:
            want, inputs = emulate_tc_model(x, self.layers[name], precision == F16_F8X2, True)
            for xr, w, b in inputs:                  # the emulator's conditions hold on these very activations
                assert_selection(selection_report(xr, w, b, precision == F16_F8X2))
            return want
        return self.ctx[precision].convert_plane(self.models[name], x, block_splitting=block_splitting)

    def close(self):
        for c in self.ctx.values():
            c.close()


@pytest.fixture(scope="module")
def ref(w2x, layers, models):
    r = Reference(w2x, layers, models)
    yield r
    r.close()


def n_of(name):
    return 4 if name in SEL or name in RANDOM else 7


def cuts(rows):
    return np.concatenate([[0], np.cumsum(rows)]).astype(int).tolist()


def slab_cuts(rows, n, n_sub):
    """w2x_slab_create's sub-band rows (the frame-row limit never binds at these sizes)"""
    if n_sub <= 0:
        n_sub = min(4, rows // 512)
    n_sub = max(1, min(n_sub, min(8, rows // (4 * n))))
    return [rows * i // n_sub for i in range(n_sub + 1)]


def mismatch(got, want, seams):
    """where two planes differ, relative to the nearest band / sub-band seam; "" when they are equal"""
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    if not len(bad):
        return ""
    r, c = (int(v) for v in bad[0])
    s = min(seams, key=lambda v: abs(r - v))
    rows = np.unique(bad[:, 0])
    return (f"{len(bad)} of {got.size} values differ in {len(rows)} rows; first at row {r} ({r - s:+d} from the seam at row {s}), "
            f"column {c}: {got[r, c]!r} != {want[r, c]!r}")


class Job:
    """cases + inputs + models for one worker run"""

    def __init__(self, layers):
        self.layers = layers
        self.cases, self.inputs = [], {}

    def add(self, case, x=None):
        if x is not None:
            self.inputs[case["id"]] = np.ascontiguousarray(x, np.float32)
        self.cases.append(case)
        return case

    def write(self, d):
        json.dump(self.cases, open(os.path.join(d, "cases.json"), "w"))
        np.savez(os.path.join(d, "inputs.npz"), **self.inputs)
        np.savez(os.path.join(d, "models.npz"), **{f"{k}/{t}{i}": (w if t == "w" else b)
                                                   for k, v in self.layers.items() for i, (w, b) in enumerate(v) for t in "wb"})


def run_worker(d, ranks=(None,), timeout=600):
    """start one worker per rank (all at once), wait, return [(outputs, log)] per rank"""
    env = dict(os.environ, **ENV)
    procs = [subprocess.Popen([sys.executable, WORKER, str(d)] + ([] if r is None else [str(r)]), env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in ranks]
    logs = [p.communicate(timeout=timeout)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(logs)
    res = []
    for r in ranks:
        k = 0 if r is None else r
        res.append((dict(np.load(os.path.join(d, f"out{k}.npz"))), json.load(open(os.path.join(d, f"log{k}.json")))))
    return res


def seeded(h, w, seed, name):
    """plane_for (the emulator's input family) for selection models, uniform noise for the others"""
    if name in SEL:
        return plane_for(h, w, seed)
    return np.random.default_rng(seed).random((h, w), dtype=np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# the cases of one worker run: bands, slabs, multi
# ---------------------------------------------------------------------------------------------------------------------
# owned rows per band: n-1, n, n+1 of the model, 1, 2, 8, 16, 17, a 1-row band at each image border
def band_groups(n):
    return [[1, n - 1, 16, n + 1, 1], [2, n, 8, 17], [17, 1], [n + 1, 8, 1, 2, 16, n - 1]]


# widths by pw = w + 2n: pw % 16 = 0, 1, 15 and pw % 4 = 2, then tiny and tile-set widths
def band_widths(n):
    return [48 - 2 * n, 49 - 2 * n, 47 - 2 * n, 50 - 2 * n, 1, 16, 17]


def band_cases():
    cases = []
    k = 0
    for name, precs in (("sel32", (F16X3, F16_F8X2)), ("sel128", (F16X3, F16_F8X2)), ("noise1", (F16X3, F16_F8X2, F16)),
                        ("scale2.0x", (F16,)), ("rand128", (F16X3, F16_F8X2, F16))):
        n = n_of(name)
        for p in precs:
            groups = band_groups(n) if name in SEL else band_groups(n)[k % 4:k % 4 + 2]
            for rows in groups:
                W = band_widths(n)[k % 7]
                cases.append(dict(id=f"band{k}", kind="band", model=name, precision=p, width=W, rows=rows, in_pad=(0, 3, 0, 5)[k % 4],
                                  out_pad=(0, 0, 7, 1)[k % 4]))
                k += 1
    return cases


# (model, precision, width, rows per slab, n_sub, order, in_pad, out_pad, pinned [input, output])
SLABS = [
    ("sel32", F16X3, 40, [50], [3], [0], 3, 1, [False, False]),          # one slab, no neighbours, 16 / 17 / 17 rows, pageable
    ("sel128", F16_F8X2, 41, [64], [8], [1], 0, 0, [True, False]),       # n_sub 8 -> 4 sub-bands of the 16-row minimum
    ("sel32", F16_F8X2, 39, [128, 48], [8, 1], [0, 1], 0, 2, [True, True]),   # 8 sub-bands of 16 rows beside K = 1
    ("sel128", F16X3, 42, [40, 70], [2, 3], [1, 0], 5, 0, [False, True]),
    ("rand128", F16, 20, [33, 34], [2, 2], [0, 0], 0, 0, [True, True]),
    ("noise1", F16, 33, [58, 57], [3, 1], [1, 1], 1, 3, [True, True]),
    ("sel32", F16X3, 20, [50, 1100, 40], [3, 0, 2], [0, 1, 0], 0, 0, [True, True]),   # automatic: 2 sub-bands of 550 rows
    ("sel128", F16_F8X2, 17, [20, 33, 64, 17], [1, 2, 0, 1], [1, 0, 1, 0], 2, 4, [True, True]),
    ("noise1", F16_F8X2, 64, [60, 61, 62, 63], [2, 2, 1, 2], [0, 1, 1, 0], 0, 0, [True, True]),
]


def slab_cases():
    return [dict(id=f"slab{k}", kind="slab", model=m, precision=p, width=W, rows=rows, n_sub=ns, order=order, in_pad=ip,
                 out_pad=op, pinned=pin) for k, (m, p, W, rows, ns, order, ip, op, pin) in enumerate(SLABS)]


def multi_cases():
    """k contexts; planes (W, H) of the model at the precision, or tile stacks (n, W, H) -> (case, {input: array})"""
    C = []

    def plane(name, p, W, H, seed, **kw):
        return dict(op="plane", model=name, precision=p, input=f"m{name}_{W}x{H}_{seed}", size=(H, W), seed=seed, **kw)

    def tiles(name, p, nt, W, H, seed):
        return dict(op="tiles", model=name, precision=p, input=f"t{name}_{nt}_{W}x{H}_{seed}", size=(nt, H, W), seed=seed)

    # k = 2: 4nk - 1 = 55 rows stays on one context, 56 is cut; a plane with >= 1024 rows per slab (automatic sub-bands)
    C.append((2, [plane("noise1", F16_F8X2, 40, 55, 1), plane("noise1", F16_F8X2, 40, 56, 2), plane("noise1", F16_F8X2, 24, 2100, 3),
                  tiles("noise1", F16_F8X2, 1, 30, 20, 4), tiles("noise1", F16_F8X2, 2, 30, 20, 5), tiles("noise1", F16_F8X2, 5, 30, 20, 6),
                  # progress lines: a plane the reference splits, with block splitting on and off, and one it does not
                  plane("noise1", F16_F8X2, 400, 1000, 7, block_splitting=True, log=True),
                  plane("noise1", F16_F8X2, 400, 1000, 7, block_splitting=False, log=True),
                  plane("noise1", F16_F8X2, 60, 90, 8, log=True)]))
    # k = 3: the plan cache -- precision, model, width and height change between calls, then back to the first plan
    C.append((3, [plane("noise1", F16_F8X2, 40, 83, 9), plane("noise1", F16_F8X2, 40, 84, 10), plane("noise1", F16X3, 40, 84, 10),
                  plane("scale2.0x", F16X3, 40, 84, 10), plane("scale2.0x", F16X3, 41, 84, 11), plane("scale2.0x", F16X3, 41, 100, 12),
                  plane("noise1", F16, 40, 84, 10), plane("noise1", F16_F8X2, 40, 84, 10),
                  tiles("noise1", F16, 2, 17, 33, 13), tiles("noise1", F16, 3, 17, 33, 14), tiles("noise1", F16, 7, 17, 33, 15)]))
    # k = 4: both sides of the rule for n = 7 and n = 4 models
    C.append((4, [plane("noise1", F16X3, 36, 111, 16), plane("noise1", F16X3, 36, 112, 17), plane("sel32", F16X3, 39, 63, 18),
                  plane("sel128", F16_F8X2, 39, 64, 19), plane("rand128", F16, 50, 200, 20),
                  tiles("sel32", F16_F8X2, 3, 20, 13, 21), tiles("sel32", F16_F8X2, 4, 20, 13, 22), tiles("rand128", F16X3, 9, 20, 13, 23)]))
    cases, inputs = [], {}
    for i, (k, calls) in enumerate(C):
        for c in calls:
            size, name = c.pop("size"), c["model"]
            seed = c.pop("seed")
            inputs[c["input"]] = (np.stack([seeded(size[1], size[2], 100 * seed + t, name) for t in range(size[0])])
                                  if c["op"] == "tiles" else seeded(*size, seed, name))
        cases.append(dict(id=f"multi{i}", kind="multi", k=k, calls=calls))
    return cases, inputs


@pytest.fixture(scope="module")
def worker_run(layers, tmp_path_factory):
    job = Job(layers)
    for c in band_cases():
        job.add(c, seeded(sum(c["rows"]), c["width"], int(c["id"][4:]), c["model"]))
    for c in slab_cases():
        job.add(c, seeded(sum(c["rows"]), c["width"], 50 + int(c["id"][4:]), c["model"]))
    mc, minputs = multi_cases()
    job.inputs.update(minputs)
    for c in mc:
        job.add(c)
    d = tmp_path_factory.mktemp("band_worker")
    job.write(d)
    (outs, log), = run_worker(d)
    return job, outs, log


def _check_passes(outs, key, want, W, seams):
    """every pass's plane equals the reference in its W columns; the row padding beyond them is untouched (NaN)"""
    fails = []
    for p in range(PASSES):
        got = outs[f"{key}.{p}"]
        msg = mismatch(got[:, :W], want, seams)
        if msg:
            fails.append(f"pass {p}: {msg}")
        if got.shape[1] > W and not np.all(np.isnan(got[:, W:])):
            fails.append(f"pass {p}: wrote into the row padding beyond column {W}")
    return fails


def test_band_run_connect_local(worker_run, ref):
    job, outs, _ = worker_run
    fails = []
    for c in (c for c in job.cases if c["kind"] == "band"):
        want = ref(c["model"], c["precision"], job.inputs[c["id"]])
        for f in _check_passes(outs, c["id"], want, c["width"], cuts(c["rows"])):
            fails.append(f"{c['id']} {c['model']} precision {c['precision']} w={c['width']} rows={c['rows']}: {f}")
    assert not fails, "\n".join(fails)


def test_slabs_connect_local(worker_run, ref):
    job, outs, _ = worker_run
    fails = []
    for c in (c for c in job.cases if c["kind"] == "slab"):
        want = ref(c["model"], c["precision"], job.inputs[c["id"]])
        r = cuts(c["rows"])
        seams = sorted({r[s] + v for s, rows in enumerate(c["rows"]) for v in slab_cuts(rows, n_of(c["model"]), c["n_sub"][s])})
        for f in _check_passes(outs, c["id"], want, c["width"], seams):
            fails.append(f"{c['id']} {c['model']} precision {c['precision']} w={c['width']} rows={c['rows']} n_sub={c['n_sub']} "
                         f"order={c['order']}: {f}")
    assert not fails, "\n".join(fails)


def _multi_seams(k, n, H):
    nd = min(k, H // (4 * n))
    if nd < 2:
        return [0, H]
    r0 = [H * i // nd for i in range(nd + 1)]
    return sorted({r0[i] + v for i in range(nd) for v in slab_cuts(r0[i + 1] - r0[i], n, 0)})


def test_multi_driver(worker_run, ref):
    job, outs, _ = worker_run
    fails = []
    for c in (c for c in job.cases if c["kind"] == "multi"):
        for j, call in enumerate(c["calls"]):
            x, got = job.inputs[call["input"]], outs[f"{c['id']}.{j}"]
            what = f"{c['id']} k={c['k']} call {j} {call['op']} {call['model']} precision {call['precision']} {x.shape}"
            if call["op"] == "tiles":
                for t in range(x.shape[0]):
                    msg = mismatch(got[t], ref(call["model"], call["precision"], x[t], block_splitting=False), [0])
                    if msg:
                        fails.append(f"{what} tile {t}: {msg}")
            else:
                want = ref(call["model"], call["precision"], x, block_splitting=call.get("block_splitting", True))
                msg = mismatch(got, want, _multi_seams(c["k"], n_of(call["model"]), x.shape[0]))
                if msg:
                    fails.append(f"{what}: {msg}")
    assert not fails, "\n".join(fails)


def test_multi_progress_lines_match_convert_plane(worker_run, ref):
    """w2x_multi_set_log: the lines of a multi call are convert_plane's for the same plane and block_splitting"""
    job, _, log = worker_run
    checked = 0
    for c in (c for c in job.cases if c["kind"] == "multi"):
        for j, call in enumerate(c["calls"]):
            if not call.get("log"):
                continue
            lines = []
            ctx = ref.ctx[call["precision"]]
            ctx.set_log(lines.append)
            try:
                ctx.convert_plane(ref.models[call["model"]], job.inputs[call["input"]], block_splitting=call.get("block_splitting", True))
            finally:
                ctx.set_log(None)
            assert log[f"{c['id']}.{j}"] == lines, (c["id"], j, call)
            checked += 1
    assert checked == 3


# ---------------------------------------------------------------------------------------------------------------------
# across processes: CUDA IPC
# ---------------------------------------------------------------------------------------------------------------------
def test_slabs_across_processes(layers, ref, tmp_path):
    """two ranks, w2x_slab_export / w2x_slab_connect, automatic n_sub (2 sub-bands of 525 rows each): bench.py's e2e path"""
    job = Job({"noise1": layers["noise1"]})
    rows = [1050, 1050]
    x = seeded(sum(rows), 48, 300, "noise1")
    job.add(dict(id="ipc", kind="slab_ipc", model="noise1", precision=[F16_F8X2, F16_F8X2], rows=rows, n_sub=0), x)
    job.write(tmp_path)
    res = run_worker(tmp_path, ranks=(0, 1))
    want = ref("noise1", F16_F8X2, x)
    seams = sorted({cuts(rows)[s] + v for s in range(2) for v in slab_cuts(rows[s], 7, 0)})
    fails = []
    for p in range(PASSES):
        got = np.concatenate([res[r][0][f"ipc.{r}.{p}"] for r in range(2)])
        msg = mismatch(got, want, seams)
        if msg:
            fails.append(f"pass {p}: {msg}")
    assert not fails, "\n".join(fails)


def test_connect_refuses_a_neighbour_in_another_precision(layers, tmp_path):
    """w2x_band_connect (IPC) refuses a neighbour session of another precision, as w2x_band_connect_local does: the rows it
    would exchange have the same size and another format"""
    job = Job({"noise1": layers["noise1"]})
    job.add(dict(id="mix", kind="slab_ipc", model="noise1", precision=[F16X3, F16_F8X2], rows=[60, 60], n_sub=0, run=False),
            seeded(120, 40, 301, "noise1"))
    job.write(tmp_path)
    res = run_worker(tmp_path, ranks=(0, 1))
    for r in range(2):
        outs, log = res[r]
        assert "mix.connect" in log, f"rank {r} connected to a neighbour in another precision"
        status, msg = log["mix.connect"]
        assert status == 1 and "precision" in msg, (r, status, msg)
        assert not outs, f"rank {r} ran"


# ---------------------------------------------------------------------------------------------------------------------
# w2x_ctx_forget_model and live band sessions
# ---------------------------------------------------------------------------------------------------------------------
def test_forget_model_refused_while_band_sessions_hold_it(layers, ref, tmp_path):
    job = Job({k: layers[k] for k in ("noise1", "scale2.0x")})
    rows = [9, 1, 50]                    # 60 rows: w2x_multi_convert_plane cuts them for two contexts (>= 4n rows each)
    x = seeded(sum(rows), 35, 302, "noise1")
    job.add(dict(id="forget", kind="forget", model="noise1", model2="scale2.0x", precision=F16_F8X2, rows=rows), x)
    job.write(tmp_path)
    (outs, log), = run_worker(tmp_path)
    st = log["forget"]
    for k in ("band open", "band open, last context", "slab open", "multi plan", "multi plan, its model"):
        status, msg = st[k]
        assert status == 1 and "band session" in msg, (k, st[k])
    for k in ("band open, other model", "band closed", "slab closed", "multi plan of the other model"):
        assert st[k] == [0, ""], (k, st[k])
    fails = _check_passes(outs, "forget", ref("noise1", F16_F8X2, x), x.shape[1], cuts(rows))
    assert not fails, "\n".join(fails)


def test_multi_keeps_the_plane_plan_beside_the_chain_plan(layers, ref, tmp_path):
    """a chain between two plane calls leaves the plane's plan in place: both plans' models are refused by w2x_ctx_forget_model
    after the chain, and the second plane call gives the first one's bits with the same launches"""
    names = ["rand128", "noise1", "scale2.0x"]
    job = Job({k: layers[k] for k in names})
    x = seeded(60, 35, 303, "noise1")     # 60 rows: the plane (n = 4) and the chain (n = 7) are both cut for two contexts
    job.add(dict(id="plans", kind="plans", models=names, precision=F16_F8X2), x)
    job.write(tmp_path)
    (outs, log), = run_worker(tmp_path)
    st = log["plans"]
    for k in ("plane's model", "chain's model"):
        status, msg = st[k]
        assert status == 1 and "band session" in msg, (k, st[k])
    msg = mismatch(outs["plans.plane"], ref("rand128", F16_F8X2, x), _multi_seams(2, 4, 60))
    assert not msg, msg
    want = ref.ctx[F16_F8X2].convert_chain([(ref.models["noise1"], False), (ref.models["scale2.0x"], True)], x)
    msg = mismatch(outs["plans.chain"], want, [0, 60, 120])
    assert not msg, msg
    assert np.array_equal(outs["plans.plane again"], outs["plans.plane"])
    assert all(st["plane launches"]) and all(st["chain launches"]), st
    assert st["plane again launches"] == st["plane launches"], st
