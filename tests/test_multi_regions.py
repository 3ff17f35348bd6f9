"""w2x_multi_convert_chain_regions (csrc/engine.cu): many windows of chains' outputs across the GPUs of a w2x_multi, each window on one
owner GPU.

Without a GPU: the placement (w2x_debug_plan_multi_regions) against a Python restatement of the rule in include/w2x_b200.h on random
window sets -- the GPUs used, every owner and every GPU's load -- with windows at every border, 1 x 1 windows, odd 2x origins and
chains of mixed depth with and without upscaling steps; the planner's refusals; the NULL handle; the binding's signatures.
On the GPU: the "GPUs" are 2, 3 and 4 contexts of device 0 (and one), driven in tests/multi_regions_worker.py (a child process with
CUDA_DEVICE_MAX_CONNECTIONS set before CUDA starts).  Every call runs twice and every window must equal, bit for bit, what
Context.convert_chain_regions gives on one context and the same window of Context.convert_chain(..., block_splitting=False); two
selection chains of test_chain_exact.py are compared with its chain emulator as well.  The cases cover the shipped models in all
three precisions and the fp32 engine, tiles of one plane whose sources and outputs are strided views of one array (pinned and
pageable, and for a plane past HostPin's 4 MiB floor, that both are registered with CUDA during the call and not after it), float64
and column-strided sources that the binding copies, NaN around every source rectangle and in the output row padding, a scratch limit
under which one GPU packs two frames and converts a window alone, one window and one context; the protocol (lines and on_step order, each context's launches against the
one-context call on the windows it owns); refusals and W2X_ERR_NOMEM, which queue nothing on any context.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_band_exchange import ENV, Job
from test_chain_exact import LAYERS as SEL_LAYERS, WINDOW_PLANES, depths, emulate_chain, spec_of, ups_of, window_cases
from test_region import odd_windows, region_windows

gpu = pytest.mark.gpu
WORKER = os.path.join(ROOT, "tests", "multi_regions_worker.py")
F16X3, F16_F8X2, F16 = 0, 1, 2
ENGINE_FP32, ENGINE_TC = 1, 2
ERR_ARG, ERR_UNSUPPORTED, ERR_NOMEM = 1, 7, 8
N1, N2, S = "noise1", "noise2", "scale2.0x"
SELS = {"selA": "A", "selB": "B", "selC": "C"}
PREC_NAMES = {F16X3: "f16x3", F16_F8X2: "f16+f8x2", F16: "f16"}


# ---------------------------------------------------------------------------------------------------------------------
# the placement, without a device
# ---------------------------------------------------------------------------------------------------------------------
def macs(model):
    return sum(9 * model.dims(layer)[0] * model.dims(layer)[1] for layer in range(len(model)))


def restated_plan(n_devices, steps, sizes, windows):
    """the rule of include/w2x_b200.h: (nd, owner, load, work)"""
    n = len(windows)
    nd = min(n_devices, n)
    layers, ups = [len(m) for m, _ in steps], [up for _, up in steps]
    work = []
    for (width, height), win in zip(sizes, windows):
        outs = region_windows(layers, ups, width, height, win)[1:]
        work.append(sum(o[2] * o[3] * macs(m) for (m, _), o in zip(steps, outs)))
    order = sorted(range(n), key=lambda i: (-work[i], i))
    load, owner = [0] * nd, [0] * n
    for i in order:
        o = min(range(nd), key=lambda o: (max(load[:o] + [load[o] + work[i]] + load[o + 1:]), load[o], o))
        owner[i] = o
        load[o] += work[i]
    return nd, owner, load, work


@pytest.fixture(scope="module")
def cpu_models(w2x):
    rng = np.random.default_rng(3)

    def model(dims):
        return w2x.Model.from_arrays([rng.standard_normal((co, ci, 3, 3)).astype(np.float32) * 0.1 for ci, co in dims],
                                     [rng.standard_normal(co) * 0.01 for _, co in dims])
    return [model([(1, 32), (32, 64), (64, 1)]), model([(1, 32), (32, 32), (32, 64), (64, 128), (128, 1)]), model([(1, 16), (16, 1)])]


def random_window(rng, W, H):
    """a window of a W x H output: the whole output, 1 x 1, at a border or corner, on odd coordinates, or anywhere"""
    kind = int(rng.integers(6))
    if kind == 0:
        return (0, 0, W, H)
    if kind == 1:
        return (int(rng.integers(W)), int(rng.integers(H)), 1, 1)
    w, h = int(rng.integers(1, W + 1)), int(rng.integers(1, H + 1))
    if kind == 2:                                   # bottom-right corner
        return (W - w, H - h, w, h)
    if kind == 3:                                   # left or top border
        return (0, int(rng.integers(H - h + 1)), w, h) if rng.integers(2) else (int(rng.integers(W - w + 1)), 0, w, h)
    x0, y0 = int(rng.integers(W - w + 1)), int(rng.integers(H - h + 1))
    if kind == 4:                                   # odd origin
        x0, y0 = min(x0 | 1, W - w) if W - w >= 1 else x0, min(y0 | 1, H - h) if H - h >= 1 else y0
    return (x0, y0, w, h)


def random_case(rng, cpu_models, trial):
    steps = [(cpu_models[int(rng.integers(len(cpu_models)))], bool(rng.integers(2))) for _ in range(int(rng.integers(1, 4)))]
    if trial % 4 == 0:
        steps = [(m, False) for m, _ in steps]      # no upscaling step
    ups = sum(1 for _, up in steps if up)
    n = int(rng.integers(1, 40)) if trial % 5 else int(rng.integers(1, 3))
    planes = [(int(rng.integers(1, 60)), int(rng.integers(1, 60))) for _ in range(int(rng.integers(1, 4)))]
    sizes, windows = [], []
    for _ in range(n):
        w, h = planes[int(rng.integers(len(planes)))]
        sizes.append((w, h))
        windows.append(random_window(rng, w << ups, h << ups))
    if trial % 7 == 0:                              # many equal windows: ties everywhere
        sizes, windows = [(16, 16)] * n, [(2, 2, 8, 8)] * n
    return steps, sizes, windows


def test_placement_matches_the_restated_rule(w2x, cpu_models):
    rng = np.random.default_rng(21)
    seen_nd, seen = set(), set()
    for trial in range(200):
        steps, sizes, windows = random_case(rng, cpu_models, trial)
        n_dev = int(rng.integers(1, 10))
        nd, owner, load = w2x.debug_plan_multi_regions(n_dev, steps, sizes, windows)
        want_nd, want_owner, want_load, work = restated_plan(n_dev, steps, sizes, windows)
        what = (trial, n_dev, [(macs(m), up) for m, up in steps], sizes, windows)
        assert nd == want_nd == min(n_dev, len(windows)), what
        assert owner.tolist() == want_owner, what
        assert load.tolist() == want_load, what
        again = [0] * nd
        for i, o in enumerate(owner.tolist()):
            again[o] += work[i]
        assert again == load.tolist(), what
        seen_nd.add(nd)
        ups = sum(1 for _, up in steps if up)
        for (w, h), win in zip(sizes, windows):
            W, H = w << ups, h << ups
            seen.add("border" if win[0] == 0 or win[1] == 0 or win[0] + win[2] == W or win[1] + win[3] == H else "inside")
            seen.add("1x1" if win[2:] == (1, 1) else "larger")
            if ups and (win[0] % 2 or win[1] % 2):
                seen.add("odd 2x origin")
        seen.add(("depths", len({len(m) for m, _ in steps}) > 1, ups > 0))
    assert len(seen_nd) >= 6
    assert {"border", "inside", "1x1", "larger", "odd 2x origin"} <= seen
    assert {("depths", a, b) for a in (False, True) for b in (False, True)} <= seen, seen


def test_plain_windows_meet_the_list_scheduling_bound(w2x, cpu_models):
    rng = np.random.default_rng(22)
    for trial in range(60):
        steps, sizes, windows = random_case(rng, cpu_models, trial)
        n_dev = int(rng.integers(2, 9))
        nd, _, load = w2x.debug_plan_multi_regions(n_dev, steps, sizes, windows)
        _, _, _, work = restated_plan(n_dev, steps, sizes, windows)
        assert nd == min(n_dev, len(windows))
        assert max(load) <= sum(work) / nd + max(work), (trial, load.tolist(), work)


def test_planner_refuses_what_the_call_refuses(w2x, cpu_models):
    m = cpu_models[0]
    cases = [(2, [(m, False)], [], [], "bad argument"),                             # no windows
             (0, [(m, False)], [(4, 4)], [(0, 0, 4, 4)], "bad argument"),
             (2, [(m, False), (m, True, True)], [(4, 4)], [(0, 0, 8, 8)], "window 0: step 1: a W2X_STEP_TTA step has no window form"),
             (2, [(m, False)], [(4, 4), (4, 4)], [(0, 0, 4, 4), (1, 1, 4, 4)], "window 1: window {1, 1, 4, 4} is not inside"),
             (2, [(m, True)], [(4, 4), (0, 4)], [(0, 0, 4, 4), (0, 0, 1, 1)], "window 1: step 0: input size")]
    for n_dev, steps, sizes, windows, want in cases:
        with pytest.raises(w2x.W2xError) as e:
            w2x.debug_plan_multi_regions(n_dev, steps, sizes, windows)
        assert e.value.status == ERR_ARG and want in e.value.message, (want, e.value.message)


def test_a_null_handle_is_refused_before_anything_else(w2x, cpu_models):
    n, models, kinds, _, _ = w2x.Context._chain_args([(cpu_models[0], True)], None)
    calls = []
    cb = w2x.capi.STEP_FN(lambda k, _u: calls.append(k))
    one = (C.c_int * 1)(8)
    win = (C.c_int * 4)(0, 0, 2, 2)
    ptr = (C.c_void_p * 1)(None)
    st = (C.c_size_t * 1)(32)
    L = w2x.lib()
    assert L.w2x_multi_convert_chain_regions(None, n, models, kinds, 1, one, one, win, ptr, st, ptr, st, cb, None) == ERR_ARG
    assert L.w2x_last_error().decode() == "w2x_multi_convert_chain_regions: NULL handle"
    assert L.w2x_convert_chain_regions(None, n, models, kinds, 1, one, one, win, ptr, st, ptr, st, cb, None) == ERR_ARG
    assert not calls


def test_binding_declares_the_multi_regions_entries(w2x):
    L = w2x.lib()
    assert L.w2x_multi_convert_chain_regions.argtypes[1:] == L.w2x_convert_chain_regions.argtypes[1:]
    assert len(L.w2x_multi_convert_chain_regions.argtypes) == 14 and len(L.w2x_debug_plan_multi_regions.argtypes) == 10
    assert "w2x_multi_convert_chain_regions" in w2x.capi.ABI_SYMBOLS
    assert callable(w2x.Multi.convert_chain_regions) and callable(w2x.debug_plan_multi_regions)


# ---------------------------------------------------------------------------------------------------------------------
# the worker run
# ---------------------------------------------------------------------------------------------------------------------
COLLECTIONS = {
    "three": [(45, 37), (30, 41), (19, 12)],
    "small": [(23, 19), (17, 26)],                  # chains with two 2x steps
    "scan": [(61, 47)],
    "pack": [(70, 64)],
    "pages": [(40, 30), (33, 21), (16, 16), (9, 25)],
    "big": [(2048, 2048)],
    "raw": [(20, 16), (17, 21)],
    "sel0": WINDOW_PLANES,                          # the planes of test_chain_exact.py's first two window cases
    "sel1": WINDOW_PLANES,
    "wide": [(1100, 1000)],                         # a 4.4 MB plane and a 17.6 MB output: their unions reach HostPin's 4 MiB
}
SHIPPED_CHAINS = [[[N1, False]], [[S, True]], [[N2, False], [S, True]], [[S, True], [S, True]], [[N1, False], [S, True], [N2, False]]]


def mixed(coll, ups):
    """windows of every plane: at every border, 1 x 1, the whole output, on odd and even 2x rows and columns"""
    wins = []
    for p, (w, h) in enumerate(COLLECTIONS[coll]):
        W, H = w << ups, h << ups
        wins += [[p, list(win)] for win in odd_windows(W, H) if win[2] > 0 and win[3] > 0]
        wins += [[p, [0, 0, 1, 1]], [p, [W - 1, H - 1, 1, 1]], [p, [W // 2 | 1, H // 2 | 1, 1, 1]]]
    return wins


def tiles(coll, ups, tw, th):
    w, h = COLLECTIONS[coll][0]
    W, H = w << ups, h << ups
    return [[0, [x, y, min(tw, W - x), min(th, H - y)]] for y in range(0, H, th) for x in range(0, W, tw)]


def patches(coll, ups, n, side, seed):
    rng = np.random.default_rng(seed)
    wins = []
    for p, (w, h) in enumerate(COLLECTIONS[coll]):
        W, H = w << ups, h << ups
        s = min(side, W, H)
        wins += [[p, [int(rng.integers(W - s + 1)), int(rng.integers(H - s + 1)), s, s]] for _ in range(n)]
    return wins


# a scratch limit of 3000 pixels of 128 channels: two 34 x 34 rectangles a frame, and the 110 x 100 windows converted alone
PACK_LIMIT = 128 * 4 * 3000
PACK_WINS = [[0, [3, 5, 110, 100]], [0, [1, 1, 20, 20]], [0, [40, 30, 20, 19]], [0, [70, 2, 21, 20]], [0, [100, 101, 20, 20]],
             [0, [9, 110, 18, 17]], [0, [20, 15, 110, 100]], [0, [0, 0, 20, 20]], [0, [120, 108, 20, 20]], [0, [57, 77, 19, 21]]]


def regions(steps, coll, wins, **kw):
    return dict(op="regions", steps=steps, coll=coll, wins=wins, **kw)


def sel_calls():
    """two selection chains of test_chain_exact.py on its window planes, in the precision the chain is emulated in"""
    calls = []
    names = {v: k for k, v in SELS.items()}
    for c, ((spec, _), prec) in enumerate(zip(window_cases("f16x3"), (F16X3, F16_F8X2))):
        steps = [[names[m], up] for m, up, _ in spec]
        calls.append(regions(steps, f"sel{c}", mixed(f"sel{c}", ups_of(spec)), precision=prec, engine=ENGINE_TC))
    return calls


def groups():
    out = []
    for k in (2, 3, 4):
        out.append((k, [regions([[N2, False], [S, True]], "three", mixed("three", 1)),
                        regions([[N1, False], [S, True]], "scan", tiles("scan", 1, 32, 24), layout="tiles", pinned=[True, True]),
                        regions([[N1, False], [S, True]], "scan", tiles("scan", 1, 32, 24), layout="tiles", pinned=[False, False])]))
    shipped = []
    for c, steps in enumerate(SHIPPED_CHAINS):
        ups = sum(1 for _, up in steps if up)
        coll = "small" if ups >= 2 else "three"
        for prec, engine in ((F16X3, ENGINE_TC), (F16, ENGINE_TC), (F16_F8X2, ENGINE_FP32)):
            shipped.append(regions(steps, coll, mixed(coll, ups), precision=prec, engine=engine))
    out.append((2, shipped + [
        regions([[N2, False], [S, True]], "three", mixed("three", 1)[::3], layout="padded", pinned=[False, True], out_pad=5),
        regions([[N2, False], [S, True]], "three", mixed("three", 1)[1::3], layout="padded", pinned=[True, False], engine=ENGINE_FP32),
        regions([[N1, False], [S, True]], "pack", PACK_WINS, scratch=PACK_LIMIT, engine=ENGINE_TC),
        regions([[N2, False], [S, True]], "three", mixed("three", 1)[::2], sources="f64"),           # sources the binding copies
        regions([[N2, False], [S, True]], "three", mixed("three", 1)[1::2], sources="colstride", pinned=[False, False]),
        regions([[N1, False], [S, True]], "scan", [[0, [5, 7, 31, 21]]]),                      # one window: nd = 1
    ]))
    out.append((3, sel_calls() + [
        regions([[S, True]], "pages", patches("pages", 1, 16, 12, 5), pinned=[False, False]),
        regions([[N1, False], [S, True]], "three", [[0, [3, 3, 40, 30]], [2, [0, 0, 38, 24]]]),   # 2 windows on 3 GPUs
        regions([[N1, False], [S, True]], "wide", tiles("wide", 1, 512, 512), layout="tiles", pinned=[False, False], probe=True),
    ]))
    out.append((4, [regions([[S, True]], "pages", patches("pages", 1, 16, 12, 6)),
                    regions([[N1, False], [S, True]], "scan", tiles("scan", 1, 16, 16), layout="tiles", pinned=[False, True])]))
    out.append((1, [regions([[N2, False], [S, True]], "three", mixed("three", 1))]))          # one context
    return out


REFUSALS = [("n_windows", ERR_ARG), ("n_steps", ERR_ARG), ("tta", ERR_ARG), ("kind", ERR_ARG), ("null_model", ERR_ARG),
            ("empty", ERR_ARG), ("outside", ERR_ARG), ("size", ERR_ARG), ("null_source", ERR_ARG), ("null_output", ERR_ARG),
            ("src_stride", ERR_ARG), ("out_stride", ERR_ARG), ("null_windows", ERR_ARG), (None, ERR_UNSUPPORTED)]
RAW_WINS = [[0, [2, 3, 10, 9]], [1, [0, 0, 34, 42]], [0, [7, 1, 1, 1]]]


def raw_calls():
    calls = []
    for bad, _ in REFUSALS:
        steps = [[N1, False], ["tiny", True]] if bad is None else [[N1, False], [S, True]]     # tiny: refused by the TC engine
        calls.append(dict(op="raw", steps=steps, coll="raw", wins=RAW_WINS, bad=bad, engine=ENGINE_TC))
    return calls


@pytest.fixture(scope="module")
def layers(oracle_models):
    out = {name: list(zip(oracle_models[name].weights, oracle_models[name].biases)) for name in (N1, N2, S)}
    out.update({k: SEL_LAYERS[v] for k, v in SELS.items()})
    rng = np.random.default_rng(4)
    out["tiny"] = [((rng.standard_normal((3, 1, 3, 3)) / 3).astype(np.float32), rng.standard_normal(3) * 0.1),
                   ((rng.standard_normal((1, 3, 3, 3)) / np.sqrt(27)).astype(np.float32), rng.standard_normal(1) * 0.1)]
    return out


def collection(name):
    """the planes of collection `name`"""
    if name.startswith("sel"):
        return list(window_cases("f16x3"))[int(name[3:])][1]
    rng = np.random.default_rng(200 + list(COLLECTIONS).index(name))
    return [rng.random((h, w), dtype=np.float32) for w, h in COLLECTIONS[name]]


@pytest.fixture(scope="module")
def worker_run(layers, tmp_path_factory):
    job = Job(layers)
    for name in COLLECTIONS:
        for i, x in enumerate(collection(name)):
            job.inputs[f"{name}/{i}"] = x
    nomem = dict(op="nomem", steps=[[N1, False], [S, True]], coll="big", wins=[[0, [1, 1, 4094, 4094]], [0, [0, 0, 64, 64]]])
    gs = groups() + [(2, raw_calls()), (2, [nomem])]
    for i, (k, calls) in enumerate(gs):
        job.add(dict(id=f"g{i}", k=k, calls=calls))
    d = tmp_path_factory.mktemp("multi_regions_worker")
    job.write(d)
    p = subprocess.run([sys.executable, WORKER, str(d)], env=dict(os.environ, **ENV), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1500)
    assert p.returncode == 0, p.stdout
    return job, dict(np.load(os.path.join(d, "out0.npz"))), json.load(open(os.path.join(d, "log0.json")))


def region_calls(job):
    for c in job.cases:
        for j, call in enumerate(c["calls"]):
            if call["op"] == "regions":
                yield c, call, f"{c['id']}.{j}"


@pytest.fixture(scope="module")
def models(w2x, layers):
    return {k: w2x.Model.from_arrays([w for w, _ in v], [b for _, b in v]) for k, v in layers.items()}


def plan(w2x, models, k, call):
    steps = [(models[m], up) for m, up in call["steps"]]
    sizes = [(collection(call["coll"])[p].shape[1], collection(call["coll"])[p].shape[0]) for p, _ in call["wins"]]
    return w2x.debug_plan_multi_regions(k, steps, sizes, [w for _, w in call["wins"]])


def crop(a, win):
    x0, y0, w, h = win
    return a[y0:y0 + h, x0:x0 + w]


def test_the_pack_case_makes_one_gpu_pack_two_frames_and_convert_a_window_alone(w2x, models):
    """the precondition of the scratch-limited GPU case: on some GPU the last step's plan of the windows it owns has two frames
    or more and a window converted alone"""
    call = regions([[N1, False], [S, True]], "pack", PACK_WINS)
    nd, owner, _ = plan(w2x, models, 2, call)
    (w, h), = COLLECTIONS["pack"]
    outs = [region_windows([7, 7], [False, True], w, h, win)[-1] for _, win in PACK_WINS]
    found = False
    for g in range(nd):
        mine = [o for o, d in zip(outs, owner.tolist()) if d == g]
        frame, _, _, _ = w2x.debug_plan_planes([o[2] for o in mine], [o[3] for o in mine], 7, 128, PACK_LIMIT)
        found = found or (frame.max() >= 1 and (frame == -1).any())
    assert nd == 2 and found, owner


def test_the_selection_chains_differ_in_depth():
    for call in sel_calls():
        spec = spec_of([[m, up, False] for m, up in call["steps"]], SELS)
        assert len(set(depths(spec))) > 1, spec


@gpu
def test_every_window_is_bit_identical_to_one_context_and_the_whole_chain(worker_run):
    """and, for the selection chains, to the chain emulator; NaN row padding and the parts of tile arrays no window covers stay NaN"""
    job, outs, log = worker_run
    fails, checked, emulated = [], 0, 0
    for c, call, key in region_calls(job):
        wins = [(p, tuple(w)) for p, w in call["wins"]]
        sel = all(m in SELS for m, _ in call["steps"])
        if sel:
            spec = spec_of([[m, up, False] for m, up in call["steps"]], SELS)
            ems = {p: emulate_chain(spec, x, PREC_NAMES[call["precision"]]) for p, x in enumerate(collection(call["coll"]))}
        assert len(log[key]["passes"]) == 2, key
        for i, (p, win) in enumerate(wins):
            ref, whole = outs[f"{key}.ref.{i}"], crop(outs[f"{key}.whole.{p}"], win)
            if not np.array_equal(ref, whole):
                fails.append(f"{key} one context window {i} {win} is not the whole chain's crop")
            if call.get("sources") and not np.array_equal(outs[f"{key}.refsrc.{i}"], ref):
                fails.append(f"{key} one context window {i} {win} from {call['sources']} sources is not the float32 call's")
            if sel:
                emulated += 1
                if not np.array_equal(ref, crop(ems[p], win)):
                    fails.append(f"{key} one context window {i} {win} is not the emulator's crop")
            for ps in range(2):
                if call.get("layout") == "tiles":
                    got = crop(outs[f"{key}.{ps}.plane{p}"], win)
                else:
                    a = outs[f"{key}.{ps}.{i}"]
                    got = a[:, :win[2]]
                    if not np.isnan(a[:, win[2]:]).all():
                        fails.append(f"{key} pass {ps} window {i}: wrote into the row padding")
                if not np.array_equal(got, ref):
                    fails.append(f"{key} k={c['k']} {call['steps']} pass {ps} window {i} {win}: not the one-context window")
                checked += 1
        if call.get("layout") == "tiles":
            for ps in range(2):
                a = outs[f"{key}.{ps}.plane0"]
                W = outs[f"{key}.whole.0"].shape[1]
                if not np.array_equal(a[:, :W], outs[f"{key}.whole.0"]) or not np.isnan(a[:, W:]).all():
                    fails.append(f"{key} pass {ps}: the tiles do not make the whole chain")
    assert checked > 1500 and emulated >= 40 and not fails, "\n".join(fails[:30])


@gpu
def test_sources_the_binding_copies_give_the_float32_bits(worker_run):
    """float64 rectangles and column-strided views are copied to float32 rows by the binding, and the copies outlive the call"""
    job, outs, _ = worker_run
    seen = set()
    for _, call, key in region_calls(job):
        if call.get("sources"):
            seen.add(call["sources"])
            for i in range(len(call["wins"])):
                assert np.array_equal(outs[f"{key}.0.{i}"][:, :call["wins"][i][1][2]], outs[f"{key}.ref.{i}"]), (key, i)
                assert np.array_equal(outs[f"{key}.refsrc.{i}"], outs[f"{key}.ref.{i}"]), (key, i)
    assert seen == {"f64", "colstride"}


@gpu
def test_pageable_buffers_are_pinned_for_the_call(worker_run):
    """the page-rounded union of the tiles' sources (views of one plane) and of their outputs (views of one array) is registered
    while the call runs, and unregistered before it returns"""
    job, _, log = worker_run
    (_, _, key), = [x for x in region_calls(job) if x[1].get("probe")]
    rec = log[key]
    assert rec["controls"] == [True, False], rec["controls"]          # the probe tells pinned memory from pageable memory
    for p in range(2):
        assert rec["probe"]["plane"][p] == [False, True, False], rec["probe"]
        assert rec["probe"]["out"][p] == [False, True, False], rec["probe"]


@gpu
def test_lines_and_on_step_order_are_the_one_context_calls(worker_run):
    job, _, log = worker_run
    for c, call, key in region_calls(job):
        want = log[key]["ref"]["events"]
        assert want[0] == "step 0" and sum(e.startswith("step ") for e in want) == len(call["steps"]), key
        assert len(want) > len(call["steps"]), key
        for p, rec in enumerate(log[key]["passes"]):
            assert rec["events"] == want, (key, p, call["steps"])


@gpu
def test_each_context_launches_the_one_context_call_on_its_windows(w2x, models, worker_run):
    job, _, log = worker_run
    seen_nd = set()
    for c, call, key in region_calls(job):
        nd, owner, _ = plan(w2x, models, c["k"], call)
        rec = log[key]
        assert rec["owner"] == owner.tolist(), key
        assert nd == min(c["k"], len(call["wins"])), key
        for p in rec["passes"]:
            assert p["launches"] == rec["owner_launches"] + [0] * (c["k"] - nd), (key, p["launches"], rec["owner_launches"])
        if nd == 1:
            assert rec["passes"][1]["launches"][0] == rec["ref"]["launches"], key
        seen_nd.add((c["k"], nd))
    assert {(2, 2), (3, 3), (4, 4), (3, 2), (2, 1), (1, 1)} <= seen_nd, seen_nd


@gpu
def test_refusals_queue_and_log_nothing(worker_run):
    job, _, log = worker_run
    g = len(groups())
    for j, (bad, status) in enumerate(REFUSALS):
        rec = log[f"g{g}.{j}"]
        got, one = rec["multi"], rec["one"]
        assert got[0] == status == one[0], (bad, rec)
        assert got[1] == one[1].replace("w2x_convert_chain_regions", "w2x_multi_convert_chain_regions"), (bad, rec)
        assert got[1].startswith("w2x_multi_convert_chain_regions: "), (bad, rec)
        assert rec["events"] == [] and rec["launches"][0] == rec["launches"][1] and rec["untouched"], (bad, rec)
    assert "W2X_STEP_TTA" in log[f"g{g}.{[b for b, _ in REFUSALS].index('tta')}"]["multi"][1]


@gpu
def test_out_of_memory_leaves_nothing_queued(worker_run):
    job, outs, log = worker_run
    key = f"g{len(groups()) + 1}.0"
    rec = log[key]
    assert rec["error"][0] == ERR_NOMEM, rec
    assert rec["launches"][0] == rec["launches"][1] and rec["untouched"] and rec["events"] == [], rec
    assert rec["after"]
    for i in range(2):
        assert np.array_equal(outs[f"{key}.after.{i}"], outs[f"{key}.ref.{i}"]), i
