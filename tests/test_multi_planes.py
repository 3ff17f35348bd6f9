"""w2x_multi_convert_planes / w2x_multi_convert_planes_chain (csrc/engine.cu): collections of planes across the GPUs of a w2x_multi,
each plane on one owner GPU, a W2X_STEP_TTA step's 8 variants of a plane spread over the GPUs.

Without a GPU: the placement (w2x_debug_plan_multi_planes) against a numpy restatement of the rule in include/w2x_b200.h on random
collections -- the GPUs used, every owner and every GPU's load -- and the balance it promises; the binding's signatures.
On the GPU: the "GPUs" are 2, 3 and 4 contexts of device 0, driven in tests/multi_planes_worker.py (a child process with
CUDA_DEVICE_MAX_CONNECTIONS set before CUDA starts).  Every call runs twice and must give, bit for bit, what Context.convert_planes_chain
gives on one context, with the same progress lines and on_step calls; step patterns S, U, SU, SUU and US with TTA on no, some and all
steps; chains of the selection models of test_chain_exact.py (n = 3, 4, 6), also compared with its chain emulator; all three
precisions and the fp32 engine; one plane (a single image's TTA across GPUs), fewer planes than GPUs, 300 planes with
sides 1-160, a plane too large to pack among small ones, row-strided pinned and pageable host planes; the one-step W2X_STEP_SAME call
against Multi.convert_planes and Context.convert_planes; a call on one GPU against the one-context call's launches; the launches of
collection A against its frames; refusals and W2X_ERR_NOMEM, which queue nothing on any context.
Peer access between distinct devices cannot be exercised on one GPU: contexts of one device always qualify.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_band_exchange import ENV, RANDOM, Job, mismatch
from test_chain_exact import LAYERS as SEL_LAYERS, emulate_chain, spec_of

gpu = pytest.mark.gpu
WORKER = os.path.join(ROOT, "tests", "multi_planes_worker.py")
F16X3, F16_F8X2, F16 = 0, 1, 2
ENGINE_FP32 = 1
NOISE, SCALE, RAND = "noise1", "scale2.0x", "rand128"
# the selection models of test_chain_exact.py (n = 3, 4, 6): their chains are compared with the chain emulator as well
SELS = {"selA": "A", "selB": "B", "selC": "C"}
PREC_NAMES = {F16X3: "f16x3", F16_F8X2: "f16+f8x2", F16: "f16"}


# ---------------------------------------------------------------------------------------------------------------------
# the placement, without a device
# ---------------------------------------------------------------------------------------------------------------------
def macs(model):
    return sum(9 * model.dims(layer)[0] * model.dims(layer)[1] for layer in range(len(model)))


def restated_plan(n_devices, steps, widths, heights):
    """the rule of include/w2x_b200.h: (nd, owner, load)"""
    n = len(widths)
    tta = any(t for _, _, t in steps)
    nd = min(n_devices, (8 if tta else 1) * n)
    plain, var = [0] * n, [0] * n
    w, h = list(widths), list(heights)
    for model, up, t in steps:
        if up:
            w, h = [2 * v for v in w], [2 * v for v in h]
        m = macs(model)
        for i in range(n):
            if t:
                var[i] += w[i] * h[i] * m
            else:
                plain[i] += w[i] * h[i] * m
    order = sorted(range(n), key=lambda i: (-(plain[i] + 8 * var[i]), i))
    load, owner = [0] * nd, [0] * n
    for i in order:
        best = None
        for o in range(nd):
            trial = list(load)
            trial[o] += plain[i]
            if tta:
                for j in range(8):
                    trial[(o + j) % nd] += var[i]
            key = (max(trial), load[o], o)
            if best is None or key < best[0]:
                best = (key, o)
        o = best[1]
        owner[i] = o
        load[o] += plain[i]
        if tta:
            for j in range(8):
                load[(o + j) % nd] += var[i]
    return nd, owner, load, plain, var


@pytest.fixture(scope="module")
def cpu_models(w2x):
    rng = np.random.default_rng(3)

    def model(dims):
        return w2x.Model.from_arrays([rng.standard_normal((co, ci, 3, 3)).astype(np.float32) * 0.1 for ci, co in dims],
                                     [rng.standard_normal(co) * 0.01 for _, co in dims])
    return [model([(1, 32), (32, 64), (64, 1)]), model([(1, 32), (32, 32), (32, 64), (64, 128), (128, 1)]), model([(1, 16), (16, 1)])]


def random_chain(rng, cpu_models, tta_p):
    return [(cpu_models[int(rng.integers(len(cpu_models)))], bool(rng.integers(2)), bool(rng.random() < tta_p))
            for _ in range(int(rng.integers(1, 4)))]


def test_placement_matches_the_restated_rule(w2x, cpu_models):
    rng = np.random.default_rng(11)
    seen_nd = set()
    for trial in range(150):
        steps = random_chain(rng, cpu_models, [0.0, 0.3, 1.0][trial % 3])
        n = int(rng.integers(1, 40)) if trial % 5 else int(rng.integers(1, 3))
        ws, hs = rng.integers(1, 200, n), rng.integers(1, 200, n)
        if trial % 7 == 0:      # many equal sizes: ties everywhere
            ws, hs = np.full(n, 16), np.full(n, 16)
        n_dev = int(rng.integers(1, 10))
        nd, owner, load = w2x.debug_plan_multi_planes(n_dev, steps, ws, hs)
        want_nd, want_owner, want_load, plain, var = restated_plan(n_dev, steps, ws.tolist(), hs.tolist())
        what = (trial, n_dev, [(macs(m), u, t) for m, u, t in steps], ws.tolist(), hs.tolist())
        assert nd == want_nd, what
        assert owner.tolist() == want_owner, what
        assert load.tolist() == want_load, what
        tta = any(t for _, _, t in steps)
        assert nd == min(n_dev, (8 if tta else 1) * n), what
        # the loads are what the owners give with variant j of plane i on (owner + j) mod nd
        again = [0] * nd
        for i, o in enumerate(owner.tolist()):
            again[o] += plain[i]
            for j in range(8 if tta else 0):
                again[(o + j) % nd] += var[i]
        assert again == load.tolist(), what
        seen_nd.add(nd)
    assert len(seen_nd) >= 6


def test_tta_only_chains_spread_evenly(w2x, cpu_models):
    rng = np.random.default_rng(12)
    for nd in (2, 4, 8):
        for trial in range(10):
            steps = [(m, u, True) for m, u, _ in random_chain(rng, cpu_models, 1.0)]
            n = int(rng.integers(1, 30))
            _, _, load = w2x.debug_plan_multi_planes(nd, steps, rng.integers(1, 300, n), rng.integers(1, 300, n))
            assert len(load) == nd and len(set(load.tolist())) == 1, (nd, trial, load)


def test_plain_chains_meet_the_list_scheduling_bound(w2x, cpu_models):
    rng = np.random.default_rng(13)
    for trial in range(60):
        steps = random_chain(rng, cpu_models, 0.0)
        n, n_dev = int(rng.integers(1, 60)), int(rng.integers(2, 9))
        ws, hs = rng.integers(1, 300, n), rng.integers(1, 300, n)
        nd, owner, load = w2x.debug_plan_multi_planes(n_dev, steps, ws, hs)
        _, _, _, plain, _ = restated_plan(n_dev, steps, ws.tolist(), hs.tolist())
        assert nd == min(n_dev, n)
        assert max(load) <= sum(plain) / nd + max(plain), (trial, load.tolist(), plain)


def test_planner_refuses_bad_arguments(w2x, cpu_models):
    with pytest.raises(w2x.W2xError):
        w2x.debug_plan_multi_planes(0, [(cpu_models[0], False, False)], [4], [4])
    with pytest.raises(w2x.W2xError):
        w2x.debug_plan_multi_planes(2, [(cpu_models[0], False, False)], [4, 0], [4, 4])


def test_binding_declares_the_multi_planes_entries(w2x):
    L = w2x.lib()
    assert L.w2x_multi_convert_planes.argtypes[1:] == L.w2x_convert_planes.argtypes[1:]
    assert L.w2x_multi_convert_planes_chain.argtypes[1:] == L.w2x_convert_planes_chain.argtypes[1:]
    assert len(L.w2x_multi_convert_planes_chain.argtypes) == 13 and len(L.w2x_debug_plan_multi_planes.argtypes) == 9
    assert {"w2x_multi_convert_planes", "w2x_multi_convert_planes_chain"} <= set(w2x.capi.ABI_SYMBOLS)
    assert callable(w2x.Multi.convert_planes) and callable(w2x.Multi.convert_planes_chain)


# ---------------------------------------------------------------------------------------------------------------------
# the worker run
# ---------------------------------------------------------------------------------------------------------------------
def sizes_with_edges(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    s = [(int(w), int(h)) for w, h in rng.integers(lo, hi + 1, size=(n, 2))]
    if n >= 5:
        s[:4] = [(1, 1), (1, hi), (hi, 1), (hi, hi)]       # 1 x 1, 1 x N, N x 1 (w, h)
    return s


COLLECTIONS = {
    "c7": sizes_with_edges(1, 7, 1, 40),
    "c12": sizes_with_edges(2, 12, 1, 48),
    "c300": sizes_with_edges(3, 300, 1, 160),
    "one": [(61, 47)],
    "two": [(40, 30), (25, 50)],
    "mix": [(300, 200)] + sizes_with_edges(4, 40, 4, 40),
    "A": [(int(w), int(h)) for w, h in np.random.default_rng(1).integers(16, 129, size=(2000, 2))],
    "big": [(2048, 2048)],
    "sel": sizes_with_edges(5, 6, 1, 16),
}
PATTERNS = {"S": [False], "U": [True], "SU": [False, True], "SUU": [False, True, True], "US": [True, False]}


def pattern(name, tta):
    """tta: "none", "some" (one step of several), "all"""
    ups = PATTERNS[name]
    flags = [tta == "all" or (tta == "some" and k == len(ups) // 2) for k in range(len(ups))]
    return [[SCALE if up else NOISE, up, t] for up, t in zip(ups, flags)]


def chain(steps, c, **kw):
    return dict(op="chain", steps=steps, coll=c, **kw)


def groups():
    out = []
    for k in (2, 3, 4):
        calls = [chain(pattern(p, t), "c12") for p in PATTERNS for t in ("none", "some", "all") if not (t == "some" and len(PATTERNS[p]) == 1)]
        calls.append(chain([[NOISE, False, True]], "one"))                                      # one image's TTA across k GPUs
        calls.append(chain([[NOISE, False, True], [SCALE, True, True]], "one"))
        out.append((k, calls))
    out.append((2, [
        chain(pattern("SU", "some"), "c12", precision=F16X3), chain(pattern("SU", "some"), "c12", precision=F16),
        chain([[RAND, False, True], [RAND, True, False]], "c12", precision=F16X3),
        chain([[NOISE, False, True], [SCALE, True, False]], "mix", scratch=8 << 20),              # the 300 x 200 plane goes alone, in bands
        chain([[NOISE, False, False], [SCALE, True, True]], "c12", pinned=[False, False], in_pad=3, out_pad=5),
        chain([[NOISE, False, False]], "c12", entry="planes"), chain([[NOISE, False, False]], "c12"),   # one W2X_STEP_SAME step
        chain([[NOISE, False, False], [SCALE, True, False]], "one"),                               # nd = 1
        chain([[SCALE, True, False]], "A"),
    ]))
    out.append((3, [
        chain([[NOISE, False, True], [SCALE, True, False]], "c7", engine=ENGINE_FP32),
        chain([[NOISE, False, False], [SCALE, True, False]], "c300"),
        chain([[NOISE, False, False], [SCALE, True, False]], "mix", scratch=8 << 20),
        chain([[SCALE, True, True], [NOISE, False, False]], "c12", in_pad=2, out_pad=1),
        chain([[NOISE, False, False]], "c12", entry="planes"),
    ]))
    out.append((4, [
        chain([[NOISE, False, False], [SCALE, True, False]], "two"),                               # 2 planes, no TTA: 2 of 4 GPUs
        chain([[SCALE, True, True]], "c300"),
    ]))
    # selection chains whose steps differ in depth (3, 4, 6) and width, TTA on the first step and on a deep step after an upscale
    out.append((2, [
        chain([["selA", False, True], ["selC", True, False]], "sel", precision=F16X3),
        chain([["selC", True, False], ["selA", False, False]], "sel", precision=F16),
    ]))
    out.append((3, [
        chain([["selB", True, False], ["selA", False, False], ["selC", False, True]], "sel", precision=F16_F8X2),
        chain([["selC", True, False], ["selB", False, False]], "sel", precision=F16X3),
    ]))
    return out


REFUSALS = ["n_steps", "null_model", "kind", "n_planes", "stride", "width"]


@pytest.fixture(scope="module")
def layers(oracle_models, oracle_mod):
    out = {name: list(zip(oracle_models[name].weights, oracle_models[name].biases)) for name in (NOISE, SCALE)}
    dims, seed = RANDOM[RAND]
    om = oracle_mod.OracleModel.random(dims, seed=seed)
    out[RAND] = list(zip(om.weights, om.biases))
    out.update({k: SEL_LAYERS[v] for k, v in SELS.items()})
    return out


def collection(name):
    """the planes of collection `name`"""
    rng = np.random.default_rng(100 + list(COLLECTIONS).index(name))
    return [rng.random((h, w), dtype=np.float32) for w, h in COLLECTIONS[name]]


def selection_planes_cases():
    """(chain, plane, precision) of every plane of every selection-model call above, for test_chain_exact.py's check of the
    emulator's conditions"""
    for _, calls in groups():
        for c in calls:
            if all(m in SELS for m, _, _ in c["steps"]):
                for x in collection(c["coll"]):
                    yield spec_of(c["steps"], SELS), x, PREC_NAMES[c.get("precision", F16_F8X2)]


@pytest.fixture(scope="module")
def worker_run(layers, tmp_path_factory):
    job = Job(layers)
    for name in COLLECTIONS:
        for i, x in enumerate(collection(name)):
            job.inputs[f"{name}/{i}"] = x
    gs = groups() + [(2, [dict(op="raw", steps=[[NOISE, False, False], [SCALE, True, True]], coll="c7", bad=b) for b in REFUSALS]),
                     (2, [dict(op="nomem", steps=[[NOISE, False, True]], coll="big")])]
    for i, (k, calls) in enumerate(gs):
        job.add(dict(id=f"g{i}", k=k, calls=calls))
    d = tmp_path_factory.mktemp("multi_planes_worker")
    job.write(d)
    p = subprocess.run([sys.executable, WORKER, str(d)], env=dict(os.environ, **ENV), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1500)
    assert p.returncode == 0, p.stdout
    return job, dict(np.load(os.path.join(d, "out0.npz"))), json.load(open(os.path.join(d, "log0.json")))


def chain_calls(job):
    for c in job.cases:
        for j, call in enumerate(c["calls"]):
            if call["op"] == "chain":
                yield c, call, f"{c['id']}.{j}"


def n_gpus(w2x, models, k, call):
    sizes = COLLECTIONS[call["coll"]]
    steps = [(models[m], up, t) for m, up, t in call["steps"]]
    return w2x.debug_plan_multi_planes(k, steps, [w for w, _ in sizes], [h for _, h in sizes])


@pytest.fixture(scope="module")
def models(w2x, layers):
    return {k: w2x.Model.from_arrays([w for w, _ in v], [b for _, b in v]) for k, v in layers.items()}


@gpu
def test_every_pass_is_bit_identical_to_one_context(worker_run):
    """and, for chains of selection models, the one-context call and every pass to the chain emulator"""
    job, outs, log = worker_run
    fails, checked, emulated = [], 0, 0
    for c, call, key in chain_calls(job):
        n = len(COLLECTIONS[call["coll"]])
        sel = all(m in SELS for m, _, _ in call["steps"])
        xs = collection(call["coll"]) if sel else None
        for i in range(n):
            if sel:
                em = emulate_chain(spec_of(call["steps"], SELS), xs[i], PREC_NAMES[call.get("precision", F16_F8X2)])
                msg = mismatch(outs[f"{key}.ref.{i}"], em, [0])
                if msg:
                    fails.append(f"{key} {call['steps']} one context plane {i} {em.shape} against the emulator: {msg}")
                emulated += 1
            for p in range(len(log[key]["passes"])):
                want, got = outs[f"{key}.ref.{i}"], outs[f"{key}.{p}.{i}"]
                W = want.shape[1]
                msg = mismatch(got[:, :W], want, [0])
                if msg:
                    fails.append(f"{key} k={c['k']} {call['steps']} {call['coll']} pass {p} plane {i} {want.shape}: {msg}")
                if sel:
                    msg = mismatch(got[:, :W], em, [0])
                    if msg:
                        fails.append(f"{key} k={c['k']} {call['steps']} pass {p} plane {i} {em.shape} against the emulator: {msg}")
                if got.shape[1] > W and not np.all(np.isnan(got[:, W:])):
                    fails.append(f"{key} pass {p} plane {i}: wrote into the row padding")
                checked += 1
        assert len(log[key]["passes"]) == 2, key
    assert checked > 2000 and emulated >= 24 and not fails, "\n".join(fails[:30])


@gpu
def test_lines_and_on_step_order_are_the_one_context_calls(worker_run):
    job, _, log = worker_run
    for c, call, key in chain_calls(job):
        want = log[key]["ref"]["events"]
        if call.get("entry") == "planes":
            want = [e for e in want if not e.startswith("step ")]
        else:
            assert want[0] == "step 0" and sum(e.startswith("step ") for e in want) == len(call["steps"]), key
        for p, rec in enumerate(log[key]["passes"]):
            assert rec["events"] == want, (key, p, call)


@gpu
def test_launches_land_on_the_gpus_used(w2x, models, worker_run):
    job, _, log = worker_run
    for c, call, key in chain_calls(job):
        nd, owner, _ = n_gpus(w2x, models, c["k"], call)
        a, b = (r["launches"] for r in log[key]["passes"])
        assert a == b, (key, a, b)
        assert not any(a[nd:]), (key, nd, a)
        busy = set(owner.tolist()) | (set(range(nd)) if any(t for _, _, t in call["steps"]) else set())
        assert all(a[d] > 0 for d in busy), (key, nd, a)


@gpu
def test_one_same_step_is_convert_planes(worker_run):
    """Multi.convert_planes against a one-step W2X_STEP_SAME chain on as many contexts, and Context.convert_planes"""
    job, outs, log = worker_run
    calls = [(c["k"], call, key) for c, call, key in chain_calls(job) if call["steps"] == [[NOISE, False, False]] and call["coll"] == "c12"]
    planes = [(k, key) for k, call, key in calls if call.get("entry") == "planes"]
    assert len(planes) == 2
    for k, key in planes:
        chained = [ck for kk, call, ck in calls if kk == k and call.get("entry") != "planes"]
        assert chained, (k, key)
        assert log[key]["ref_planes"]["equal"] and log[key]["ref_planes"]["launches"] == log[key]["ref"]["launches"]
        for i in range(12):
            assert np.array_equal(outs[f"{key}.0.{i}"], outs[f"{chained[0]}.0.{i}"]), (key, i)
        assert log[key]["passes"][1]["launches"] == log[chained[0]]["passes"][1]["launches"]


@gpu
def test_one_gpu_used_is_the_one_context_call(w2x, models, worker_run):
    job, _, log = worker_run
    seen = 0
    for c, call, key in chain_calls(job):
        nd, _, _ = n_gpus(w2x, models, c["k"], call)
        if nd == 1:
            for rec in log[key]["passes"][1:]:
                assert rec["launches"] == [log[key]["ref"]["launches"]] + [0] * (c["k"] - 1), (key, rec)
            seen += 1
    assert seen == 1


@gpu
def test_launches_grow_with_frames_not_planes(w2x, models, worker_run):
    """collection A at scale2.0x: each GPU launches at most n + 1 kernels per frame of its planes (pack, n layers with the gather)"""
    job, _, log = worker_run
    (c, call, key), = [x for x in chain_calls(job) if x[1]["coll"] == "A"]
    sizes = COLLECTIONS["A"]
    nd, owner, _ = n_gpus(w2x, models, c["k"], call)
    bound = []
    for d in range(nd):
        mine = [sizes[i] for i in range(len(sizes)) if owner[i] == d]
        frame, _, _, dims = w2x.debug_plan_planes([2 * w for w, _ in mine], [2 * h for _, h in mine], 7, 128, 1 << 30)   # the worker's limit
        assert (frame >= 0).all()
        bound.append((7 + 1) * len(dims))
    launches = log[key]["passes"][1]["launches"]
    assert nd == 2 and all(0 < a <= b for a, b in zip(launches, bound)), (launches, bound)
    assert sum(launches) <= sum(bound) < len(sizes)


@gpu
def test_refusals_queue_and_log_nothing(worker_run):
    job, outs, log = worker_run
    g = len(groups())
    for j, bad in enumerate(REFUSALS):
        rec = log[f"g{g}.{j}"]
        status, msg = rec["multi"]
        assert status in (1, 7) and status == rec["one"][0], (bad, rec)
        assert msg == rec["one"][1].replace("w2x_convert_planes_chain", "w2x_multi_convert_planes_chain"), (bad, rec)
        assert rec["events"] == [] and rec["launches"][0] == rec["launches"][1] and rec["untouched"], (bad, rec)


@gpu
def test_out_of_memory_leaves_nothing_queued(worker_run):
    job, outs, log = worker_run
    rec = log[f"g{len(groups()) + 1}.0"]
    assert rec["error"][0] == 8, rec
    assert rec["launches"][0] == rec["launches"][1] and rec["untouched"], rec
    assert rec["after"] and np.array_equal(outs[f"g{len(groups()) + 1}.0.after.0"], outs[f"g{len(groups()) + 1}.0.ref.0"])
