"""w2x_multi_convert_chain (csrc/engine_band.cu): noise and 2x scaling chains with the plane's row bands kept on their GPUs
between the steps, on ONE device, bit for bit against Context.convert_chain on one context in the same precision.

The "GPUs" are k contexts of device 0 (see tests/test_band_exchange.py); the cases run in tests/multi_chain_worker.py, a child
process with CUDA_DEVICE_MAX_CONNECTIONS set before CUDA initialises, and this module builds the inputs and references and
compares.  Every chain call runs three passes (flags, events and the cached plan are reused); every pass must give the
reference's bits.

  * k = 2, 3, 4; chains [noise], [scale^], [noise, scale^], [noise, scale^, scale^], [scale^, noise], the shipped n = 7 models,
    the random n = 4 model of test_band_exchange.py and a chain mixing both depths, and chains of the selection models of
    test_chain_exact.py (n = 3, 4, 6), whose reference is the chain emulator (which one-context convert_chain must match too);
    all three precisions; odd sizes; cuts on odd and even rows; step-0 frame widths with (w + 2n) % 4 in {1, 2, 3}; heights on both sides of the height / (4 n) rule; a plane
    whose later steps get several sub-bands per GPU; row-strided pinned and pageable host planes.
  * progress lines and on_step order; a one-step W2X_STEP_SAME chain against Multi.convert_plane; the plan cache; refusals;
    w2x_ctx_forget_model against the chain plan.
  * launch_pad alone against a numpy restatement of its frame.
  * the CLI with W2X_DEVICES=0,0 against its one-GPU run.
Without a GPU: the binding's signature, the numpy restatement's own sanity and the W2X_DEVICES parsing of host/w2xc.hpp.
"""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_band_exchange import ENV, RANDOM, Job, mismatch, slab_cuts
from test_chain_exact import LAYERS as SEL_LAYERS, emulate_chain, spec_of

gpu = pytest.mark.gpu
PKG = os.path.join(ROOT, "waifu2x-converter-cpp_b200")
CLI = os.path.join(PKG, "w2x-converter")
WORKER = os.path.join(ROOT, "tests", "multi_chain_worker.py")
PASSES = 3
F16X3, F16_F8X2, F16 = 0, 1, 2
N_OF = {"noise1": 7, "scale2.0x": 7, "rand128": 4, "selA": 3, "selB": 4, "selC": 6}
# the selection models of test_chain_exact.py (n = 3, 4, 6): their chains are compared with the chain emulator as well
SELS = {"selA": "A", "selB": "B", "selC": "C"}
PREC_NAMES = {F16X3: "f16x3", F16_F8X2: "f16+f8x2", F16: "f16"}

NOISE, SCALE, RAND = "noise1", "scale2.0x", "rand128"
S = lambda m, up=False, tta=False: [m, up, tta]   # noqa: E731  (a step)


def chain(steps, p, W, H, seed, **kw):
    return dict(op="chain", steps=steps, precision=p, input=f"x{W}x{H}_{seed}", size=(H, W), seed=seed, **kw)


def plane(model, p, W, H, seed, **kw):
    return dict(op="plane", model=model, precision=p, input=f"x{W}x{H}_{seed}", size=(H, W), seed=seed, **kw)


# (k, calls).  Frame widths at step 0 are w + 2n (a SAME step) or 2w + 2n (an upscaling one).
CASES = [
    (2, [
        # one W2X_STEP_SAME step is w2x_multi_convert_plane: calls 0 and 1 must agree in bits, lines and launches
        chain([S(NOISE)], F16_F8X2, 40, 56, 1), plane(NOISE, F16_F8X2, 40, 56, 1),
        chain([S(SCALE, True)], F16_F8X2, 33, 57, 2),                                           # cut at row 28; 16-byte frame rows (80)
        chain([S(NOISE), S(SCALE, True)], F16X3, 35, 61, 3, pinned=[False, False], in_pad=3, out_pad=5),   # 49 % 4 = 1, pageable
        chain([S(NOISE), S(SCALE, True)], F16, 37, 58, 4, in_pad=1, out_pad=2),                 # 51 % 4 = 3, cut at the odd row 29
        chain([S(SCALE, True), S(NOISE)], F16, 30, 59, 5),                                      # a SAME step after an upscale; 74 % 4 = 2
        # 260 rows per GPU: one sub-band at steps 0 and 1, two (1040 rows) at step 2 -- overlap rows read through the resize, both walks
        chain([S(NOISE), S(SCALE, True), S(SCALE, True)], F16_F8X2, 24, 520, 6, passes=2),
        # the cut uses the deeper model: 56 rows are cut (n = 7), 55 run on the first context
        chain([S(RAND), S(SCALE, True)], F16_F8X2, 37, 56, 7), chain([S(RAND), S(SCALE, True)], F16_F8X2, 37, 55, 8),
        chain([S(RAND, True), S(RAND)], F16X3, 21, 32, 9), chain([S(RAND, True), S(RAND)], F16X3, 21, 31, 10),
        # a plane the reference splits into blocks, with block splitting on and off
        chain([S(NOISE), S(SCALE, True)], F16_F8X2, 400, 1000, 11, passes=1), chain([S(NOISE), S(SCALE, True)], F16_F8X2, 400, 1000, 11, passes=1, block_splitting=False),
    ]),
    (3, [
        chain([S(NOISE), S(SCALE, True)], F16_F8X2, 40, 100, 12),                               # cuts at rows 33 and 66
        # the plan cache: the same call again, then another model, kind list, size and precision, then the first plan again
        chain([S(NOISE), S(SCALE, True)], F16_F8X2, 40, 100, 12, passes=1), chain([S(SCALE), S(SCALE, True)], F16_F8X2, 40, 100, 12, passes=1),
        chain([S(SCALE, True), S(SCALE, True)], F16_F8X2, 40, 100, 12, passes=1), chain([S(SCALE, True), S(SCALE, True)], F16_F8X2, 41, 101, 13, passes=1),
        chain([S(SCALE, True), S(SCALE, True)], F16X3, 41, 101, 13, passes=1), chain([S(NOISE), S(SCALE, True)], F16_F8X2, 40, 100, 12, passes=1),
        chain([S(RAND, True), S(RAND, True)], F16X3, 21, 50, 14),
    ]),
    (4, [
        chain([S(NOISE), S(SCALE, True), S(SCALE, True)], F16, 20, 113, 15),                    # cuts at rows 28, 56 and 84
        chain([S(RAND), S(RAND, True)], F16_F8X2, 19, 70, 16), chain([S(SCALE, True)], F16X3, 17, 111, 17),   # 111 rows: 3 of the 4 contexts
    ]),
    # selection chains whose steps differ in depth (3, 4, 6) and width, shallow -> deep and deep -> shallow; every height cuts
    # for every context (height / (4 n_max) >= k)
    (2, [
        chain([S("selA"), S("selC", True)], F16X3, 23, 50, 40), chain([S("selC", True), S("selA")], F16, 19, 49, 41),
    ]),
    (3, [
        chain([S("selC", True), S("selA")], F16_F8X2, 17, 75, 42), chain([S("selB", True), S("selA", True), S("selC")], F16X3, 9, 72, 43),
    ]),
]
# refusals (k = 2): status, the step named in the message, nothing logged, no on_step call
REFUSALS = [
    (chain([S(NOISE), S(SCALE, True, True)], F16_F8X2, 40, 56, 1), 1, "step 1", "multi-GPU"),
    (chain([S(NOISE, False, True)], F16_F8X2, 40, 56, 1), 1, "step 0", "multi-GPU"),
    (chain([S(NOISE), S(None, True)], F16_F8X2, 40, 56, 1), 1, "step 1", "NULL model"),
    (chain([], F16_F8X2, 40, 56, 1), 1, "n_steps", ""),
    (dict(op="raw", steps=[S(NOISE), S(SCALE, True)], input="x40x56_1", in_stride=40 * 4 + 2), 1, "step 0", "stride"),
    (dict(op="raw", steps=[S(NOISE), S(SCALE, True)], input="x40x56_1", out_stride=80 * 4 - 4), 1, "step 1", "stride"),
]
# w2x_ctx_forget_model against the chain plan (k = 2): (call, expected status or None)
FORGET = [
    (chain([S(NOISE), S(SCALE, True)], F16_F8X2, 40, 56, 1, passes=1), None),
    (dict(op="forget", model=NOISE), 1), (dict(op="forget", model=SCALE), 1), (dict(op="forget", model=RAND), 0),
    (chain([S(RAND, True)], F16_F8X2, 40, 56, 1, passes=1), None),           # a new plan: the old one's sessions are gone
    (dict(op="forget", model=NOISE), 0), (dict(op="forget", model=SCALE), 0), (dict(op="forget", model=RAND), 1),
    (dict(op="reopen"), None), (dict(op="forget", model=RAND), 0),
]


# ---------------------------------------------------------------------------------------------------------------------
# the numpy restatement of launch_pad's frame (FrameSource, csrc/kernels.h)
# ---------------------------------------------------------------------------------------------------------------------
def frame_of(src, row0, col0, w, h, pad_x, pad_top, rows_above, rows_below, up2x, cols_left, cols_right, pw, ph):
    """the pw x ph frame whose pixel (fy, fx) is the plane's pixel (clamp(fy - pad_top, -rows_above, h - 1 + rows_below),
    clamp(fx - pad_x, -cols_left, w - 1 + cols_right)); the plane's pixel (y, x) is src[row0 + y][col0 + x], or with up2x (the
    nearest 2x resize of src) src[row0 + (y >> 1)][col0 + (x >> 1)]"""
    sh = 1 if up2x else 0
    sy = row0 + (np.clip(np.arange(ph) - pad_top, -rows_above, h - 1 + rows_below) >> sh)
    sx = col0 + (np.clip(np.arange(pw) - pad_x, -cols_left, w - 1 + cols_right) >> sh)
    assert sy.min() >= 0 and sx.min() >= 0, "the real rows and columns must exist"
    return src[np.ix_(sy, sx)]


def selection_chain_cases():
    """(chain, input, precision) of every selection-model chain call above, for test_chain_exact.py's check of the emulator's
    conditions"""
    for _, calls in CASES:
        for c in calls:
            if c["op"] == "chain" and all(m in SELS for m, _, _ in c["steps"]):
                yield spec_of(c["steps"], SELS), np.random.default_rng(c["seed"]).random(c["size"], dtype=np.float32), PREC_NAMES[c["precision"]]


def test_frame_restatement_by_hand():
    src = np.arange(12, dtype=np.float32).reshape(4, 3)          # rows 0..3; the 2x plane has rows 0 0 1 1 2 2 3 3
    f = frame_of(src, 2, 0, 6, 4, 1, 3, 3, 0, True, 0, 0, 8, 8)  # band = 2x rows 4..7 (source rows 2, 3); 3 real rows above: 2x rows 1, 2, 3
    assert f.shape == (8, 8)
    assert [r[1] for r in f.tolist()] == [0, 3, 3, 6, 6, 9, 9, 9]             # source rows 0 1 1 | 2 2 3 3 | replicated 3
    assert f[3].tolist() == [6, 6, 6, 7, 7, 8, 8, 8]
    g = frame_of(src, 1, 0, 6, 4, 2, 2, 0, 0, True, 0, 0, 10, 8)  # image borders on both sides: replicate the band's own rows
    assert [r[2] for r in g.tolist()] == [3, 3, 3, 3, 6, 6, 6, 6] and g.shape == (8, 10)
    h = frame_of(src, 0, 0, 5, 2, 0, 0, 0, 1, True, 0, 0, 5, 3)  # an odd width cuts the 2x plane; one real row below
    assert h.tolist() == [[0, 0, 1, 1, 2], [0, 0, 1, 1, 2], [3, 3, 4, 4, 5]]
    # no resize: the plane is src[1:3, 1:2], one real row and column on each side, pads of 2 left and right, 1 above and below
    e = frame_of(src, 1, 1, 1, 2, 2, 1, 1, 1, False, 1, 1, 5, 4)
    assert e.tolist() == [[0, 0, 1, 2, 2], [3, 3, 4, 5, 5], [6, 6, 7, 8, 8], [9, 9, 10, 11, 11]]
    # a window of 2x columns [1, 3) with pad 2: it widens by one (the first copy of source column 0), its left pad and real columns
    # one smaller, so that no pad shows 2x column 0
    assert frame_of(src, 0, 0, 3, 1, 1, 0, 0, 0, True, -1, 0, 6, 1).tolist() == [[0, 0, 0, 1, 1, 1]]


def test_binding_declares_the_multi_chain_and_pad_entries(w2x):
    L = w2x.lib()
    assert len(L.w2x_multi_convert_chain.argtypes) == len(L.w2x_convert_chain.argtypes) == 13
    assert L.w2x_multi_convert_chain.argtypes[1:] == L.w2x_convert_chain.argtypes[1:]
    assert len(L.w2x_debug_pad.argtypes) == 20
    assert callable(w2x.Multi.convert_chain)


def test_device_list_parsing(w2x, tmp_path):
    """W2X_DEVICES of w2xc::gpuRuntime: the list's syntax, and that it overrides --gpus / W2X_GPUS in the planned GPU count"""
    exe = str(tmp_path / "test_device_list")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(PKG, "host"),
                           os.path.join(ROOT, "tests", "cpp", "test_device_list.cpp"), "-o", exe, "-L", PKG, "-lw2x_b200", f"-Wl,-rpath,{PKG}"])
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 0 and "ALL OK" in p.stdout, p.stdout + p.stderr


def pad_case(ctx, rng, w, h, pad_x, pad_top, ra, rb, up2x, cl, cr, pw, ph, y0, rows):
    """launch_pad against frame_of on a source whose every row and column outside the clamps' reach is NaN: "" when they agree"""
    sh = 1 if up2x else 0
    r_lo, r_hi, c_lo, c_hi = -ra >> sh, (h - 1 + rb) >> sh, -cl >> sh, (w - 1 + cr) >> sh     # what the clamps reach, in src units
    row0, col0 = 1 - r_lo, 2 - c_lo
    src = np.full((row0 + r_hi + 2, col0 + c_hi + 4), np.nan, np.float32)
    src[row0 + r_lo:row0 + r_hi + 1, col0 + c_lo:col0 + c_hi + 1] = rng.random((r_hi - r_lo + 1, c_hi - c_lo + 1), dtype=np.float32)
    want = frame_of(src, row0, col0, w, h, pad_x, pad_top, ra, rb, up2x, cl, cr, pw, ph)
    out = np.full(want.shape, -7.0, np.float32)
    ctx.debug_pad(src, row0, col0, w, h, pad_x, pad_top, ra, rb, up2x, cl, cr, out, y0, rows)
    want[:y0] = -7.0
    want[y0 + rows:] = -7.0
    return mismatch(out, want, [y0, y0 + rows])


@gpu
def test_pad_against_numpy(w2x):
    ctx = w2x.Context(0)
    rng = np.random.default_rng(5)
    fails, checked = [], 0
    try:
        # row bands of a 2x plane: (source width, w2): even and odd 2x widths; (5, 10) with pad_x = 7 gives a 24-float frame row (the
        # 16-byte stores); a neighbour's side has one halo row, which the band's store window leaves out
        for (ws, w2), n in itertools.product(((1, 2), (1, 1), (2, 4), (2, 3), (3, 6), (5, 10), (5, 9), (9, 18)), (4, 7)):
            for ra, rb, st, sb in itertools.product((0, 1, n), (0, 1, n), (0, 1), (0, 1)):
                pt, pb = (1 if st else n), (1 if sb else n)
                if ra > pt or rb > pb:
                    continue
                ph = 6 + pt + pb
                bad = pad_case(ctx, rng, w2, 6, n, pt, ra, rb, True, 0, 0, w2 + 2 * n, ph, st, ph - st - sb)
                checked += 1
                if bad:
                    fails.append(f"w2={w2} n={n} rows_above={ra} rows_below={rb} skip={st},{sb}: {bad}")
        # with and without the resize: (left pad, right pad, cols_left, cols_right) and (top pad, bottom pad, rows_above, rows_below),
        # among them real columns and rows beyond the plane, a right pad other than the left one, and the odd pads of windows
        # starting on an odd 2x column / row (the plane one wider, its pad and real columns / rows before it one smaller: -1 when
        # there are none); store windows that leave out rows at the top, the bottom, or both
        for up2x, n, w in itertools.product((False, True), (4, 7), (5, 8, 10)):
            for (pl, pr, cl, cr), (pt, pb, ra, rb) in itertools.product(
                    ((n, n, 0, 0), (n, n, 2, n), (n - 1, n, -1, 0), (n - 1, n, n - 1, 1), (1, n, 1, 0), (n, 2, 0, 3)),
                    ((n, n, 0, 0), (n - 1, n, -1, 0), (n - 1, n, n - 1, n), (1, n, 1, 0), (n, 1, 3, 1), (n, n, n, n))):
                h = 7
                pw, ph = w + pl + pr, h + pt + pb
                for y0, rows in ((0, ph), (1, ph - 2), (3, ph - 5), (ph - 4, 4), (0, 2)):
                    bad = pad_case(ctx, rng, w, h, pl, pt, ra, rb, up2x, cl, cr, pw, ph, y0, rows)
                    checked += 1
                    if bad:
                        fails.append(f"up2x={up2x} w={w} h={h} x={pl, pr, cl, cr} y={pt, pb, ra, rb} window={y0, rows}: {bad}")
        # a taller band than one block of row pairs, odd pad, real rows on both sides
        bad = pad_case(ctx, rng, 26, 60, 7, 7, 7, 7, True, 0, 0, 40, 74, 0, 74)
        assert not bad, bad
    finally:
        ctx.close()
    assert checked >= 1500 and not fails, "\n".join(fails[:20])


# ---------------------------------------------------------------------------------------------------------------------
# the worker run
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def layers(oracle_models, oracle_mod):
    out = {name: list(zip(oracle_models[name].weights, oracle_models[name].biases)) for name in (NOISE, SCALE)}
    dims, seed = RANDOM[RAND]
    om = oracle_mod.OracleModel.random(dims, seed=seed)
    out[RAND] = list(zip(om.weights, om.biases))
    out.update({k: SEL_LAYERS[v] for k, v in SELS.items()})
    return out


@pytest.fixture(scope="module")
def models(w2x, layers):
    return {k: w2x.Model.from_arrays([w for w, _ in v], [b for _, b in v]) for k, v in layers.items()}


@pytest.fixture(scope="module")
def worker_run(layers, tmp_path_factory):
    job = Job(layers)
    groups = [(k, calls) for k, calls in CASES] + [(2, [c for c, *_ in REFUSALS]), (2, [c for c, _ in FORGET])]
    for i, (k, calls) in enumerate(groups):
        calls = [dict(c) for c in calls]
        for c in calls:
            if "size" in c:
                job.inputs[c["input"]] = np.random.default_rng(c.pop("seed")).random(c.pop("size"), dtype=np.float32)
        job.add(dict(id=f"g{i}", k=k, calls=calls))
    d = tmp_path_factory.mktemp("multi_chain_worker")
    job.write(d)
    p = subprocess.run([sys.executable, WORKER, str(d)], env=dict(os.environ, **ENV), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    import json
    return job, dict(np.load(os.path.join(d, "out0.npz"))), json.load(open(os.path.join(d, "log0.json")))


class Reference:
    """Context.convert_chain on one context per precision, with its lines, on_step calls and launch count; for a chain of
    selection models the planes are the chain emulator's, which the one-context call must give as well"""

    def __init__(self, w2x, models):
        self.models = models
        self.ctx = {}
        for p in (F16X3, F16_F8X2, F16):
            self.ctx[p] = w2x.Context(0)
            self.ctx[p].set_precision(p)
        self.memo = {}

    def __call__(self, call, x):
        key = (repr(call["steps"]), call["precision"], call["input"], call.get("block_splitting", True))
        if key not in self.memo:
            ctx, events = self.ctx[call["precision"]], []
            steps = [(self.models[m], up, tta) for m, up, tta in call["steps"]]
            ctx.convert_chain(steps, x, block_splitting=call.get("block_splitting", True))         # the models are on the device now
            ctx.set_log(events.append)
            before = ctx.launch_count()
            try:
                y = ctx.convert_chain(steps, x, block_splitting=call.get("block_splitting", True), on_step=lambda k: events.append(f"step {k}"))
            finally:
                ctx.set_log(None)
            if all(m in SELS for m, _, _ in call["steps"]):
                want = emulate_chain(spec_of(call["steps"], SELS), x, PREC_NAMES[call["precision"]])
                msg = mismatch(y, want, [0])
                assert not msg, f"one-context convert_chain {call['steps']} against the emulator: {msg}"
                y = want
            self.memo[key] = (y, events, ctx.launch_count() - before)
        return self.memo[key]

    def close(self):
        for c in self.ctx.values():
            c.close()


@pytest.fixture(scope="module")
def ref(w2x, models):
    r = Reference(w2x, models)
    yield r
    r.close()


def gpus_of(k, call, H):
    return min(k, H // (4 * max(N_OF[m] for m, _, _ in call["steps"])))


def seams_of(k, call, H):
    """the output rows where a GPU's band or one of its sub-bands starts"""
    nd, u = gpus_of(k, call, H), sum(1 for s in call["steps"] if s[1])
    if nd < 2:
        return [0, H << u]
    r0 = [H * i // nd for i in range(nd + 1)]
    n = N_OF[call["steps"][-1][0]]
    return sorted({(r0[i] << u) + (v & ~1) for i in range(nd) for v in slab_cuts((r0[i + 1] - r0[i]) << u, n, 0)})


def chain_calls(job, n_groups=len(CASES)):
    for c in job.cases[:n_groups]:
        for j, call in enumerate(c["calls"]):
            if call["op"] == "chain":
                yield c, j, call, f"{c['id']}.{j}"


@gpu
def test_every_pass_is_bit_identical_to_one_context(worker_run, ref):
    job, outs, log = worker_run
    fails, checked = [], 0
    for c, j, call, key in chain_calls(job):
        x = job.inputs[call["input"]]
        want, _, _ = ref(call, x)
        W = want.shape[1]
        what = f"{key} k={c['k']} {call['steps']} precision {call['precision']} {x.shape}"
        assert isinstance(log[key], list), (what, log[key])
        for p in range(call.get("passes", PASSES)):
            got = outs[f"{key}.{p}"]
            msg = mismatch(got[:, :W], want, seams_of(c["k"], call, x.shape[0]))
            if msg:
                fails.append(f"{what} pass {p}: {msg}")
            if got.shape[1] > W and not np.all(np.isnan(got[:, W:])):
                fails.append(f"{what} pass {p}: wrote into the row padding beyond column {W}")
            checked += 1
    assert checked >= 40 and not fails, "\n".join(fails)


@gpu
def test_lines_and_on_step_order_are_convert_chains(worker_run, ref):
    job, _, log = worker_run
    for c, j, call, key in chain_calls(job):
        _, events, _ = ref(call, job.inputs[call["input"]])
        assert events[0] == "step 0" and len(events) > len(call["steps"])
        for p, rec in enumerate(log[key]):
            assert rec["events"] == events, (key, p, call)


@gpu
def test_launch_counts(worker_run, ref):
    """a cut plane launches on every GPU it uses and the same on every pass once the plan exists; a plane too small to cut launches
    what one context launches, on the first context only"""
    job, _, log = worker_run
    small = 0
    for c, j, call, key in chain_calls(job):
        H = job.inputs[call["input"]].shape[0]
        nd = gpus_of(c["k"], call, H)
        recs = log[key]
        if nd < 2:
            _, _, n_ref = ref(call, job.inputs[call["input"]])
            for rec in recs[1:]:                       # the first pass may upload a model
                assert rec["launches"] == [n_ref] + [0] * (c["k"] - 1), (key, rec)
            small += 1
            continue
        if len(call["steps"]) > 1 or call["steps"][0][1]:
            for rec in recs:
                assert all(v > 0 for v in rec["launches"][:nd]) and not any(rec["launches"][nd:]), (key, rec)
                assert len(set(rec["launches"][1:nd - 1])) <= 1, (key, rec)       # inner GPUs do the same work
        for rec in recs[2:]:
            assert rec["launches"] == recs[1]["launches"], (key, recs)
    assert small == 2


@gpu
def test_one_same_step_is_multi_convert_plane(worker_run):
    job, outs, log = worker_run
    a, b = log["g0.0"], log["g0.1"]
    for p in range(PASSES):
        assert np.array_equal(outs[f"g0.0.{p}"], outs[f"g0.1.{p}"])
        assert a[p]["events"] == ["step 0"] + b[p]["events"] and len(b[p]["events"]) == 7
    assert a[1]["launches"] == b[1]["launches"] == a[2]["launches"] and all(a[1]["launches"])


@gpu
def test_refusals_queue_and_log_nothing(worker_run):
    job, outs, log = worker_run
    g = len(CASES)
    for j, (call, status, names, word) in enumerate(REFUSALS):
        rec = log[f"g{g}.{j}"]
        assert isinstance(rec, dict) and rec["error"][0] == status, (call, rec)
        msg = rec["error"][1]
        assert "w2x_multi_convert_chain" in msg and names in msg and word in msg, (call, msg)
        assert rec["events"] == [], (call, rec)
        assert not any(k.startswith(f"g{g}.{j}.") for k in outs)


@gpu
def test_forget_model_and_the_chain_plan(worker_run):
    job, _, log = worker_run
    g = len(CASES) + 1
    for j, (call, status) in enumerate(FORGET):
        if call["op"] != "forget":
            continue
        got = log[f"g{g}.{j}"]
        assert got[0] == status, (j, call, got)
        assert ("band session" in got[1]) == (status == 1), (j, call, got)


# ---------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("args", [["-m", "noise_scale"], ["-m", "scale", "--scale_ratio", "4"]], ids=["noise_scale", "scale4"])
def test_cli_two_gpus_write_the_one_gpu_png(w2x, json_models, tmp_path, args):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    cv2.imwrite(str(tmp_path / "in.png"), _test_image(40, 60))           # 60 rows: cut for two GPUs
    runs = []
    for name, env in (("one", {}), ("two", dict(ENV, W2X_DEVICES="0,0"))):
        d = tmp_path / name
        d.mkdir()
        r = subprocess.run([CLI, "-i", str(tmp_path / "in.png"), "-o", str(d / "out.png"), "--model_dir", os.path.dirname(json_models["scale2.0x"]), *args],
                           capture_output=True, text=True, env=dict(os.environ, **env))
        assert r.returncode == 0, r.stdout + r.stderr
        runs.append((r.stdout, open(d / "out.png", "rb").read()))
    assert runs[0][0] == runs[1][0] and "2x scaling" in runs[0][0]
    assert runs[0][1] == runs[1][1]


@gpu
def test_cli_tta_with_a_device_list_writes_nothing(w2x, json_models, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    cv2.imwrite(str(tmp_path / "in.png"), _test_image(20, 16))
    r = subprocess.run([CLI, "-i", "in.png", "--tta", "1", "--model_dir", os.path.dirname(json_models["scale2.0x"])],
                       capture_output=True, text=True, cwd=tmp_path, env=dict(os.environ, **ENV, W2X_DEVICES="0,0"))
    assert r.returncode == 1 and "--tta" in r.stderr and r.stdout == ""
    assert os.listdir(tmp_path) == ["in.png"]
    r = subprocess.run([CLI, "-i", "in.png", "--gpus", "3", "--model_dir", os.path.dirname(json_models["scale2.0x"])],
                       capture_output=True, text=True, cwd=tmp_path, env=dict(os.environ, **ENV, W2X_DEVICES="0,0"))
    assert r.returncode != 0 and "W2X_DEVICES names 2 device(s) but 3" in r.stderr
    assert os.listdir(tmp_path) == ["in.png"]
