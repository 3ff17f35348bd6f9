"""Every step-table entry point bit for bit against the exact emulators, on chains whose steps differ in depth and width.

The chain, planes, region, regions and TTA calls share one machinery (the step table, the frame description FrameSource /
window_frame and the pack and gather kernels), and their other tests compare one call of it with another.  Here each call is
compared with the emulators of tests/exact_arith.py and test_edge_exact.py, which give the one correct bit pattern:

  * step k maps P to the emulated model applied to U_k(P), U_k the identity or the nearest 2x resize (np.repeat on both axes);
    the model is emulate_tc_model(fused=True) in f16x3 and f16+f8x2, the same with xh_only in f16, fp32_convert on the fp32
    engine;
  * a TTA step emulates the 8 variants V_j(U_k(P)) (the index map of include/w2x_b200.h, test_tta.variant), carries each output
    back, sums them j = 0..7 in float32 and multiplies by 0.125f;
  * a window is the crop of the emulated whole output.

The selection models have different depths n (3, 4, 6), widest activations (32, 128) and first-layer widths (32, 64, 128), and
the chains order them shallow -> deep and deep -> shallow, so that a value taken from the wrong step (the frame pad, the context
clamp of window_frame, the pad of the pack and gather kernels, chain_host's context rows, the scratch sizes) changes bits.  On
the fp32 engine narrow random models of depths 2, 3 and 5 play that part; 1-8-16-1 is no tensor-core model, so an automatic
context runs it on the fp32 engine inside a chain whose other steps run on tensor cores.

Without a GPU: the selection conditions (assert_selection) on every middle-layer input of every step of every GPU case below and
of the selection cases of test_multi_chain.py and test_multi_planes.py, the chains' mix of depths and widths, and the frame
plans the scratch-limit cases rely on.
"""
import numpy as np
import pytest

from exact_arith import F32, fp32_convert
from test_edge_exact import assert_selection, emulate_tc_model, plane_for, sel_model, selection_report
from test_region import crop, device_region, region_windows
from test_regions import device_regions, mixed_windows, sources
from test_tta import dense, device_chain, device_planes_chain, mean8, unvariant, up2, variant

gpu = pytest.mark.gpu
TC_CONFIGS = ["f16x3", "f16+f8x2", "f16"]
CONFIGS = TC_CONFIGS + ["fp32"]


# ---------------------------------------------------------------------------------------------------------------------
# models and chains
# ---------------------------------------------------------------------------------------------------------------------
def random_layers(widths, seed):
    """narrow random layers for the fp32 engine: w ~ N(0, 1 / (9 cin)), b ~ N(0, 0.01)"""
    rng = np.random.default_rng(seed)
    out = []
    for ci, co in zip(widths[:-1], widths[1:]):
        out.append(((rng.standard_normal((co, ci, 3, 3)) / np.sqrt(9 * ci)).astype(F32), rng.standard_normal(co) * 0.1))
    return out


# selection models: A n = 3, 32 channels at most; B n = 4, 128 at most; C n = 6, 128 at most, first_layer_kernel<128>
LAYERS = {
    "A": sel_model((32, 32), 0, 11),
    "B": sel_model((64, 128, 32), 1, 7),
    "C": sel_model((128, 64, 32, 64, 32), 2, 23),
    # fp32 engine: F1 n = 3 (no tensor-core model: 8 and 16 channels), F2 n = 5, F3 n = 2
    "F1": random_layers((1, 8, 16, 1), 31),
    "F2": random_layers((1, 6, 12, 8, 4, 1), 32),
    "F3": random_layers((1, 8, 1), 33),
}
SEL = {"A", "B", "C"}
S, U = False, True


def ch(*steps):
    """a chain: (model name, upscale[, tta]) per step"""
    return tuple((s[0], s[1], s[2] if len(s) > 2 else False) for s in steps)


SEL_CHAINS = [ch(("A", S), ("C", U)), ch(("C", U), ("A", S)), ch(("B", U), ("A", U), ("C", S))]
FP32_CHAINS = [ch(("F1", S), ("F2", U)), ch(("F2", U), ("F1", S)), ch(("F3", U), ("F1", U), ("F2", S))]
# an automatic context: the selection steps on tensor cores, F1 on the fp32 engine
MIXED_ENGINE_CHAINS = [ch(("C", S), ("F1", U)), ch(("F1", U), ("B", S))]
TTA_SEL = [ch(("C", S, True), ("A", U)), ch(("A", S), ("B", U), ("C", S, True))]
TTA_FP32 = [ch(("F2", S, True), ("F1", U)), ch(("F1", S), ("F3", U), ("F2", S, True))]


def chains_for(config):
    return FP32_CHAINS if config == "fp32" else SEL_CHAINS + MIXED_ENGINE_CHAINS


def window_chains_for(config):
    return FP32_CHAINS[:2] if config == "fp32" else SEL_CHAINS[:2] + MIXED_ENGINE_CHAINS[:1]


def ups_of(spec):
    return sum(1 for _, up, _ in spec if up)


def depths(spec):
    return [len(LAYERS[m]) for m, _, _ in spec]


def widest(name):
    return max(max(w.shape[0], w.shape[1]) for w, _ in LAYERS[name])


# ---------------------------------------------------------------------------------------------------------------------
# the chain emulator
# ---------------------------------------------------------------------------------------------------------------------
def spec_of(steps, names):
    """a chain of the multi-GPU workers ([model, upscale, tta] per step, its models named by `names`) in this module's terms"""
    return ch(*[(names[m], up, tta) for m, up, tta in steps])


def emulate_model(name, plane, config):
    """the plane through one model -> (output, the middle layers' inputs for selection_report)"""
    layers = LAYERS[name]
    if config == "fp32" or name not in SEL:
        return fp32_convert(plane, [w for w, _ in layers], [b for _, b in layers]), []
    return emulate_tc_model(plane, layers, config == "f16+f8x2", True, config == "f16")


def emulate_step(name, plane, config, up, tta):
    src = up2(plane) if up else plane
    if not tta:
        return emulate_model(name, src, config)
    outs, inputs = [], []
    for j in range(8):
        o, i = emulate_model(name, dense(variant(src, j)), config)
        outs.append(unvariant(o, j))
        inputs += i
    return mean8(outs), inputs


def emulate_chain(spec, plane, config, check=False):
    """the chain's output; check: assert the selection conditions on every middle-layer input of every step (and variant)"""
    y = np.asarray(plane, F32)
    for name, up, tta in spec:
        y, inputs = emulate_step(name, y, config, up, tta)
        if check:
            for xr, w, b in inputs:
                assert_selection(selection_report(xr, w, b, config == "f16+f8x2"))
    return y


class Emulated:
    """emulate_chain, memoised per (chain, plane, config)"""

    def __init__(self):
        self.memo = {}

    def __call__(self, spec, x, config):
        key = (spec, x.shape, x.tobytes(), config)
        if key not in self.memo:
            self.memo[key] = emulate_chain(spec, x, config)
        return self.memo[key]


# ---------------------------------------------------------------------------------------------------------------------
# the GPU cases (shared with the CPU test of their selection conditions)
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [(1, 1), (2, 3), (7, 5), (45, 37)]                   # (w, h)
SIZES_UU = [(1, 1), (2, 3), (7, 5), (23, 19)]                # chains with two 2x steps
TALL = (5, 512)                                              # 2x: 1024 rows, two copy bands of chain_host
PLANE_SIZES = [(1, 1), (1, 23), (23, 1), (9, 7), (30, 21), (2, 3)]
PLANE_SIZES_UU = [(1, 1), (1, 9), (9, 1), (7, 5)]
PACK_SIZES = [(60, 50), (1, 17), (17, 1), (9, 7), (12, 10), (2, 3), (20, 14)]
PACK_LIMITS = [1 << 19, 1 << 20]
TILES = (5, 20, 13)                                          # n, w, h
WINDOW_PLANES = [(45, 37), (30, 21)]
TTA_SIZES = [(13, 9), (1, 7), (6, 1)]
TTA_PLANES = [(13, 9), (1, 7), (6, 1), (5, 8)]


def chain_cases(config):
    for c, spec in enumerate(chains_for(config)):
        for k, (w, h) in enumerate(SIZES if ups_of(spec) < 2 else SIZES_UU):
            yield spec, plane_for(h, w, 10 * c + k)


def tall_case(config):
    return chains_for(config)[0], plane_for(TALL[1], TALL[0], 3)


def band_case(config):
    return chains_for(config)[0], plane_for(37, 45, 5)


def planes_cases(config):
    for c, spec in enumerate(chains_for(config)):
        sizes = PLANE_SIZES if ups_of(spec) < 2 else PLANE_SIZES_UU
        yield spec, [plane_for(h, w, 100 + 10 * c + i) for i, (w, h) in enumerate(sizes)]


def pack_case(config):
    return chains_for(config)[0], [plane_for(h, w, 200 + i) for i, (w, h) in enumerate(PACK_SIZES)]


def single_model_cases(config):
    """convert_planes of one model, convert_tiles of another"""
    a, b = ("F2", "F1") if config == "fp32" else ("B", "C")
    n, w, h = TILES
    return (a, [plane_for(h_, w_, 300 + i) for i, (w_, h_) in enumerate(PLANE_SIZES)],
            b, np.stack([plane_for(h, w, 310 + t) for t in range(n)]))


def window_cases(config):
    for c, spec in enumerate(window_chains_for(config)):
        yield spec, [plane_for(h, w, 400 + 10 * c + i) for i, (w, h) in enumerate(WINDOW_PLANES)]


def tta_cases(config):
    for c, spec in enumerate(TTA_FP32 if config == "fp32" else TTA_SEL):
        yield spec, [plane_for(h, w, 500 + 10 * c + i) for i, (w, h) in enumerate(TTA_PLANES)]


def selection_cases(config):
    """every (chain, plane) the GPU tests of this module emulate in config"""
    out = list(chain_cases(config)) + [tall_case(config), band_case(config)]
    for spec, planes in list(planes_cases(config)) + [pack_case(config)] + list(window_cases(config)) + list(tta_cases(config)):
        out += [(spec, x) for x in planes]
    a, planes, b, tiles = single_model_cases(config)
    out += [(ch((a, S)), x) for x in planes] + [(ch((b, S)), t) for t in tiles]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("config", TC_CONFIGS)
def test_selection_conditions_hold_on_every_gpu_case(config):
    """assert_selection on every middle-layer input, of every step and TTA variant, of every selection case here and in
    test_multi_chain.py / test_multi_planes.py: step k + 1 reads step k's float32 output, so the conditions are checked there too"""
    from test_multi_chain import selection_chain_cases
    from test_multi_planes import selection_planes_cases
    cases = [c for c in selection_cases(config) if any(m in SEL for m, _, _ in c[0])]
    cases += [c for c in selection_chain_cases() if c[2] == config] + [c for c in selection_planes_cases() if c[2] == config]
    for spec, x, *_ in cases:
        emulate_chain(spec, x, config, check=True)
    assert len(cases) > 40


def test_chains_mix_depths_and_widths():
    """every chain has steps of different depth, both orders occur, and the widest activation and first-layer width vary"""
    assert [len(LAYERS[m]) for m in ("A", "B", "C", "F1", "F2", "F3")] == [3, 4, 6, 3, 5, 2]
    assert [widest(m) for m in ("A", "B", "C")] == [32, 128, 128]
    assert [LAYERS[m][0][0].shape[0] for m in ("A", "B", "C")] == [32, 64, 128]
    for chains in (SEL_CHAINS, FP32_CHAINS, MIXED_ENGINE_CHAINS, TTA_SEL, TTA_FP32):
        for spec in chains:
            assert len(set(depths(spec))) > 1, spec
        assert any(depths(s)[0] < depths(s)[-1] for s in chains) and any(depths(s)[0] > depths(s)[-1] for s in chains)
    assert any(spec[0][2] for spec in TTA_SEL) and any(spec[-1][2] and ups_of(spec) for spec in TTA_SEL)


def test_mixed_engine_chains_need_both_engines():
    """F1's inner widths 8 and 16 make it no tensor-core model (1 -> {32, 64, 128} ... -> 1), so an automatic context runs it on
    the fp32 engine, and every one of these chains has a step on each engine"""
    assert [w.shape[0] for w, _ in LAYERS["F1"][:-1]] == [8, 16]
    for spec in MIXED_ENGINE_CHAINS:
        assert {m in SEL for m, _, _ in spec} == {True, False}


@pytest.mark.parametrize("limit", PACK_LIMITS)
def test_pack_plans_change_between_steps(w2x, limit):
    """the scratch-limited planes chain: some step packs two frames or more, some step converts a plane alone, and the two steps'
    plans differ (each planned with its own n and widest activation)"""
    plans = pack_plans(w2x, chains_for("f16x3")[0], PACK_SIZES, limit)
    assert any(len(dims) >= 2 for _, dims in plans), plans
    assert any((frame == -1).any() for frame, _ in plans), plans
    assert plans[0][0].tolist() != plans[1][0].tolist()


def test_window_plan_has_frames_and_a_window_alone(w2x):
    spec, x = band_case("f16x3")
    _, limit, outs = window_pack(spec, x)
    frame, _, _, _ = w2x.debug_plan_planes([w[2] for w in outs], [w[3] for w in outs], depths(spec)[-1], widest(spec[-1][0]), limit)
    assert frame.max() >= 1 and (frame == -1).any(), frame


def pack_plans(w2x, spec, sizes, limit):
    """each step's frame plan (frame per plane, frame sizes) for planes of sizes"""
    plans, ws, hs = [], [w for w, _ in sizes], [h for _, h in sizes]
    for name, up, _ in spec:
        if up:
            ws, hs = [2 * v for v in ws], [2 * v for v in hs]
        frame, _, _, dims = w2x.debug_plan_planes(ws, hs, len(LAYERS[name]), widest(name), limit)
        plans.append((frame, dims))
    return plans


def window_pack(spec, x):
    """windows of one plane, a scratch limit giving the last step two frames and a window converted alone, the output windows"""
    wins = [(0, (3, 5, 80, 60)), (0, (1, 1, 20, 20)), (0, (40, 30, 20, 19)), (0, (61, 2, 21, 20)), (0, (69, 53, 21, 21)),
            (0, (9, 55, 18, 17))]
    limit = 128 * 4 * 3000
    H, W = x.shape
    outs = [region_windows(depths(spec), [up for _, up, _ in spec], W, H, w)[-1] for _, w in wins]
    return wins, limit, outs


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models(w2x):
    return {k: w2x.Model.from_arrays([w for w, _ in v], [b for _, b in v]) for k, v in LAYERS.items()}


@pytest.fixture(scope="module")
def ctxs(w2x):
    out = {}
    for config in CONFIGS:
        if config == "fp32":
            out[config] = w2x.Context(0, engine=w2x.ENGINE_FP32)
        else:
            out[config] = w2x.Context(0)           # automatic: F1 runs on the fp32 engine
            out[config].set_precision(TC_CONFIGS.index(config))
    yield out
    for c in out.values():
        c.close()


@pytest.fixture(scope="module")
def em():
    return Emulated()


def steps_of(models, spec):
    return [(models[m], up, tta) for m, up, tta in spec]


def mismatch(got, want):
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    bad = np.argwhere(got != want)
    if not len(bad):
        return ""
    i = tuple(bad[0])
    return f"{len(bad)} of {got.size} differ, first at {i}: {got[i]!r} != {want[i]!r}"


class Fails(list):
    def check(self, what, got, want):
        msg = mismatch(np.asarray(got), want)
        if msg:
            self.append(f"{what}: {msg}")

    def done(self):
        assert not self, "\n".join(self[:30])


def name_of(spec):
    return "".join(f"[{m},{'U' if up else 'S'}{',T' if t else ''}]" for m, up, t in spec)


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_convert_chain(w2x, models, ctxs, em, config):
    """convert_chain and convert_chain_device on 1 x 1, 2 x 3, odd and ~45 x 37 planes"""
    ctx, fails = ctxs[config], Fails()
    for spec, x in chain_cases(config):
        steps, want = steps_of(models, spec), em(spec, x, config)
        fails.check(f"host {name_of(spec)} {x.shape}", ctx.convert_chain(steps, x), want)
        fails.check(f"device {name_of(spec)} {x.shape}", device_chain(ctx, steps, x, pad_in=3, pad_out=5), want)
    fails.done()


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_convert_chain_bands_and_blocks(w2x, models, ctxs, em, config):
    """a 2x plane of 1024 rows (chain_host's copy bands, their context rows the last step's n), scratch bands of 16 and 23 rows
    on an upscaling last step, and the literal block walk with 32 x 32 blocks on both steps"""
    ctx, fails = ctxs[config], Fails()
    spec, x = tall_case(config)
    steps = steps_of(models, spec)
    want = em(spec, x, config)
    assert want.shape[0] >= 1024
    fails.check("tall host", ctx.convert_chain(steps, x), want)
    fails.check("tall device", device_chain(ctx, steps, x), want)
    spec, x = band_case(config)
    steps, want = steps_of(models, spec), em(spec, x, config)
    n, w2 = depths(spec)[-1], 2 * x.shape[1]
    try:
        for rows in (16, 23):
            ctx.set_scratch_limit(widest(spec[-1][0]) * (w2 + 2 * n) * 4 * (rows + 2 * n))
            fails.check(f"scratch bands of {rows} rows host", ctx.convert_chain(steps, x), want)
            fails.check(f"scratch bands of {rows} rows device", device_chain(ctx, steps, x), want)
    finally:
        ctx.set_scratch_limit(0)
    bw, bh = w2x.get_block_size()
    try:
        w2x.set_block_size(32, 32)
        assert w2x.requires_splitting(x.shape[1], x.shape[0]) and w2x.requires_splitting(w2, 2 * x.shape[0])
        ctx.set_block_walk(w2x.WALK_BLOCKS)
        for spec_ in chains_for(config)[:2]:
            fails.check(f"literal walk {name_of(spec_)}", ctx.convert_chain(steps_of(models, spec_), x), em(spec_, x, config))
    finally:
        ctx.set_block_walk(w2x.WALK_FUSED)
        w2x.set_block_size(bw, bh)
    fails.done()


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_convert_planes_and_tiles(w2x, models, ctxs, em, config):
    """convert_planes (1 x N and N x 1 among them) and convert_tiles, batched and two tiles a pass"""
    ctx, fails = ctxs[config], Fails()
    a, planes, b, tiles = single_model_cases(config)
    want = [em(ch((a, S)), x, config) for x in planes]
    for i, (g, e) in enumerate(zip(ctx.convert_planes(models[a], planes), want)):
        fails.check(f"convert_planes {a} plane {i} {planes[i].shape}", g, e)
    want = np.stack([em(ch((b, S)), t, config) for t in tiles])
    fails.check(f"convert_tiles {b}", ctx.convert_tiles(models[b], tiles), want)
    n = len(LAYERS[b])
    try:
        ctx.set_scratch_limit(widest(b) * (tiles.shape[2] + 2 * n) * (tiles.shape[1] + 2 * n) * 4 * 2)
        fails.check(f"convert_tiles {b} grouped", ctx.convert_tiles(models[b], tiles), want)
    finally:
        ctx.set_scratch_limit(0)
    fails.done()


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_convert_planes_chain(w2x, models, ctxs, em, config):
    """convert_planes_chain and convert_planes_chain_device on collections with 1 x N and N x 1 planes"""
    ctx, fails = ctxs[config], Fails()
    for spec, planes in planes_cases(config):
        steps = steps_of(models, spec)
        want = [em(spec, x, config) for x in planes]
        for entry, got in (("host", ctx.convert_planes_chain(steps, planes)), ("device", device_planes_chain(ctx, steps, planes))):
            for i, (g, e) in enumerate(zip(got, want)):
                fails.check(f"{entry} {name_of(spec)} plane {i} {planes[i].shape}", g, e)
    fails.done()


@gpu
@pytest.mark.parametrize("config", TC_CONFIGS)
def test_planes_chain_frames_and_planes_alone(w2x, models, ctxs, em, config):
    """scratch limits under which one step packs two frames or more and another converts a plane alone (the plans are asserted
    by test_pack_plans_change_between_steps)"""
    ctx, fails = ctxs[config], Fails()
    spec, planes = pack_case(config)
    steps = steps_of(models, spec)
    want = [em(spec, x, config) for x in planes]
    try:
        for limit in PACK_LIMITS:
            ctx.set_scratch_limit(limit)
            for entry, got in (("host", ctx.convert_planes_chain(steps, planes)), ("device", device_planes_chain(ctx, steps, planes))):
                for i, (g, e) in enumerate(zip(got, want)):
                    fails.check(f"limit {limit} {entry} plane {i} {planes[i].shape}", g, e)
    finally:
        ctx.set_scratch_limit(0)
    fails.done()


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_chain_region_and_regions(w2x, models, ctxs, em, config):
    """convert_chain_region(_device) on every window of mixed_windows (every border, 1 x 1, odd 2x rows and columns) and
    convert_chain_regions(_device) on the windows of two planes in one call"""
    import torch
    ctx, fails = ctxs[config], Fails()
    for spec, planes in window_cases(config):
        steps = steps_of(models, spec)
        wholes = [em(spec, x, config) for x in planes]
        wins = mixed_windows(planes, ups_of(spec))
        srcs, sizes = sources(w2x, steps, planes, wins)
        want = [crop(wholes[p], win) for p, win in wins]
        d_planes = [torch.from_numpy(x).cuda() for x in planes]
        for (p, win), s, size, e in zip(wins, srcs, sizes, want):
            fails.check(f"region {name_of(spec)} plane {p} window {win}", ctx.convert_chain_region(steps, s, size, win), e)
            fails.check(f"region device {name_of(spec)} plane {p} window {win}", device_region(w2x, ctx, steps, d_planes[p], size, win), e)
        got = ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins])
        for (p, win), g, e in zip(wins, got, want):
            fails.check(f"regions {name_of(spec)} plane {p} window {win}", g, e)
        got = device_regions(w2x, ctx, steps, d_planes, wins)
        for (p, win), g, e in zip(wins, got, want):
            fails.check(f"regions device {name_of(spec)} plane {p} window {win}", g, e)
    fails.done()


@gpu
@pytest.mark.parametrize("config", TC_CONFIGS)
def test_regions_frames_and_a_window_alone(w2x, models, ctxs, em, config):
    """a scratch limit under which the last step packs two frames and converts a window alone (test_window_plan_has_frames_and_a_window_alone)"""
    import torch
    ctx, fails = ctxs[config], Fails()
    spec, x = band_case(config)
    steps = steps_of(models, spec)
    wins, limit, _ = window_pack(spec, x)
    whole = em(spec, x, config)
    want = [crop(whole, w) for _, w in wins]
    srcs, sizes = sources(w2x, steps, [x], wins)
    try:
        ctx.set_scratch_limit(limit)
        for (_, win), g, e in zip(wins, ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins]), want):
            fails.check(f"host window {win}", g, e)
        for (_, win), g, e in zip(wins, device_regions(w2x, ctx, steps, [torch.from_numpy(x).cuda()], wins), want):
            fails.check(f"device window {win}", g, e)
    finally:
        ctx.set_scratch_limit(0)
    fails.done()


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_tta_steps_in_mixed_chains(w2x, models, ctxs, em, config):
    """TTA on the first step, and on a deep step after an upscale: convert_chain(_device) and convert_planes_chain(_device) on
    non-square planes"""
    ctx, fails = ctxs[config], Fails()
    for spec, planes in tta_cases(config):
        steps = steps_of(models, spec)
        want = [em(spec, x, config) for x in planes]
        for x, e in zip(planes, want):
            if (x.shape[1], x.shape[0]) in TTA_SIZES:
                fails.check(f"chain {name_of(spec)} {x.shape}", ctx.convert_chain(steps, x), e)
                fails.check(f"chain device {name_of(spec)} {x.shape}", device_chain(ctx, steps, x), e)
        for entry, got in (("host", ctx.convert_planes_chain(steps, planes)), ("device", device_planes_chain(ctx, steps, planes))):
            for i, (g, e) in enumerate(zip(got, want)):
                fails.check(f"planes {entry} {name_of(spec)} plane {i} {planes[i].shape}", g, e)
    fails.done()
