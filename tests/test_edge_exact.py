"""Bit-exact tests of the kernels around the tensor-core layer, and of the fp32 engine, on ordinary inputs.

Every kernel here has a fully specified float32 order, so tests/exact_arith.py repeats it with correctly rounded float32
operations and the GPU result must match bit for bit: a different fma order, an encoding taken from the wrong operand or
a tap order change moves outputs by 1e-7 to 1e-5, inside every tolerance of tests/test_gpu_parity.py.

fp32 engine (conv3x3_planar_fp32<1/4/32>): the emulator without contraction equals the CPU oracle (the reference's
association built with -ffp-contract=off) bit for bit, so the FMA contraction in the 9-tap sum is the only difference
between the engine and the reference.

Tensor-core engine: a wgmma layer cannot be emulated on general activations (HGMMA's accumulation order and truncation are
not specified), except on a selection layer: output o has one nonzero weight, +-2^-j or +-2^-j (1 - 2^-12) at input
channel pi(o), tap tau(o).  With the packer's wscale 2^11, wh = 2^(11-j) and wl in {0, -+2^(-1-j)} are exact in fp16 and
their e4m3 copies, and the accumulator of output o receives at most three nonzero products:
  f16x3      xh wh, xl wh, xh wl                        -- every partial sum fits float32 (checked below);
  f16+f8x2   xh wh in the main accumulator, xl8 wh8 + xh8 wl8 in the correction buffer, which is added with an ordinary
             float32 add -- the buffer must hold the two products' sum exactly (checked below).
(2^-j (1 + 2^-11) would not do: xh (wh + wl) then carries into the next binade and needs 25 bits when xl ends on the
activation's last bit.)  The epilogue after the sums is specified, so the record encodings (fp16 hi, fp16 lo or e4m3 xh8 /
xl8), the first layer, planar_to_nhwc / nhwc_to_planar and both last-layer kernels are compared bit for bit on the real
output of a first layer with random weights.  selection_report() checks these conditions on the very activations a test
feeds in.

Hardware behaviour these tests rest on, measured with them on an H100 80GB HBM3 (700 W power limit): the tensor cores
multiply fp16 and e4m3 subnormal operands exactly (the small-activation channels of first_layer_params() and the
fp16-subnormal planes of tie_planes() give subnormal xl8 routinely), and a correction group of two e4m3 products spanning
up to 13 bits (the largest these inputs reach) comes out of the e4m3 accumulator unrounded.
"""
import itertools

import numpy as np
import pytest
import torch

import tc_numerics_model as T
from exact_arith import (F8_A, F8_C, F32, add32, e4m3, emulate_first_layer, emulate_last_fused, emulate_last_separate, f16,
                         fp32_convert, fp32_filter, mul32, readback, record_xh8, tc_activation)

PRECISIONS = ["f16x3", "f16+f8x2"]
SHAPES = [(32, 32), (32, 64), (32, 128), (64, 32), (64, 64), (64, 128), (128, 32), (128, 64), (128, 128)]
NUM_SMS = [0, 1, 3]                # 0 = every SM
SEL_WSCALE = 2.0 ** 11             # max |w| = 1/2: floor(log2(1024 / (1/2))) = 11
GROUP_SPAN_MAX = 24                # f16+f8x2: bits between the correction group's top bit and its lowest set bit


def _mismatch(got, want):
    bad = np.argwhere(got != want)
    i = tuple(bad[0])
    return f"{len(bad)} of {got.size} differ, first at {i}: {got[i]!r} != {want[i]!r}"


# ---------------------------------------------------------------------------------------------------------------------
# ordinary inputs
# ---------------------------------------------------------------------------------------------------------------------
def ordinary_planes(c, h, w, seed):
    """seeded values: normal * 1.5 (negatives, some >= 1), about 10 % exact zeros, a few tiny values"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((c, h, w)) * 1.5
    x[rng.random((c, h, w)) < 0.1] = 0.0
    tiny = rng.random((c, h, w)) < 0.05
    x[tiny] *= 2.0 ** -14
    return x.astype(F32)


def tie_planes(c, h, w, seed):
    """planes whose x16 values are fp16 rounding ties (odd multiples of half an fp16 ulp), their neighbours, values whose
    fp16 residual is an e4m3 subnormal after the 2^10 scale, and fp16 subnormals"""
    rng = np.random.default_rng(seed)
    e = rng.integers(-3, 4, (c, h, w)).astype(np.float64)
    m = rng.integers(1024, 2048, (c, h, w)).astype(np.float64)
    kind = rng.integers(0, 5, (c, h, w))
    x16 = (m + 0.5) * 2.0 ** (e - 10)                                 # ties
    x16 = np.where(kind == 1, (m + 0.5 + 2.0 ** -12) * 2.0 ** (e - 10), x16)          # just past a tie
    x16 = np.where(kind == 2, (m + 2.0 ** -9 * rng.integers(1, 8, (c, h, w))) * 2.0 ** (e - 10), x16)  # small residual
    x16 = np.where(kind == 3, rng.integers(1, 1024, (c, h, w)) * 2.0 ** -24 * 1.25, x16)  # fp16 subnormal range
    x16 = np.where(kind == 4, 0.0, x16)
    x16 *= rng.choice([-1.0, 1.0], (c, h, w))
    return (x16 / 16).astype(F32)


def first_layer_params(c, seed):
    """random first-layer weights and biases; per channel scale 1/3 (most), 2^-10 (small activations: subnormal xl8),
    2^-20 (fp16-subnormal activations) or 0 with bias 0 (exact zeros)"""
    rng = np.random.default_rng(seed)
    scale = rng.choice([1 / 3, 2.0 ** -10, 2.0 ** -20], size=c, p=[0.7, 0.2, 0.1])
    scale[c - 1] = 0.0
    w0 = (rng.standard_normal((c, 1, 3, 3)) * scale[:, None, None, None]).astype(F32)
    b0 = (rng.standard_normal(c) * 0.1 * scale * 3).astype(F32).astype(np.float64)
    return w0, b0


def selection_layer(cin, cout, case, seed):
    """w [Cout, Cin, 3, 3] with one nonzero weight per output: at channel pi(o) = (o + case Cout (+ case)) mod Cin,
    tap tau(o) = (o + case) mod 9, value +-2^-j or +-2^-j (1 - 2^-12), j in 1..5 (j = 1 at output 0: wscale 2^11)"""
    rng = np.random.default_rng(seed)
    o = np.arange(cout)
    pi = (o + case * cout + (case if cout >= cin else 0)) % cin
    tau = (o + case) % 9
    j = rng.integers(1, 6, cout)
    j[0] = 1
    val = rng.choice([-1.0, 1.0], cout) * 2.0 ** -j * np.where(rng.random(cout) < 0.5, 1 - 2.0 ** -12, 1.0)
    w = np.zeros((cout, cin, 3, 3), F32)
    w[o, pi, tau // 3, tau % 3] = val
    b = (rng.standard_normal(cout) * 0.1).astype(F32).astype(np.float64)
    return w, b


# ---------------------------------------------------------------------------------------------------------------------
# selection-layer emulator and its conditions
# ---------------------------------------------------------------------------------------------------------------------
def _selection(w):
    o, i, ky, kx = np.nonzero(w)
    assert np.array_equal(o, np.arange(w.shape[0])), "exactly one nonzero weight per output"
    return i, ky, kx


def selection_terms(x16r, w, f8):
    """The nonzero products output o's accumulators receive, as float64 [Cout, H, W] (exact), with the e4m3 copies'
    power-of-two scales taken out: (main, c1, c2) = (xh wh, xl wh, xh wl), in f16+f8x2 (xh wh, xl8 wh8, xh8 wl8).
    x16r: activations * 16 ([Cin, H + 2, W + 2], the ring the layer reads included)."""
    i, ky, kx = _selection(w)
    h, wd = x16r.shape[1] - 2, x16r.shape[2] - 2
    xin = np.stack([x16r[i[o], ky[o]:ky[o] + h, kx[o]:kx[o] + wd] for o in range(w.shape[0])]).astype(F32)
    ws = T.wscale_of(w)
    wsc = (w[np.arange(w.shape[0]), i, ky, kx] * F32(ws)).astype(F32)
    wh = f16(wsc)
    wl = wsc - wh
    xh = f16(xin).astype(np.float64)
    if f8:
        xl = e4m3((xin - f16(xin)).astype(np.float64) * 2.0 ** F8_A) * 2.0 ** -F8_A
        xh_c = record_xh8(xin)
        wh_c = e4m3(wh * 2.0 ** -F8_A) * 2.0 ** F8_A
        wl_c = e4m3(wl * 2.0 ** F8_C) * 2.0 ** -F8_C
    else:
        xl = f16(xin - f16(xin)).astype(np.float64)
        xh_c, wh_c, wl_c = xh, wh, f16(wl)
    col = lambda v: np.asarray(v, np.float64)[:, None, None]          # noqa: E731
    return (xh * col(wh), xl * col(wh_c), xh_c * col(wl_c)), ws, (wh, wl, wh_c, wl_c)


def selection_acc(terms, f8):
    """the float32 accumulator: f16x3 the exact sum; f16+f8x2 the main product plus the correction buffer (one add)"""
    main, c1, c2 = terms
    if f8:
        return add32(main.astype(F32), (c1 + c2).astype(F32))
    return (main + c1 + c2).astype(F32)


def emulate_selection(x16r, w, b, f8):
    """a selection layer on the tensor-core engine: activations * 16 out ([Cout, H, W])"""
    terms, ws, _ = selection_terms(x16r, w, f8)
    return tc_activation(selection_acc(terms, f8), ws, b)


def _units(arrs):
    """the arrays as int64 multiples of their common grain (exact), and the grain"""
    nz = np.concatenate([np.abs(a[a != 0]) for a in arrs] + [np.ones(1)])
    m, e = np.frexp(nz)
    mi = (m * 2.0 ** 53).astype(np.int64)
    _, low = np.frexp((mi & -mi).astype(np.float64))
    g = 2.0 ** int((e - 53 + low - 1).min())
    out = [np.rint(a / g).astype(np.int64) for a in arrs]
    assert max(int(np.abs(u).max()) for u in out) < 2 ** 60
    assert all(np.array_equal(u * g, a) for u, a in zip(out, arrs))
    return out, g


def _fits_f32(units):
    """every element's odd part has at most 24 bits: the value is a float32 (no exponent is near float32's limits here)"""
    u = np.abs(units[units != 0])
    return bool(np.all(u // (u & -u) < 2 ** 24))


def selection_report(x16r, w, b, f8):
    """Checks a selection layer's conditions on activations x16r and returns what it measured."""
    rep = {}
    terms, ws, (wh, wl, wh_c, wl_c) = selection_terms(x16r, w, f8)
    rep["wscale"] = ws
    rep["splits exact"] = bool(np.array_equal(f16(wl), wl) and np.all(wh != 0) and
                               np.array_equal(wh_c, wh) and np.array_equal(wl_c, wl))
    (main, c1, c2), _ = _units(list(terms))
    sums = ([main, c1, c2, main + c1, main + c2, c1 + c2, main + c1 + c2] if not f8 else [main, c1, c2, c1 + c2])
    rep["partial sums fit float32"] = all(_fits_f32(s) for s in sums)
    if f8:   # the correction group: bits from the top of the largest of |c1|, |c2|, |c1 + c2| down to the lowest set bit
        both = (c1 != 0) & (c2 != 0)
        lo = np.minimum(np.where(c1 != 0, c1 & -c1, 2 ** 62), np.where(c2 != 0, c2 & -c2, 2 ** 62))
        top = np.maximum(np.maximum(np.abs(c1), np.abs(c2)), np.abs(c1 + c2))
        span = np.where(both, np.frexp(top.astype(np.float64))[1] - np.frexp(lo.astype(np.float64))[1] + 1, 0)
        rep["group_span"] = int(span.max())
        rep["group_span_hist"] = {int(k): int(v) for k, v in zip(*np.unique(span[both], return_counts=True))}
    v = emulate_selection(x16r, w, b, f8)
    rep["v_max"] = float(np.abs(v).max())
    # what the activations exercise
    x = np.asarray(x16r, F32)
    d = x - f16(x)
    up, down = (np.asarray(x, np.float64) * (1 + s * 2.0 ** -20) for s in (1, -1))
    rep["fp16 ties"] = int(np.sum((d != 0) & (up.astype(np.float16) != down.astype(np.float16))))
    xl8 = e4m3(d.astype(np.float64) * 2.0 ** F8_A)
    rep["subnormal xl8"] = int(np.sum((xl8 != 0) & (np.abs(xl8) < 2.0 ** -6)))
    rep["zeros"] = int(np.sum(x == 0))
    rep["negative"] = int(np.sum(x < 0))
    return rep


def assert_selection(rep):
    assert rep["wscale"] == SEL_WSCALE, rep
    assert rep["splits exact"], rep
    assert rep["partial sums fit float32"], rep
    assert rep.get("group_span", 0) <= GROUP_SPAN_MAX, rep
    assert rep["v_max"] < 448, rep                                  # xh8 = e4m3(v / 2) and xl8 stay below saturation


def emulate_tc_model(plane, layers, f8, fused):
    """Context.convert_plane of 1 -> C1 -> selection layers -> 1 on the tensor-core engine; also returns the middle layers'
    inputs (with their zero ring) for selection_report"""
    n = len(layers)
    x16 = emulate_first_layer(np.pad(np.asarray(plane, F32), n, mode="edge"), *layers[0])
    inputs = []
    for w, b in layers[1:-1]:
        xr = np.pad(x16, ((0, 0), (1, 1), (1, 1)))                     # the TMA loads zero-fill outside the frame
        inputs.append((xr, w, b))
        x16 = emulate_selection(xr, w, b, f8)
    w2, b2 = layers[-1]
    out = emulate_last_fused(x16, w2, b2, n) if fused else emulate_last_separate(x16, w2, b2, n, f8)
    return out, inputs


def last_layer(c, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((1, c, 3, 3)) * 0.05).astype(F32), np.array([F32(rng.standard_normal() * 0.05)], np.float64)


def sel_model(widths, case, seed):
    """1 -> widths[0] -> ... -> widths[-1] -> 1: random first layer, selection layers, random last layer"""
    layers = [first_layer_params(widths[0], seed)]
    for k, (ci, co) in enumerate(zip(widths[:-1], widths[1:])):
        layers.append(selection_layer(ci, co, case, seed + 10 * k + 1))
    layers.append(last_layer(widths[-1], seed + 99))
    return layers


def _model(w2x, layers):
    return w2x.Model.from_arrays([t[0] for t in layers], [t[1] for t in layers])


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cin,cout", [(1, 4), (3, 5), (13, 17), (48, 33), (9, 1)])
def test_fp32_emulator_without_contraction_is_the_oracle(oracle_mod, cin, cout):
    """the emulator's association with a rounded multiply and add per tap = OracleModel.filter (the reference's order,
    -ffp-contract=off), bit for bit, on odd plane sizes"""
    om = oracle_mod.OracleModel.random([(cin, cout)], seed=cin * 100 + cout)
    for k, (h, w) in enumerate([(1, 1), (5, 3), (9, 31), (17, 40)]):
        x = ordinary_planes(cin, h, w, seed=k + cin)
        want = om.filter(0, x, n_job=2)
        got = fp32_filter(x, om.weights[0], om.biases[0], contract=False)
        assert np.array_equal(got, want), (h, w, _mismatch(got, want))
        fused = fp32_filter(x, om.weights[0], om.biases[0])
        assert np.abs(fused - want).max() <= 1e-5 * max(1.0, float(np.abs(want).max()))     # contraction: last bits only


def test_fp32_emulator_contraction_changes_bits():
    """the fma and the no-fma emulations differ on ordinary inputs, so comparing with the contracted one has teeth"""
    rng = np.random.default_rng(0)
    w = (rng.standard_normal((8, 8, 3, 3)) / 8).astype(F32)
    b = np.zeros(8)
    x = ordinary_planes(8, 20, 20, 1)
    assert not np.array_equal(fp32_filter(x, w, b), fp32_filter(x, w, b, contract=False))


def test_selection_layer_packs_as_designed(w2x):
    """the packer's wscale and fp16 hi / lo weights are the generator's for a selection layer (layer 1 of a model)"""
    layers = sel_model((64, 128), 0, 5)
    model = _model(w2x, layers)
    data, n_chunk, kblocks, ws = model.debug_tc_pack(1)
    assert ws == SEL_WSCALE
    w = layers[1][0]
    wsc = (w * F32(ws)).astype(F32)
    img = np.abs(data.view(np.float16).astype(np.float64))            # the hi and lo images of every (chunk, tap)
    wh, wl = f16(wsc), wsc - f16(wsc)
    assert np.array_equal(np.sort(img[img >= 1]), np.sort(np.abs(wh[wh != 0]).astype(np.float64)))
    assert np.array_equal(np.sort(img[(img > 0) & (img < 1)]), np.sort(np.abs(wl[wl != 0]).astype(np.float64)))
    assert set(np.abs(wh[wh != 0]).tolist()) <= {2.0 ** (11 - j) for j in range(1, 6)}
    assert set(np.abs(wl[wl != 0]).tolist()) <= {2.0 ** (-1 - j) for j in range(1, 6)} and np.count_nonzero(wl) > 0


def _filter_cases():
    for k, (cin, cout) in enumerate(SHAPES):
        w, b = selection_layer(cin, cout, k, 300 + k)
        for s, (wd, h) in enumerate([(1, 1), (7, 5), (17, 16), (33, 9)]):
            maker = tie_planes if s % 2 else ordinary_planes
            yield (cin, cout), w, b, maker(cin, h, wd, seed=1000 * k + s)


def _model_cases(c1, c2):
    for case, (wd, h) in enumerate(MODEL_SIZES):
        layers = sel_model((c1, c2), case, 10 * c1 + c2 + case)
        yield case, (wd, h), layers, plane_for(h, wd, case)


def plane_for(h, w, seed):
    """an input plane: uniform [0, 1) noise, or a smooth u8 / 255 image with flat runs"""
    rng = np.random.default_rng(seed)
    if seed % 2:
        return rng.random((h, w), dtype=F32)
    yy, xx = np.mgrid[0:h, 0:w]
    return (np.round(127 + 100 * np.sin(xx / 5.0 + seed) * np.cos(yy / 3.0)) / 255).astype(F32)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_selection_conditions_hold(prec):
    """selection_report on the inputs of every GPU case below"""
    f8 = prec != "f16x3"
    reps = []
    for _, w, b, x in _filter_cases():
        reps.append(selection_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w, b, f8))
    for c1, c2 in SHAPES:
        for _, _, layers, x in _model_cases(c1, c2):
            for xr, w, b in emulate_tc_model(x, layers, f8, True)[1]:
                reps.append(selection_report(xr, w, b, f8))
    for widths in CHAINS:
        for case, (wd, h) in enumerate(MODEL_SIZES[:3]):
            for xr, w, b in emulate_tc_model(plane_for(h, wd, case), sel_model(widths, case, sum(widths) + case), f8, True)[1]:
                reps.append(selection_report(xr, w, b, f8))
    layers, x = _geometry_model(), plane_for(70, 60, 3)
    for xr, w, b in emulate_tc_model(x, layers, f8, True)[1]:
        reps.append(selection_report(xr, w, b, f8))
    for rep in reps:
        assert_selection(rep)
    total = {k: sum(r[k] for r in reps) for k in ("fp16 ties", "subnormal xl8", "zeros", "negative")}
    print(prec, total, "max group span", max(r.get("group_span", 0) for r in reps))
    assert all(v > 0 for v in total.values()), total


def test_model_cases_select_every_channel_and_tap():
    for c1, c2 in SHAPES:
        chans, taps = set(), set()
        for _, _, layers, _ in _model_cases(c1, c2):
            i, ky, kx = _selection(layers[1][0])
            chans |= set(i.tolist())
            taps |= set((3 * ky + kx).tolist())
        assert chans == set(range(c1)) and taps == set(range(9)), (c1, c2)


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests: fp32 engine
# ---------------------------------------------------------------------------------------------------------------------
# CT = 1 (Cout = 1), 4 (2..16) and 32 (> 16); partial last groups (3, 5, 17, 31, 33, 48) and input chunks (1, 3, 7, 9, 17)
FP32_LAYERS = [(1, 3), (3, 5), (7, 17), (9, 31), (17, 33), (3, 48), (9, 1), (1, 16), (17, 2), (128, 128)]
FP32_SIZES = [(1, 1), (1, 8), (7, 1), (31, 7), (32, 8), (33, 9), (40, 17)]      # (w, h) around the 32 x 8 block


@pytest.fixture(scope="module")
def fp32_ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_FP32)
    yield c
    c.close()


@pytest.fixture(scope="module")
def tc_ctxs(w2x):
    c = {}
    for p, prec in zip(PRECISIONS, (w2x.PRECISION_F16X3, w2x.PRECISION_F16_F8X2)):
        c[p] = w2x.Context(0, engine=w2x.ENGINE_TC)
        c[p].set_precision(prec)
    yield c
    for v in c.values():
        v.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", FP32_LAYERS)
def test_fp32_filter_layer_is_bit_exact(w2x, fp32_ctx, cin, cout):
    rng = np.random.default_rng(cin * 1000 + cout)
    w = (rng.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(F32)
    b = (rng.standard_normal(cout) * 0.1).astype(F32).astype(np.float64)
    model = w2x.Model.from_arrays([w], [b])
    fails = []
    for k, (wd, h) in enumerate(FP32_SIZES if cin * cout < 10000 else FP32_SIZES[3:]):
        x = ordinary_planes(cin, h, wd, seed=k)
        want = fp32_filter(x, w, b)
        got = fp32_ctx.filter_layer(model, 0, x)
        if not np.array_equal(got, want):
            fails.append(f"{wd}x{h}: {_mismatch(got, want)}")
    assert not fails, "\n".join(fails)


FP32_MODELS = [(1, 3, 5, 1), (1, 17, 1), (1, 48, 33, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dims", FP32_MODELS, ids=lambda d: "-".join(map(str, d)))
def test_fp32_convert_plane_is_bit_exact(w2x, fp32_ctx, oracle_mod, dims):
    """copyMakeBorder + layers + crop (pad_replicate_kernel, conv3x3_planar_fp32, crop_kernel); a plane that block-splits
    (64 x 64 blocks) in the fused and the literal walk (copy2d_kernel); convert_tiles"""
    om = oracle_mod.OracleModel.random(list(zip(dims[:-1], dims[1:])), seed=sum(dims))
    model = w2x.Model.from_arrays(om.weights, om.biases)
    fails = []
    for k, (wd, h) in enumerate([(1, 1), (5, 3), (33, 9), (40, 17)]):
        x = plane_for(h, wd, k)
        want = fp32_convert(x, om.weights, om.biases)
        got = fp32_ctx.convert_plane(model, x)
        if not np.array_equal(got, want):
            fails.append(f"{wd}x{h}: {_mismatch(got, want)}")
    x = plane_for(90, 100, 1)
    want = fp32_convert(x, om.weights, om.biases)
    bw, bh = w2x.get_block_size()
    try:
        w2x.set_block_size(64, 64)
        assert w2x.requires_splitting(100, 90)
        for walk in (w2x.WALK_FUSED, w2x.WALK_BLOCKS):
            fp32_ctx.set_block_walk(walk)
            got = fp32_ctx.convert_plane(model, x)
            if not np.array_equal(got, want):
                fails.append(f"split walk={walk}: {_mismatch(got, want)}")
    finally:
        fp32_ctx.set_block_walk(w2x.WALK_FUSED)
        w2x.set_block_size(bw, bh)
    tiles = np.stack([plane_for(13, 20, 10 + t) for t in range(3)])
    got = fp32_ctx.convert_tiles(model, tiles)
    for t in range(3):
        want = fp32_convert(tiles[t], om.weights, om.biases)
        if not np.array_equal(got[t], want):
            fails.append(f"tile {t}: {_mismatch(got[t], want)}")
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests: tensor-core engine through selection layers
# ---------------------------------------------------------------------------------------------------------------------
# convert_plane frames of a 3-layer model (w + 6) x (h + 6): around the first layer's 32 x 8 block and the 16 x 16 tile-set
MODEL_SIZES = [(10, 3), (26, 10), (27, 11), (25, 27), (58, 34)]
# two selection layers: the middle one's epilogue writes records of 64, 32 and 128 channels, the last_layer_kernel reads
# 128, 64 and 32
CHAINS = [(32, 64, 128), (128, 32, 64), (64, 128, 32)]


def _f8_detail(x16r, w, f8, got, want, fmt):
    """where a correction group is involved, its span at the first mismatches (evidence for the hardware's e4m3 sums)"""
    if not f8:
        return ""
    (_, c1, c2), _, _ = selection_terms(x16r, w, True)
    bad = np.argwhere(fmt(got) != fmt(want))[:5]
    return " groups at first mismatches: " + "; ".join(f"{tuple(i)} c1={c1[tuple(i)]!r} c2={c2[tuple(i)]!r}" for i in bad)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_filter_layer_selection_is_bit_exact(w2x, tc_ctxs, prec):
    """planar_to_nhwc (x16, fp16 split, e4m3 copies, replicate ring) -> one selection layer (every shape) ->
    nhwc_to_planar, on ordinary planes and on planes of fp16 ties and small residuals, at every, one and three SMs"""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    fails = []
    try:
        for (cin, cout), w, b, x in _filter_cases():
            model = w2x.Model.from_arrays([w], [b])
            xr = mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
            want = readback(emulate_selection(xr, w, b, f8), f8)
            for sms in NUM_SMS:
                ctx.debug_set_num_sms(sms)
                got = ctx.filter_layer(model, 0, x)
                if not np.array_equal(got, want):
                    fails.append(f"{cin}->{cout} {x.shape} sms={sms}: {_mismatch(got, want)}" +
                                 _f8_detail(xr, w, f8, got, want, lambda a: a))
    finally:
        ctx.debug_set_num_sms(0)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("c1,c2", SHAPES)
@pytest.mark.parametrize("prec", PRECISIONS)
def test_first_layer_is_bit_exact(w2x, tc_ctxs, c1, c2, prec):
    """first_layer_kernel<C1, F8> with random weights and biases, its records read by a selection layer
    tc_conv3x3_kernel<C1, C2>, the last layer fused (last_gather) and separate (last_layer_kernel<C2>)"""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    fails = []
    try:
        for case, (wd, h), layers, x in _model_cases(c1, c2):
            model = _model(w2x, layers)
            for fused in (True, False):
                want = emulate_tc_model(x, layers, f8, fused)[0]
                ctx.debug_set_fuse_last(fused)
                for sms in NUM_SMS:
                    ctx.debug_set_num_sms(sms)
                    got = ctx.convert_plane(model, x)
                    if not np.array_equal(got, want):
                        fails.append(f"{wd}x{h} fused={fused} sms={sms}: {_mismatch(got, want)}")
    finally:
        ctx.debug_set_num_sms(0)
        ctx.debug_set_fuse_last(True)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("widths", CHAINS, ids=lambda c: "-".join(map(str, c)))
@pytest.mark.parametrize("prec", PRECISIONS)
def test_epilogue_records_are_bit_exact(w2x, tc_ctxs, widths, prec):
    """1 -> C1 -> C2 -> C3 -> 1 with two selection layers: the second reads the first's epilogue records (hi / lo or
    hi / xh8 / xl8); the last layer fused into the second (last_gather) or separate (last_layer_kernel<C3> reads the
    records back)"""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    fails = []
    try:
        for case, (wd, h) in enumerate(MODEL_SIZES[:3]):
            layers = sel_model(widths, case, sum(widths) + case)
            model = _model(w2x, layers)
            x = plane_for(h, wd, case)
            for fused in (True, False):
                want = emulate_tc_model(x, layers, f8, fused)[0]
                ctx.debug_set_fuse_last(fused)
                for sms in NUM_SMS:
                    ctx.debug_set_num_sms(sms)
                    got = ctx.convert_plane(model, x)
                    if not np.array_equal(got, want):
                        fails.append(f"{wd}x{h} fused={fused} sms={sms}: {_mismatch(got, want)}")
    finally:
        ctx.debug_set_num_sms(0)
        ctx.debug_set_fuse_last(True)
    assert not fails, "\n".join(fails)


def _geometry_model():
    return sel_model((32, 64, 32), 0, 4242)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_geometry_entry_points_are_bit_exact(w2x, tc_ctxs, prec):
    """convert_plane around the 32 x 8 block and the 16 x 16 tile-set, a block-splitting plane in both walks, scratch-limit
    bands down to 16 rows, host copy bands, convert_band_device halos, batched and grouped convert_tiles and Band
    sessions with 1 to 17 owned rows -- each against the emulator, 1 -> 32 -> 64 -> 32 -> 1 (n = 4)"""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    layers = _geometry_model()
    model = _model(w2x, layers)
    n = len(layers)
    em = lambda p: emulate_tc_model(p, layers, f8, True)[0]            # noqa: E731
    fails = []

    def check(name, got, want):
        if not np.array_equal(got, want):
            fails.append(f"{name}: {_mismatch(got, want)}")

    for k, (wd, h) in enumerate([(1, 1), (2, 3), (24, 1), (25, 9), (8, 8), (9, 10), (40, 17), (57, 24)]):
        x = plane_for(h, wd, k)
        check(f"convert_plane {wd}x{h}", ctx.convert_plane(model, x), em(x))
    W, H = 60, 70
    x = plane_for(H, W, 3)
    whole = em(x)
    bw, bh = w2x.get_block_size()
    try:
        w2x.set_block_size(32, 32)
        assert w2x.requires_splitting(W, H)
        for walk in (w2x.WALK_FUSED, w2x.WALK_BLOCKS):
            ctx.set_block_walk(walk)
            check(f"block split walk={walk}", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_block_walk(w2x.WALK_FUSED)
        w2x.set_block_size(bw, bh)
    try:
        for rows in (16, 17, 23):
            ctx.set_scratch_limit(64 * (W + 2 * n) * 4 * (rows + 2 * n))
            check(f"scratch bands of {rows} rows", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_scratch_limit(0)
    try:
        for nb in (2, 3, 8):
            ctx.debug_set_host_bands(nb)
            check(f"host bands {nb}", ctx.convert_plane(model, x), whole)
    finally:
        ctx.debug_set_host_bands(0)
    d_in = torch.from_numpy(x).cuda()
    y0, bh_ = 20, 25
    for above, below in itertools.product((0, n, n + 3), repeat=2):
        out = torch.empty((bh_, W), device="cuda")
        ctx.convert_band_device(model, d_in[y0 - above:].data_ptr(), W, bh_, above, below, W * 4, out.data_ptr(), W * 4)
        ctx.synchronize()
        want = em(x[y0 - above:y0 + bh_ + below])[above:above + bh_]
        check(f"band rows_above={above} rows_below={below}", out.cpu().numpy(), want)
    tiles = np.stack([plane_for(13, 20, 20 + t) for t in range(5)])
    want = np.stack([em(t) for t in tiles])
    check("convert_tiles batched", ctx.convert_tiles(model, tiles), want)
    try:
        ctx.set_scratch_limit(64 * (20 + 2 * n) * (13 + 2 * n) * 4 * 2)     # two tiles per pass
        check("convert_tiles grouped", ctx.convert_tiles(model, tiles), want)
    finally:
        ctx.set_scratch_limit(0)
    # Band sessions: owned rows 1, 2, 7, 8, 9, 16, 17
    cuts = np.concatenate([[0], np.cumsum([1, 2, 7, 8, 9, 16, 17])])
    Hb = int(cuts[-1])
    xb = plane_for(Hb, W, 5)
    d_in = torch.from_numpy(xb).cuda()
    bands, outs = [], []
    try:
        for b in range(len(cuts) - 1):
            r0, r1 = int(cuts[b]), int(cuts[b + 1])
            up, down = b > 0, b < len(cuts) - 2
            band = w2x.Band(ctx, model, W, r1 - r0, up, down)
            bands.append(band)
            band.load(d_in[r0 - (1 if up else 0):].data_ptr(), W * 4)
            outs.append(torch.empty((r1 - r0, W), device="cuda"))

        def dev(ptr, nb):
            return torch.as_tensor(w2x.DevBytes(ptr, nb), device="cuda")

        for k in range(bands[0].steps):
            for band in bands:
                band.step(k)
            halos = [band.halo(k) for band in bands]
            ctx.synchronize()
            for b in range(len(bands) - 1):
                for seg in range(len(halos[b])):
                    _, _, sd, rd, nb = halos[b][seg]
                    su, ru, _, _, _ = halos[b + 1][seg]
                    dev(ru, nb).copy_(dev(sd, nb))
                    dev(rd, nb).copy_(dev(su, nb))
            torch.cuda.synchronize()
        for band, o in zip(bands, outs):
            band.finish(o.data_ptr(), W * 4)
        ctx.synchronize()
        check("band sessions", torch.cat(outs).cpu().numpy(), em(xb))
    finally:
        for band in bands:
            band.close()
    assert not fails, "\n".join(fails)
