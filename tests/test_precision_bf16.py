"""W2X_PRECISION_BF16X3: the tensor-core engine's three split products on bf16 operands, x*w = xh*wh + xl*wh + xh*wl with
h = the bf16 rounding, in fp32 accumulators.

bf16 has fp32's exponent range.  The records hold hi = bf16(16 a), lo = bf16(16 a - hi) and the weights pack at wscale 1 as
wh = bf16(w), wl = bf16(w - wh), so nothing saturates or underflows until fp32 itself does: the relative error is the same at
every activation and model scale, and a power-of-two rescaling of a model (tests/test_model_scale.py) moves every operand,
product and partial sum by the same power of two.  Its outputs are then bit-identical to the shipped model's.

CPU: the packed weight image, an emulation of the precision on the shipped models across six decades of input scale, the
constants.  GPU: the layer kernels (conv3x3_bf16x3_kernel) bit for bit on a bf16 lattice, the edge kernels against emulators,
the golden outputs, the activation range, the rescalings, every entry point against convert_plane, the CLI.
"""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_activation_range as AR
import test_model_scale as MS
from conftest import golden_path
from exact_arith import F32, add32, emulate_first_layer, emulate_last_fused, fma32, leaky_last, mul32, tc_activation
from test_tc_exact import LAYER_SIZES, MODEL_SIZES, NUM_SMS, SHAPES, _mismatch, _tilesets, accumulate, accumulate_units, binary_plane

MODELS = ["scale2.0x", "noise1", "noise2"]
BF16_MAX = float.fromhex("0x1.fep127")
# The relative error (max-abs / max(1, max |reference|)) include/w2x_b200.h states for bf16x3: the CPU emulation of the
# shipped models reaches 9.4e-6 over input scales x1 to x1e6, the H100 1.45e-5 (test_activation_range, noise2 at x1000); the
# bound keeps a margin of two over the GPU and three over the emulation.
BF16X3_BOUND = 3e-5
SCALES = [1, 100, 1e4, 1e6]
GPU_SCALES = AR.SCALES + [1e6]
Q = 2.0 ** -11                     # the lattice's product quantum


# ---------------------------------------------------------------------------------------------------------------------
# bf16 arithmetic and emulators
# ---------------------------------------------------------------------------------------------------------------------
def bf16(x):
    """round to bf16 (nearest, ties to even), saturating at +-0x1.fep127 as cvt.rn.satfinite.bf16x2.f32 does (NaN stays
    NaN), as float32"""
    x = np.clip(np.asarray(x, F32), -BF16_MAX, BF16_MAX)
    return torch.from_numpy(np.ascontiguousarray(x)).to(torch.bfloat16).to(torch.float32).numpy()


def bf16_bits(x):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, F32))).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16)


def bf16_operands(x16, w):
    """[(xh, wh), (xl, wh), (xh, wl)] as float64: the record split of x16 (activations * 16) and the weight image's (wscale 1)"""
    wf = np.asarray(w, F32)
    wh = bf16(wf)
    wl = bf16(wf - wh)                                               # the difference is exact
    xh = bf16(x16)
    xl = bf16(np.asarray(x16, F32) - xh)
    return [(np.asarray(a, np.float64), np.asarray(b, np.float64)) for a, b in ((xh, wh), (xl, wh), (xh, wl))]


def bf16_readback(v):
    """nhwc_bf16_to_planar: (hi + lo) / 16"""
    hi = bf16(v)
    return mul32(add32(hi, bf16(np.asarray(v, F32) - hi)), F32(1.0 / 16))


def emulate_bf16_filter_layer(planes, w, b, exact=True):
    """Context.filter_layer: planar_to_nhwc_bf16 (replicate ring, x16, split) -> the layer -> nhwc_bf16_to_planar"""
    x16 = mul32(np.pad(planes, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
    return bf16_readback(tc_activation(accumulate(bf16_operands(x16, w), exact), 1.0, b))


def emulate_bf16_last_separate(a1, w2, b2, n):
    """last_layer_kernel on bf16 records: (hi + lo) / 16, then per group of 8 channels eight partial sums over the taps"""
    c2, ph, pw = a1.shape
    w2 = np.asarray(w2, F32)
    hi = bf16(a1)
    a = mul32(add32(hi, bf16(a1 - hi)), F32(1.0 / 16))
    acc = np.zeros((ph - 2 * n, pw - 2 * n), F32)
    for c8 in range(c2 // 8):
        cs = slice(8 * c8, 8 * c8 + 8)
        t = np.zeros((8,) + acc.shape, F32)
        for ky in range(3):
            for kx in range(3):
                t = fma32(w2[0, cs, ky, kx][:, None, None], a[cs, n - 1 + ky:ph - n - 1 + ky, n - 1 + kx:pw - n - 1 + kx], t)
        for e in range(8):
            acc = add32(acc, t[e])
    return leaky_last(add32(acc, F32(b2[0])))


def emulate_bf16_model(plane, model, fused):
    """Context.convert_plane of a 1 -> C1 -> C2 -> 1 lattice model"""
    (w0, b0), (w1, b1), (w2, b2) = model
    n = 3
    x16 = emulate_first_layer(np.pad(plane, n, mode="edge"), w0, b0)
    zpad = [(np.pad(a, ((0, 0), (1, 1), (1, 1))), b) for a, b in bf16_operands(x16, w1)]   # the TMA loads zero-fill
    a1 = tc_activation(accumulate(zpad), 1.0, b1)
    return emulate_last_fused(a1, w2, b2, n) if fused else emulate_bf16_last_separate(a1, w2, b2, n)


def bf16x3_forward(plane, weights, biases):
    """the engine's arithmetic off the lattice: first layer in fp32, every tensor-core layer as the three bf16 products summed
    in float64 and rounded once to fp32, the fp32 epilogue on x16, the last layer on the fp32 activations (fused)"""
    n = len(weights)
    x = torch.from_numpy(np.pad(plane.astype(F32), n, mode="edge"))[None, None]
    act = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), torch.from_numpy(weights[0])) + \
        torch.from_numpy(biases[0].astype(F32))[None, :, None, None]
    act = torch.where(act < 0, act * np.float32(0.1), act) * 16.0
    for li in range(1, n - 1):
        pairs = bf16_operands(act[0].numpy(), weights[li])
        acc = sum(F.conv2d(torch.from_numpy(a)[None], torch.from_numpy(bw), padding=1) for a, bw in pairs).float()
        v = acc + torch.from_numpy(mul32(biases[li].astype(F32), F32(16)))[None, :, None, None]
        act = torch.where(v < 0, v * np.float32(0.1), v)
    out = F.conv2d(act / 16.0, torch.from_numpy(weights[-1]), padding=1) + np.float32(biases[-1][0])
    out = torch.where(out < 0, out * np.float32(0.1), out)
    return out[0, 0, n:-n, n:-n].numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the bf16 lattice
# ---------------------------------------------------------------------------------------------------------------------
# activations x16 = n + k 2^-10, n in {+-1, +-2}, k in {-1, 0, 1}: xh = bf16(x16) = n (bf16 keeps 8 bits: 1 +- 2^-9 would be
#     a rounding tie), xl = k 2^-10;
# weights w = wh + wl, wh in {0, +-1/2}, wl in {0, +-2^-11}, nonzero only where wh is: wh = bf16(w), wl = w - wh exactly;
# so every product is a multiple of Q = 2^-11 and bf16_lattice_report checks that the sums of the positive and of the
# negative terms stay within 2^22 Q: every partial sum, in any order, is exact in fp32.
def bf16_lattice_layer(cin, cout, seed):
    rng = np.random.default_rng(seed)
    shape = (cout, cin, 3, 3)
    nz = rng.random(shape) < 0.25
    wh = np.where(nz, rng.choice([-0.5, 0.5], size=shape), 0.0)
    wl = np.where(nz, rng.choice([-Q, 0.0, Q], size=shape, p=[0.125, 0.75, 0.125]), 0.0)
    wh[0, 0, 1, 1], wl[0, 0, 1, 1] = 0.5, Q
    b = rng.integers(-256, 257, cout) * 2.0 ** -10                    # 16 b on a 2^-6 grid
    return (wh + wl).astype(F32), b


def bf16_lattice_planes(c, h, w, seed):
    rng = np.random.default_rng(seed)
    n = rng.choice([-2.0, -1.0, 1.0, 2.0], size=(c, h, w))
    k = rng.choice([-1, 0, 1], size=(c, h, w), p=[0.125, 0.75, 0.125])
    return ((n + k * 2.0 ** -10) / 16).astype(F32)


def bf16_lattice_model(c1, c2, seed):
    """1 -> C1 -> C2 -> 1: one first-layer tap 16 w = +-1 per channel and 16 b = (1 or 2) + k 2^-10, so on a binary plane the
    first layer's outputs are {1, 2} + k 2^-10; the middle layer is a lattice layer; the last layer has ordinary weights"""
    rng = np.random.default_rng(seed)
    w0 = np.zeros((c1, 1, 3, 3), F32)
    tap, sign = rng.integers(0, 9, c1), rng.choice([-1.0, 1.0], c1)
    w0[np.arange(c1), 0, tap // 3, tap % 3] = sign / 16
    b0 = (np.where(sign > 0, 1.0, 2.0) + rng.integers(-1, 2, c1) * 2.0 ** -10) / 16
    w1, b1 = bf16_lattice_layer(c1, c2, seed + 1)
    w2 = (rng.standard_normal((1, c2, 3, 3)) * 0.05).astype(F32)
    b2 = np.array([F32(rng.standard_normal() * 0.05)], np.float64)
    return [(w0, b0), (w1, b1), (w2, b2)]


def bf16_lattice_report(x16_ring, w):
    """the splits are exact, the quantum is Q and the positive and negative term sums stay within 2^22 Q"""
    x = np.asarray(x16_ring, F32)
    wf = np.asarray(w, F32)
    xh, wh = bf16(x), bf16(wf)
    xl, wl = x - xh, wf - wh
    pairs = bf16_operands(x, w)
    units, q = accumulate_units(pairs)
    mag, _ = accumulate_units([(np.abs(a), np.abs(b)) for a, b in pairs])
    return {"splits exact": bool(np.array_equal(bf16(xl), xl) and np.array_equal(bf16(wl), wl)),
            "q": q, "sum_max_q": float(max((mag + units).max(), (mag - units).max())) / 2}


def assert_bf16_lattice(rep):
    assert rep["splits exact"], rep
    assert rep["q"] == Q, rep
    assert rep["sum_max_q"] <= 2 ** 22, rep


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------------
def test_constants_agree(w2x):
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "w2x_b200.h")).read()
    assert int(re.search(r"#define W2X_PRECISION_BF16X3 (\d+)", header).group(1)) == w2x.PRECISION_BF16X3 == 4
    assert "#define W2X_PRECISION_BF16X3 4" in header and not re.search(r"#define W2X_PRECISION_\w+ 3\b", header)


def _pack_reference(w):
    """bf16(w) / bf16(w - bf16(w)) in debug_tc_pack's layout: [chunk][tap][hi | lo][n_out rows of 64 B, SWIZZLE_64B]"""
    cout, cin = w.shape[:2]
    wf = np.asarray(w, F32)
    hi = bf16(wf)
    img = np.zeros((cin // 32, 9, 2, cout * 32), np.uint16)
    n, k = np.meshgrid(np.arange(cout), np.arange(32), indexing="ij")
    logical = n * 64 + 2 * k
    off = (logical ^ (((logical >> 7) & 3) << 4)) // 2
    for c in range(cin // 32):
        for t in range(9):
            blk = wf[:, 32 * c:32 * c + 32, t // 3, t % 3]
            hb = hi[:, 32 * c:32 * c + 32, t // 3, t % 3]
            img[c, t, 0, off] = bf16_bits(blk)
            img[c, t, 1, off] = bf16_bits(blk - hb)
    return img.reshape(-1)


@pytest.mark.parametrize("name", MODELS)
def test_pack_image(w2x, oracle_models, name):
    """every tensor-core layer's bf16 image, of the shipped model and of its x2^17 overflow rescaling (unpacked for the fp16
    precisions), is bf16(w) / bf16(w - bf16(w)) in the f16x3 layout at wscale 1"""
    om = oracle_models[name]
    over = MS.overflow_layer(om.weights)
    c = [1.0] * len(om.weights)
    c[over] = 2.0 ** MS.OVERFLOW_K
    for label, (ws, bs) in (("shipped", (om.weights, om.biases)), ("x2^17", MS.rescale(om.weights, om.biases, c))):
        m = w2x.Model.from_arrays(ws, bs)
        for li in range(1, len(ws) - 1):
            got = m.debug_tc_pack_bf16(li)
            assert got is not None, (label, li)
            assert np.array_equal(got, _pack_reference(ws[li])), (label, li)
        assert m.debug_tc_pack_bf16(0) is None and m.debug_tc_pack_bf16(len(ws) - 1) is None
        if label == "x2^17":
            assert m.debug_tc_pack(over)[0] is None                  # past the fp16 limit: no fp16 image


@pytest.fixture(scope="module")
def emulated(oracle_mod, oracle_models):
    x = oracle_mod.seeded_plane(96, 96, 1, "uniform")
    res = {}
    for name in MODELS:
        om = oracle_models[name]
        for s in SCALES:
            xs = (x * np.float32(s)).astype(F32)
            ref, _ = AR.f64_forward(xs, om.weights, om.biases)
            res[(name, s)] = AR.rel_err(bf16x3_forward(xs, om.weights, om.biases), ref)
    return res


def test_emulated_accuracy_is_flat_across_input_scale(emulated):
    """the emulated precision within the stated bound at input scales x1 to x1e6, on every shipped model"""
    print({k: f"{v:.2e}" for k, v in emulated.items()})
    bad = {k: v for k, v in emulated.items() if not v <= BF16X3_BOUND}
    assert not bad, bad
    assert BF16X3_BOUND < 1e-4


def test_lattice_emulator_is_the_float_emulator_on_the_lattice():
    w, b = bf16_lattice_layer(64, 128, seed=9)
    x = bf16_lattice_planes(64, 13, 21, seed=10)
    assert_bf16_lattice(bf16_lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w))
    assert np.array_equal(emulate_bf16_filter_layer(x, w, b, exact=True), emulate_bf16_filter_layer(x, w, b, exact=False))


def test_new_layer_kernels_have_no_stack_frame(w2x):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    r = subprocess.run(["cuobjdump", "-res-usage", w2x.lib_path()], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump could not read the library")
    found = re.findall(r"Function (\S*conv3x3_bf16x3_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", r.stdout)
    assert len(found) == 18, len(found)                   # 9 shapes x (plain, fused last layer)
    assert not [(n, s) for n, _, s in found if int(s) != 0]


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    c.set_precision(w2x.PRECISION_BF16X3)
    yield c
    c.close()


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", SHAPES)
def test_single_layer_is_bit_exact(w2x, bctx, cin, cout):
    """conv3x3_bf16x3_kernel<Cin, Cout, false> and the planar converters through filter_layer, at frame sizes around the
    tile-set and the M-tile, on every SM, one SM and three SMs"""
    w, b = bf16_lattice_layer(cin, cout, seed=100 * cin + cout)
    model = w2x.Model.from_arrays([w], [b])
    fails = []
    try:
        for i, (wd, h) in enumerate(LAYER_SIZES):
            x = bf16_lattice_planes(cin, h, wd, seed=1000 * i + cin + cout)
            assert_bf16_lattice(bf16_lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w))
            want = emulate_bf16_filter_layer(x, w, b)
            for sms in NUM_SMS:
                bctx.debug_set_num_sms(sms)
                got = bctx.filter_layer(model, 0, x)
                if not np.array_equal(got, want):
                    fails.append(f"{wd}x{h} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        bctx.debug_set_num_sms(0)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("c1,c2", SHAPES)
def test_whole_model_is_bit_exact(w2x, bctx, c1, c2):
    """1 -> C1 -> C2 -> 1 through convert_plane: first_layer_kernel<C1, BF16>, conv3x3_bf16x3_kernel<C1, C2, FUSE> + last_gather
    and, unfused, last_layer_kernel<C2, BF16>; the profile counters show that the CTAs covered every tile-set once"""
    m = bf16_lattice_model(c1, c2, seed=10 * c1 + c2)
    weights, biases = [t[0] for t in m], [t[1] for t in m]
    model = w2x.Model.from_arrays(weights, biases)
    all_sms = torch.cuda.get_device_properties(0).multi_processor_count
    fails = []
    try:
        for i, (wd, h) in enumerate(MODEL_SIZES):
            x = binary_plane(h, wd, seed=i + c1 + c2)
            frame16 = emulate_first_layer(np.pad(x, 3, mode="edge"), *m[0])
            assert_bf16_lattice(bf16_lattice_report(np.pad(frame16, ((0, 0), (1, 1), (1, 1))), m[1][0]))
            n_ts = _tilesets(wd + 6, h + 6)
            for fused in (True, False):
                want = emulate_bf16_model(x, m, fused)
                bctx.debug_set_fuse_last(fused)
                for sms in NUM_SMS:
                    bctx.debug_set_num_sms(sms)
                    bctx.debug_tc_profile_enable(True)
                    got = bctx.convert_plane(model, x)
                    prof = bctx.debug_tc_profile_read(1)
                    if prof["ctas"] != min(n_ts, sms or all_sms) or round(prof["tilesets"] * prof["ctas"]) != n_ts:
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {prof['ctas']} CTAs x {prof['tilesets']} tile-sets")
                    if not np.array_equal(got, want):
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        bctx.debug_set_num_sms(0)
        bctx.debug_set_fuse_last(True)
        bctx.debug_tc_profile_enable(False)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [32, 64, 128])
def test_first_layer_forms_and_converters_are_bit_exact(w2x, bctx, c):
    """first_layer_kernel<C, BF16, UP2X> read back through a selection layer (one weight 1 per output channel: the output is
    the input record's value) against the emulated first layer, for the plain and the folded 2x form; and the planar
    converters on values across the bf16 range, 1e-30 to 1e30"""
    rng = np.random.default_rng(c)
    sel = np.zeros((c, c, 3, 3), F32)
    sel[np.arange(c), rng.permutation(c), 1, 1] = 1.0
    w0 = (rng.standard_normal((c, 1, 3, 3)) * 0.3).astype(F32)
    b0 = rng.standard_normal(c) * 0.1
    w2 = (rng.standard_normal((1, c, 3, 3)) * 0.05).astype(F32)
    model = w2x.Model.from_arrays([w0, sel, w2], [b0, np.zeros(c), np.zeros(1)])
    x = rng.random((21, 30), dtype=np.float32)
    up = np.repeat(np.repeat(x, 2, 0), 2, 1)
    for fused in (True, False):
        bctx.debug_set_fuse_last(fused)
        try:
            for plane, got in ((x, bctx.convert_plane(model, x)), (up, bctx.convert_chain([(model, True)], x))):
                a0 = emulate_first_layer(np.pad(plane, 3, mode="edge"), w0, b0)
                pairs = [(np.pad(a, ((0, 0), (1, 1), (1, 1))), bw) for a, bw in bf16_operands(a0, sel)]
                a1 = tc_activation(accumulate(pairs, exact=False), 1.0, np.zeros(c))
                want = emulate_last_fused(a1, w2, np.zeros(1), 3) if fused else emulate_bf16_last_separate(a1, w2, np.zeros(1), 3)
                assert np.array_equal(got, want), (fused, plane.shape, _mismatch(got, want))
        finally:
            bctx.debug_set_fuse_last(True)
    planes = (np.exp(rng.uniform(-69, 69, (c, 9, 11))) * rng.choice([-1, 1], (c, 9, 11))).astype(F32)
    got = bctx.filter_layer(model, 1, planes)
    x16 = mul32(np.pad(planes, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
    want = bf16_readback(tc_activation(accumulate(bf16_operands(x16, sel), exact=False), 1.0, np.zeros(c)))
    assert np.array_equal(got, want), _mismatch(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind", [("scale2.0x", "uniform"), ("scale2.0x", "smooth"), ("noise1", "uniform"), ("noise2", "uniform")])
def test_golden_parity(bctx, shipped, oracle_mod, name, kind):
    """the 256x256 golden outputs of the reference's OpenCV path"""
    x = oracle_mod.seeded_plane(256, 256, 0, kind)
    g = np.load(golden_path(f"cfg1_{name}_{kind}.npy"))
    err = float(np.abs(bctx.convert_plane(shipped[name], x) - g).max())
    print(name, kind, f"max-abs {err:.2e}")
    assert err <= BF16X3_BOUND, err


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_activation_range(bctx, shipped, oracle_mod, oracle_models, name):
    """input scales x1 to x20000 (where f16x3 saturates) and x1e6: relative error within the bound against float64"""
    om = oracle_models[name]
    x = oracle_mod.seeded_plane(64, 56, 7, "uniform")
    report = []
    for s in GPU_SCALES:
        xs = (x * np.float32(s)).astype(F32)
        ref, _ = AR.f64_forward(xs, om.weights, om.biases)
        e = AR.rel_err(bctx.convert_plane(shipped[name], xs), ref)
        report.append(f"x{s:g} {e:.2e}")
        assert e <= BF16X3_BOUND, report
    print(name, ", ".join(report))


def _extra_patterns(weights):
    n = len(weights)
    pats = []
    for k in (-30, 30):
        c = [1.0] * n
        c[1] = 2.0 ** k
        pats.append((f"layer 1 x2^{k}", c))
    for k in (MS.OVERFLOW_K, 40):
        c = [1.0] * n
        c[MS.overflow_layer(weights)] = 2.0 ** k
        pats.append((f"overflow layer x2^{k}", c))
    return pats


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_every_rescaling_is_bit_identical(w2x, bctx, oracle_mod, oracle_models, name):
    """every pattern of tests/test_model_scale.py, one layer x2^+-30 and the overflow layer x2^17 and x2^40: bit-identical to
    the shipped model's bf16x3 output, fused and separate last layer"""
    om = oracle_models[name]
    x = MS.gpu_plane(oracle_mod)
    fails = []
    for fused in (True, False):
        bctx.debug_set_fuse_last(fused)
        try:
            want = None
            for label, c in MS.patterns(om.weights) + _extra_patterns(om.weights):
                got = bctx.convert_plane(w2x.Model.from_arrays(*MS.rescale(om.weights, om.biases, c)), x)
                if want is None:
                    want = got
                elif not np.array_equal(got, want):
                    fails.append(f"fused={fused} {label}: {_mismatch(got, want)}")
        finally:
            bctx.debug_set_fuse_last(True)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_auto_runs_the_overflow_model_on_the_tensor_cores_in_bf16x3_only(w2x, oracle_mod, oracle_models, name):
    om = oracle_models[name]
    c = [1.0] * len(om.weights)
    c[MS.overflow_layer(om.weights)] = 2.0 ** MS.OVERFLOW_K
    model = w2x.Model.from_arrays(*MS.rescale(om.weights, om.biases, c))
    x = MS.gpu_plane(oracle_mod)
    n = len(om.weights)
    ctx = w2x.Context(0, engine=w2x.ENGINE_AUTO)
    try:
        ctx.set_timing(True)
        for prec in (w2x.PRECISION_F16X3, w2x.PRECISION_F16_F8X2, w2x.PRECISION_F16):
            ctx.set_precision(prec)
            ctx.convert_plane(model, x)
            assert [t[2] for t in ctx.layer_times()] == ["fp32_direct"] * n, prec
        ctx.set_precision(w2x.PRECISION_BF16X3)
        ctx.convert_plane(model, x)
        names = [t[2] for t in ctx.layer_times()]
        assert names == ["first_1xN"] + ["wgmma_bf16x3"] * (n - 3) + ["wgmma_bf16x3+last", "last_gather"], names
        ctx.set_engine(w2x.ENGINE_TC)
        ctx.set_precision(w2x.PRECISION_F16X3)
        with pytest.raises(w2x.W2xError) as e:
            ctx.convert_plane(model, x)
        assert e.value.status == 7                                          # W2X_ERR_UNSUPPORTED
    finally:
        ctx.close()


@pytest.mark.gpu
def test_every_entry_point_equals_convert_plane(w2x, bctx, shipped, oracle_mod):
    """host and device buffers, the fused and the literal block walk, scratch-limited bands, convert_tiles, convert_planes,
    convert_chain (host and device), convert_planes_chain with a TTA step, convert_chain_regions and caller-exchange Band
    sessions: bit-identical to convert_plane in bf16x3"""
    ctx, model, up = bctx, shipped["noise2"], shipped["scale2.0x"]
    n = len(model)
    W, H = 90, 100
    x = oracle_mod.seeded_plane(W, H, 4, "uniform")
    whole = ctx.convert_plane(model, x)
    fails = []

    def check(what, got, want):
        if not np.array_equal(got, want):
            fails.append(f"{what}: {_mismatch(got, want)}")

    d_in = torch.from_numpy(x).cuda()
    d_out = torch.empty_like(d_in)
    ctx.convert_plane_device(model, d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
    ctx.synchronize()
    check("device buffers", d_out.cpu().numpy(), whole)
    bw, bh = w2x.get_block_size()
    try:
        w2x.set_block_size(48, 48)
        for walk in (w2x.WALK_FUSED, w2x.WALK_BLOCKS):
            ctx.set_block_walk(walk)
            check(f"block split walk={walk}", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_block_walk(w2x.WALK_FUSED)
        w2x.set_block_size(bw, bh)
    try:
        ctx.set_scratch_limit(128 * (W + 2 * n) * 4 * (23 + 2 * n))
        check("scratch bands", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_scratch_limit(0)
    tiles = np.stack([oracle_mod.seeded_plane(40, 30, 20 + t, "uniform") for t in range(5)])
    want = [ctx.convert_plane(model, t, block_splitting=False) for t in tiles]
    check("convert_tiles", ctx.convert_tiles(model, tiles), np.stack(want))
    planes = [oracle_mod.seeded_plane(wd, h, 40 + i, "uniform") for i, (wd, h) in enumerate([(40, 30), (17, 50), (64, 9)])]
    for i, (got, p) in enumerate(zip(ctx.convert_planes(model, planes), planes)):
        check(f"convert_planes {i}", got, ctx.convert_plane(model, p, block_splitting=False))
    # a chain: noise2, then scale2.0x with the folded 2x resize
    mid = ctx.convert_plane(model, x, block_splitting=False)
    chain = ctx.convert_plane(up, np.repeat(np.repeat(mid, 2, 0), 2, 1), block_splitting=False)
    steps = [(model, False), (up, True)]
    check("convert_chain", ctx.convert_chain(steps, x, block_splitting=False), chain)
    d_c = torch.empty((2 * H, 2 * W), device="cuda")
    ctx.convert_chain_device(steps, d_in.data_ptr(), W, H, W * 4, d_c.data_ptr(), 2 * W * 4, block_splitting=False)
    ctx.synchronize()
    check("convert_chain_device", d_c.cpu().numpy(), chain)
    win = (13, 21, 70, 64)
    src = w2x.chain_region_source(steps, (W, H), win)
    got = ctx.convert_chain_regions(steps, [x[src[1]:src[1] + src[3], src[0]:src[0] + src[2]]], [(W, H)], [win])[0]
    check("convert_chain_regions", got, chain[win[1]:win[1] + win[3], win[0]:win[0] + win[2]])
    # TTA: the mean of the 8 variants' conversions, each as convert_plane computes it
    tta = ctx.convert_planes_chain([(model, False, True)], planes[:2])
    for i, p in enumerate(planes[:2]):
        outs = []
        for j in range(8):
            v = p.T if j & 4 else p
            v = v[::-1] if j & 2 else v
            v = v[:, ::-1] if j & 1 else v
            o = ctx.convert_plane(model, np.ascontiguousarray(v), block_splitting=False)
            o = o[:, ::-1] if j & 1 else o
            o = o[::-1] if j & 2 else o
            outs.append(o.T if j & 4 else o)
        acc = outs[0]
        for o in outs[1:]:
            acc = add32(acc, o)
        check(f"convert_planes_chain TTA {i}", tta[i], mul32(acc, F32(0.125)))
    # Band sessions, the halo rows moved by the caller after every step
    cuts = [0, 7, 30, 61, H]
    bands, outs = [], []
    try:
        for b in range(len(cuts) - 1):
            r0, r1 = cuts[b], cuts[b + 1]
            u, dn = b > 0, b < len(cuts) - 2
            band = w2x.Band(ctx, model, W, r1 - r0, u, dn)
            bands.append(band)
            band.load(d_in[r0 - (1 if u else 0):].data_ptr(), W * 4)
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
        check("band sessions", torch.cat(outs).cpu().numpy(), whole)
    finally:
        for band in bands:
            band.close()
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_workers_bands_and_multi_on_one_device(w2x, bctx, shipped, oracle_models, oracle_mod):
    """in-library exchange band groups and a w2x_multi of contexts 0, 0 (tests/band_worker.py): bit-identical to convert_plane"""
    from test_band_exchange import Job, run_worker
    om = oracle_models["noise1"]
    job = Job({"noise1": list(zip(om.weights, om.biases))})
    x = oracle_mod.seeded_plane(70, 60, 3, "uniform")
    big = oracle_mod.seeded_plane(96, 400, 5, "uniform")
    job.add({"id": "bands", "kind": "band", "model": "noise1", "width": 70, "precision": 4, "rows": [17, 9, 34],
             "in_pad": 0, "out_pad": 0}, x)
    job.add({"id": "big", "kind": "multi", "k": 2, "model": "noise1", "width": 96,
             "calls": [{"op": "plane", "model": "noise1", "precision": 4, "input": "big2"}]})
    job.inputs["big2"] = big
    with tempfile.TemporaryDirectory() as d:
        job.write(d)
        (outs, _), = run_worker(d)
    want = bctx.convert_plane(shipped["noise1"], x)
    for p in range(3):
        assert np.array_equal(outs[f"bands.{p}"], want), p
    assert np.array_equal(outs["big.0"], bctx.convert_plane(shipped["noise1"], big))


@pytest.mark.gpu
def test_a_bf16x3_band_refuses_an_f16x3_neighbour(w2x, shipped):
    model = shipped["noise1"]
    ctxs = [w2x.Context(0, engine=w2x.ENGINE_TC) for _ in range(2)]
    ctxs[0].set_precision(w2x.PRECISION_BF16X3)
    ctxs[1].set_precision(w2x.PRECISION_F16X3)
    bands = []
    try:
        bands = [w2x.Band(ctxs[0], model, 50, 30, False, True), w2x.Band(ctxs[1], model, 50, 30, True, False)]
        with pytest.raises(w2x.W2xError) as e:
            bands[0].connect_local(None, bands[1])
        assert e.value.status == 1 and "precision" in str(e.value)
        with pytest.raises(w2x.W2xError):
            bands[0].connect(None, bands[1].export())
    finally:
        for b in bands:
            b.close()
        for c in ctxs:
            c.close()


@pytest.mark.gpu
def test_interface(w2x, shipped, oracle_mod, monkeypatch):
    monkeypatch.setenv("W2X_PRECISION", "bf16x3")
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        assert c.get_precision() == w2x.PRECISION_BF16X3 == 4
        c.set_timing(True)
        c.convert_plane(shipped["scale2.0x"], oracle_mod.seeded_plane(64, 48, 0, "uniform"))
        assert [t[2] for t in c.layer_times()] == ["first_1xN"] + ["wgmma_bf16x3"] * 4 + ["wgmma_bf16x3+last", "last_gather"]
        c.debug_set_fuse_last(False)
        c.convert_plane(shipped["scale2.0x"], oracle_mod.seeded_plane(64, 48, 0, "uniform"))
        assert [t[2] for t in c.layer_times()] == ["first_1xN"] + ["wgmma_bf16x3"] * 5 + ["last_Nx1"]
        with pytest.raises(w2x.W2xError):
            c.set_precision(3)
    finally:
        c.close()


@pytest.fixture(scope="module")
def cli(w2x):
    from test_cli import CLI                              # skips where cv2 is missing, like tests/test_cli.py
    w2x.build()
    assert os.path.exists(CLI)
    return CLI


@pytest.mark.gpu
@pytest.mark.parametrize("mode,level,ratio,name", [("noise_scale", 1, 2.0, "in(noise_scale)(Level1)(x2.000000).png"),
                                                  ("scale", 1, 3.0, "in(scale)(x3.000000).png"),
                                                  ("noise", 2, 2.0, "in(noise)(Level2).png")])
def test_cli_with_the_environment_value(cli, tmp_path, json_models, oracle_models, ncpu, mode, level, ratio, name):
    """the drop-in CLI with W2X_PRECISION=bf16x3 against the reference pipeline: the same file name, every output byte
    within 1 LSB"""
    import cv2
    from test_cli import _reference_pipeline, _test_image
    bgr = _test_image(45, 33, 11)
    cv2.imwrite(str(tmp_path / "in.png"), bgr)
    mdir = os.path.dirname(json_models["scale2.0x"])
    r = subprocess.run([cli, "-i", str(tmp_path / "in.png"), "-m", mode, "--noise_level", str(level), "--scale_ratio", str(ratio),
                        "--model_dir", mdir, "-j", "2"], capture_output=True, text=True, env=dict(os.environ, W2X_PRECISION="bf16x3"))
    assert r.returncode == 0, r.stdout + r.stderr
    out = cv2.imread(str(tmp_path / name), cv2.IMREAD_COLOR)
    assert out is not None, os.listdir(tmp_path)
    ref = _reference_pipeline(bgr, mode, level, ratio, oracle_models, ncpu)
    assert out.shape == ref.shape
    diff = np.abs(out.astype(int) - ref.astype(int))
    print(mode, f"8-bit max diff {diff.max()}, changed {100 * (diff > 0).mean():.2f} %")
    assert diff.max() <= 1
