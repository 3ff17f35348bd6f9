"""Bit-exact tests of the tensor-core engine on exactly representable operands.

The tensor-core layer's arithmetic is deterministic up to the order in which the tensor cores add products.  On operands
where every product and every partial sum is exact, that order cannot matter, and exactly one output bit pattern is
correct.  A dropped, doubled or misrouted tap, 64-column slice, m64 half, 32-channel chunk or tile-set then fails every
time, where the tolerance tests (tests/test_gpu_parity.py) would let it through: one tap's e4m3 corrections dropped on one
slice of one half moves a whole-model output by less than F8_TOL.

The lattice (Q = 2^-4 is the quantum every product is a multiple of):
  activations x16 = x * 16 = n + k * 2^-13,  n in {+-1, +-2}, k in {-1, 0, 1}:  xh = fp16(x16) = n, xl = k * 2^-13
      (with 2^-12, -1 + 2^-12 would be a rounding tie);  xl8 = e4m3(xl * 2^10), xh8 = e4m3(xh / 2) are exact;
  weights w * wscale = wh + wl,  wh in {0, +-512},  wl in {0, +-1/8} and nonzero only where wh is (a lone wl would become
      its own wh, whose wh8 = e4m3(wh * 2^-10) underflows);  about three quarters of the weights are zero, and one
      |w| > 0.5 makes wscale = 2^10;  wh8 = e4m3(wh * 2^-10) and wl8 = e4m3(wl * 2) are exact;
so every correction product equals the true xl * wh or xh * wl.  lattice_report() checks, on the very inputs a test uses:
  (a) every operand split above is exact;
  (b) per output, the sums P of the positive and N of the negative terms stay within 2^22 Q: any partial sum in any order
      lies in [N, P], two bits inside fp32's 24, so neither HGMMA order nor truncation can round;
  (c) each e4m3 correction group (one tap, one 32-channel chunk: K = 64) adds up to at most GROUP_MAX_Q quanta in
      absolute value -- Hopper's e4m3 accumulation precision is not documented, so nothing may rest on it;
  (d) |16 (conv + bias)| < 1024, so the epilogue's fp16 and xl8 conversions do not saturate;
  (e) the wscale the packer picks (floor(log2(1024 / max|w|)), clamped to [0, 14]) is the 2^10 the lattice is built for.

The emulator computes from weights and planes (not from the packed images) what the kernels compute: the operand splits,
an exact accumulation in int64 units of Q, the epilogue's fmaf / leaky-ReLU / fp16 and e4m3 stores and the read-back.
Where the float32 sums are not exact (the fused last layer, last_gather, last_layer_kernel) it repeats them in the
kernels' own order with correctly rounded float32 operations.
"""
import fractions

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tc_numerics_model as T
from exact_arith import (F8_A, F8_C, F32, e4m3, emulate_first_layer, emulate_last_fused, emulate_last_separate,
                         f16, fma32, mul32, readback, tc_activation)

SHAPES = [(32, 32), (32, 64), (32, 128), (64, 32), (64, 64), (64, 128), (128, 32), (128, 64), (128, 128)]
PRECISIONS = ["f16x3", "f16+f8x2"]
Q = 2.0 ** -4
SUM_MAX_Q = 2 ** 22                # (b); the cases below reach 2^21.3 (128 input channels)
GROUP_MAX_Q = 64                   # (c); the cases below reach 45
LATTICE_WSCALE = 2.0 ** 10


# ---------------------------------------------------------------------------------------------------------------------
# emulator
# ---------------------------------------------------------------------------------------------------------------------
def operands(x16, w, f8):
    """The three factor pairs a tensor-core layer multiplies, as float64 with the e4m3 copies' power-of-two scales taken
    out (scaling by 2^k commutes with the products): [(xh, wh), (xl, wh), (xh, wl)], and wscale.  x16: activations * 16
    (float32 [C, ...]); w: raw weights [Cout, Cin, 3, 3]."""
    ws = T.wscale_of(w)
    wsc = (np.asarray(w, F32) * F32(ws)).astype(F32)                 # exact: a power of two
    wh = f16(wsc)
    wl = wsc - wh                                                     # exact
    xh = f16(x16)
    xl = np.asarray(x16, F32) - xh
    if f8:
        pairs = [(xh, wh),
                 (e4m3(xl * 2.0 ** F8_A) * 2.0 ** -F8_A, e4m3(wh * 2.0 ** -F8_A) * 2.0 ** F8_A),     # xl8 * wh8
                 (e4m3(xh * 2.0 ** -F8_C) * 2.0 ** F8_C, e4m3(wl * 2.0 ** F8_C) * 2.0 ** -F8_C)]     # xh8 * wl8
    else:
        pairs = [(xh, wh), (f16(xl), wh), (xh, f16(wl))]
    return [(np.asarray(a, np.float64), np.asarray(b, np.float64)) for a, b in pairs], ws


def grain(a):
    """the largest power of two that divides every element of a (float64); None if a is all zeros"""
    nz = np.abs(a[a != 0])
    if nz.size == 0:
        return None
    m, e = np.frexp(nz)
    mi = (m * 2.0 ** 53).astype(np.int64)
    _, low = np.frexp((mi & -mi).astype(np.float64))
    return 2.0 ** int((e - 53 + low - 1).min())


def conv_valid_int(x, w):
    """out[o, y, x] = sum_{i, ky, kx} w[o, i, ky, kx] * x[i, y + ky, x + kx] for integer x, w (x already holds the 1-pixel
    ring), as int64.  The products are summed by float64 matrix products: with every |partial sum| below 2^53 they are
    integers held exactly, in any order."""
    ci, hp, wp = x.shape
    h, wd = hp - 2, wp - 2
    assert np.abs(x).max() * np.abs(w).max() * 9 * ci < 2 ** 53
    xf, wf = x.astype(np.float64), w.astype(np.float64)
    out = np.zeros((w.shape[0], h * wd), np.float64)
    for ky in range(3):
        for kx in range(3):
            out += wf[:, :, ky, kx] @ xf[:, ky:ky + h, kx:kx + wd].reshape(ci, -1)
    return out.astype(np.int64).reshape(w.shape[0], h, wd)


def accumulate_units(pairs):
    """Exact sum of the three convolutions, in int64 units of the common quantum q: (units, q).  Raises if the operands
    are not on a lattice coarse enough for exact integer sums."""
    grains = [(grain(a), grain(b)) for a, b in pairs]
    q = min(ga * gb for ga, gb in grains if ga is not None and gb is not None)
    total = None
    for (a, b), (ga, gb) in zip(pairs, grains):
        if ga is None or gb is None:
            continue
        A, B = np.rint(a / ga).astype(np.int64), np.rint(b / gb).astype(np.int64)
        f = int(round(ga * gb / q))
        if int(np.abs(A).max()) * int(np.abs(B).max()) * f * 9 * a.shape[0] >= 2 ** 53:
            raise ValueError("operands too fine for an exact integer accumulation")
        t = conv_valid_int(A, B) * f
        total = t if total is None else total + t
    return total, q


def accumulate(pairs, exact=True):
    """the layer's fp32 accumulator: exact (lattice operands; then rounded once to float32, which (b) makes exact), or a
    float64 sum for operands off the lattice"""
    if exact:
        units, q = accumulate_units(pairs)
        return (units.astype(np.float64) * q).astype(F32)
    acc = sum(F.conv2d(torch.from_numpy(a)[None], torch.from_numpy(b))[0] for a, b in pairs)
    return acc.numpy().astype(F32)








def emulate_filter_layer(planes, w, b, f8, exact=True):
    """Context.filter_layer on the tensor-core engine: planar_to_nhwc (replicate ring, x16, split) -> layer -> nhwc_to_planar"""
    x16 = mul32(np.pad(planes, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
    pairs, ws = operands(x16, w, f8)
    return readback(tc_activation(accumulate(pairs, exact), ws, b), f8)




def emulate_model(plane, model, f8, fused):
    """Context.convert_plane of a 1 -> C1 -> C2 -> 1 model on the tensor-core engine"""
    (w0, b0), (w1, b1), (w2, b2) = model
    n = 3
    frame = np.pad(plane, n, mode="edge")
    x16 = emulate_first_layer(frame, w0, b0)
    pairs, ws = operands(x16, w1, f8)
    zpad = [(np.pad(a, ((0, 0), (1, 1), (1, 1))), b) for a, b in pairs]     # the TMA loads zero-fill outside the frame
    a1 = tc_activation(accumulate(zpad), ws, b1)                      # [C2, ph, pw], activations * 16
    return emulate_last_fused(a1, w2, b2, n) if fused else emulate_last_separate(a1, w2, b2, n, f8)


# ---------------------------------------------------------------------------------------------------------------------
# lattice generator and its conditions
# ---------------------------------------------------------------------------------------------------------------------
def lattice_layer(cin, cout, seed):
    """raw fp32 weights [Cout, Cin, 3, 3] with w * 2^10 = wh + wl on the lattice, and fp64 biases with 16 b on a 2^-6 grid"""
    rng = np.random.default_rng(seed)
    shape = (cout, cin, 3, 3)
    nz = rng.random(shape) < 0.25
    wh = np.where(nz, rng.choice([-512.0, 512.0], size=shape), 0.0)
    wl = np.where(nz, rng.choice([-0.125, 0.0, 0.125], size=shape, p=[0.125, 0.75, 0.125]), 0.0)
    wh[0, 0, 1, 1], wl[0, 0, 1, 1] = 512.0, 0.125                     # |w| = 0.5 + 2^-13 > 0.5: wscale = 2^10
    w = ((wh + wl) * 2.0 ** -10).astype(F32)
    b = rng.integers(-256, 257, cout) * 2.0 ** -10
    return w, b


def lattice_planes(c, h, w, seed):
    """input planes x = (n + k 2^-13) / 16"""
    rng = np.random.default_rng(seed)
    n = rng.choice([-2.0, -1.0, 1.0, 2.0], size=(c, h, w))
    k = rng.choice([-1, 0, 1], size=(c, h, w), p=[0.125, 0.75, 0.125])
    return ((n + k * 2.0 ** -13) / 16).astype(F32)


def lattice_model(c1, c2, seed):
    """1 -> C1 -> C2 -> 1: the first layer has one tap 16 w = +-1 per channel and 16 b = (1 or 2) + k 2^-13, so on a
    binary plane its outputs are {1, 2} + k 2^-13 (the leaky-ReLU's positive branch); the middle layer is a lattice
    layer; the last layer has ordinary random weights (its float32 sums are emulated in the kernels' order)"""
    rng = np.random.default_rng(seed)
    w0 = np.zeros((c1, 1, 3, 3), F32)
    tap, sign = rng.integers(0, 9, c1), rng.choice([-1.0, 1.0], c1)
    w0[np.arange(c1), 0, tap // 3, tap % 3] = sign / 16
    b0 = (np.where(sign > 0, 1.0, 2.0) + rng.integers(-1, 2, c1) * 2.0 ** -13) / 16
    w1, b1 = lattice_layer(c1, c2, seed + 1)
    w2 = (rng.standard_normal((1, c2, 3, 3)) * 0.05).astype(F32)
    b2 = np.array([F32(rng.standard_normal() * 0.05)], np.float64)
    return [(w0, b0), (w1, b1), (w2, b2)]


def binary_plane(h, w, seed):
    return (np.random.default_rng(seed).random((h, w)) < 0.5).astype(F32)


def lattice_report(x16_ring, w, b):
    """Checks conditions (a)-(e) for one layer on activations x16_ring ([Cin, H + 2, W + 2], the ring the layer reads
    included) and returns what it measured."""
    rep = {}
    x = np.asarray(x16_ring, F32)
    xh = f16(x)
    xl = x - xh
    ws = T.wscale_of(w)
    wsc = (w * F32(ws)).astype(F32)
    wh = f16(wsc)
    wl = wsc - wh
    exact = lambda v, r: bool(np.array_equal(np.asarray(v, np.float64), np.asarray(r, np.float64)))  # noqa: E731
    rep["a"] = {"xl fp16": exact(f16(xl), xl), "xl8": exact(e4m3(xl * 2.0 ** F8_A), xl * 2.0 ** F8_A),
                "xh8": exact(e4m3(xh * 2.0 ** -F8_C), xh * 2.0 ** -F8_C), "wl fp16": exact(f16(wl), wl),
                "wh8": exact(e4m3(wh * 2.0 ** -F8_A), wh * 2.0 ** -F8_A), "wl8": exact(e4m3(wl * 2.0 ** F8_C), wl * 2.0 ** F8_C),
                "no lone wl": bool(np.all((wl == 0) | (wh != 0)))}
    pairs = [(xh.astype(np.float64), wh.astype(np.float64)), (xl.astype(np.float64), wh.astype(np.float64)),
             (xh.astype(np.float64), wl.astype(np.float64))]
    units, q = accumulate_units(pairs)
    rep["q"] = q
    # (b): the sums of the positive and of the negative terms, P = (sum |t| + sum t) / 2 and -N = (sum |t| - sum t) / 2
    mag, q_mag = accumulate_units([(np.abs(a), np.abs(b_)) for a, b_ in pairs])
    assert q_mag == q
    rep["sum_max_q"] = float(max((mag + units).max(), (mag - units).max())) / 2
    # (c): one e4m3 group = one tap of one 32-channel chunk, both corrections; sum of the absolute terms
    h, wd = x.shape[1] - 2, x.shape[2] - 2
    g = 0.0
    for c in range(x.shape[0] // 32):
        cs = slice(32 * c, 32 * c + 32)
        for ky in range(3):
            for kx in range(3):
                s = (np.einsum("oi,ihw->ohw", np.abs(wh[:, cs, ky, kx]).astype(np.float64), np.abs(xl[cs, ky:ky + h, kx:kx + wd]).astype(np.float64)) +
                     np.einsum("oi,ihw->ohw", np.abs(wl[:, cs, ky, kx]).astype(np.float64), np.abs(xh[cs, ky:ky + h, kx:kx + wd]).astype(np.float64)))
                g = max(g, float(s.max()))
    rep["group_max_q"] = g / q
    # (d): the epilogue's input to the fp16 / e4m3 stores
    v = fma32((units.astype(np.float64) * q).astype(F32), F32(1.0 / ws), mul32(np.asarray(b, np.float64).astype(F32), F32(16))[:, None, None])
    rep["v_max"] = float(np.abs(v).max())
    rep["wscale"] = ws
    return rep


def assert_lattice(rep):
    assert all(rep["a"].values()), rep["a"]
    assert rep["q"] == Q, rep["q"]
    assert rep["sum_max_q"] <= SUM_MAX_Q, rep["sum_max_q"]
    assert rep["group_max_q"] <= GROUP_MAX_Q, rep["group_max_q"]
    assert rep["v_max"] < 1024, rep["v_max"]
    assert rep["wscale"] == LATTICE_WSCALE, rep["wscale"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the generator's conditions and the emulator
# ---------------------------------------------------------------------------------------------------------------------
def test_e4m3_helper_agrees_with_torch():
    """every e4m3 value, the midpoints between neighbours (ties) and points on either side, within +-448"""
    vals = np.unique(torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float64).numpy())
    vals = vals[np.isfinite(vals)]
    mids = (vals[:-1] + vals[1:]) / 2
    probe = np.concatenate([vals, mids, mids * (1 + 2.0 ** -20), mids * (1 - 2.0 ** -20), [2.0 ** -12, 3e-4]])
    probe = probe[np.abs(probe) <= 448]
    ref = torch.from_numpy(probe).to(torch.float8_e4m3fn).to(torch.float64).numpy()
    assert np.array_equal(e4m3(probe), ref)
    assert e4m3(np.array([460.0, -1e4]))[0] == 448 and e4m3(np.array([-1e4]))[0] == -448    # satfinite


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal(400) * 2.0 ** rng.integers(-8, 8, 400)).astype(F32)
    b = (rng.standard_normal(400)).astype(F32)
    c = np.concatenate([(-(a[:200].astype(np.float64) * b[:200]) * (1 + rng.standard_normal(200) * 2.0 ** -20)).astype(F32),   # cancellation
                        (rng.standard_normal(200) * 4).astype(F32)])
    got = fma32(a, b, c)
    for ai, bi, ci, gi in zip(a, b, c, got):
        exact = fractions.Fraction(float(ai)) * fractions.Fraction(float(bi)) + fractions.Fraction(float(ci))
        cand = [F32(float(exact)), np.nextafter(F32(float(exact)), F32(np.inf)), np.nextafter(F32(float(exact)), F32(-np.inf))]
        best = min(cand, key=lambda f: (abs(fractions.Fraction(float(f)) - exact), int(np.array(f).view(np.int32)) & 1))
        assert gi == best, (ai, bi, ci, gi, best)


@pytest.mark.parametrize("cin,cout", SHAPES)
def test_lattice_conditions_hold(cin, cout):
    """(a)-(e) on a single-layer case (replicate ring) and on the middle layer of a whole-model case (zero ring)"""
    w, b = lattice_layer(cin, cout, seed=cin + cout)
    x = lattice_planes(cin, 21, 30, seed=cin * cout)
    rep = lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w, b)
    print(cin, cout, {k: v for k, v in rep.items() if k != "a"})
    assert_lattice(rep)
    m = lattice_model(cin, cout, seed=7 * cin + cout)
    x16 = emulate_first_layer(np.pad(binary_plane(20, 13, 3), 3, mode="edge"), *m[0])
    assert set(np.unique(x16).tolist()) <= {n + k * 2.0 ** -13 for n in (1, 2) for k in (-1, 0, 1)}
    rep = lattice_report(np.pad(x16, ((0, 0), (1, 1), (1, 1))), *m[1])
    assert_lattice(rep)


@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("f8", [False, True], ids=PRECISIONS)
def test_int64_accumulation_equals_float64_conv(cin, cout, f8):
    w, _ = lattice_layer(cin, cout, seed=cin + cout)
    x16 = mul32(np.pad(lattice_planes(cin, 11, 17, seed=cin * cout), ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
    pairs, ws = operands(x16, w, f8)
    assert ws == LATTICE_WSCALE
    units, q = accumulate_units(pairs)
    assert q == Q
    ref = sum(F.conv2d(torch.from_numpy(a)[None], torch.from_numpy(b_))[0] for a, b_ in pairs).numpy()
    assert np.array_equal(units.astype(np.float64) * q, ref)
    assert np.abs(units).max() < 2 ** 24                              # held exactly by an fp32 accumulator


def test_emulator_matches_the_numerics_model_off_the_lattice():
    """A random (non-lattice) layer in f16x3, the emulator with a float64 accumulation against tests/tc_numerics_model.py's
    arithmetic for the same layer (fp16 split, wide accumulation, fp32 epilogue, hi + lo read-back).  They differ only in
    roundings of about 2^-24 relative (fmaf vs a separate multiply and add, the fp32 cast of the accumulator)."""
    rng = np.random.default_rng(4)
    cin, cout = 64, 128
    w = (rng.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(F32)
    b = rng.standard_normal(cout).astype(F32).astype(np.float64) * 0.05
    x = rng.random((cin, 19, 23), dtype=F32)
    got = emulate_filter_layer(x, w, b, f8=False, exact=False)
    xt = F.pad(torch.from_numpy(x)[None], (1, 1, 1, 1), mode="replicate")
    ws = T.wscale_of(w)
    wh, wl = T.split16(torch.from_numpy(w) * ws)
    xh, xl = T.split16(xt * T.ACT_SCALE)
    xh, xl, wh, wl = (t.double() for t in (xh, xl, wh, wl))
    acc = F.conv2d(xh, wh) + F.conv2d(xl, wh) + F.conv2d(xh, wl)
    v = T.leaky(acc.float() * np.float32(1.0 / ws) + torch.from_numpy((b * 16).astype(F32))[None, :, None, None])
    hi, lo = T.split16(v)
    ref = ((hi.float() + lo.float()) / T.ACT_SCALE)[0].numpy()
    err = float(np.abs(got - ref).max())
    assert err <= 2.0 ** -20 * max(1.0, float(np.abs(ref).max())), err
    assert err > 0 or np.array_equal(got, ref)


@pytest.mark.parametrize("cin,cout", SHAPES)
def test_packer_splits_the_lattice_weights_as_the_generator_does(w2x, cin, cout):
    """the library's wscale and its fp16 hi / lo weight images equal the generator's split (layer 1 of a 1->C1->C2->1 model)"""
    m = lattice_model(cin, cout, seed=cin + 3 * cout)
    model = w2x.Model.from_arrays([t[0] for t in m], [t[1] for t in m])
    data, n_chunk, kblocks, ws = model.debug_tc_pack(1)
    assert ws == T.wscale_of(m[1][0]) == LATTICE_WSCALE
    assert n_chunk == cin // 32 and kblocks == 1
    wsc = (m[1][0] * F32(ws)).astype(F32)
    wh = f16(wsc)
    wl = wsc - wh
    assert np.array_equal(f16(wl), wl)
    n, k = np.meshgrid(np.arange(cout), np.arange(32), indexing="ij")
    logical = n * 64 + 2 * k
    off = (logical ^ (((logical >> 7) & 3) << 4)) // 2                # SWIZZLE_64B rows of 64 B
    blk = cout * 32
    for c in range(n_chunk):
        for t in range(9):
            base = (c * 9 + t) * 2 * blk
            hi = data[base:base + blk][off].view(np.float16).astype(F32)
            lo = data[base + blk:base + 2 * blk][off].view(np.float16).astype(F32)
            assert np.array_equal(hi, wh[:, 32 * c:32 * c + 32, t // 3, t % 3]), (c, t)
            assert np.array_equal(lo, wl[:, 32 * c:32 * c + 32, t // 3, t % 3]), (c, t)


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
NUM_SMS = [0, 1, 3]                # 0 = every SM
# filter_layer planes: the frame (w + 2) x (h + 2) has Wp mod 16 in {8 (Wp < 16), 0, 1, 7, 8, 9, 15, 14} and
# Hp mod 16 in {7 (Hp < 16), 1, 8, 0, 0, 9 (Hp < 16), 9, 10}; 60 x 40 has 12 tile-sets, all in one CTA at one SM
LAYER_SIZES = [(6, 5), (14, 15), (15, 22), (21, 14), (22, 30), (23, 7), (29, 23), (60, 40)]
# convert_plane planes of a 3-layer model: frame (w + 6) x (h + 6) = 16x9, 17x24, 23x16, 31x33, 60x40
MODEL_SIZES = [(10, 3), (11, 18), (17, 10), (25, 27), (54, 34)]


def _tilesets(pw, ph):
    return -(-pw // 16) * -(-ph // 16)


@pytest.fixture(scope="module")
def tc_ctxs(w2x):
    c = {}
    for p, prec in zip(PRECISIONS, (w2x.PRECISION_F16X3, w2x.PRECISION_F16_F8X2)):
        c[p] = w2x.Context(0, engine=w2x.ENGINE_TC)
        c[p].set_precision(prec)
    yield c
    for v in c.values():
        v.close()


def _mismatch(got, want):
    bad = np.argwhere(got != want)
    i = tuple(bad[0])
    return f"{len(bad)} of {got.size} differ, first at {i}: {got[i]!r} != {want[i]!r}"


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("prec", PRECISIONS)
def test_single_layer_is_bit_exact(w2x, tc_ctxs, cin, cout, prec):
    """tc_conv3x3_kernel<Cin, Cout, FUSE = false, F8> through filter_layer, at frame widths / heights around the 16-pixel
    tile-set and the 8-pixel M-tile, on every SM, one SM and three SMs"""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    w, b = lattice_layer(cin, cout, seed=100 * cin + cout)
    model = w2x.Model.from_arrays([w], [b])
    fails = []
    try:
        for i, (wd, h) in enumerate(LAYER_SIZES):
            x = lattice_planes(cin, h, wd, seed=1000 * i + cin + cout)
            assert_lattice(lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w, b))
            want = emulate_filter_layer(x, w, b, f8)
            for sms in NUM_SMS:
                ctx.debug_set_num_sms(sms)
                got = ctx.filter_layer(model, 0, x)
                if not np.array_equal(got, want):
                    fails.append(f"{wd}x{h} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        ctx.debug_set_num_sms(0)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("c1,c2", SHAPES)
@pytest.mark.parametrize("prec", PRECISIONS)
def test_whole_model_is_bit_exact(w2x, tc_ctxs, c1, c2, prec):
    """1 -> C1 -> C2 -> 1 through convert_plane: first_layer_kernel<C1>, tc_conv3x3_kernel<C1, C2, FUSE> + last_gather and,
    with the last layer not fused, tc_conv3x3_kernel<C1, C2> + last_layer_kernel<C2>.  The profile counters show that the
    CTAs covered every tile-set once: tile-sets x CTAs = the layer's tile-set count, CTAs = min(tile-sets, SMs)."""
    ctx, f8 = tc_ctxs[prec], prec != "f16x3"
    m = lattice_model(c1, c2, seed=10 * c1 + c2)
    model = w2x.Model.from_arrays([t[0] for t in m], [t[1] for t in m])
    all_sms = torch.cuda.get_device_properties(0).multi_processor_count
    fails = []
    try:
        ctx.debug_tc_profile_enable(True)
        for i, (wd, h) in enumerate(MODEL_SIZES):
            x = binary_plane(h, wd, seed=i + c1 + c2)
            frame16 = emulate_first_layer(np.pad(x, 3, mode="edge"), *m[0])
            assert_lattice(lattice_report(np.pad(frame16, ((0, 0), (1, 1), (1, 1))), *m[1]))
            n_ts = _tilesets(wd + 6, h + 6)
            for fused in (True, False):
                want = emulate_model(x, m, f8, fused)
                ctx.debug_set_fuse_last(fused)
                for sms in NUM_SMS:
                    ctx.debug_set_num_sms(sms)
                    ctx.debug_tc_profile_enable(True)                 # zero the counters
                    got = ctx.convert_plane(model, x)
                    prof = ctx.debug_tc_profile_read(1)
                    if prof["ctas"] != min(n_ts, sms or all_sms) or round(prof["tilesets"] * prof["ctas"]) != n_ts:
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {prof['ctas']} CTAs x {prof['tilesets']} tile-sets, "
                                     f"want {n_ts} tile-sets")
                    if not np.array_equal(got, want):
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        ctx.debug_set_num_sms(0)
        ctx.debug_set_fuse_last(True)
        ctx.debug_tc_profile_enable(False)
    assert not fails, "\n".join(fails)


# every (Cin, Cout) pair once as a middle layer: 32-32-64-64-128-128-32-128-64-32
CHAIN = [32, 32, 64, 64, 128, 128, 32, 128, 64, 32]


def _grid_models(oracle_mod, oracle_models):
    ms = {n: (om.weights, om.biases) for n, om in oracle_models.items()}
    dims = [(1, CHAIN[0])] + list(zip(CHAIN[:-1], CHAIN[1:])) + [(CHAIN[-1], 1)]
    om = oracle_mod.OracleModel.random(dims, seed=77)
    ms["chain"] = (om.weights, om.biases)
    for c1, c2 in SHAPES:                                             # every shape as the fused last tensor-core layer
        om = oracle_mod.OracleModel.random([(1, c1), (c1, c2), (c2, 1)], seed=c1 + 3 * c2)
        ms[f"1-{c1}-{c2}-1"] = (om.weights, om.biases)
    return ms


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_output_does_not_depend_on_the_grid(w2x, tc_ctxs, oracle_mod, oracle_models, prec):
    """On ordinary inputs a tile-set's result must not depend on which CTA computed it or on what that CTA computed
    before (accumulator reset, staging-tile reuse, barrier parity): the three shipped models, a random chain with every
    shape as a middle layer (fused and separate last layer) and a random 1 -> C1 -> C2 -> 1 model per shape, 200 x 150
    planes, bit-identical at 1, 2, 7 and 64 SMs to the full grid"""
    ctx = tc_ctxs[prec]
    x = oracle_mod.seeded_plane(200, 150, 9, "uniform")
    fails = []
    try:
        for name, (ws, bs) in _grid_models(oracle_mod, oracle_models).items():
            model = w2x.Model.from_arrays(ws, bs)
            for fused in ((True, False) if name == "chain" else (True,)):
                ctx.debug_set_fuse_last(fused)
                ctx.debug_set_num_sms(0)
                ref = ctx.convert_plane(model, x)
                assert np.isfinite(ref).all(), name
                for sms in (1, 2, 7, 64):
                    ctx.debug_set_num_sms(sms)
                    got = ctx.convert_plane(model, x)
                    if not np.array_equal(got, ref):
                        fails.append(f"{name} fused={fused} num_sms={sms}: {_mismatch(got, ref)}")
    finally:
        ctx.debug_set_num_sms(0)
        ctx.debug_set_fuse_last(True)
    assert not fails, "\n".join(fails)
