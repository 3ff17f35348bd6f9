"""Both engines bit for bit at the benchmark's plane sizes, against small planes they are the periodic extension of.

Every output pixel of a step depends only on the (2n + 1)^2 neighbourhood of its input pixel, with replicate padding only at
the plane's border, and every entry point computes it from the same operands in the same order wherever the pixel lies.  So
take an H x W plane X[y][x] = T[y mod p][x mod q] of a random p x q tile T, and the small plane x of h x w pixels with the
same rule, h = H (mod p), h >= p + 2M and w = W (mod q), w >= q + 2M, where M is the sum of the steps' layer counts (input
pixels, conservative) and s = 2^u for u upscaling steps.  Output row Y of the big plane is output row m(Y) of the small one:
  m(Y) = Y                            for Y < s M            (the top border and its replicate padding)
  m(Y) = Y - s (H - h)                for Y >= s (H - M)     (the bottom border: h = H mod p keeps the phase)
  m(Y) = s M + ((Y - s M) mod s p)    otherwise              (the interior, periodic with period s p)
and columns likewise with q and w.  The expected big output is one gather of the small output, so a conversion of about
120 x 180 pixels checks every pixel of a 4096^2 or 8192^2 one bit for bit: every tile-set of every CTA, frames past 2^32
bytes, scratch bands and the host copy pipeline's bands, where the tolerance tests let through anything under 6e-5.

The periods are odd primes, so the tile-set (16 x 16), M-tile (8) and 32-pixel geometry meets every phase of T.  The small
plane's reference is absolute where an emulator exists (lattice operands on the tensor-core engine, tests/test_tc_exact.py;
the fp32 engine, tests/exact_arith.py) and otherwise the same context's conversion of the small plane, itself held to the
oracle at the tolerances of tests/test_gpu_parity*.py so that the relation cannot hold trivially.
"""
import math
import time

import numpy as np
import pytest
import torch

from exact_arith import F32, add32, fma32, fp32_convert, leaky_last, mul32
from test_tc_exact import (SHAPES, assert_lattice, binary_plane, emulate_filter_layer, emulate_first_layer, emulate_model,
                           lattice_layer, lattice_model, lattice_planes, lattice_report)

P, Q = 97, 89                      # row and column periods
PRECISIONS = {"f16x3": 0, "f16+f8x2": 1, "f16": 2}       # W2X_PRECISION_*
DEFAULT_PRECISION = "f16+f8x2"
F8_TOL, TC_TOL, F16_TOL = 6e-5, 2e-5, 1.5e-3       # tests/test_gpu_parity.py, tests/test_precision_f16.py
ORACLE_TOL = {"f16x3": TC_TOL, "f16+f8x2": F8_TOL, "f16": F16_TOL}
N_LAYERS = 7                       # the shipped models

LAYER_PLANE = (2045, 1277)         # W x H: frame 2047 x 1279, 128 x 80 tile-sets with partial ones at the right and bottom
MODEL_PLANE = (4096, 4096)         # bench.py's plane; 128-channel record frames of 4102^2 pixels pass 2^32 bytes
BIG_PLANE = (8192, 8192)           # config 4
TILES = (64, 512)                  # config 5: 64 tiles of 512^2
CHAIN_PLANE = (1920, 1080)         # config 2: noise1, then 2x and scale2.0x
SIZES = [*LAYER_PLANE, *MODEL_PLANE, *BIG_PLANE, TILES[1], *CHAIN_PLANE]


# ---------------------------------------------------------------------------------------------------------------------
# the periodic extension
# ---------------------------------------------------------------------------------------------------------------------
def small_size(n, period, m):
    """the smallest size >= period + 2 m that is congruent to n modulo period"""
    return period + 2 * m + (n - period - 2 * m) % period


def source_index(n, period, m, s, shift=0):
    """m(Y) for the s n output rows (or columns) of a plane of n input rows: the small plane's row that equals row Y.
    shift moves the interior's residue (the negative control)."""
    ns = small_size(n, period, m)
    assert n >= ns, (n, ns)
    y = np.arange(s * n)
    mid = s * m + (y - s * m + shift) % (s * period)
    return np.where(y < s * m, y, np.where(y >= s * (n - m), y - s * (n - ns), mid))


def periodic(tile, h, w):
    """X[..., y, x] = tile[..., y mod p, x mod q] of size h x w"""
    return np.take(np.take(tile, np.arange(h) % tile.shape[-2], axis=-2), np.arange(w) % tile.shape[-1], axis=-1)


class Extension:
    """a big plane of W x H input pixels and its small plane, for steps of m layers in all and s = 2^upscales"""

    def __init__(self, W, H, m, s=1):
        self.W, self.H, self.m, self.s = W, H, m, s
        self.w, self.h = small_size(W, Q, m), small_size(H, P, m)

    def index(self, shift=0):
        return (source_index(self.H, P, self.m, self.s, shift), source_index(self.W, Q, self.m, self.s, shift))

    def gather(self, small_out):
        """the expected big output from the small one (numpy or a torch tensor, [..., s h, s w])"""
        my, mx = self.index()
        if isinstance(small_out, torch.Tensor):
            my, mx = (torch.from_numpy(i).to(small_out.device) for i in (my, mx))
            return small_out.index_select(-2, my).index_select(-1, mx)
        return np.take(np.take(small_out, my, axis=-2), mx, axis=-1)


def expand_on_device(tile, H, W):
    """periodic(tile, H, W) built on the GPU from the tile"""
    t = torch.from_numpy(np.ascontiguousarray(tile, F32)).cuda()
    iy = torch.arange(H, device="cuda") % tile.shape[-2]
    ix = torch.arange(W, device="cuda") % tile.shape[-1]
    return t.index_select(-2, iy).index_select(-1, ix).contiguous()


def is_odd_prime(n):
    return n > 2 and n % 2 == 1 and all(n % d for d in range(3, math.isqrt(n) + 1, 2))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the mapping against the oracle
# ---------------------------------------------------------------------------------------------------------------------
# chains of 7-layer models (8 channels: the mapping depends on the layer count, not on the width); True = 2x first
CPU_CHAINS = {"noise1": [False], "noise1+scale2x": [False, True], "noise1+2xscale2x": [False, True, True]}
# about 3 periods per side, each with another H mod p and W mod q
CPU_PLANES = [(3 * Q + 80, 3 * P + 5), (3 * Q + 1, 3 * P + 60), (3 * Q + 44, 3 * P + 96)]


def _toy_model(oracle_mod, seed):
    return oracle_mod.OracleModel.random([(1, 8)] + [(8, 8)] * (N_LAYERS - 2) + [(8, 1)], seed=seed)


def _oracle_chain(oracle_mod, ups, x, ncpu):
    for k, up in enumerate(ups):
        if up:
            x = np.ascontiguousarray(np.repeat(np.repeat(x, 2, axis=0), 2, axis=1))
        x = _toy_model(oracle_mod, 5 + k).convert(x, block_splitting=False, n_job=ncpu)
    return x


_cpu_cache = {}


def _cpu_case(oracle_mod, ncpu, chain, plane):
    """(extension, big output, small output) of a chain on a periodic plane, the oracle computing both"""
    key = (chain, plane)
    if key not in _cpu_cache:
        ups = CPU_CHAINS[chain]
        ext = Extension(*plane, m=N_LAYERS * len(ups), s=2 ** sum(ups))
        tile = np.random.default_rng(plane[0] + plane[1]).random((P, Q), dtype=F32)
        big = _oracle_chain(oracle_mod, ups, periodic(tile, ext.H, ext.W), ncpu)
        small = _oracle_chain(oracle_mod, ups, periodic(tile, ext.h, ext.w), ncpu)
        _cpu_cache[key] = ext, big, small
    return _cpu_cache[key]


@pytest.mark.parametrize("plane", CPU_PLANES, ids=lambda p: f"{p[0]}x{p[1]}")
@pytest.mark.parametrize("chain", list(CPU_CHAINS))
def test_the_mapping_holds_on_the_oracle(oracle_mod, ncpu, chain, plane):
    """a plane of about 3 periods per side, converted whole, equals the gather from its small plane bit for bit: both
    borders of each axis, the corners and the interior"""
    ext, big, small = _cpu_case(oracle_mod, ncpu, chain, plane)
    assert big.shape == (ext.s * ext.H, ext.s * ext.W) and small.shape == (ext.s * ext.h, ext.s * ext.w)
    assert ext.h < ext.H and ext.w < ext.W
    my, mx = ext.index()
    for idx, n, period in ((my, ext.H, P), (mx, ext.W, Q)):      # each of the three pieces of m() is used
        y = np.arange(ext.s * n)
        assert (idx == y).sum() >= ext.s * ext.m and (idx < y).sum() >= ext.s * ext.m
        assert len(np.unique(idx)) >= ext.s * (period + 2 * ext.m)
    want = ext.gather(small)
    assert np.array_equal(big, want), f"{np.sum(big != want)} of {big.size} differ"


@pytest.mark.parametrize("chain", list(CPU_CHAINS))
def test_a_shifted_residue_differs(oracle_mod, ncpu, chain):
    """negative control: the gather with the interior's residue shifted by one row or one column does not match"""
    ext, big, small = _cpu_case(oracle_mod, ncpu, chain, CPU_PLANES[0])
    for shift in (1, -1):
        my, mx = ext.index()
        sy, sx = ext.index(shift)
        assert not np.array_equal(big, np.take(np.take(small, sy, axis=-2), mx, axis=-1)), shift
        assert not np.array_equal(big, np.take(np.take(small, my, axis=-2), sx, axis=-1)), shift


def test_the_periods_share_no_factor_with_the_geometry():
    """odd primes: no tile-set, M-tile or 32-pixel boundary keeps the same phase of T, and no plane of the cases here is a
    whole number of periods"""
    for period in (P, Q):
        assert is_odd_prime(period)
        for g in (8, 16, 32):
            assert math.gcd(period, g) == 1 and g % period != 0
        for n in SIZES + [d for p in CPU_PLANES for d in p]:
            assert n % period != 0, (n, period)
            assert n >= small_size(n, period, 2 * N_LAYERS)


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 engine's emulator on torch tensors (exact_arith.fp32_convert, on the GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _fma32_t(a, b, c):
    """exact_arith.fma32 on float32 tensors"""
    a, b, c = a.double(), b.double(), c.double()
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(torch.int64) & 1) == 0
    away = torch.nextafter(s, torch.where(err > 0, torch.full_like(s, math.inf), torch.full_like(s, -math.inf)))
    return torch.where((err != 0) & even, away, s).float()


def fp32_convert_t(plane, weights, biases, device, chunk=16):
    """exact_arith.fp32_convert (Model::filter per layer: tap 0 a rounded multiply, fmaf over taps 1..8, inputs summed in
    ascending order, + bias, leaky) with torch operations on `device`"""
    n = len(weights)
    x = torch.nn.functional.pad(torch.as_tensor(np.asarray(plane, F32), device=device)[None, None], (n,) * 4,
                                mode="replicate")[0]
    for w, b in zip(weights, biases):
        w = torch.from_numpy(np.asarray(w, F32)).to(device)
        cout, cin = w.shape[:2]
        h, wd = x.shape[1:]
        p = torch.nn.functional.pad(x[None], (1, 1, 1, 1), mode="replicate")[0]
        acc = torch.zeros((cout, h, wd), dtype=torch.float32, device=device)
        for i0 in range(0, cin, chunk):
            i1 = min(cin, i0 + chunk)
            t = None
            for k in range(9):
                ky, kx = divmod(k, 3)
                v = p[None, i0:i1, ky:ky + h, kx:kx + wd]
                wk = w[:, i0:i1, ky, kx][:, :, None, None]
                t = wk * v if t is None else _fma32_t(wk, v, t)
            for i in range(i1 - i0):
                acc = acc + t[:, i]
        bias = torch.from_numpy(np.asarray(b, np.float64).astype(F32)).to(device)[:, None, None]
        r = acc + bias
        x = torch.clamp(r, max=0) * F32(0.1) + torch.clamp(r, min=0)
    return x[0, n:-n, n:-n]


def test_torch_fp32_emulator_equals_exact_arith(oracle_mod):
    """the torch port computes exact_arith.fp32_convert's bits (on the CPU here), so the GPU case below rests on it"""
    om = oracle_mod.OracleModel.random([(1, 32), (32, 40), (40, 1)], seed=3)
    x = np.random.default_rng(2).random((23, 31), dtype=F32) * F32(4) - F32(1)
    want = fp32_convert(x, om.weights, om.biases)
    got = fp32_convert_t(x, om.weights, om.biases, "cpu").numpy()
    assert np.array_equal(got, want), f"{np.sum(got != want)} of {got.size} differ"
    r = (np.random.default_rng(4).standard_normal(1000) * 3).astype(F32)
    assert np.array_equal(leaky_last(r), (torch.clamp(torch.from_numpy(r), max=0) * F32(0.1) +
                                           torch.clamp(torch.from_numpy(r), min=0)).numpy())
    a, b, c = (np.random.default_rng(k).standard_normal(4000).astype(F32) for k in (5, 6, 7))
    c[:2000] = -(a[:2000].astype(np.float64) * b[:2000]).astype(F32)          # cancellation
    assert np.array_equal(_fma32_t(*(torch.from_numpy(v) for v in (a, b, c))).numpy(), fma32(a, b, c))
    assert np.array_equal((torch.from_numpy(a) + torch.from_numpy(b)).numpy(), add32(a, b))
    assert np.array_equal((torch.from_numpy(a) * torch.from_numpy(b)).numpy(), mul32(a, b))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
COMPARED = {}                      # case -> pixels compared bit for bit
PEAK = [0]                         # device memory in use (torch.cuda.mem_get_info), the largest seen after a conversion


def _note_memory():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    PEAK[0] = max(PEAK[0], total - free)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.perf_counter()
    yield
    if COMPARED:
        print(f"\ntest_periodic_scale: {time.perf_counter() - t0:.1f} s, peak device memory in use {PEAK[0] / 2 ** 30:.2f} GiB")
        for k, v in COMPARED.items():
            print(f"  {k}: {v} pixels bit for bit")


def _compare(fails, label, got, want, pad):
    """got == want bit for bit (torch tensors [..., H, W]); on a mismatch, a line with the count, the first positions as
    frame coordinates (the plane + pad on each side) and 16 x 16 tile-set indices, and the largest difference"""
    want = want.to(got.device)
    assert got.shape == want.shape, (label, got.shape, want.shape)
    COMPARED[label] = COMPARED.get(label, 0) + got.numel()
    bad = got != want
    n = int(bad.sum())
    if n == 0:
        return
    tiles_x = -(-(got.shape[-1] + 2 * pad) // 16)
    where = []
    for i in bad.nonzero()[:4].tolist():
        fy, fx = i[-2] + pad, i[-1] + pad
        where.append(f"{tuple(i)} frame ({fy}, {fx}) tile-set {fy // 16 * tiles_x + fx // 16}")
    d = float((got[bad].double() - want[bad].double()).abs().max())
    fails.append(f"{label}: {n} of {got.numel()} differ, max |diff| {d:.3e}, first at " + "; ".join(where))


@pytest.fixture
def tc(w2x):
    """a tensor-core context per test, so that at most one context's scratch buffers (two of at most 16 GiB) are held"""
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


def _flags(prec):
    """(f8, xh_only) of the emulators for a precision"""
    return prec == "f16+f8x2", prec == "f16"


# ---- 1. lattice layers and models, against the emulator ------------------------------------------------------------
MODEL_SHAPES = [(128, 128), (64, 32)]       # the first in every precision, the others in the default one


def _layer_case(cin, cout):
    """a lattice layer and its input tile"""
    w, b = lattice_layer(cin, cout, seed=100 * cin + cout)
    return w, b, lattice_planes(cin, P, Q, seed=cin * cout + 1)


def _model_case(c1, c2):
    """a 1 -> C1 -> C2 -> 1 lattice model and its binary tile"""
    return lattice_model(c1, c2, seed=10 * c1 + c2), binary_plane(P, Q, seed=c1 + c2)


@pytest.mark.parametrize("cin,cout", SHAPES)
def test_lattice_conditions_hold_on_the_small_planes(cin, cout):
    """(a)-(e) of tests/test_tc_exact.py on the small planes of the GPU cases below, which hold every neighbourhood of the
    big planes: a layer's input with its replicate ring, and a model's middle layer on the first layer's frame"""
    w, b, tile = _layer_case(cin, cout)
    ext = Extension(*LAYER_PLANE, m=1)
    x = periodic(tile, ext.h, ext.w)
    assert_lattice(lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w, b))
    if (cin, cout) in MODEL_SHAPES:
        m, tile = _model_case(cin, cout)
        ext = Extension(*MODEL_PLANE, m=3)
        frame16 = emulate_first_layer(np.pad(periodic(tile, ext.h, ext.w), 3, mode="edge"), *m[0])
        assert_lattice(lattice_report(np.pad(frame16, ((0, 0), (1, 1), (1, 1))), *m[1]))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("prec", list(PRECISIONS))
def test_lattice_layers_at_scale_are_bit_exact(w2x, tc, prec):
    """every (Cin, Cout) through filter_layer_device on a 2045 x 1277 plane: about 78 tile-sets per CTA on the full grid,
    partial tile-sets on the right and bottom edges, and in the default precision once more on 3 SMs (3400 per CTA).  The
    inputs are those test_lattice_conditions_hold_on_the_small_planes checks."""
    W, H = LAYER_PLANE
    ext = Extension(W, H, m=1)
    f8, xh_only = _flags(prec)
    fails = []
    tc.set_precision(PRECISIONS[prec])
    try:
        for cin, cout in SHAPES:
            w, b, tile = _layer_case(cin, cout)
            x = periodic(tile, ext.h, ext.w)
            want = ext.gather(torch.from_numpy(emulate_filter_layer(x, w, b, f8, xh_only=xh_only)).cuda())
            model = w2x.Model.from_arrays([w], [b])
            d_in = expand_on_device(tile, H, W)
            d_out = torch.empty((cout, H, W), device="cuda")
            for sms in ((0, 3) if prec == DEFAULT_PRECISION else (0,)):
                tc.debug_set_num_sms(sms)
                d_out.fill_(math.nan)
                tc.filter_layer_device(model, 0, d_in.data_ptr(), d_out.data_ptr(), W, H)
                _note_memory()
                _compare(fails, f"filter_layer {cin}->{cout} {prec} {W}x{H} num_sms={sms}", d_out, want, 1)
            del d_in, d_out, want
    finally:
        tc.debug_set_num_sms(0)
        tc.set_precision(PRECISIONS[DEFAULT_PRECISION])
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("prec", list(PRECISIONS))
def test_lattice_models_at_4096_are_bit_exact(w2x, tc, prec):
    """1 -> C1 -> C2 -> 1 lattice models through convert_plane_device at 4096^2, the last layer fused and separate; with
    C1 = 128 the first layer's record frame passes 2^32 bytes and each CTA runs about 500 tile-sets.  The inputs are those
    test_lattice_conditions_hold_on_the_small_planes checks."""
    W, H = MODEL_PLANE
    ext = Extension(W, H, m=3)
    f8, xh_only = _flags(prec)
    fails = []
    tc.set_precision(PRECISIONS[prec])
    try:
        for c1, c2 in MODEL_SHAPES if prec == DEFAULT_PRECISION else MODEL_SHAPES[:1]:
            m, tile = _model_case(c1, c2)
            model = w2x.Model.from_arrays([t[0] for t in m], [t[1] for t in m])
            x = periodic(tile, ext.h, ext.w)
            d_in = expand_on_device(tile, H, W)
            d_out = torch.empty((H, W), device="cuda")
            for fused in (True, False):
                want = ext.gather(torch.from_numpy(emulate_model(x, m, f8, fused, xh_only)).cuda())
                tc.debug_set_fuse_last(fused)
                d_out.fill_(math.nan)
                tc.convert_plane_device(model, d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
                _note_memory()
                _compare(fails, f"lattice 1-{c1}-{c2}-1 {prec} fused={fused} {W}x{H}", d_out, want, 3)
            del d_in, d_out
    finally:
        tc.debug_set_fuse_last(True)
        tc.set_precision(PRECISIONS[DEFAULT_PRECISION])
    assert not fails, "\n".join(fails)


# ---- 2. the benchmark's workloads with the shipped models, against the same context on the small plane --------------
def _tile(seed):
    return np.random.default_rng(seed).random((P, Q), dtype=F32)


def _small_reference(ctx, model, om, x, prec, ncpu):
    """the context's conversion of the small plane, held to the oracle"""
    small = ctx.convert_plane(model, x)
    err = float(np.abs(small - om.convert(x, n_job=ncpu)).max())
    assert err <= ORACLE_TOL[prec], (prec, err)
    return small


@pytest.mark.gpu
@pytest.mark.slow
def test_scale2x_at_4096_is_bit_exact(tc, shipped, oracle_models, ncpu):
    """bench.py's pass: scale2.0x on 4096^2 through the device entry (its `value`) in all three precisions and through the
    host entry (its `e2e`: the copy pipeline's bands) in the default one"""
    W, H = MODEL_PLANE
    ext = Extension(W, H, m=N_LAYERS)
    tile = _tile(41)
    x = periodic(tile, ext.h, ext.w)
    model, om = shipped["scale2.0x"], oracle_models["scale2.0x"]
    fails = []
    d_in = expand_on_device(tile, H, W)
    d_out = torch.empty((H, W), device="cuda")
    try:
        for prec in [DEFAULT_PRECISION] + [p for p in PRECISIONS if p != DEFAULT_PRECISION]:
            tc.set_precision(PRECISIONS[prec])
            want = ext.gather(torch.from_numpy(_small_reference(tc, model, om, x, prec, ncpu)).cuda())
            d_out.fill_(math.nan)
            tc.convert_plane_device(model, d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
            _note_memory()
            _compare(fails, f"scale2.0x {prec} {W}x{H} device", d_out, want, N_LAYERS)
            if prec == DEFAULT_PRECISION:
                got = tc.convert_plane(model, d_in.cpu().numpy())
                _note_memory()
                _compare(fails, f"scale2.0x {prec} {W}x{H} host", torch.from_numpy(got).cuda(), want, N_LAYERS)
    finally:
        tc.set_precision(PRECISIONS[DEFAULT_PRECISION])
    del d_in, d_out
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("name", ["noise1", "scale2.0x"])
def test_8192_plane_is_bit_exact(tc, shipped, oracle_models, ncpu, name):
    """config 4: one 8192^2 plane in the default precision, in scratch bands under the default 16 GiB limit and under a
    1 GiB one"""
    W, H = BIG_PLANE
    ext = Extension(W, H, m=N_LAYERS)
    tile = _tile(42 + len(name))
    want = ext.gather(torch.from_numpy(_small_reference(tc, shipped[name], oracle_models[name], periodic(tile, ext.h, ext.w),
                                                        DEFAULT_PRECISION, ncpu)).cuda())
    d_in = expand_on_device(tile, H, W)
    d_out = torch.empty((H, W), device="cuda")
    fails = []
    try:
        for limit in (0, 1 << 30):
            tc.set_scratch_limit(limit)
            d_out.fill_(math.nan)
            tc.convert_plane_device(shipped[name], d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
            _note_memory()
            _compare(fails, f"{name} {W}x{H} scratch_limit={limit}", d_out, want, N_LAYERS)
    finally:
        tc.set_scratch_limit(0)
    del d_in, d_out, want
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.slow
def test_64_tiles_of_512_are_bit_exact(tc, shipped, oracle_models, ncpu):
    """config 5: 64 noise2 tiles of 512^2 through convert_tiles (pipelined groups), each tile the extension of its own T;
    the small tiles go through convert_tiles too, two of them held to the oracle"""
    n, S = TILES
    ext = Extension(S, S, m=N_LAYERS)
    tiles = [_tile(1000 + t) for t in range(n)]
    small = tc.convert_tiles(shipped["noise2"], np.stack([periodic(t, ext.h, ext.w) for t in tiles]))
    for t in (0, n - 1):
        err = float(np.abs(small[t] - oracle_models["noise2"].convert(periodic(tiles[t], ext.h, ext.w), n_job=ncpu)).max())
        assert err <= F8_TOL, (t, err)
    got = tc.convert_tiles(shipped["noise2"], np.stack([periodic(t, S, S) for t in tiles]))
    _note_memory()
    fails = []
    _compare(fails, f"noise2 {n} tiles of {S}x{S}", torch.from_numpy(got), torch.from_numpy(ext.gather(small)), N_LAYERS)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.slow
def test_1080p_noise_scale_chain_is_bit_exact(tc, shipped, oracle_models, ncpu):
    """config 2: noise1, then 2x and scale2.0x on 1920 x 1080 through convert_chain and convert_chain_device (s = 2)"""
    W, H = CHAIN_PLANE
    ext = Extension(W, H, m=2 * N_LAYERS, s=2)
    steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
    tile = _tile(43)
    x = periodic(tile, ext.h, ext.w)
    small = tc.convert_chain(steps, x)
    d = oracle_models["noise1"].convert(x, n_job=ncpu)
    ref = oracle_models["scale2.0x"].convert(np.ascontiguousarray(np.repeat(np.repeat(d, 2, axis=0), 2, axis=1)), n_job=ncpu)
    err = float(np.abs(small - ref).max())
    assert err <= 1.5 * F8_TOL, err                                   # two passes, as tests/test_gpu_parity_large.py
    want = ext.gather(torch.from_numpy(small).cuda())
    fails = []
    got = tc.convert_chain(steps, periodic(tile, H, W))
    _note_memory()
    _compare(fails, f"noise1+scale2.0x {W}x{H} convert_chain", torch.from_numpy(got).cuda(), want, N_LAYERS)
    d_in = expand_on_device(tile, H, W)
    d_out = torch.full((2 * H, 2 * W), math.nan, device="cuda")
    tc.convert_chain_device(steps, d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), 2 * W * 4)
    _note_memory()
    _compare(fails, f"noise1+scale2.0x {W}x{H} convert_chain_device", d_out, want, N_LAYERS)
    assert not fails, "\n".join(fails)


# ---- 3. the fp32 engine, against its emulator ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.slow
def test_fp32_engine_at_4096_is_bit_exact(w2x, shipped, oracle_models):
    """scale2.0x on 4096^2 on the fp32 engine, under the default scratch limit and in bands under a 1 GiB one, against
    fp32_convert of the small plane (run with torch on the GPU)"""
    W, H = MODEL_PLANE
    ext = Extension(W, H, m=N_LAYERS)
    tile = _tile(44)
    om = oracle_models["scale2.0x"]
    want = ext.gather(fp32_convert_t(periodic(tile, ext.h, ext.w), om.weights, om.biases, "cuda"))
    d_in = expand_on_device(tile, H, W)
    d_out = torch.empty((H, W), device="cuda")
    fails = []
    ctx = w2x.Context(0, engine=w2x.ENGINE_FP32)
    try:
        for limit in (0, 1 << 30):
            ctx.set_scratch_limit(limit)
            d_out.fill_(math.nan)
            ctx.convert_plane_device(shipped["scale2.0x"], d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
            _note_memory()
            _compare(fails, f"fp32 engine scale2.0x {W}x{H} scratch_limit={limit}", d_out, want, N_LAYERS)
    finally:
        ctx.close()
    del d_in, d_out, want
    torch.cuda.empty_cache()
    assert not fails, "\n".join(fails)
