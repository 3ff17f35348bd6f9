"""Planes, bands, slabs, tile batches and filter layers on both sides of the frame-row limit.

The CUDA-core kernels at the edges of the tensor-core engine (the first layer, the separate last layer, the gathers, the pack)
tile a frame in 32 x 8-pixel blocks on grid.y <= 65535, so a frame may have at most 8 * 65535 = 524280 rows.  Every driver
must cut taller work into frames within that limit (scratch bands, tile groups, slab sub-bands), refuse a band session it
cannot run before anything is queued, and the fp32 kernels must cover any height.

The model is test_edge_exact's selection model 1 -> 32 -> 64 -> 32 -> 1 (n = 4 layers, a frame is h + 8 rows): its output has
exactly one correct bit pattern, given by emulate_tc_model in both precisions and by fp32_convert on the fp32 engine.  A 10^6-row
plane is too large to emulate whole, so rows [a, b) are compared with the emulator run on input rows [a - n, b + n) (less at the
image border): an output row depends on input rows within n of it only, which test_window_identity checks on the CPU.  The
windows sit at the top, the bottom, every seam a driver here chooses and frame row 524280; every row is compared, bit for bit,
with one run of the same engine at a small scratch limit (bands of 100 000 rows), which the windows check as well.
"""
import ctypes as C
import itertools
import math

import numpy as np
import pytest
import torch

from exact_arith import F32, fp32_convert, fp32_filter, mul32, readback
from test_edge_exact import (PRECISIONS, _geometry_model, _mismatch, assert_selection, emulate_selection, emulate_tc_model,
                             ordinary_planes, plane_for, selection_layer, selection_report)
from test_gpu_parity import F8_TOL

LIMIT = 8 * 65535                        # rows a frame may have
LAYERS = _geometry_model()
N = len(LAYERS)                          # 4
MAXC = 64
HEIGHTS = [LIMIT - 2 * N, LIMIT - 2 * N + 1, 1_100_000]     # the tallest one-frame plane, the first that needs two, three bands
WIDTHS = [1, 5]
SMALL_BAND = 100_000                     # rows per band of the reference run
HALO = N + 3                             # rows of real context around the convert_band_device bands
FILTER_H = LIMIT + 20                    # row blocks 65535.. of the fp32 kernels run in their second pass


# ---------------------------------------------------------------------------------------------------------------------
# inputs, windows and emulators
# ---------------------------------------------------------------------------------------------------------------------
def tall_plane(h, w, salt=0):
    """uniform noise (w = 1) or a smooth u8 / 255 image (w = 5)"""
    return plane_for(h, w, (1 if w == 1 else 2) + 2 * salt)


def tc_em(prec):
    f8 = prec != "f16x3"
    return lambda p: emulate_tc_model(p, LAYERS, f8, True)[0]


def fp32_em(p):
    return fp32_convert(p, [t[0] for t in LAYERS], [t[1] for t in LAYERS])


def window_input(x, a, b, n=N):
    """the input rows output rows [a, b) depend on, and where row a lies in them"""
    lo, hi = max(0, a - n), min(x.shape[0], b + n)
    return x[lo:hi], a - lo


def window_want(em, x, a, b, n=N):
    xi, k = window_input(x, a, b, n)
    return em(xi)[k:k + b - a]


def seams(h):
    """every output row at which some driver below starts a band, sub-band or block, and frame row LIMIT of a whole frame"""
    s = set(range(LIMIT - 2 * N, h, LIMIT - 2 * N))           # scratch bands at the default limit
    s |= {h * i // 4 for i in (1, 2, 3)}                       # host copy bands, slab sub-bands (n_sub = 4)
    s |= {h * i // 3 for i in (1, 2)}                          # slab sub-bands (n_sub = 3)
    s |= {504, (h - 1) // 504 * 504}                           # the literal walk's first and last block seams (512 - 2n)
    s.add(LIMIT - N)
    return s


def windows(h, centres, half):
    out = []
    for c in sorted({0, h} | set(centres)):
        a, b = max(0, c - half), min(h, c + half)
        if a < b and (a, b) not in out:
            out.append((a, b))
    return out


def tc_windows(h):
    return windows(h, seams(h) | set(range(SMALL_BAND, h, SMALL_BAND)), 12)


def fp32_windows(h):
    """fewer and shorter: the fp32 emulator is slow"""
    return windows(h, {s for s in seams(h) if s % (LIMIT - 2 * N) == 0 or s in (LIMIT - N, h // 4, h // 2)}, 6)


def band_windows(h):
    """output rows of a convert_band_device band: its ends and the scratch-band seams"""
    return windows(h, set(range(LIMIT - 2 * N, h, LIMIT - 2 * N)), 6)


def tile_pool(prec):
    """1 x 1 tiles: 512 values and their emulated outputs (a 1 x 1 tile's output depends only on its value)"""
    vals = np.random.default_rng(77).random(512, dtype=F32)
    em = tc_em(prec)
    return vals, np.array([em(np.full((1, 1), v, F32))[0, 0] for v in vals], F32)


def tile_pool_3x2(prec):
    tiles = np.stack([plane_for(2, 3, 40 + k) for k in range(48)])
    em = tc_em(prec)
    return tiles, np.stack([em(t) for t in tiles])


def tc_filter_case(seed=5):
    w, b = selection_layer(32, 32, 1, seed)
    return w, b, ordinary_planes(32, FILTER_H, 1, seed)


def filter_windows():
    return [(0, 8), (LIMIT - 8, LIMIT + 8), (FILTER_H - 8, FILTER_H)]


def filter_input(x, a, b):
    """the input rows of filter_layer's output rows [a, b) (one row of context), and where row a lies in them"""
    lo, hi = max(0, a - 1), min(x.shape[1], b + 1)
    return x[:, lo:hi], a - lo


def tc_filter_inputs(x):
    """what the selection layer reads for each window: activations * 16 with the replicate ring"""
    for a, b in filter_windows():
        yield mul32(np.pad(filter_input(x, a, b)[0], ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w", [1, 5, 20])
def test_window_identity(w):
    """every window of 1, 3 and 8 output rows, emulated on its input rows with n rows of context (less at the border),
    equals the whole plane's rows bit for bit, for both tensor-core emulators and the fp32 one; with n - 1 rows of context
    some window differs, so n is what the identity needs"""
    h = 16
    x = plane_for(h, w, w)
    for name, em in [("f16x3", tc_em("f16x3")), ("f16+f8x2", tc_em("f16+f8x2")), ("fp32", fp32_em)]:
        whole = em(x)
        for k in ((1, 3, 8) if name != "fp32" else (8,)):       # the fp32 emulator is slow
            for a in range(0, h - k + 1):
                got = window_want(em, x, a, a + k)
                assert np.array_equal(got, whole[a:a + k]), (name, w, a, a + k, _mismatch(got, whole[a:a + k]))
        assert any(not np.array_equal(window_want(em, x, a, a + 8, N - 1), whole[a:a + 8]) for a in range(1, h - 8)), name


def _window_inputs():
    """every input a tensor-core window below is emulated on"""
    for w in WIDTHS:
        for h in HEIGHTS:
            x = tall_plane(h, w)
            for a, b in tc_windows(h):
                yield window_input(x, a, b)[0]
            xe = tall_plane(h + 2 * HALO, w, 1)
            for a, b in band_windows(h):
                yield window_input(xe, a + HALO, b + HALO)[0]
    for v in tile_pool("f16x3")[0]:
        yield np.full((1, 1), v, F32)
    yield from tile_pool_3x2("f16x3")[0]


@pytest.mark.parametrize("prec", PRECISIONS)
def test_selection_conditions_hold_on_every_window(prec):
    f8 = prec != "f16x3"
    count = 0
    for x in _window_inputs():
        for xr, w, b in emulate_tc_model(x, LAYERS, f8, True)[1]:
            assert_selection(selection_report(xr, w, b, f8))
            count += 1
    w, b, x = tc_filter_case()
    for xr in tc_filter_inputs(x):
        assert_selection(selection_report(xr, w, b, f8))
    assert count > 1000


def test_limits_of_the_cases():
    """the heights and tile counts below sit on the two sides of the limit"""
    assert HEIGHTS[0] + 2 * N == LIMIT and HEIGHTS[1] + 2 * N == LIMIT + 1
    assert LIMIT // (1 + 2 * N) == 58253 and LIMIT // (2 + 2 * N) == 52428
    assert FILTER_H > LIMIT and math.ceil(HEIGHTS[2] / (LIMIT - 2 * N)) == 3


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model(w2x):
    return w2x.Model.from_arrays([t[0] for t in LAYERS], [t[1] for t in LAYERS])


@pytest.fixture(scope="module")
def engines(w2x):
    c = {}
    for p, prec in zip(PRECISIONS, (w2x.PRECISION_F16X3, w2x.PRECISION_F16_F8X2)):
        c[p] = w2x.Context(0, engine=w2x.ENGINE_TC)
        c[p].set_precision(prec)
    c["fp32"] = w2x.Context(0, engine=w2x.ENGINE_FP32)
    yield c
    for v in c.values():
        v.close()


def device_convert(ctx, model, x, **kw):
    h, w = x.shape
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_out = torch.empty_like(d_in)
    torch.cuda.synchronize()
    ctx.convert_plane_device(model, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), w * 4, **kw)
    ctx.synchronize()
    return d_out.cpu().numpy()


def small_scratch_run(ctx, model, x, maxc=MAXC, n=N):
    """convert_plane_device in scratch bands of SMALL_BAND rows"""
    ctx.set_scratch_limit(maxc * (x.shape[1] + 2 * n) * 4 * (SMALL_BAND + 2 * n))
    try:
        return device_convert(ctx, model, x)
    finally:
        ctx.set_scratch_limit(0)


class Checker:
    """compares outputs with the emulator in windows (cached per input) and with a whole reference output"""

    def __init__(self, em):
        self.em, self.cache, self.fails = em, {}, []

    def windows(self, name, got, x, wins, off=0):
        for a, b in wins:
            key = (id(x), a + off, b + off)
            if key not in self.cache:
                self.cache[key] = window_want(self.em, x, a + off, b + off)
            if not np.array_equal(got[a:b], self.cache[key]):
                self.fails.append(f"{name}: rows [{a}, {b}): {_mismatch(got[a:b], self.cache[key])}")

    def whole(self, name, got, ref):
        if not np.array_equal(got, ref):
            self.fails.append(f"{name}: whole output: {_mismatch(got, ref)}")

    def done(self):
        assert not self.fails, "\n".join(self.fails)


def plane_entry_points(w2x, ctx, model, em, wins, w, h):
    """convert_plane_device, convert_plane with one and with the default host bands, convert_band_device with halos of n and
    n + 3 rows, and both block walks on a plane the reference splits (default 512 x 512 blocks), with their progress lines"""
    chk = Checker(em)
    x = tall_plane(h, w)
    ref = small_scratch_run(ctx, model, x)
    chk.windows("small scratch limit", ref, x, wins)
    got = device_convert(ctx, model, x)
    chk.windows("convert_plane_device", got, x, wins)
    chk.whole("convert_plane_device", got, ref)
    try:
        for nb in (1, 0):
            ctx.debug_set_host_bands(nb)
            got = ctx.convert_plane(model, x)
            chk.windows(f"convert_plane host bands={nb}", got, x, wins)
            chk.whole(f"convert_plane host bands={nb}", got, ref)
    finally:
        ctx.debug_set_host_bands(0)
    xe = tall_plane(h + 2 * HALO, w, 1)
    ref_e = small_scratch_run(ctx, model, xe)[HALO:HALO + h]
    d_in = torch.from_numpy(xe).cuda()
    torch.cuda.synchronize()
    for halo in (N, HALO):
        out = torch.empty((h, w), device="cuda")
        ctx.convert_band_device(model, d_in[HALO - halo:].data_ptr(), w, h, halo, halo, w * 4, out.data_ptr(), w * 4)
        ctx.synchronize()
        got = out.cpu().numpy()
        chk.windows(f"convert_band_device halo={halo}", got, xe, band_windows(h), off=HALO)
        chk.whole(f"convert_band_device halo={halo}", got, ref_e)
    del d_in
    assert w2x.requires_splitting(w, h)
    n_blocks = len(w2x.block_table(w, h, N)[0])
    lines = []
    ctx.set_log(lines.append)
    try:
        for walk in (w2x.WALK_BLOCKS, w2x.WALK_FUSED):
            ctx.set_block_walk(walk)
            lines.clear()
            got = ctx.convert_plane(model, x)
            chk.windows(f"walk={walk}", got, x, wins)
            chk.whole(f"walk={walk}", got, ref)
            starts = sum(line.startswith("start process block") for line in lines)
            if starts != n_blocks or len(lines) != n_blocks * (N + 1):
                chk.fails.append(f"walk={walk}: {starts} block lines, {len(lines)} lines for {n_blocks} blocks")
    finally:
        ctx.set_block_walk(w2x.WALK_FUSED)
        ctx.set_log(None)
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("prec", PRECISIONS)
def test_tc_plane_entry_points(w2x, engines, model, prec, w, h):
    plane_entry_points(w2x, engines[prec], model, tc_em(prec), tc_windows(h), w, h)


@pytest.mark.gpu
@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("w", WIDTHS)
def test_fp32_plane_entry_points(w2x, engines, model, w, h):
    plane_entry_points(w2x, engines["fp32"], model, fp32_em, fp32_windows(h), w, h)


@pytest.mark.gpu
@pytest.mark.parametrize("h", HEIGHTS)
def test_planes_with_a_tall_plane(w2x, engines, model, h):
    """convert_planes and convert_planes_device on [a tall plane, small ones]: each plane equals convert_plane_device of that
    plane, and the progress lines are the single-plane calls' lines"""
    ctx = engines["f16+f8x2"]
    planes = [tall_plane(h, 5)] + [plane_for(hh, ww, 30 + k) for k, (ww, hh) in enumerate([(1, 1), (7, 3), (40, 17), (5, 60)])]
    lines = []
    ctx.set_log(lines.append)
    try:
        want, dev_lines, host_lines = [], [], []
        for x in planes:
            lines.clear()
            want.append(device_convert(ctx, model, x, block_splitting=False))
            dev_lines += lines
            lines.clear()
            ctx.convert_plane(model, x, block_splitting=False)
            host_lines += lines
        assert len(dev_lines) == N * (math.ceil(h / (LIMIT - 2 * N)) + len(planes) - 1)
        lines.clear()
        got = ctx.convert_planes(model, planes)
        assert lines == host_lines
        bad = [k for k in range(len(planes)) if not np.array_equal(got[k], want[k])]
        assert not bad, ("host", bad)
        d_in = [torch.from_numpy(x).cuda() for x in planes]
        d_out = [torch.empty_like(d) for d in d_in]
        torch.cuda.synchronize()
        lines.clear()
        ctx.convert_planes_device(model, [d.data_ptr() for d in d_in], [x.shape[1] for x in planes], [x.shape[0] for x in planes],
                                  [x.shape[1] * 4 for x in planes], [d.data_ptr() for d in d_out], [x.shape[1] * 4 for x in planes])
        ctx.synchronize()
        assert lines == dev_lines
        bad = [k for k in range(len(planes)) if not np.array_equal(d_out[k].cpu().numpy(), want[k])]
        assert not bad, ("device", bad)
    finally:
        ctx.set_log(None)


def tiles_async(w2x, ctx, model, tiles):
    n, th, tw = tiles.shape
    out = np.empty_like(tiles)
    ip = (C.c_void_p * n)(*range(tiles.ctypes.data, tiles.ctypes.data + n * tiles.strides[0], tiles.strides[0]))
    op = (C.c_void_p * n)(*range(out.ctypes.data, out.ctypes.data + n * out.strides[0], out.strides[0]))
    L = w2x.lib()
    rc = L.w2x_convert_tiles_async(ctx._h, model._h, ip, op, n, tw, th, tw * 4, tw * 4)
    if rc:
        raise w2x.W2xError(rc, L.w2x_last_error().decode())
    ctx.synchronize()
    return out


def frames_for(n_tiles, th):
    return math.ceil(n_tiles / (LIMIT // (th + 2 * N)))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_tiles_across_the_limit(w2x, engines, model, prec):
    """convert_tiles_device, convert_tiles_async and host convert_tiles on 1 x 1 tiles (58253 per frame) and 3 x 2 tiles (52428
    per frame) on both sides of a frame's capacity, and a host batch whose groups of a quarter each pass the limit: every
    tile against the emulator and against convert_planes_device, and (n + 1) launches per frame"""
    ctx = engines[prec]
    rng = np.random.default_rng(3)
    fails = []
    vals, vout = tile_pool(prec)
    tiles3, tout3 = tile_pool_3x2(prec)
    cases = []
    for n_tiles in (58253, 58254):
        idx = rng.integers(0, len(vals), n_tiles)
        cases.append((f"1x1 n={n_tiles}", vals[idx].reshape(-1, 1, 1), vout[idx].reshape(-1, 1, 1)))
    for n_tiles in (52428, 52429):
        idx = rng.integers(0, len(tiles3), n_tiles)
        cases.append((f"3x2 n={n_tiles}", tiles3[idx], tout3[idx]))
    for name, tiles, want in cases:
        n_tiles, th, tw = tiles.shape
        d_in = torch.from_numpy(tiles).cuda()
        d_out, d_out2 = torch.empty_like(d_in), torch.empty_like(d_in)
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        ctx.convert_tiles_device(model, d_in.data_ptr(), d_out.data_ptr(), n_tiles, tw, th)
        ctx.synchronize()
        if ctx.launch_count() - n0 != (N + 1) * frames_for(n_tiles, th):
            fails.append(f"{name} device: {ctx.launch_count() - n0} launches")
        got = d_out.cpu().numpy()
        if not np.array_equal(got, want):
            fails.append(f"{name} device: {_mismatch(got, want)}")
        n0 = ctx.launch_count()
        got = tiles_async(w2x, ctx, model, tiles)
        if ctx.launch_count() - n0 != (N + 1) * frames_for(n_tiles, th):
            fails.append(f"{name} async: {ctx.launch_count() - n0} launches")
        if not np.array_equal(got, want):
            fails.append(f"{name} async: {_mismatch(got, want)}")
        step = th * tw * 4
        ctx.convert_planes_device(model, list(range(d_in.data_ptr(), d_in.data_ptr() + n_tiles * step, step)), [tw] * n_tiles,
                                  [th] * n_tiles, [tw * 4] * n_tiles, list(range(d_out2.data_ptr(), d_out2.data_ptr() + n_tiles * step, step)),
                                  [tw * 4] * n_tiles)
        ctx.synchronize()
        got = d_out2.cpu().numpy()
        if not np.array_equal(got, want):
            fails.append(f"{name} convert_planes_device: {_mismatch(got, want)}")
        del d_in, d_out, d_out2
    # host: four groups of 60000 1 x 1 tiles, each group two frames
    n_tiles = 240_000
    idx = rng.integers(0, len(vals), n_tiles)
    n0 = ctx.launch_count()
    got = ctx.convert_tiles(model, vals[idx].reshape(-1, 1, 1))
    groups = [n_tiles * (g + 1) // 4 - n_tiles * g // 4 for g in range(4)]
    if ctx.launch_count() - n0 != (N + 1) * sum(frames_for(k, 1) for k in groups) or min(groups) <= 58253:
        fails.append(f"host 1x1 n={n_tiles}: {ctx.launch_count() - n0} launches")
    if not np.array_equal(got, vout[idx].reshape(-1, 1, 1)):
        fails.append(f"host 1x1 n={n_tiles}: {_mismatch(got, vout[idx].reshape(-1, 1, 1))}")
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_fp32_filter_layer_past_the_limit(w2x, engines):
    """filter_layer of FILTER_H rows on the fp32 engine (conv3x3_planar_fp32 with 4 and 32 output planes per block) against
    fp32_filter in windows: the top, frame row LIMIT (the second pass of the row-block loop) and the bottom"""
    ctx = engines["fp32"]
    fails = []
    for k, (cin, cout, wd) in enumerate([(3, 5, 5), (8, 33, 1)]):
        rng = np.random.default_rng(k)
        w = (rng.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(F32)
        b = (rng.standard_normal(cout) * 0.1).astype(F32).astype(np.float64)
        x = ordinary_planes(cin, FILTER_H, wd, seed=k)
        got = ctx.filter_layer(w2x.Model.from_arrays([w], [b]), 0, x)
        for a, c in filter_windows():
            xi, k = filter_input(x, a, c)
            want = fp32_filter(xi, w, b)[:, k:k + c - a]
            if not np.array_equal(got[:, a:c], want):
                fails.append(f"{cin}->{cout} rows [{a}, {c}): {_mismatch(got[:, a:c], want)}")
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_tc_filter_layer_past_the_limit(w2x, engines, prec):
    """filter_layer of FILTER_H rows on the tensor-core engine (planar_to_nhwc, a 32 -> 32 selection layer, nhwc_to_planar)
    against emulate_selection in windows"""
    ctx, f8 = engines[prec], prec != "f16x3"
    w, b, x = tc_filter_case()
    got = ctx.filter_layer(w2x.Model.from_arrays([w], [b]), 0, x)
    fails = []
    for (a, c), xr in zip(filter_windows(), tc_filter_inputs(x)):
        k = filter_input(x, a, c)[1]
        want = readback(emulate_selection(xr, w, b, f8), f8)[:, k:k + c - a]
        if not np.array_equal(got[:, a:c], want):
            fails.append(f"rows [{a}, {c}): {_mismatch(got[:, a:c], want)}")
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_band_session_at_the_limit(w2x, engines, model, prec):
    """an unconnected Band session whose frame has exactly LIMIT rows: load, steps, finish"""
    ctx = engines[prec]
    h = LIMIT - 2 * N
    x = tall_plane(h, 1)
    d_in = torch.from_numpy(x).cuda()
    out = torch.empty_like(d_in)
    torch.cuda.synchronize()
    band = w2x.Band(ctx, model, 1, h, False, False)
    try:
        band.load(d_in.data_ptr(), 4)
        for k in range(band.steps):
            band.step(k)
        band.finish(out.data_ptr(), 4)
        ctx.synchronize()
    finally:
        band.close()
    chk = Checker(tc_em(prec))
    got = out.cpu().numpy()
    chk.windows("band session", got, x, tc_windows(h))
    chk.whole("band session", got, small_scratch_run(ctx, model, x))
    chk.done()


@pytest.mark.gpu
def test_band_create_refuses_frames_past_the_limit(w2x, engines, model):
    """for every pair of edge kinds, a band one row taller than its frame allows is refused with W2X_ERR_ARG, naming the limit,
    before any device memory is taken"""
    ctx = engines["f16+f8x2"]
    ctx.synchronize()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for up, down in itertools.product((0, 1, 2), repeat=2):
        rows = LIMIT - (1 if up == 1 else N) - (1 if down == 1 else N) + 1
        with pytest.raises(w2x.W2xError) as e:
            w2x.Band(ctx, model, 1, rows, up, down)
        assert e.value.status == 1 and str(LIMIT) in e.value.message, (up, down, e.value)
    assert torch.cuda.mem_get_info()[0] == free0


@pytest.mark.gpu
def test_slab_raises_n_sub(w2x, engines, model):
    """an unconnected Slab of 1.1 million rows asked for one sub-band runs as three"""
    ctx = engines["f16+f8x2"]
    h, w = HEIGHTS[2], 5
    x = tall_plane(h, w)
    out = np.empty_like(x)
    slab = w2x.Slab(ctx, model, w, h, False, False, n_sub=1)
    try:
        slab.convert(x, out)
    finally:
        slab.close()
    chk = Checker(tc_em("f16+f8x2"))
    chk.windows("slab", out, x, tc_windows(h))
    chk.whole("slab", out, small_scratch_run(ctx, model, x))
    chk.done()


@pytest.mark.gpu
def test_shipped_model_one_row_past_the_limit(w2x, oracle_models):
    """scale2.0x (n = 7) in the default precision on a 1 x 524267 plane (frame LIMIT + 1 rows) through convert_plane_device:
    windows within F8_TOL of the CPU oracle, every row equal to a small-scratch-limit run"""
    om = oracle_models["scale2.0x"]
    model = w2x.Model.from_arrays(om.weights, om.biases)
    n = len(om.weights)
    h = LIMIT - 2 * n + 1
    x = plane_for(h, 1, 9)
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        got = device_convert(ctx, model, x)
        ref = small_scratch_run(ctx, model, x, maxc=128, n=n)
    finally:
        ctx.close()
    errs = []
    for a, b in windows(h, {LIMIT - 2 * n, LIMIT - n, SMALL_BAND}, 12):
        xi, k = window_input(x, a, b, n)
        errs.append(float(np.abs(got[a:b] - om.convert(xi, n_job=4)[k:k + b - a]).max()))
    assert max(errs) <= F8_TOL, errs
    assert np.array_equal(got, ref), _mismatch(got, ref)
