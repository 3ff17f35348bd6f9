"""The progress lines (w2x_ctx_set_log) of every conversion entry point, computed here from w2x.block_table and the rules below
and compared with what the library prints.  A plane, as w2x_convert_plane or w2x_convert_plane_device converts it, gets:

  1. when block splitting is on and the reference would split it: per block of block_table, "start process block (c,r) ..." and
     "Iteration #1..." to "#n";
  2. otherwise, from host memory through w2x_convert_plane's copy pipeline cut into bands: "Iteration #1..#n" once;
  3. otherwise: "Iteration #1..#n" once per scratch band of the plane.

w2x_convert_planes* print each plane's lines in order, as the single-plane call with block splitting off; w2x_convert_chain* print
on_step(k) and then step k's plane lines; the tiles calls print "Iteration #1..#n" per packed frame, or per tile when frames are not
packed.  A call rejected by its argument checks prints no line and launches nothing.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_UNSUPPORTED = 1, 7
STEP_FN = C.CFUNCTYPE(None, C.c_int, C.c_void_p)
FRAME_ROWS = 8 * 65535
ENGINES = ["tc", "fp32"]
WALKS = ["fused", "blocks"]
# regime -> plane size (w, h), block size, host copy bands, scratch limit in rows of the widest 128-channel activation
REGIMES = {
    "plain": ((40, 30), None, 0, None),
    "split": ((120, 100), (64, 64), 0, None),
    "host_bands": ((60, 90), None, 3, None),
    "scratch": ((50, 100), None, 0, 40),
}


def its(n):
    return [f"Iteration #{k}..." for k in range(1, n + 1)]


def max_channels(model):
    return max(max(model.dims(i)[:2]) for i in range(len(model)))


class Settings:
    """what the lines depend on besides the plane: the context's scratch limit and host copy bands"""

    def __init__(self, limit=16 << 30, host_bands=0):
        self.limit, self.host_bands = limit, host_bands

    def host_copy_bands(self, n, h):
        nb = min(self.host_bands if self.host_bands > 0 else min(4, h // 512), 8)
        return 1 if nb < 2 or h // nb < 2 * n else nb

    def scratch_band_rows(self, model, w, h):
        n = len(model)
        per_row = max_channels(model) * (w + 2 * n) * 4
        return min(h, max(16, min(self.limit // per_row, FRAME_ROWS) - 2 * n))

    def plane_lines(self, w2x, model, w, h, block_splitting, host):
        n = len(model)
        if block_splitting and w2x.requires_splitting(w, h):
            tab, _, _ = w2x.block_table(w, h, n)
            return [line for r, c in tab[:, :2] for line in [f"start process block ({c},{r}) ..."] + its(n)]
        if host and self.host_copy_bands(n, h) > 1:
            return its(n)
        return its(n) * math.ceil(h / self.scratch_band_rows(model, w, h))

    def tile_frames(self, model, n_tiles, w, h, packed):
        if not packed:
            return n_tiles
        n = len(model)
        per_tile = max_channels(model) * (w + 2 * n) * (h + 2 * n) * 4
        group = max(1, min(n_tiles, self.limit // per_tile, FRAME_ROWS // (h + 2 * n)))
        return math.ceil(n_tiles / group)


@pytest.fixture(scope="module")
def models(w2x, oracle_models):
    ms = {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}
    rng = np.random.default_rng(5)

    def random_model(chans):
        ws = [rng.normal(0, 0.3, (co, ci, 3, 3)).astype(np.float32) for ci, co in zip(chans, chans[1:])]
        return w2x.Model.from_arrays(ws, [rng.normal(0, 0.1, co) for co in chans[1:]])
    ms["one_to_two"] = random_model([1, 32, 64, 2])
    ms["no_tc"] = random_model([1, 8, 16, 1])     # the tensor-core engine needs 1 -> {32,64,128}... -> 1
    return ms


@pytest.fixture
def ctx(w2x):
    c = w2x.Context(0)
    yield c
    c.set_log(None)
    c.close()
    w2x.set_block_size(512, 512)


def setup_ctx(w2x, ctx, engine, walk, regime, model):
    (w, h), block, host_bands, limit_rows = REGIMES[regime]
    ctx.set_engine(w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    ctx.set_block_walk(w2x.WALK_BLOCKS if walk == "blocks" else w2x.WALK_FUSED)
    s = Settings(host_bands=host_bands)
    ctx.debug_set_host_bands(host_bands)
    if limit_rows is not None:
        s.limit = max_channels(model) * (w + 2 * len(model)) * 4 * limit_rows
        ctx.set_scratch_limit(s.limit)
    if block is not None:
        w2x.set_block_size(*block)
    return w, h, s


def dev(x):
    d = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    torch.cuda.synchronize()
    return d


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("walk", WALKS)
@pytest.mark.parametrize("engine", ENGINES)
def test_plane_entry_points(w2x, ctx, models, engine, walk, regime):
    model = models["noise2"]
    w, h, s = setup_ctx(w2x, ctx, engine, walk, regime, model)
    n = len(model)
    rng = np.random.default_rng(1)
    x = rng.random((h, w), dtype=np.float32)
    got = []
    ctx.set_log(got.append)

    def check(name, want, call):
        got.clear()
        call()
        ctx.synchronize()
        assert got == want, name

    for bs in (True, False):
        check(f"plane bs={bs}", s.plane_lines(w2x, model, w, h, bs, True), lambda: ctx.convert_plane(model, x, block_splitting=bs))
        d_in, d_out = dev(x), dev(np.zeros_like(x))
        check(f"plane_device bs={bs}", s.plane_lines(w2x, model, w, h, bs, False),
              lambda: ctx.convert_plane_device(model, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), w * 4, block_splitting=bs))

    a, b = h // 4, h - h // 4                       # a band with n real rows of context on both sides
    assert a >= n
    d_in, d_out = dev(x), dev(np.zeros_like(x))
    check("band_device", s.plane_lines(w2x, model, w, b - a, False, False),
          lambda: ctx.convert_band_device(model, d_in.data_ptr() + (a - n) * w * 4, w, b - a, n, n, w * 4, d_out.data_ptr(), w * 4))

    planes = [x, rng.random((9, 17), dtype=np.float32), rng.random((40, 5), dtype=np.float32)]
    for host in (True, False):
        want = [line for p in planes for line in s.plane_lines(w2x, model, p.shape[1], p.shape[0], False, host)]
        if host:
            check("planes", want, lambda: ctx.convert_planes(model, planes))
        else:
            d_in = [dev(p) for p in planes]
            d_out = [dev(np.zeros_like(p)) for p in planes]
            ws, hs = [p.shape[1] for p in planes], [p.shape[0] for p in planes]
            check("planes_device", want, lambda: ctx.convert_planes_device(model, [d.data_ptr() for d in d_in], ws, hs, [v * 4 for v in ws],
                                                                           [d.data_ptr() for d in d_out], [v * 4 for v in ws]))

    # a noise step on the half-size plane, then an upscaling step back to (about) the regime's size
    steps = [(models["noise1"], False), (models["scale2.0x"], True)]
    x0 = x[: h // 2, : w // 2]
    h0, w0 = x0.shape
    if regime == "split":
        assert not w2x.requires_splitting(w0, h0) and w2x.requires_splitting(2 * w0, 2 * h0)
    for bs in (True, False):
        for host in (True, False):
            want = [("step", 0)] + s.plane_lines(w2x, steps[0][0], w0, h0, bs, host)
            want += [("step", 1)] + s.plane_lines(w2x, steps[1][0], 2 * w0, 2 * h0, bs, host)
            on_step = lambda k: got.append(("step", k))
            if host:
                check(f"chain bs={bs}", want, lambda: ctx.convert_chain(steps, x0, block_splitting=bs, on_step=on_step))
            else:
                d_in, d_out = dev(x0), dev(np.zeros((2 * h0, 2 * w0), np.float32))
                check(f"chain_device bs={bs}", want, lambda: ctx.convert_chain_device(steps, d_in.data_ptr(), w0, h0, w0 * 4, d_out.data_ptr(),
                                                                                      2 * w0 * 4, block_splitting=bs, on_step=on_step))


def tiles_async(w2x, ctx, model, tiles, out):
    n, th, tw = tiles.shape
    ip = (C.c_void_p * n)(*[tiles[i].ctypes.data for i in range(n)])
    op = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    rc = w2x.lib().w2x_convert_tiles_async(ctx._h, model._h, ip, op, n, tw, th, tw * 4, tw * 4)
    if rc:
        raise w2x.W2xError(rc, w2x.lib().w2x_last_error().decode())


@pytest.mark.parametrize("frames", ["one", "several"])
@pytest.mark.parametrize("engine", ENGINES)
def test_tiles(w2x, ctx, models, engine, frames):
    """10 tiles: the host call runs them as 2 copy groups of 5; a small scratch limit packs 2 tiles per frame"""
    model = models["noise2"]
    n = len(model)
    n_tiles, T = 10, 16
    ctx.set_engine(w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    s = Settings()
    if frames == "several":
        s.limit = 2 * max_channels(model) * (T + 2 * n) ** 2 * 4
        ctx.set_scratch_limit(s.limit)
    packed = engine == "tc"
    assert s.tile_frames(model, n_tiles, T, T, packed) == (n_tiles if not packed else 1 if frames == "one" else 5)
    tiles = np.random.default_rng(2).random((n_tiles, T, T), dtype=np.float32)
    got = []
    ctx.set_log(got.append)
    host_frames = sum(s.tile_frames(model, 5, T, T, packed) for _ in range(2))
    ctx.convert_tiles(model, tiles)
    assert got == its(n) * host_frames, "host"
    got.clear()
    out = np.empty_like(tiles)
    tiles_async(w2x, ctx, model, tiles, out)
    ctx.synchronize()
    assert got == its(n) * s.tile_frames(model, n_tiles, T, T, packed), "async"
    got.clear()
    d_in, d_out = dev(tiles), dev(np.zeros_like(tiles))
    ctx.convert_tiles_device(model, d_in.data_ptr(), d_out.data_ptr(), n_tiles, T, T)
    ctx.synchronize()
    assert got == its(n) * s.tile_frames(model, n_tiles, T, T, packed), "device"


def plane_calls(w2x, ctx, model, x, null):
    """every plane entry point on x, with a NULL input pointer when `null`; each returns the library's status"""
    L = w2x.lib()
    h, w = x.shape
    out = np.zeros((2 * h, 2 * w), np.float32)
    d_in, d_out = dev(x), dev(out)
    xp = None if null else x.ctypes.data
    dp = None if null else d_in.data_ptr()
    n = len(model)
    pi, ps, pp = C.c_int * 1, C.c_size_t * 1, C.c_void_p * 1
    steps = (C.c_void_p * 1)(model._h)
    same = (C.c_int * 1)(w2x.STEP_SAME)
    return {
        "plane": lambda: L.w2x_convert_plane(ctx._h, model._h, xp, w, h, w * 4, out.ctypes.data, w * 4, 1),
        "plane_device": lambda: L.w2x_convert_plane_device(ctx._h, model._h, dp, w, h, w * 4, d_out.data_ptr(), w * 4, 1),
        "band_device": lambda: L.w2x_convert_band_device(ctx._h, model._h, dp, w, h - 2 * n, n, n, w * 4, d_out.data_ptr(), w * 4),
        "planes": lambda: L.w2x_convert_planes(ctx._h, model._h, 1, pp(xp), pi(w), pi(h), ps(w * 4), pp(out.ctypes.data), ps(w * 4)),
        "planes_device": lambda: L.w2x_convert_planes_device(ctx._h, model._h, 1, pp(dp), pi(w), pi(h), ps(w * 4), pp(d_out.data_ptr()),
                                                             ps(w * 4)),
        "chain": lambda: L.w2x_convert_chain(ctx._h, 1, steps, same, xp, w, h, w * 4, out.ctypes.data, w * 4, 1, STEP_FN(), None),
        "chain_device": lambda: L.w2x_convert_chain_device(ctx._h, 1, steps, same, dp, w, h, w * 4, d_out.data_ptr(), w * 4, 1,
                                                           STEP_FN(), None),
    }


def assert_rejected(ctx, got, calls, want_status, case):
    ctx.synchronize()
    for name, call in calls.items():
        got.clear()
        n0 = ctx.launch_count()
        status = call()
        ctx.synchronize()
        assert (status, got, ctx.launch_count() - n0) == (want_status, [], 0), (case, name)


@pytest.mark.parametrize("case", ["null", "one_to_two", "tc_refuses"])
def test_rejected_calls_print_nothing(w2x, ctx, models, case):
    """also with the host copy pipeline cutting the plane into bands, which used to print the lines before the engine check"""
    x = np.random.default_rng(3).random((90, 60), dtype=np.float32)
    model = models[{"null": "noise2", "one_to_two": "one_to_two", "tc_refuses": "no_tc"}[case]]
    if case == "tc_refuses":
        ctx.set_engine(w2x.ENGINE_TC)
    got = []
    ctx.set_log(got.append)
    want = ERR_UNSUPPORTED if case == "tc_refuses" else ERR_ARG
    for host_bands in (1, 3):
        ctx.debug_set_host_bands(host_bands)
        assert_rejected(ctx, got, plane_calls(w2x, ctx, model, x, case == "null"), want, (case, host_bands))


def misfit_block_size(w2x, w, h, n):
    """a non-square block size whose literal walk on a w x h plane runs one block or more before one does not fit"""
    for bh in range(2 * n + 2, 200):
        w2x.set_block_size(64, bh)
        if not w2x.requires_splitting(w, h):
            continue
        tab, _, _ = w2x.block_table(w, h, n)
        fits = [t[6] + (t[3] - t[2]) - 2 * n <= h and t[7] + (t[5] - t[4]) - 2 * n <= w for t in tab]
        if fits[0] and not all(fits):
            return 64, bh
    raise AssertionError("no such block size")


@pytest.mark.parametrize("engine", ENGINES)
def test_literal_walk_that_does_not_fit(w2x, ctx, models, engine):
    model = models["noise2"]
    x = np.random.default_rng(4).random((100, 120), dtype=np.float32)
    w2x.set_block_size(*misfit_block_size(w2x, 120, 100, len(model)))
    ctx.set_engine(w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    ctx.set_block_walk(w2x.WALK_BLOCKS)
    got = []
    ctx.set_log(got.append)
    calls = plane_calls(w2x, ctx, model, x, False)
    assert_rejected(ctx, got, {k: calls[k] for k in ("plane", "plane_device", "chain", "chain_device")}, ERR_ARG, engine)
