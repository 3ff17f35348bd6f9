"""Windows of a chain's output: w2x_chain_region_source, w2x_convert_chain_region and w2x_convert_chain_region_device.

A window of the output is computed from the source rectangle alone and must equal, bit for bit, the same window of
w2x_convert_chain(..., block_splitting = 0) on the whole plane: every step converts only its output window, reading the real
neighbours the previous window holds and replicating only at the plane's own border.  The CPU part checks the window arithmetic
against a restatement of it here; the GPU part checks the bits on both engines and every precision, through the host and the
device entry points, with row bands forced by the scratch limit, with NaN around the source rectangle, against the exact emulator
of the first layer, and the call protocol: on_step, progress lines, launches, refusals and W2X_ERR_NOMEM."""
import ctypes as C
import itertools

import numpy as np
import pytest

gpu = pytest.mark.gpu
ERR_ARG, ERR_UNSUPPORTED, ERR_NOMEM = 1, 7, 8


def region_windows(layers, ups, width, height, window):
    """[source rectangle, step 0's output window, ..., window]: a step's input window is its output window grown by its model's
    layer count and clamped to its input plane, then for an upscaling step halved, floor at the top-left and ceil at the
    bottom-right"""
    W, H = width << sum(ups), height << sum(ups)
    x0, y0, w, h = window
    x1, y1 = x0 + w, y0 + h
    wins = [tuple(window)]
    for n, up in reversed(list(zip(layers, ups))):
        x0, y0, x1, y1 = max(0, x0 - n), max(0, y0 - n), min(W, x1 + n), min(H, y1 + n)
        if up:
            x0, y0, x1, y1 = x0 // 2, y0 // 2, -(-x1 // 2), -(-y1 // 2)
            W, H = W // 2, H // 2
        wins.insert(0, (x0, y0, x1 - x0, y1 - y0))
    return wins


def crop(a, win):
    x0, y0, w, h = win
    return a[y0:y0 + h, x0:x0 + w]


def border_windows(W, H):
    """windows touching 0, 1, 2, 3 and 4 of the plane's borders, 1 x 1 windows and odd coordinates"""
    wins = [(W // 3 | 1, H // 3 | 1, max(1, W // 4), max(1, H // 5)),   # interior, odd corner
            (0, H // 4 | 1, max(1, W // 3), max(1, H // 3)),              # left border
            (W - max(1, W // 3), H - max(1, H // 2), max(1, W // 3), max(1, H // 2)),   # bottom-right corner
            (0, 0, W, max(1, H // 3)),                                     # top strip: three borders
            (0, 0, W, H),                                                  # the whole output
            (0, 0, 1, 1), (W - 1, H - 1, 1, 1), (W // 2 | 1, H // 2 | 1, 1, 1)]
    return [w for w in wins if w[0] + w[2] <= W and w[1] + w[3] <= H]


def small_model(w2x, widths, seed):
    rng = np.random.default_rng(seed)
    ws, bs = [], []
    for ci, co in zip(widths[:-1], widths[1:]):
        ws.append((rng.standard_normal((co, ci, 3, 3)) / np.sqrt(9 * ci)).astype(np.float32))
        bs.append(rng.standard_normal(co) * 0.1)
    return w2x.Model.from_arrays(ws, bs)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the window arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def test_region_source_matches_the_window_arithmetic(w2x):
    models = [(small_model(w2x, (1, 4, 1), 1), 2), (small_model(w2x, (1, 3, 5, 1), 2), 3), (small_model(w2x, (1, 2, 2, 2, 2, 2, 2, 1), 3), 7)]
    checked = 0
    for n_steps in (1, 2, 3):
        for ups in itertools.product((False, True), repeat=n_steps):
            for rot in range(len(models)):
                chosen = [models[(rot + k) % len(models)] for k in range(n_steps)]
                steps = [(m, up) for (m, _), up in zip(chosen, ups)]
                layers = [n for _, n in chosen]
                for width, height in ((13, 9), (1, 1), (40, 27)):
                    W, H = width << sum(ups), height << sum(ups)
                    for win in border_windows(W, H):
                        wins = region_windows(layers, ups, width, height, win)
                        assert w2x.chain_region_source(steps, (width, height), win) == wins[0], (layers, ups, width, height, win)
                        checked += 1
    assert checked > 500, checked


def test_region_source_refusals(w2x):
    m = small_model(w2x, (1, 4, 1), 1)
    steps = [(m, False), (m, True)]
    cases = [([(m, False), (m, True, True)], (2, 2, 3, 3), "step 1"),
             ([(m, True, True), (m, True)], (2, 2, 3, 3), "step 0"),
             (steps, (2, 2, 0, 3), "empty window"),
             (steps, (2, 2, 3, -1), "empty window"),
             (steps, (-1, 2, 3, 3), "not inside"),
             (steps, (2, 2, 19, 3), "not inside"),           # the output is 20 x 18
             (steps, (2, 16, 3, 3), "not inside")]
    for st, win, want in cases:
        with pytest.raises(w2x.W2xError) as e:
            w2x.chain_region_source(st, (10, 9), win)
        assert e.value.status == ERR_ARG and want in e.value.message, (win, e.value.message)
    n, models, kinds, _, _ = w2x.Context._chain_args(steps, None)
    src = (C.c_int * 4)()
    assert w2x.lib().w2x_chain_region_source(n, models, kinds, 10, 9, None, src) == ERR_ARG
    assert b"NULL window" in w2x.lib().w2x_last_error()
    bad_kinds = (C.c_int * 2)(0, 2)
    assert w2x.lib().w2x_chain_region_source(n, models, bad_kinds, 10, 9, (C.c_int * 4)(0, 0, 1, 1), src) == ERR_ARG
    assert b"step 1" in w2x.lib().w2x_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bits, reads, kernels and protocol
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


def chains(shipped):
    N1, N2, S = shipped["noise1"], shipped["noise2"], shipped["scale2.0x"]
    return [[(N1, False)], [(S, True)], [(N2, False), (S, True)], [(S, True), (S, True)], [(N1, False), (S, True), (N2, False)]]


def odd_windows(W, H):
    """windows at even and odd 2x rows and columns, at the borders and in the interior"""
    wins = [(0, 0, W, H), (1, 1, 5, 3), (W - 7, H - 4, 7, 4), (W - 1, 0, 1, H), (0, H - 1, W, 1), (W // 2 | 1, H // 3 | 1, 23, 17),
            (2, 3, 32, 9), (W // 4 * 2, H // 4 * 2, 9, 8)]
    return [(x0, y0, min(w, W - x0), min(h, H - y0)) for x0, y0, w, h in wins]


CONFIGS = ["default", "f16x3", "f16", "fp32"]


def make_ctx(w2x, config):
    if config == "fp32":
        return w2x.Context(0, engine=w2x.ENGINE_FP32)
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    if config == "f16x3":
        c.set_precision(w2x.PRECISION_F16X3)
    elif config == "f16":
        c.set_precision(w2x.PRECISION_F16)
    return c


def device_region(w2x, ctx, steps, d_x, size, win, pad_out=3):
    """convert_chain_region_device on a whole plane held on the device, the output row stride padded by pad_out floats"""
    import torch
    sx0, sy0, _, _ = w2x.chain_region_source(steps, size, win)
    W = size[0]
    out = torch.full((win[3], win[2] + pad_out), -7.5, device="cuda")
    ctx.convert_chain_region_device(steps, d_x.data_ptr() + (sy0 * W + sx0) * 4, size, win, W * 4, out.data_ptr(), out.stride(0) * 4)
    ctx.synchronize()
    o = out.cpu().numpy()
    assert (o[:, win[2]:] == -7.5).all()
    return o[:, :win[2]]


@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_windows_are_bit_identical_to_the_whole_chain(w2x, shipped, oracle_mod, config):
    import torch
    ctx = make_ctx(w2x, config)
    fails = []
    try:
        for c, steps in enumerate(chains(shipped)):
            ups = sum(1 for _, up in steps if up)
            width, height = (23, 19) if ups >= 2 else (45, 37)
            x = oracle_mod.seeded_plane(width, height, c, "uniform")
            whole = ctx.convert_chain(steps, x, block_splitting=False)
            W, H = width << ups, height << ups
            d_x = torch.from_numpy(x).cuda()
            for win in odd_windows(W, H):
                sx0, sy0, sw, sh = w2x.chain_region_source(steps, (width, height), win)
                want = crop(whole, win)
                got = ctx.convert_chain_region(steps, x[sy0:sy0 + sh, sx0:sx0 + sw], (width, height), win)   # a strided view
                if not np.array_equal(got, want):
                    fails.append(f"host chain {c} window {win}")
                if not np.array_equal(device_region(w2x, ctx, steps, d_x, (width, height), win), want):
                    fails.append(f"device chain {c} window {win}")
    finally:
        ctx.close()
    assert not fails, fails


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_windows_in_scratch_bands(w2x, shipped, oracle_mod, config):
    """a scratch limit that cuts every step's window into 16-row bands changes no bit"""
    import torch
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        width, height = 41, 53
        x = oracle_mod.seeded_plane(width, height, 5, "uniform")
        whole = ctx.convert_chain(steps, x, block_splitting=False)
        d_x = torch.from_numpy(x).cuda()
        for win in [(3, 5, 61, 90), (0, 0, 82, 106), (1, 17, 40, 61)]:
            ctx.set_scratch_limit(128 * (win[2] + 14) * 4 * (16 + 14))
            sx0, sy0, sw, sh = w2x.chain_region_source(steps, (width, height), win)
            assert np.array_equal(ctx.convert_chain_region(steps, x[sy0:sy0 + sh, sx0:sx0 + sw], (width, height), win), crop(whole, win)), win
            assert np.array_equal(device_region(w2x, ctx, steps, d_x, (width, height), win), crop(whole, win)), win
    finally:
        ctx.set_scratch_limit(0)
        ctx.close()


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_nothing_outside_the_rectangle_is_read(w2x, shipped, oracle_mod, config):
    """the source rectangle inside a buffer that is NaN everywhere else: the window still matches and holds no NaN"""
    import torch
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise2"], False), (shipped["scale2.0x"], True)]
        width, height = 37, 29
        x = oracle_mod.seeded_plane(width, height, 9, "uniform")
        whole = ctx.convert_chain(steps, x, block_splitting=False)
        for win in [(5, 7, 31, 21), (0, 0, 74, 58), (73, 1, 1, 57), (11, 0, 9, 3)]:
            sx0, sy0, sw, sh = w2x.chain_region_source(steps, (width, height), win)
            buf = np.full((sh + 10, sw + 12), np.nan, np.float32)
            buf[5:5 + sh, 6:6 + sw] = x[sy0:sy0 + sh, sx0:sx0 + sw]
            got = ctx.convert_chain_region(steps, buf[5:5 + sh, 6:6 + sw], (width, height), win)
            assert not np.isnan(got).any() and np.array_equal(got, crop(whole, win)), win
            d_buf = torch.from_numpy(buf).cuda()
            out = torch.empty((win[3], win[2]), device="cuda")
            ctx.convert_chain_region_device(steps, d_buf.data_ptr() + (5 * buf.shape[1] + 6) * 4, (width, height), win, buf.shape[1] * 4,
                                            out.data_ptr(), win[2] * 4)
            ctx.synchronize()
            got = out.cpu().numpy()
            assert not np.isnan(got).any() and np.array_equal(got, crop(whole, win)), win
    finally:
        ctx.close()


@gpu
@pytest.mark.parametrize("prec", ["f16x3", "f16+f8x2"])
def test_first_layer_column_context_is_bit_exact(w2x, prec):
    """first_layer_kernel with real columns left and right of the window, and the up2x form on odd 2x columns and rows, against the
    exact emulator of the whole plane (1 -> 32 -> 64 -> 32 -> 1 with selection layers, as test_edge_exact checks row bands)"""
    from test_edge_exact import _model, emulate_tc_model, plane_for, sel_model
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    ctx.set_precision(w2x.PRECISION_F16X3 if prec == "f16x3" else w2x.PRECISION_F16_F8X2)
    f8 = prec != "f16x3"
    layers = sel_model((32, 64, 32), 0, 4242)
    model = _model(w2x, layers)
    fails = []
    try:
        width, height = 45, 37
        x = plane_for(height, width, 7)
        for up, plane in ((False, x), (True, np.repeat(np.repeat(x, 2, 0), 2, 1))):
            steps = [(model, up)]
            want = emulate_tc_model(plane, layers, f8, True)[0]
            H, W = plane.shape
            for win in [(5, 3, 17, 11), (0, 6, 9, 20), (W - 13, 2, 13, 9), (3, 5, 21, 13), (W - 7, 1, 7, 9), (1, H - 5, 19, 5), (7, 9, 1, 1)]:
                sx0, sy0, sw, sh = w2x.chain_region_source(steps, (width, height), win)
                got = ctx.convert_chain_region(steps, x[sy0:sy0 + sh, sx0:sx0 + sw], (width, height), win)
                if not np.array_equal(got, crop(want, win)):
                    fails.append(f"up2x={up} window {win}")
    finally:
        ctx.close()
    assert not fails, fails


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_region_protocol(w2x, shipped, oracle_mod, config):
    """on_step(k) before step k, then the lines and launches of convert_plane_device(block_splitting=False) on a plane the size of
    step k's output window -- with and without scratch bands"""
    import torch
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True), (shipped["scale2.0x"], True)]
        width, height = 30, 26
        x = oracle_mod.seeded_plane(width, height, 3, "uniform")
        d_x = torch.from_numpy(x).cuda()
        win = (37, 21, 50, 61)
        wins = region_windows([7, 7, 7], [False, True, True], width, height, win)
        for limit in (0, 128 * (wins[2][2] + 14) * 4 * (16 + 14)):
            ctx.set_scratch_limit(limit)
            want, want_launches = [], []
            for k, (m, _) in enumerate(steps):
                ow, oh = wins[k + 1][2], wins[k + 1][3]
                d_in, d_out = torch.zeros((oh, ow), device="cuda"), torch.empty((oh, ow), device="cuda")
                lines = [("step", k)]
                ctx.set_log(lines.append)
                n0 = ctx.launch_count()
                ctx.convert_plane_device(m, d_in.data_ptr(), ow, oh, ow * 4, d_out.data_ptr(), ow * 4, block_splitting=False)
                want_launches.append(ctx.launch_count() - n0)
                ctx.synchronize()
                want += lines
            got, at = [], []

            def on_step(k):
                got.append(("step", k))
                at.append(ctx.launch_count())
            ctx.set_log(got.append)
            sx0, sy0, sw, sh = wins[0]
            for entry in ("host", "device"):
                got.clear()
                at.clear()
                if entry == "host":
                    ctx.convert_chain_region(steps, x[sy0:sy0 + sh, sx0:sx0 + sw], (width, height), win, on_step=on_step)
                else:
                    out = torch.empty((win[3], win[2]), device="cuda")
                    ctx.convert_chain_region_device(steps, d_x.data_ptr() + (sy0 * width + sx0) * 4, (width, height), win, width * 4,
                                                    out.data_ptr(), win[2] * 4, on_step=on_step)
                    ctx.synchronize()
                at.append(ctx.launch_count())
                assert got == want, (entry, limit, got[:8], want[:8])
                assert [b - a for a, b in zip(at, at[1:])] == want_launches, (entry, limit)
            ctx.set_log(None)
    finally:
        ctx.set_scratch_limit(0)
        ctx.close()


@gpu
def test_region_refusals_queue_nothing(w2x, shipped, oracle_mod):
    import torch
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        N, S = shipped["noise1"], shipped["scale2.0x"]
        steps = [(N, False), (S, True)]
        width, height = 20, 16
        x = torch.from_numpy(oracle_mod.seeded_plane(width, height, 1, "uniform")).cuda()
        out = torch.full((32, 40), -3.0, device="cuda")
        lines, calls = [], []
        ctx.set_log(lines.append)
        lib = w2x.lib()
        n0 = ctx.launch_count()
        cb = w2x.capi.STEP_FN(lambda k, _u: calls.append(k))

        def call(st, win=(2, 3, 10, 9), src=x.data_ptr(), sst=width * 4, dst=out.data_ptr(), dstst=40 * 4, size=(width, height)):
            n, models, kinds, _, _ = w2x.Context._chain_args(st, None)
            w = (C.c_int * 4)(*win) if win is not None else None
            rc = lib.w2x_convert_chain_region_device(ctx._h, n, models, kinds, size[0], size[1], w, C.c_void_p(src), sst, C.c_void_p(dst),
                                                     dstst, cb, None)
            return rc, lib.w2x_last_error().decode()

        cases = [(dict(st=[(N, False), (S, True, True)]), ERR_ARG, "step 1"),
                 (dict(st=[(N, False, True), (S, True)]), ERR_ARG, "step 0"),
                 (dict(st=[]), ERR_ARG, "n_steps"),
                 (dict(st=steps, win=None), ERR_ARG, "NULL window"),
                 (dict(st=steps, win=(2, 3, 0, 9)), ERR_ARG, "empty window"),
                 (dict(st=steps, win=(35, 3, 6, 9)), ERR_ARG, "not inside"),
                 (dict(st=steps, win=(2, -1, 6, 9)), ERR_ARG, "not inside"),
                 (dict(st=steps, src=0), ERR_ARG, "NULL source"),
                 (dict(st=steps, dst=0), ERR_ARG, "NULL output"),
                 (dict(st=steps, sst=4), ERR_ARG, "source row stride"),
                 (dict(st=steps, sst=width * 4 + 2), ERR_ARG, "source row stride"),
                 (dict(st=steps, dstst=9 * 4), ERR_ARG, "output row stride"),
                 (dict(st=steps, dstst=40 * 4 + 1), ERR_ARG, "output row stride"),
                 (dict(st=steps, size=(0, 16)), ERR_ARG, "input size"),
                 (dict(st=[(N, False), (small_model(w2x, (1, 3, 1), 4), True)]), ERR_UNSUPPORTED, "step 1")]
        for kw, status, want in cases:
            rc, msg = call(**kw)
            assert rc == status and want in msg, (kw, rc, msg)
        rc = lib.w2x_convert_chain_region(None, 1, *w2x.Context._chain_args(steps[:1], None)[1:3], width, height, (C.c_int * 4)(0, 0, 1, 1),
                                          None, 4, None, 4, cb, None)
        assert rc == ERR_ARG
        ctx.synchronize()
        assert ctx.launch_count() == n0 and not lines and not calls
        assert (out == -3.0).all().item()
    finally:
        ctx.set_log(None)
        ctx.close()


@gpu
def test_out_of_memory_leaves_nothing_queued(w2x, shipped, oracle_mod):
    """with the device all but full, a window whose buffers cannot be reserved returns W2X_ERR_NOMEM before any copy or launch"""
    import torch
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    filler = None
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        small = oracle_mod.seeded_plane(16, 16, 1, "uniform")
        ctx.convert_chain_region(steps, small, (16, 16), (0, 0, 32, 32))     # the models' device copies exist
        w = h = 2048
        win = (1, 1, 2 * w - 2, 2 * h - 2)
        d_in = torch.from_numpy(oracle_mod.seeded_plane(w, h, 2, "uniform")).cuda()
        d_out = torch.full((win[3], win[2]), -3.25, device="cuda")
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        n0, calls = ctx.launch_count(), []
        with pytest.raises(w2x.W2xError) as e:
            ctx.convert_chain_region_device(steps, d_in.data_ptr(), (w, h), win, w * 4, d_out.data_ptr(), win[2] * 4, on_step=calls.append)
        assert e.value.status == ERR_NOMEM, e.value.message
        assert ctx.launch_count() == n0 and not calls
        ctx.synchronize()
        del filler
        filler = None
        torch.cuda.empty_cache()
        assert (d_out == -3.25).all().item()
    finally:
        del filler
        ctx.close()
