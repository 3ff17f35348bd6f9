"""Many windows of chains' outputs in one call: w2x_convert_chain_regions and w2x_convert_chain_regions_device.

Each step packs the windows' step outputs into frames, each rectangle holding its window's real neighbours as padding, so every window
must equal, bit for bit, w2x_convert_chain_region on that window alone and the same window of w2x_convert_chain(..., block_splitting
= 0) on its whole plane.  The CPU part checks the refusals that need no device; the GPU part checks the bits on both engines and
every precision, through the host and the device entry points, for tiles of one plane, with NaN around every source rectangle, with
frames and windows converted alone forced by the scratch limit, and the call protocol: on_step, progress lines, launches, refusals
and W2X_ERR_NOMEM."""
import ctypes as C

import numpy as np
import pytest
from test_region import CONFIGS, chains, crop, make_ctx, odd_windows, region_windows, small_model

gpu = pytest.mark.gpu
ERR_ARG, ERR_UNSUPPORTED, ERR_NOMEM = 1, 7, 8


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


def sources(w2x, steps, planes, wins):
    """windows as (plane index, window) -> the source rectangles as strided views of their planes, and the planes' sizes"""
    srcs, sizes = [], []
    for p, win in wins:
        x = planes[p]
        size = (x.shape[1], x.shape[0])
        sx0, sy0, sw, sh = w2x.chain_region_source(steps, size, win)
        srcs.append(x[sy0:sy0 + sh, sx0:sx0 + sw])
        sizes.append(size)
    return srcs, sizes


def device_regions(w2x, ctx, steps, d_planes, wins, pad_out=3, on_step=None):
    """convert_chain_regions_device on whole planes held on the device, every output's row stride padded by pad_out floats, checked
    untouched"""
    import torch
    d_src, sizes, strides, outs = [], [], [], []
    for p, win in wins:
        d = d_planes[p]
        H, W = d.shape
        sx0, sy0, _, _ = w2x.chain_region_source(steps, (W, H), win)
        d_src.append(d.data_ptr() + (sy0 * W + sx0) * 4)
        sizes.append((W, H))
        strides.append(W * 4)
        outs.append(torch.full((win[3], win[2] + pad_out), -7.5, device="cuda"))
    ctx.convert_chain_regions_device(steps, d_src, sizes, [w for _, w in wins], strides, [o.data_ptr() for o in outs],
                                     [o.stride(0) * 4 for o in outs], on_step=on_step)
    ctx.synchronize()
    got = []
    for o, (_, win) in zip(outs, wins):
        o = o.cpu().numpy()
        assert (o[:, win[2]:] == -7.5).all()
        got.append(o[:, :win[2]])
    return got


def mixed_windows(planes, ups):
    """windows of every plane: at every border, 1 x 1, the whole output, on odd and even 2x rows and columns"""
    wins = []
    for p, x in enumerate(planes):
        W, H = x.shape[1] << ups, x.shape[0] << ups
        wins += [(p, w) for w in odd_windows(W, H) if w[2] > 0 and w[3] > 0]
        wins += [(p, (0, 0, 1, 1)), (p, (W - 1, H - 1, 1, 1)), (p, (W // 2 | 1, H // 2 | 1, 1, 1))]
    return wins


# ---------------------------------------------------------------------------------------------------------------------
# CPU: refusals before any device work
# ---------------------------------------------------------------------------------------------------------------------
def test_regions_refuse_a_null_context(w2x):
    m = small_model(w2x, (1, 4, 1), 1)
    n, models, kinds, cb, _ = w2x.Context._chain_args([(m, True)], None)
    one = (C.c_int * 1)(8)
    win = (C.c_int * 4)(0, 0, 2, 2)
    src = (C.c_void_p * 1)(None)
    st = (C.c_size_t * 1)(32)
    for fn in (w2x.lib().w2x_convert_chain_regions, w2x.lib().w2x_convert_chain_regions_device):
        assert fn(None, n, models, kinds, 1, one, one, win, src, st, src, st, cb, None) == ERR_ARG


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bits, reads, frames and protocol
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_regions_are_bit_identical_to_the_whole_chain_and_to_one_window(w2x, shipped, oracle_mod, config):
    import torch
    ctx = make_ctx(w2x, config)
    fails = []
    try:
        for c, steps in enumerate(chains(shipped)):
            ups = sum(1 for _, up in steps if up)
            dims = [(23, 19), (17, 26)] if ups >= 2 else [(45, 37), (30, 41), (19, 12)]
            planes = [oracle_mod.seeded_plane(w, h, 10 * c + i, "uniform") for i, (w, h) in enumerate(dims)]
            wholes = [ctx.convert_chain(steps, x, block_splitting=False) for x in planes]
            wins = mixed_windows(planes, ups)
            srcs, sizes = sources(w2x, steps, planes, wins)
            want = [crop(wholes[p], win) for p, win in wins]
            for i, ((p, win), s, size) in enumerate(zip(wins, srcs, sizes)):
                if not np.array_equal(ctx.convert_chain_region(steps, s, size, win), want[i]):
                    fails.append(f"one window: chain {c} plane {p} window {win}")
            got = ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins])
            fails += [f"host: chain {c} plane {p} window {w}" for (p, w), g, e in zip(wins, got, want) if not np.array_equal(g, e)]
            d_planes = [torch.from_numpy(x).cuda() for x in planes]
            got = device_regions(w2x, ctx, steps, d_planes, wins)
            fails += [f"device: chain {c} plane {p} window {w}" for (p, w), g, e in zip(wins, got, want) if not np.array_equal(g, e)]
    finally:
        ctx.close()
    assert not fails, fails


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_tiles_of_one_plane_make_the_whole_chain(w2x, shipped, oracle_mod, config):
    """tiles covering the output exactly, from overlapping source rectangles of one host array, put together"""
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        width, height = 61, 47
        x = oracle_mod.seeded_plane(width, height, 4, "uniform")
        whole = ctx.convert_chain(steps, x, block_splitting=False)
        H, W = whole.shape
        wins = [(0, (tx, ty, min(32, W - tx), min(24, H - ty))) for ty in range(0, H, 24) for tx in range(0, W, 32)]
        srcs, sizes = sources(w2x, steps, [x], wins)
        out = np.full_like(whole, np.nan)
        ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins], out=[crop(out, w) for _, w in wins])
        assert np.array_equal(out, whole)
    finally:
        ctx.close()


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_nothing_outside_the_rectangles_is_read(w2x, shipped, oracle_mod, config):
    """every source rectangle inside its own buffer that is NaN everywhere else: every window still matches and holds no NaN"""
    import torch
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise2"], False), (shipped["scale2.0x"], True)]
        planes = [oracle_mod.seeded_plane(37, 29, 9, "uniform"), oracle_mod.seeded_plane(20, 33, 8, "uniform")]
        wholes = [ctx.convert_chain(steps, x, block_splitting=False) for x in planes]
        wins = [(0, (5, 7, 31, 21)), (0, (0, 0, 74, 58)), (1, (39, 1, 1, 57)), (0, (11, 0, 9, 3)), (1, (3, 4, 30, 50))]
        srcs, sizes = sources(w2x, steps, planes, wins)
        views, d_bufs = [], []
        for s in srcs:
            sh, sw = s.shape
            buf = np.full((sh + 10, sw + 12), np.nan, np.float32)
            buf[5:5 + sh, 6:6 + sw] = s
            views.append(buf[5:5 + sh, 6:6 + sw])
            d_bufs.append(torch.from_numpy(buf).cuda())
        want = [crop(wholes[p], w) for p, w in wins]
        got = ctx.convert_chain_regions(steps, views, sizes, [w for _, w in wins])
        for g, e, win in zip(got, want, wins):
            assert not np.isnan(g).any() and np.array_equal(g, e), win
        outs = [torch.empty((w[3], w[2]), device="cuda") for _, w in wins]
        ctx.convert_chain_regions_device(steps, [d.data_ptr() + (5 * d.shape[1] + 6) * 4 for d in d_bufs], sizes, [w for _, w in wins],
                                         [d.shape[1] * 4 for d in d_bufs], [o.data_ptr() for o in outs], [w[2] * 4 for _, w in wins])
        ctx.synchronize()
        for o, e, win in zip(outs, want, wins):
            g = o.cpu().numpy()
            assert not np.isnan(g).any() and np.array_equal(g, e), win
    finally:
        ctx.close()


@gpu
def test_frames_and_windows_converted_alone(w2x, shipped, oracle_mod):
    """a scratch limit under which the last step's plan has two frames and a window converted alone changes no bit"""
    import torch
    ctx = make_ctx(w2x, "default")
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        width, height = 70, 64
        x = oracle_mod.seeded_plane(width, height, 12, "uniform")
        whole = ctx.convert_chain(steps, x, block_splitting=False)
        wins = [(0, (3, 5, 110, 100)), (0, (1, 1, 20, 20)), (0, (40, 30, 20, 19)), (0, (70, 2, 21, 20)), (0, (100, 101, 20, 20)),
                (0, (9, 110, 18, 17))]
        limit = 128 * 4 * 3000                              # 3000 pixels of 128 channels: two 34 x 34 rectangles a frame
        outs = [region_windows([7, 7], [False, True], width, height, w)[-1] for _, w in wins]
        frame, _, _, _ = w2x.debug_plan_planes([w[2] for w in outs], [w[3] for w in outs], 7, 128, limit)
        assert frame.max() >= 1 and (frame == -1).any(), frame
        ctx.set_scratch_limit(limit)
        srcs, sizes = sources(w2x, steps, [x], wins)
        want = [crop(whole, w) for _, w in wins]
        got = ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins])
        assert all(np.array_equal(g, e) for g, e in zip(got, want))
        got = device_regions(w2x, ctx, steps, [torch.from_numpy(x).cuda()], wins)
        assert all(np.array_equal(g, e) for g, e in zip(got, want))
    finally:
        ctx.set_scratch_limit(0)
        ctx.close()


@gpu
@pytest.mark.parametrize("config", ["default", "fp32"])
def test_regions_protocol(w2x, shipped, oracle_mod, config):
    """on_step(k) before step k; step k's lines are the one-window calls' lines at step k, window by window; its launches are those
    of convert_planes_device on planes of the step's output-window sizes, fewer than the one-window calls' when windows pack"""
    import torch
    ctx = make_ctx(w2x, config)
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True), (shipped["scale2.0x"], True)]
        planes = [oracle_mod.seeded_plane(30, 26, 3, "uniform"), oracle_mod.seeded_plane(19, 22, 4, "uniform")]
        wins = [(0, (37, 21, 50, 61)), (1, (0, 0, 76, 88)), (0, (81, 3, 39, 40)), (1, (7, 9, 1, 1))]
        srcs, sizes = sources(w2x, steps, planes, wins)
        d_planes = [torch.from_numpy(x).cuda() for x in planes]
        n_steps = len(steps)

        def run(fn):
            """fn(on_step) -> (lines per step, launches per step)"""
            got, at = [], []

            def on_step(k):
                got.append(("step", k))
                at.append(ctx.launch_count())
            ctx.set_log(got.append)
            fn(on_step)
            ctx.synchronize()
            at.append(ctx.launch_count())
            ctx.set_log(None)
            cut = [i for i, v in enumerate(got) if isinstance(v, tuple)] + [len(got)]
            assert [got[i] for i in cut[:-1]] == [("step", k) for k in range(n_steps)], got[:4]
            return [got[a + 1:b] for a, b in zip(cut, cut[1:])], [b - a for a, b in zip(at, at[1:])]

        want_lines, loop_launches = [[] for _ in range(n_steps)], [0] * n_steps
        for s, size, (_, win) in zip(srcs, sizes, wins):
            lines, launches = run(lambda cb: ctx.convert_chain_region(steps, s, size, win, on_step=cb))
            for k in range(n_steps):
                want_lines[k] += lines[k]
                loop_launches[k] += launches[k]
        want_launches = []
        for k in range(n_steps):
            ow = [region_windows([7, 7, 7], [False, True, True], *size, w)[k + 1] for size, (_, w) in zip(sizes, wins)]
            d_in = [torch.zeros((o[3], o[2]), device="cuda") for o in ow]
            d_out = [torch.empty((o[3], o[2]), device="cuda") for o in ow]
            n0 = ctx.launch_count()
            ctx.convert_planes_device(steps[k][0], [t.data_ptr() for t in d_in], [o[2] for o in ow], [o[3] for o in ow],
                                      [o[2] * 4 for o in ow], [t.data_ptr() for t in d_out], [o[2] * 4 for o in ow])
            ctx.synchronize()
            want_launches.append(ctx.launch_count() - n0)
        host = run(lambda cb: ctx.convert_chain_regions(steps, srcs, sizes, [w for _, w in wins], on_step=cb))
        device = run(lambda cb: device_regions(w2x, ctx, steps, d_planes, wins, on_step=cb))
        for entry, (lines, launches) in (("host", host), ("device", device)):
            assert lines == want_lines, (entry, [len(v) for v in lines], [len(v) for v in want_lines])
            assert launches == want_launches, (entry, launches, want_launches)
        if config == "default":
            assert sum(want_launches) < sum(loop_launches), (want_launches, loop_launches)
        else:
            assert want_launches == loop_launches
    finally:
        ctx.set_log(None)
        ctx.close()


@gpu
def test_regions_refusals_queue_nothing(w2x, shipped, oracle_mod):
    import torch
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        N, S = shipped["noise1"], shipped["scale2.0x"]
        steps = [(N, False), (S, True)]
        width, height = 20, 16
        x = torch.from_numpy(oracle_mod.seeded_plane(width, height, 1, "uniform")).cuda()
        out = torch.full((3, 32, 40), -3.0, device="cuda")
        lines, calls = [], []
        ctx.set_log(lines.append)
        lib = w2x.lib()
        n0 = ctx.launch_count()
        cb = w2x.capi.STEP_FN(lambda k, _u: calls.append(k))
        good = [(2, 3, 10, 9), (0, 0, 40, 32), (7, 1, 1, 1)]

        def call(st, wins=good, nw=3, sizes=None, src=None, sst=None, dst=None, dstst=None, null=None, host=False):
            n, models, kinds, _, _ = w2x.Context._chain_args(st, None)
            sizes = sizes or [(width, height)] * nw
            src = src or [x.data_ptr()] * nw
            sst = sst or [width * 4] * nw
            dst = dst or [out[i].data_ptr() for i in range(nw)]
            dstst = dstst or [40 * 4] * nw
            args = [(C.c_int * nw)(*[s[0] for s in sizes]), (C.c_int * nw)(*[s[1] for s in sizes]),
                    (C.c_int * (4 * nw))(*[v for w in wins for v in w]), (C.c_void_p * nw)(*src), (C.c_size_t * nw)(*sst),
                    (C.c_void_p * nw)(*dst), (C.c_size_t * nw)(*dstst)]
            if null is not None:
                args[null] = None
            fn = lib.w2x_convert_chain_regions if host else lib.w2x_convert_chain_regions_device
            rc = fn(ctx._h, n, models, kinds, nw, *args, cb, None)
            return rc, lib.w2x_last_error().decode()

        small = small_model(w2x, (1, 3, 1), 4)
        cases = [(dict(st=steps, nw=0, wins=[]), ERR_ARG, "n_windows"),
                 (dict(st=[(N, False), (S, True, True)]), ERR_ARG, "step 1"),
                 (dict(st=[(N, False, True), (S, True)]), ERR_ARG, "step 0"),
                 (dict(st=[]), ERR_ARG, "n_steps"),
                 (dict(st=steps, wins=[good[0], (2, 3, 0, 9), good[2]]), ERR_ARG, "window 1: empty window"),
                 (dict(st=steps, wins=[good[0], good[1], (35, 3, 6, 9)]), ERR_ARG, "window 2: window {35, 3, 6, 9} is not inside"),
                 (dict(st=steps, wins=[good[0], good[1], (2, -1, 6, 9)]), ERR_ARG, "window 2: window"),
                 (dict(st=steps, src=[x.data_ptr(), 0, x.data_ptr()]), ERR_ARG, "window 1: NULL source"),
                 (dict(st=steps, dst=[out[0].data_ptr(), out[1].data_ptr(), 0]), ERR_ARG, "window 2: NULL output"),
                 (dict(st=steps, sst=[width * 4, 4, width * 4]), ERR_ARG, "window 1: the source row stride"),
                 (dict(st=steps, sst=[width * 4 + 2] * 3), ERR_ARG, "window 0: the source row stride"),
                 (dict(st=steps, dstst=[40 * 4, 39 * 4, 40 * 4]), ERR_ARG, "window 1: the output row stride"),
                 (dict(st=steps, dstst=[40 * 4, 40 * 4, 40 * 4 + 1]), ERR_ARG, "window 2: the output row stride"),
                 (dict(st=steps, sizes=[(width, height), (0, 16), (width, height)]), ERR_ARG, "window 1: step 0: input size"),
                 (dict(st=[(N, False), (small, True)]), ERR_UNSUPPORTED, "step 1"),
                 (dict(st=[(N, False), (small, True)], host=True), ERR_UNSUPPORTED, "step 1"),
                 (dict(st=steps, wins=[good[0], (2, 3, 0, 9), good[2]], host=True), ERR_ARG, "window 1: empty window")]
        cases += [(dict(st=steps, null=i), ERR_ARG, "NULL array") for i in range(7)]
        for kw, status, want in cases:
            rc, msg = call(**kw)
            assert rc == status and want in msg, (kw, rc, msg)
            assert msg.startswith("w2x_convert_chain_regions" + ("" if kw.get("host") else "_device") + ":") or status != ERR_ARG, msg
        ctx.synchronize()
        assert ctx.launch_count() == n0 and not lines and not calls
        assert (out == -3.0).all().item()
    finally:
        ctx.set_log(None)
        ctx.close()


@gpu
def test_out_of_memory_leaves_nothing_queued(w2x, shipped, oracle_mod):
    """with the device all but full, windows whose buffers cannot be reserved give W2X_ERR_NOMEM before any copy or launch"""
    import torch
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    filler = None
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        small = oracle_mod.seeded_plane(16, 16, 1, "uniform")
        ctx.convert_chain_regions(steps, [small, small], [(16, 16)] * 2, [(0, 0, 32, 32), (0, 0, 32, 32)])   # the models' device copies exist
        w = h = 2048
        wins = [(1, 1, 2 * w - 2, 2 * h - 2), (0, 0, 64, 64)]
        d_in = torch.from_numpy(oracle_mod.seeded_plane(w, h, 2, "uniform")).cuda()
        d_out = [torch.full((win[3], win[2]), -3.25, device="cuda") for win in wins]
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        n0, calls, lines = ctx.launch_count(), [], []
        ctx.set_log(lines.append)
        with pytest.raises(w2x.W2xError) as e:
            ctx.convert_chain_regions_device(steps, [d_in.data_ptr()] * 2, [(w, h)] * 2, wins, [w * 4] * 2, [d.data_ptr() for d in d_out],
                                             [win[2] * 4 for win in wins], on_step=calls.append)
        assert e.value.status == ERR_NOMEM, e.value.message
        assert ctx.launch_count() == n0 and not calls and not lines
        ctx.synchronize()
        del filler
        filler = None
        torch.cuda.empty_cache()
        assert all((d == -3.25).all().item() for d in d_out)
    finally:
        ctx.set_log(None)
        del filler
        ctx.close()
