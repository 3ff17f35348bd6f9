"""A context's calls across stream switches, on the caller's stream, and from two host threads.

Every call on a context shares its scratch (activation frames, padded planes, host staging, chain and TTA planes, frame tables), and
only the order of the context's stream keeps two calls apart.  w2x_ctx_set_stream therefore makes the new stream wait for everything
queued on the old one.  Every result here equals, bit for bit (np.array_equal), the same call made on an idle context.  Before a
racing pair, every call of the pair runs once on the idle context in the same order: that gives the expected outputs, and it grows
every scratch buffer to its final size (a grow frees the old block, and cudaFree waits for the whole device, which would hide an
overlap).  The contexts run the tensor-core engine at the default precision.

  * Waits after a switch: w2x_ctx_synchronize and w2x_ctx_layer_times, called on a new stream, cover the work queued on the old one.
  * Scratch across a switch: a noise + 2x chain queued on one torch stream, then each entry point that shares the scratch on a
    second torch stream (device entry points) or on the context's own stream (host entry points), each held back by the same short
    sleep so that the two would overlap; and one sequence over three streams.
  * The caller's stream: the input written by a torch op, the call (which uploads a model the context has not seen), the output
    read by a torch op, all on one stream behind a sleep, with no host synchronise between them.
  * Two contexts on one device, driven from two host threads at once, and w2x_last_error kept per thread.
"""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LONG = 1 << 28            # torch.cuda._sleep cycles: roughly 0.1-0.2 s
SHORT = 1 << 22           # a few ms: both calls of a racing pair are queued before either starts
A_W, A_H = 1920, 1080     # the chain every racing pair starts with; the other call of a pair is no larger
ERR_ARG = 1


class Call:
    """One entry point: run(ctx, models) queues it, reading `ins` and writing `outs` -- device tensors, or numpy arrays for a host
    entry point, which returns once its outputs have landed."""

    def __init__(self, run, ins, outs, host=False):
        self.run, self.ins, self.outs, self.host = run, ins, outs, host

    def clear(self):
        for o in self.outs:
            if isinstance(o, np.ndarray):
                o.fill(np.nan)
            else:
                o.fill_(float("nan"))

    def results(self):
        return [o.copy() if isinstance(o, np.ndarray) else o.cpu().numpy() for o in self.outs]


def steps(M, pattern, tta=False):
    return [(M["noise1"], False, tta) if c == "S" else (M["scale2.0x"], True, tta) for c in pattern]


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def empty(*shape):
    import torch
    return torch.empty(shape, dtype=torch.float32, device="cuda")


def ptrs(ts):
    return [t.data_ptr() for t in ts]


def rand(rng, *shape):
    return rng.random(shape, dtype=np.float32)


def sizes(rng, n, lo, hi):
    return [(int(w), int(h)) for w, h in rng.integers(lo, hi + 1, size=(n, 2))]


def chain_su(rng):
    x, y = dev(rand(rng, A_H, A_W)), empty(2 * A_H, 2 * A_W)
    return Call(lambda c, M: c.convert_chain_device(steps(M, "SU"), x.data_ptr(), A_W, A_H, A_W * 4, y.data_ptr(), 2 * A_W * 4), [x], [y])


def plane_device(rng):
    w, h = 1600, 900
    x, y = dev(rand(rng, h, w)), empty(h, w)
    return Call(lambda c, M: c.convert_plane_device(M["noise2"], x.data_ptr(), w, h, w * 4, y.data_ptr(), w * 4), [x], [y])


def band_device(rng):
    w, h, y0, rows, halo = 1600, 1000, 300, 500, 16     # rows [300, 800) with 16 rows of context on either side
    x, y = dev(rand(rng, h, w)), empty(rows, w)
    return Call(lambda c, M: c.convert_band_device(M["noise2"], x.data_ptr() + (y0 - halo) * w * 4, w, rows, halo, halo, w * 4,
                                                   y.data_ptr(), w * 4), [x], [y])


def tiles_device(rng):
    n, t = 16, 256
    x, y = dev(rand(rng, n, t, t)), empty(n, t, t)
    return Call(lambda c, M: c.convert_tiles_device(M["noise2"], x.data_ptr(), y.data_ptr(), n, t, t), [x], [y])


def planes_device(rng):
    sz = sizes(rng, 12, 40, 300)
    xs, ys = [dev(rand(rng, h, w)) for w, h in sz], [empty(h, w) for w, h in sz]
    ws, hs, st = [w for w, _ in sz], [h for _, h in sz], [w * 4 for w, _ in sz]
    return Call(lambda c, M: c.convert_planes_device(M["noise1"], ptrs(xs), ws, hs, st, ptrs(ys), st), xs, ys)


def chain_tta(rng):
    w, h = 480, 270
    x, y = dev(rand(rng, h, w)), empty(h, w)
    return Call(lambda c, M: c.convert_chain_device(steps(M, "S", tta=True), x.data_ptr(), w, h, w * 4, y.data_ptr(), w * 4), [x], [y])


def planes_chain_device(rng):
    sz = sizes(rng, 10, 40, 200)
    xs, ys = [dev(rand(rng, h, w)) for w, h in sz], [empty(2 * h, 2 * w) for w, h in sz]
    ws, hs = [w for w, _ in sz], [h for _, h in sz]
    return Call(lambda c, M: c.convert_planes_chain_device(steps(M, "SU"), ptrs(xs), ws, hs, [w * 4 for w in ws], ptrs(ys),
                                                           [w * 8 for w in ws]), xs, ys)


def filter_layer_device(rng):
    w, h = 512, 384                                       # noise2's layer 1 is 32 -> 32
    x, y = dev(rand(rng, 32, h, w)), empty(32, h, w)
    return Call(lambda c, M: c.filter_layer_device(M["noise2"], 1, x.data_ptr(), y.data_ptr(), w, h), [x], [y])


def plane(rng):
    x, y = rand(rng, 900, 1600), np.empty((900, 1600), np.float32)
    return Call(lambda c, M: c.convert_plane(M["noise2"], x, out=y), [x], [y], host=True)


def tiles(rng):
    x = rand(rng, 16, 256, 256)                           # 4 copy groups
    y = np.empty_like(x)
    return Call(lambda c, M: c.convert_tiles(M["noise2"], x, out=y), [x], [y], host=True)


def planes(rng):
    xs = [rand(rng, h, w) for w, h in sizes(rng, 20, 40, 300)]
    ys = [np.empty_like(x) for x in xs]
    return Call(lambda c, M: c.convert_planes(M["noise1"], xs, out=ys), xs, ys, host=True)


def chain(rng):
    x, y = rand(rng, 270, 480), np.empty((540, 960), np.float32)
    return Call(lambda c, M: c.convert_chain(steps(M, "SU"), x, out=y), [x], [y], host=True)


MAKERS = [chain_su, plane_device, band_device, tiles_device, planes_device, chain_tta, planes_chain_device, filter_layer_device,
          plane, tiles, planes, chain]
B_ARMS = ["plane_device", "band_device", "tiles_device", "planes_device", "chain_tta", "planes_chain_device", "filter_layer_device",
          "plane", "tiles", "planes", "chain"]
C_ARMS = ["plane_device", "band_device", "tiles_device", "planes_device", "filter_layer_device", "chain_tta"]


@pytest.fixture(scope="module")
def models(w2x, oracle_models):
    M = {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}
    assert M["noise2"].dims(1)[:2] == (32, 32)
    return M


@pytest.fixture(scope="module")
def ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.close()


@pytest.fixture(scope="module")
def calls(ctx):
    rng = np.random.default_rng(17)
    return {f.__name__: f(rng) for f in MAKERS}


def on_idle(ctx, M, seq):
    """Each call of seq on the context's own stream, one after the other, each once the one before has finished -> their outputs."""
    import torch
    ctx.set_stream(0)
    want = []
    for call in seq:
        call.clear()
        torch.cuda.synchronize()
        call.run(ctx, M)
        ctx.synchronize()
        want.append(call.results())
    return want


def queue(ctx, M, call, stream):
    """A device call on `stream` right after a short sleep there; a host call on the context's own stream, at once."""
    import torch
    if call.host:
        ctx.set_stream(0)
        call.run(ctx, M)
        return
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SHORT)
        ctx.set_stream(stream.cuda_stream)
        call.run(ctx, M)


def mismatches(got, want):
    return [i for i, (g, w) in enumerate(zip(got, want)) if not np.array_equal(g, w)]


def tiles_async(w2x, ctx, model, x, out):
    n, th, tw = x.shape
    ip = (C.c_void_p * n)(*[x[i].ctypes.data for i in range(n)])
    op = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    L = w2x.lib()
    rc = L.w2x_convert_tiles_async(ctx._h, model._h, ip, op, n, tw, th, tw * 4, tw * 4)
    if rc:
        raise w2x.W2xError(rc, L.w2x_last_error().decode())


# ---- waits that must cover the previous stream ---------------------------------------------------------------------------------
def test_synchronize_covers_the_previous_stream(w2x, ctx, models):
    import torch
    n, t = 16, 512
    pinned = torch.empty((n, t, t), dtype=torch.float32).pin_memory()
    pinned_out = torch.empty((n, t, t), dtype=torch.float32).pin_memory()
    x, out = pinned.numpy(), pinned_out.numpy()
    x[...] = rand(np.random.default_rng(5), n, t, t)
    ctx.set_stream(0)
    tiles_async(w2x, ctx, models["noise2"], x, out)
    ctx.synchronize()
    want = out.copy()
    out.fill(np.nan)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        with torch.cuda.stream(s1):
            torch.cuda._sleep(LONG)
            ctx.set_stream(s1.cuda_stream)
            tiles_async(w2x, ctx, models["noise2"], x, out)
        ctx.set_stream(s2.cuda_stream)
        ctx.synchronize()
        landed = np.array_equal(out, want)        # read at once: nothing but w2x_ctx_synchronize has waited
        unwritten = int(np.isnan(out).sum())
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(0)
    assert landed, f"{unwritten} pixels not written when w2x_ctx_synchronize returned"


def test_layer_times_cover_the_previous_stream(ctx, models, calls):
    import torch
    call = calls["plane_device"]
    want = on_idle(ctx, models, [call])[0]
    ctx.layer_times(reset=True)
    call.clear()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        ctx.set_timing(True)
        with torch.cuda.stream(s1):
            torch.cuda._sleep(LONG)
            ctx.set_stream(s1.cuda_stream)
            call.run(ctx, models)
        ctx.set_stream(s2.cuda_stream)
        times = ctx.layer_times(reset=True)
    finally:
        ctx.set_timing(False)
        torch.cuda.synchronize()
        ctx.set_stream(0)
        ctx.layer_times(reset=True)
    assert len(times) == len(models["noise2"])
    assert [cnt for _, cnt, _ in times] == [1] * len(times)
    assert all(ms > 0 for ms, _, _ in times), [ms for ms, _, _ in times]
    assert not mismatches(call.results(), want)


# ---- scratch shared across a switch --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", B_ARMS)
def test_scratch_across_a_switch(ctx, models, calls, b):
    """A = noise1 + scale2.0x chain on s1; B on s2 (device entry points) or on the context's own stream (host entry points)"""
    import torch
    seq = [calls["chain_su"], calls[b]]
    want = on_idle(ctx, models, seq)
    for call in seq:
        call.clear()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        queue(ctx, models, seq[0], s1)
        queue(ctx, models, seq[1], s2)
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(0)
    bad = {k: mismatches(call.results(), w) for k, call, w in zip("AB", seq, want)}
    assert not any(bad.values()), bad


def test_ordering_through_two_switches(ctx, models, calls):
    """A on s1, a plane on s2, tiles on the context's own stream; w2x_ctx_synchronize on the last stream covers all three"""
    import torch
    seq = [calls["chain_su"], calls["plane_device"], calls["tiles_device"]]
    want = on_idle(ctx, models, seq)
    for call in seq:
        call.clear()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        queue(ctx, models, seq[0], s1)
        queue(ctx, models, seq[1], s2)
        ctx.set_stream(0)
        seq[2].run(ctx, models)
        ctx.synchronize()
        got = [call.results() for call in seq]
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(0)
    bad = {k: mismatches(g, w) for k, g, w in zip(("s1", "s2", "own"), got, want)}
    assert not any(bad.values()), bad


# ---- ordering on the caller's stream, with no host synchronise -----------------------------------------------------------------
@pytest.mark.parametrize("arm", C_ARMS)
def test_order_on_the_callers_stream(w2x, oracle_models, ctx, models, calls, arm):
    import torch
    call = calls[arm]
    want = on_idle(ctx, models, [call])[0]
    unseen = {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}   # uploaded inside the call
    vals = [t.clone() for t in call.ins]
    for t in call.ins:
        t.fill_(float("nan"))
    call.clear()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    try:
        with torch.cuda.stream(s):
            torch.cuda._sleep(LONG)
            for t, v in zip(call.ins, vals):
                t.copy_(v)
            ctx.set_stream(s.cuda_stream)
            call.run(ctx, unseen)
            read = [o.clone() for o in call.outs]
        s.synchronize()
        got = [r.cpu().numpy() for r in read]
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(0)
        for t, v in zip(call.ins, vals):
            t.copy_(v)
        torch.cuda.synchronize()
        for m in unseen.values():
            ctx.forget_model(m)
    assert not mismatches(got, want)


# ---- two contexts, two host threads --------------------------------------------------------------------------------------------
def thread_data(rng):
    w, h = 800, 600
    return {"plane": rand(rng, 768, 1024), "planes": [rand(rng, h, w) for w, h in sizes(rng, 20, 40, 300)],
            "chain": rand(rng, 300, 400), "x": dev(rand(rng, h, w)), "y": empty(h, w), "wh": (w, h)}


def sequence(ctx, M, d, stream):
    """host plane, host planes, host noise + 2x chain, then a device plane on `stream`"""
    import torch
    outs = [ctx.convert_plane(M["noise2"], d["plane"])]
    outs += ctx.convert_planes(M["noise1"], d["planes"])
    outs.append(ctx.convert_chain(steps(M, "SU"), d["chain"]))
    w, h = d["wh"]
    with torch.cuda.stream(stream):
        d["y"].fill_(float("nan"))
        ctx.set_stream(stream.cuda_stream)
        ctx.convert_plane_device(M["noise2"], d["x"].data_ptr(), w, h, w * 4, d["y"].data_ptr(), w * 4)
        ctx.synchronize()
    ctx.set_stream(0)
    outs.append(d["y"].cpu().numpy())
    return outs


def test_two_contexts_on_two_threads(w2x, ctx, models):
    import torch
    rng = np.random.default_rng(23)
    data = [thread_data(rng) for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    torch.cuda.synchronize()
    want = [sequence(ctx, models, d, s) for d, s in zip(data, streams)]   # serial, on one idle context
    L = w2x.lib()
    x = rand(rng, 4, 16, 16)
    out = np.empty_like(x)
    barrier = threading.Barrier(2, timeout=120)
    got, failed, errors = [None, None], [None, None], []
    ctxs = [w2x.Context(0, engine=w2x.ENGINE_TC) for _ in range(2)]

    def worker(i):
        try:
            got[i] = [sequence(ctxs[i], models, data[i], streams[i]) for _ in range(2)]
            ip = (C.c_void_p * 4)(*[x[t].ctypes.data for t in range(4)])
            op = (C.c_void_p * 4)(*[out[t].ctypes.data if t != i else None for t in range(4)])
            barrier.wait()
            rc = L.w2x_convert_tiles(ctxs[i]._h, models["noise2"]._h, ip, op, 4, 16, 16, 64, 64)
            barrier.wait()                        # the other thread's call has failed too
            failed[i] = (rc, L.w2x_last_error().decode())
        except BaseException as e:                # reported by the main thread
            errors.append((i, repr(e)))
            barrier.abort()

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        torch.cuda.synchronize()
        for c in ctxs:
            c.close()
    assert not errors, errors
    for i in range(2):
        for r in range(2):
            assert not mismatches(got[i][r], want[i]), (i, r, mismatches(got[i][r], want[i]))
        assert failed[i] == (ERR_ARG, f"w2x_convert_tiles: NULL tile {i}"), failed[i]
