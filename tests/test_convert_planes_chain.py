"""w2x_convert_planes_chain / w2x_convert_planes_chain_device: the noise and 2x scale chain of w2x_convert_chain on a whole
collection of planes of different sizes, each step packing the planes into frames as w2x_convert_planes does, and an upscaling step
packing straight from the half-resolution planes.

Every output is checked bit for bit (np.array_equal) against the per-plane convert_chain(block_splitting=False) and against the
per-step loop of convert_planes on the resized planes: in all three precisions, on patterns U, SU, UU, SUU and US, with the shipped
models and random 1 -> C1 -> C2 -> 1 models of different widths, on collections of 1 to 300 planes with sides from 1 to 160.  Also:
plans that change between steps, both entry points with strided planes and a torch stream, the fp32 engine and the fuse-off probe,
the one-step case against convert_planes, launch counts, on_step calls and progress lines, rejected calls, W2X_ERR_NOMEM, and the CPU
oracle.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_convert_chain import steps_for, up2
from test_convert_planes import planes_for, random_model
from test_gpu_parity import TC_TOL

pytestmark = pytest.mark.gpu

PRECISIONS = [0, 1, 2]   # f16x3, f16+f8x2, f16
PATTERNS = ["U", "SU", "UU", "SUU", "US"]
EDGES = [(1, 1), (1, 37), (37, 1), (1, 160), (160, 1), (160, 160), (15, 13)]
COUNTS = {"U": 1, "SU": 7, "UU": 60, "SUU": 300, "US": 25}   # planes per collection
ERR_ARG, ERR_UNSUPPORTED, ERR_NOMEM = 1, 7, 8
STEP_FN = C.CFUNCTYPE(None, C.c_int, C.c_void_p)


def sizes_for(seed, n, hi=160, edges=True):
    rng = np.random.default_rng(seed)
    out = (EDGES if edges else []) + [(int(w), int(h)) for w, h in rng.integers(1, hi + 1, size=(n, 2))]
    return out[:n]


def chain_loop(ctx, steps, planes):
    """the per-plane reference"""
    return [ctx.convert_chain(steps, x, block_splitting=False) for x in planes]


def step_loop(ctx, steps, planes, on_step=None):
    """the per-step reference: convert_planes on the resized planes"""
    ys = planes
    for k, (model, up) in enumerate(steps):
        if on_step is not None:
            on_step(k)
        ys = ctx.convert_planes(model, [up2(y) if up else y for y in ys])
    return ys


def dev(xs):
    ds = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]
    torch.cuda.synchronize()
    return ds


def ptrs(ds):
    return [d.data_ptr() for d in ds]


def device_chain(ctx, steps, planes, on_step=None):
    ups = sum(up for _, up in steps)
    d_in = dev(planes)
    d_out = [torch.empty((x.shape[0] << ups, x.shape[1] << ups), device="cuda") for x in planes]
    torch.cuda.synchronize()
    ctx.convert_planes_chain_device(steps, ptrs(d_in), [x.shape[1] for x in planes], [x.shape[0] for x in planes],
                                    [x.shape[1] * 4 for x in planes], ptrs(d_out), [(x.shape[1] << ups) * 4 for x in planes], on_step)
    ctx.synchronize()
    return [d.cpu().numpy() for d in d_out]


def device_step_loop(ctx, steps, planes, on_step=None):
    """the per-step reference on the device: convert_planes_device, repeat_interleave between steps -> (outputs, launches)"""
    ys, launches = dev(planes), 0
    for k, (model, up) in enumerate(steps):
        xs = [y.repeat_interleave(2, 0).repeat_interleave(2, 1).contiguous() if up else y for y in ys]
        outs = [torch.empty_like(x) for x in xs]
        torch.cuda.synchronize()
        if on_step is not None:
            on_step(k)
        n0 = ctx.launch_count()
        ctx.convert_planes_device(model, ptrs(xs), [x.shape[1] for x in xs], [x.shape[0] for x in xs], [x.shape[1] * 4 for x in xs],
                                  ptrs(outs), [x.shape[1] * 4 for x in xs])
        launches += ctx.launch_count() - n0
        ctx.synchronize()
        ys = outs
    return [y.cpu().numpy() for y in ys], launches


def assert_all_equal(got, want, what):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if not np.array_equal(g, w)]
    assert len(got) == len(want) and not bad, (what, bad[:10])


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.fixture(scope="module")
def randoms(w2x):
    return random_model(w2x, 32, 64, 21), random_model(w2x, 128, 32, 22)


@pytest.fixture
def ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.set_log(None)
    c.close()


# ---- results, bit for bit ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("models", ["shipped", "random"])
def test_patterns_and_collections(ctx, shipped, randoms, oracle_mod, precision, models):
    ctx.set_precision(precision)
    same, scale = (shipped["noise1"], shipped["scale2.0x"]) if models == "shipped" else randoms
    for j, pattern in enumerate(PATTERNS):
        planes = planes_for(oracle_mod, sizes_for(10 * precision + j, COUNTS[pattern]), 100 * j)
        steps = steps_for(pattern, same, scale)
        want = chain_loop(ctx, steps, planes)
        got = ctx.convert_planes_chain(steps, planes)
        assert_all_equal(got, want, (pattern, "per-plane chain"))
        assert_all_equal(step_loop(ctx, steps, planes), want, (pattern, "per-step loop"))
        if COUNTS[pattern] <= 60:
            assert_all_equal(device_chain(ctx, steps, planes), want, (pattern, "device"))


def test_plans_that_change_between_steps(w2x, ctx, shipped, oracle_mod):
    """a 100 x 100 plane packs at step 0 and goes alone once doubled; then a limit that cuts every step into many frames"""
    same, scale = shipped["noise1"], shipped["scale2.0x"]
    n = len(same)
    limit = 8 << 20
    sizes = [(100, 100)] + sizes_for(3, 30, 40, edges=False)     # no wide plane widens the frames
    frame0 = w2x.debug_plan_planes([w for w, _ in sizes], [h for _, h in sizes], n, 128, limit)[0]
    frame1 = w2x.debug_plan_planes([2 * w for w, _ in sizes], [2 * h for _, h in sizes], n, 128, limit)[0]
    assert frame0[0] >= 0 and frame1[0] == -1
    planes = planes_for(oracle_mod, sizes, 40)
    steps = steps_for("SU", same, scale)
    ctx.set_scratch_limit(limit)
    want = chain_loop(ctx, steps, planes)
    assert_all_equal(ctx.convert_planes_chain(steps, planes), want, "host, one plane alone after 2x")
    assert_all_equal(device_chain(ctx, steps, planes), want, "device, one plane alone after 2x")

    sizes = sizes_for(4, 80, 24, edges=False)
    for k, s in enumerate((1, 2, 4)):
        frame, _, _, dims = w2x.debug_plan_planes([s * w for w, _ in sizes], [s * h for _, h in sizes], n, 128, limit)
        assert len(dims) >= 5 and (frame >= 0).all(), (k, len(dims))
    planes = planes_for(oracle_mod, sizes, 80)
    steps = steps_for("SUU", same, scale)
    want = chain_loop(ctx, steps, planes)
    assert_all_equal(ctx.convert_planes_chain(steps, planes), want, "host, many frames")
    assert_all_equal(device_chain(ctx, steps, planes), want, "device, many frames")


def test_strided_planes_and_a_torch_stream(ctx, shipped, oracle_mod):
    steps = steps_for("SU", shipped["noise1"], shipped["scale2.0x"])
    planes = planes_for(oracle_mod, sizes_for(5, 40, 90), 500)
    want = chain_loop(ctx, steps, planes)
    sentinel = np.float32(12345.5)
    ins, outs, bufs = [], [], []
    for x in planes:
        h, w = x.shape
        b = np.full((h, w + 5), -7.0, np.float32)
        b[:, :w] = x
        ins.append(b[:, :w])
        o = np.full((2 * h, 2 * w + 3), sentinel, np.float32)
        bufs.append(o)
        outs.append(o[:, :2 * w])
    ctx.convert_planes_chain(steps, ins, out=outs)
    assert_all_equal(outs, want, "host strided")
    assert all((b[:, o.shape[1]:] == sentinel).all() for o, b in zip(outs, bufs))

    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            d_in = [torch.full((x.shape[0], x.shape[1] + 3), -7.0, device="cuda") for x in planes]
            for d, x in zip(d_in, planes):
                d[:, :x.shape[1]] = torch.from_numpy(x).cuda()
            d_out = [torch.full((2 * x.shape[0], 2 * x.shape[1] + 9), float(sentinel), device="cuda") for x in planes]
            ctx.convert_planes_chain_device(steps, ptrs(d_in), [x.shape[1] for x in planes], [x.shape[0] for x in planes],
                                            [d.stride(0) * 4 for d in d_in], ptrs(d_out), [d.stride(0) * 4 for d in d_out])
            got = [d.cpu().numpy() for d in d_out]      # ordered after the chain on the same stream
        assert_all_equal([g[:, :2 * x.shape[1]] for g, x in zip(got, planes)], want, "device strided, torch stream")
        assert all((g[:, 2 * x.shape[1]:] == sentinel).all() for g, x in zip(got, planes))
    finally:
        ctx.set_stream(0)


@pytest.mark.parametrize("mode", ["fp32", "fuse_off"])
def test_engines_that_do_not_pack(w2x, shipped, oracle_mod, mode):
    c = w2x.Context(0, engine=w2x.ENGINE_FP32 if mode == "fp32" else w2x.ENGINE_TC)
    try:
        if mode == "fuse_off":
            c.debug_set_fuse_last(0)
        planes = planes_for(oracle_mod, sizes_for(6, 16, 70), 600)
        for pattern in ("SU", "US"):
            steps = steps_for(pattern, shipped["noise1"], shipped["scale2.0x"])
            want = chain_loop(c, steps, planes)
            assert_all_equal(c.convert_planes_chain(steps, planes), want, (mode, pattern, "host"))
            assert_all_equal(device_chain(c, steps, planes), want, (mode, pattern, "device"))
    finally:
        c.close()


@pytest.mark.parametrize("engine", ["tc", "fp32"])
def test_one_step_is_convert_planes(w2x, shipped, oracle_mod, engine):
    c = w2x.Context(0, engine=w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    try:
        model = shipped["noise2"]
        planes = planes_for(oracle_mod, sizes_for(7, 30, 100) + [(300, 280)], 700)
        c.set_scratch_limit(6 << 20)      # several frames and a plane converted alone
        lines = []
        c.set_log(lines.append)
        results = {}
        for name, call in (("planes", lambda: c.convert_planes(model, planes)),
                           ("chain", lambda: c.convert_planes_chain([(model, False)], planes)),
                           ("planes_device", lambda: device_step_loop(c, [(model, False)], planes)[0]),
                           ("chain_device", lambda: device_chain(c, [(model, False)], planes))):
            lines.clear()
            n0 = c.launch_count()
            out = call()
            results[name] = (out, list(lines), c.launch_count() - n0)
        for host, dev_ in (("planes", "chain"), ("planes_device", "chain_device")):
            assert_all_equal(results[dev_][0], results[host][0], dev_)
            assert results[dev_][1] == results[host][1] and results[dev_][2] == results[host][2], dev_
        assert results["planes"][1] and results["planes"][2] > 0
    finally:
        c.close()


@pytest.mark.parametrize("limit", [16 << 30, 3 << 20])
def test_launch_count_is_the_per_step_sum(ctx, shipped, oracle_mod, limit):
    ctx.set_scratch_limit(limit)
    steps = steps_for("SUU", shipped["noise1"], shipped["scale2.0x"])
    planes = planes_for(oracle_mod, sizes_for(8, 50, 64), 800)
    want, per_step = device_step_loop(ctx, steps, planes)
    n0 = ctx.launch_count()
    got = device_chain(ctx, steps, planes)
    assert ctx.launch_count() - n0 == per_step
    n0 = ctx.launch_count()
    ctx.convert_planes_chain(steps, planes)
    assert ctx.launch_count() - n0 == per_step
    assert_all_equal(got, want, "device per-step loop")


@pytest.mark.parametrize("engine", ["tc", "fp32"])
def test_on_step_and_progress_lines(w2x, shipped, oracle_mod, engine):
    c = w2x.Context(0, engine=w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    try:
        c.set_scratch_limit(8 << 20)       # the 2x planes of 150 x 120 go alone, in scratch bands
        steps = steps_for("SUS", shipped["noise1"], shipped["scale2.0x"])
        planes = planes_for(oracle_mod, [(150, 120), (9, 17), (40, 5), (1, 1)], 900)
        got = []
        c.set_log(got.append)
        on_step = lambda k: got.append(("step", k))
        step_loop(c, steps, planes, on_step)
        want = list(got)
        got.clear()
        c.convert_planes_chain(steps, planes, on_step=on_step)
        assert got == want, "host"
        assert [g for g in want if isinstance(g, tuple)] == [("step", k) for k in range(3)]
        got.clear()
        device_step_loop(c, steps, planes, on_step)
        want = list(got)
        got.clear()
        device_chain(c, steps, planes, on_step)
        assert got == want, "device"
    finally:
        c.close()


# ---- rejected calls -----------------------------------------------------------------------------------------------------------
def test_rejected_calls(w2x, ctx, shipped):
    L = w2x.lib()
    rng = np.random.default_rng(5)
    one_to_two = w2x.Model.from_arrays([rng.normal(0, 0.3, (co, ci, 3, 3)).astype(np.float32) for ci, co in ((1, 32), (32, 64), (64, 2))],
                                       [rng.normal(0, 0.1, co) for co in (32, 64, 2)])
    no_tc = w2x.Model.from_arrays([rng.normal(0, 0.3, (co, ci, 3, 3)).astype(np.float32) for ci, co in ((1, 8), (8, 16), (16, 1))],
                                  [rng.normal(0, 0.1, co) for co in (8, 16, 1)])
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    n = 4
    planes = [np.full((8, 8), 0.5, np.float32) for _ in range(n)]
    sentinel = np.float32(-3.25)
    outs = [np.full((16, 16), sentinel, np.float32) for _ in range(n)]
    d_in = dev(planes)
    d_out = [torch.full((16, 16), float(sentinel), device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    lines = []
    ctx.set_log(lines.append)

    def call(host, models=(noise, scale), kinds=(0, 1), n_steps=2, n_planes=n, ws=(8,) * n, hs=(8,) * n, ist=(32,) * n,
             ost=(64,) * n, null_in=None, null_out=None, null_array=None):
        ins = [x.ctypes.data for x in planes] if host else ptrs(d_in)
        os_ = [o.ctypes.data for o in outs] if host else ptrs(d_out)
        if null_in is not None:
            ins[null_in] = None
        if null_out is not None:
            os_[null_out] = None
        args = {"models": (C.c_void_p * 2)(*[m._h if m is not None else None for m in models]), "kinds": (C.c_int * 2)(*kinds),
                "in": (C.c_void_p * n)(*ins), "ws": (C.c_int * n)(*ws), "hs": (C.c_int * n)(*hs), "ist": (C.c_size_t * n)(*ist),
                "out": (C.c_void_p * n)(*os_), "ost": (C.c_size_t * n)(*ost)}
        if null_array is not None:
            args[null_array] = None
        fn = L.w2x_convert_planes_chain if host else L.w2x_convert_planes_chain_device
        return fn(ctx._h, n_steps, args["models"], args["kinds"], n_planes, args["in"], args["ws"], args["hs"], args["ist"], args["out"],
                  args["ost"], STEP_FN(), None)

    cases = [
        ("n_steps", ERR_ARG, "n_steps", dict(n_steps=0)),
        ("n_planes", ERR_ARG, "n_planes", dict(n_planes=0)),
        ("no models array", ERR_ARG, "step 0", dict(null_array="models")),
        ("no kinds array", ERR_ARG, "step 0", dict(null_array="kinds")),
        ("no widths array", ERR_ARG, "NULL array", dict(null_array="ws")),
        ("no out strides array", ERR_ARG, "NULL array", dict(null_array="ost")),
        ("null model", ERR_ARG, "step 1", dict(models=(noise, None))),
        ("unknown kind", ERR_ARG, "step 1", dict(kinds=(0, 2))),
        ("1 -> 2 model", ERR_ARG, "step 1", dict(models=(noise, one_to_two))),
        ("null input plane", ERR_ARG, "plane 2", dict(null_in=2)),
        ("null output plane", ERR_ARG, "plane 3", dict(null_out=3)),
        ("empty plane", ERR_ARG, "plane 1", dict(ws=(8, 0, 8, 8))),
        ("overflow", ERR_ARG, "plane 1", dict(kinds=(1, 1), ws=(8, 1 << 29, 8, 8), hs=(8, 1, 8, 8), ost=(128,) * n)),
        ("input stride not a multiple of 4", ERR_ARG, "plane 1", dict(ist=(32, 34, 32, 32))),
        ("input stride short", ERR_ARG, "plane 0", dict(ist=(28, 32, 32, 32))),
        ("output stride short of the 2x row", ERR_ARG, "plane 2", dict(ost=(64, 64, 32, 64))),
        ("engine refuses", ERR_UNSUPPORTED, "step 1", dict(models=(noise, no_tc))),
    ]
    for host in (True, False):
        for name, status, where, kw in cases:
            ctx.synchronize()
            lines.clear()
            n0 = ctx.launch_count()
            rc = call(host, **kw)
            ctx.synchronize()
            msg = L.w2x_last_error().decode()
            assert (rc, lines, ctx.launch_count() - n0) == (status, [], 0), (host, name, msg)
            assert where in msg, (host, name, msg)
    assert all((o == sentinel).all() for o in outs)
    assert all(bool((d == float(sentinel)).all()) for d in d_out)
    assert call(True) == 0 and call(False) == 0      # the same arguments, unbroken, go through


def test_out_of_memory_leaves_nothing_queued(w2x, shipped, oracle_mod):
    """with the device all but full, a collection whose frame has its buffers already but whose plane converted alone cannot reserve
    its scratch returns W2X_ERR_NOMEM before any on_step call, progress line or launch, the frame's included"""
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    filler = None
    try:
        steps = [(shipped["noise1"], False)]
        c.set_scratch_limit(256 << 20)      # frames of at most 256 MiB / (128 channels x 4 bytes) = 512 Ki pixels
        small, large = planes_for(oracle_mod, [(64, 64), (1024, 1024)], 7)   # padded 78 x 78 packs, 1038 x 1038 does not
        device_chain(c, steps, [small])     # the model's device copy and the frame's buffers exist
        d_in = dev([small, large])
        d_out = [torch.full(x.shape, -3.25, device="cuda") for x in (small, large)]
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        lines, calls = [], []
        c.set_log(lines.append)
        n0 = c.launch_count()
        with pytest.raises(w2x.W2xError) as e:
            c.convert_planes_chain_device(steps, ptrs(d_in), [64, 1024], [64, 1024], [64 * 4, 1024 * 4], ptrs(d_out), [64 * 4, 1024 * 4],
                                          calls.append)
        assert e.value.status == ERR_NOMEM, e.value.message
        assert c.launch_count() == n0 and not calls and not lines
        c.synchronize()
        assert all(bool((d == -3.25).all()) for d in d_out)
    finally:
        c.set_log(None)
        del filler
        torch.cuda.empty_cache()
        c.close()


def test_against_the_oracle(ctx, shipped, oracle_models, oracle_mod):
    """each step of a noise1 + scale2.0x collection against the CPU oracle on the GPU's previous step"""
    ctx.set_precision(0)   # f16x3, the precision TC_TOL states
    planes = planes_for(oracle_mod, [(1, 1), (15, 13), (40, 7), (33, 48)], 950)
    steps = [("noise1", False), ("scale2.0x", True)]
    prev = planes
    for k in range(len(steps)):
        got = ctx.convert_planes_chain([(shipped[m], up) for m, up in steps[:k + 1]], planes)
        name, up = steps[k]
        for x, y in zip(prev, got):
            ref = oracle_models[name].convert(up2(x) if up else x, n_job=4)
            assert np.abs(y - ref).max() <= TC_TOL, (k, x.shape)
        prev = got
