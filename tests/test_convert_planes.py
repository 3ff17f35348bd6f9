"""w2x_convert_planes / w2x_convert_planes_device: independent planes of any sizes packed side by side into frames.

  * CPU: the frame planner (w2x_debug_plan_planes, no device) -- rectangles never overlap and lie inside their frame, every
    frame stays within the scratch limit and the row limit, every plane is placed exactly once or converted alone;
  * GPU: every plane bit for bit (np.array_equal) against convert_plane on that plane alone, in all three tensor-core
    precisions, on the shipped and random 1 -> C1 -> C2 -> 1 models, through the host and the device entry point, with strided
    inputs and outputs, many frames, a plane too large to pack, the fp32 engine and the fuse-off probe; one mix against the CPU
    oracle; the launch count (n + 1 per frame); argument errors; the progress lines.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_parity import TC_TOL

MAX_ROWS = 8 * 65535
FIXED_SIZES = [(1, 1), (1, 300), (300, 1), (15, 13), (16, 16), (17, 9), (129, 77), (511, 3), (512, 512), (700, 300)]


def random_sizes(seed, n=200, lo=1, hi=160):
    rng = np.random.default_rng(seed)
    return [(int(w), int(h)) for w, h in rng.integers(lo, hi + 1, size=(n, 2))]


def check_plan(w2x, sizes, n_layers, maxc, limit):
    ws, hs = [s[0] for s in sizes], [s[1] for s in sizes]
    frame, x0, y0, dims = w2x.debug_plan_planes(ws, hs, n_layers, maxc, limit)
    px_limit = limit // (maxc * 4)
    dims = dims.astype(np.int64)
    for fw, fh in dims:
        assert fw >= 1 and fh >= 1
        assert fw * fh * maxc * 4 <= limit, (fw, fh)          # tc::act_bytes(maxc, fw, fh) within the scratch limit
        assert fh <= MAX_ROWS
    occupancy = [np.zeros((fh, fw), np.uint8) for fw, fh in dims]
    for i, (w, h) in enumerate(sizes):
        pw, ph = w + 2 * n_layers, h + 2 * n_layers
        f = frame[i]
        if f < 0:   # converted alone: only when its rectangle cannot fit a frame
            assert pw * ph > px_limit or ph > MAX_ROWS or ph * max(pw, dims[:, 0].max(initial=0)) > px_limit, (w, h)
            continue
        assert 0 <= f < len(dims)
        fw, fh = dims[f]
        assert 0 <= x0[i] and x0[i] + pw <= fw and 0 <= y0[i] and y0[i] + ph <= fh, (i, w, h, x0[i], y0[i], fw, fh)
        occupancy[f][y0[i]:y0[i] + ph, x0[i]:x0[i] + pw] += 1
    for occ in occupancy:
        assert occ.max() <= 1                                  # rectangles never overlap
        assert occ.any()                                       # no empty frame
    return frame, dims


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("limit_mb", [16 << 10, 64, 8])
def test_plan_invariants(w2x, seed, limit_mb):
    sizes = FIXED_SIZES + [(1, 2000), (2000, 1)] + random_sizes(seed)
    frame, dims = check_plan(w2x, sizes, 7, 128, limit_mb << 20)
    if limit_mb == 16 << 10:   # the default limit: everything packs, into one frame
        assert (frame >= 0).all() and len(dims) == 1
        # without the 2000-pixel strips (whose shelf is mostly empty) the frame wastes little
        sizes = FIXED_SIZES + random_sizes(seed)
        frame, dims = check_plan(w2x, sizes, 7, 128, limit_mb << 20)
        area = sum((w + 14) * (h + 14) for w, h in sizes)
        assert len(dims) == 1 and dims[0, 0] * dims[0, 1] <= 1.3 * area


def test_plan_small_limits_and_single_path(w2x):
    sizes = random_sizes(5, 300, 1, 200)
    for n_layers, maxc in ((7, 128), (3, 32), (5, 64)):
        for limit in (1 << 20, 3 << 20, 1 << 26):
            check_plan(w2x, sizes, n_layers, maxc, limit)
    # one plane too large for any frame: placed nowhere, the others packed
    frame, dims = check_plan(w2x, [(100, 100), (800, 800), (50, 20)], 7, 128, 16 << 20)
    assert list(frame >= 0) == [True, False, True]
    # a tall thin plane with more rows than a frame may have
    frame, _ = check_plan(w2x, [(1, MAX_ROWS), (10, 10)], 7, 32, 1 << 40)
    assert list(frame >= 0) == [False, True]


def test_plan_arguments(w2x):
    with pytest.raises(w2x.W2xError):
        w2x.debug_plan_planes([], [])
    with pytest.raises(w2x.W2xError, match="plane 1"):
        w2x.debug_plan_planes([4, 0], [4, 4])


# ================================================================================================ GPU
PRECISIONS = [0, 1, 2]   # f16x3, f16+f8x2, f16


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


def random_model(w2x, c1, c2, seed):
    rng = np.random.default_rng(seed)
    ws = [rng.normal(0, 1 / 3, (c1, 1, 3, 3)), rng.normal(0, 1 / np.sqrt(9 * c1), (c2, c1, 3, 3)),
          rng.normal(0, 1 / np.sqrt(9 * c2), (1, c2, 3, 3))]
    bs = [rng.normal(0, 0.1, c1), rng.normal(0, 0.1, c2), rng.normal(0, 0.1, 1)]
    return w2x.Model.from_arrays([w.astype(np.float32) for w in ws], bs)


def planes_for(oracle_mod, sizes, seed):
    return [oracle_mod.seeded_plane(w, h, seed + i, "uniform") for i, (w, h) in enumerate(sizes)]


def assert_each_equal(ctx, model, planes, got):
    bad = [i for i, x in enumerate(planes) if not np.array_equal(got[i], ctx.convert_plane(model, x, block_splitting=False))]
    assert not bad, [(i, planes[i].shape) for i in bad[:10]]


@pytest.fixture
def ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_sizes_equal_plane_by_plane(w2x, ctx, shipped, oracle_mod, precision):
    ctx.set_precision(precision)
    planes = planes_for(oracle_mod, FIXED_SIZES + random_sizes(precision), 1000)
    models = list(shipped.values()) + [random_model(w2x, c1, c2, 7 * c1 + c2) for c1, c2 in ((32, 32), (64, 128), (128, 32))]
    for model in models:
        assert_each_equal(ctx, model, planes, ctx.convert_planes(model, planes))


@pytest.mark.gpu
def test_many_frames_and_a_plane_too_large(w2x, ctx, shipped, oracle_mod):
    model = shipped["noise2"]
    limit = 6 << 20
    ctx.set_scratch_limit(limit)
    sizes = random_sizes(11, 60, 1, 64) + [(300, 280)]
    frame, _, _, dims = w2x.debug_plan_planes([s[0] for s in sizes], [s[1] for s in sizes], 7, 128, limit)
    assert len(dims) >= 3 and frame[-1] == -1 and (frame[:-1] >= 0).all()
    planes = planes_for(oracle_mod, sizes, 50)
    for precision in PRECISIONS:
        ctx.set_precision(precision)
        assert_each_equal(ctx, model, planes, ctx.convert_planes(model, planes))


def strided_views(planes, pad, fill):
    """Each plane inside a wider buffer (row stride = width + pad floats), plus an output view of the same layout."""
    ins, outs, bufs = [], [], []
    for x in planes:
        h, w = x.shape
        b = np.full((h, w + pad), -7.0, np.float32)
        b[:, :w] = x
        ins.append(b[:, :w])
        o = np.full((h, w + pad), fill, np.float32)
        bufs.append(o)
        outs.append(o[:, :w])
    return ins, outs, bufs


@pytest.mark.gpu
def test_strided_host_and_device(w2x, ctx, shipped, oracle_mod):
    import torch
    model = shipped["scale2.0x"]
    sizes = FIXED_SIZES[:8] + random_sizes(3, 40)
    planes = planes_for(oracle_mod, sizes, 300)
    want = [ctx.convert_plane(model, x, block_splitting=False) for x in planes]
    sentinel = np.float32(12345.5)
    ins, outs, bufs = strided_views(planes, 5, sentinel)
    ctx.convert_planes(model, ins, out=outs)
    for i, (o, b) in enumerate(zip(outs, bufs)):
        assert np.array_equal(o, want[i]), i
        assert (b[:, o.shape[1]:] == sentinel).all(), i      # the stride padding is untouched
    # device planes with strides, asynchronous on the context's stream
    d_in = [torch.from_numpy(np.ascontiguousarray(b)).cuda() for b in strided_views(planes, 3, 0)[2]]
    for d, x in zip(d_in, planes):
        d[:, :x.shape[1]] = torch.from_numpy(x).cuda()
    d_out = [torch.full((x.shape[0], x.shape[1] + 9), float(sentinel), device="cuda") for x in planes]
    torch.cuda.synchronize()
    ctx.convert_planes_device(model, [d.data_ptr() for d in d_in], [x.shape[1] for x in planes], [x.shape[0] for x in planes],
                              [d.stride(0) * 4 for d in d_in], [d.data_ptr() for d in d_out], [d.stride(0) * 4 for d in d_out])
    ctx.synchronize()
    for i, (d, x) in enumerate(zip(d_out, planes)):
        got = d.cpu().numpy()
        assert np.array_equal(got[:, :x.shape[1]], want[i]), i
        assert (got[:, x.shape[1]:] == sentinel).all(), i


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fuse_off"])
def test_plane_by_plane_cases(w2x, shipped, oracle_mod, mode):
    c = w2x.Context(0, engine=w2x.ENGINE_FP32 if mode == "fp32" else w2x.ENGINE_TC)
    try:
        if mode == "fuse_off":
            c.debug_set_fuse_last(0)
        planes = planes_for(oracle_mod, FIXED_SIZES[:6] + random_sizes(9, 20, 1, 90), 700)
        model = shipped["noise1"]
        assert_each_equal(c, model, planes, c.convert_planes(model, planes))
    finally:
        c.close()


@pytest.mark.gpu
def test_against_the_oracle(ctx, shipped, oracle_models, oracle_mod):
    ctx.set_precision(0)   # f16x3, the precision TC_TOL states
    sizes = [(1, 1), (15, 13), (40, 7), (64, 64), (97, 33)]
    planes = planes_for(oracle_mod, sizes, 900)
    om = oracle_models["scale2.0x"]
    got = ctx.convert_planes(shipped["scale2.0x"], planes)
    for x, y in zip(planes, got):
        assert np.abs(y - om.convert(x, n_job=4)).max() <= TC_TOL


@pytest.mark.gpu
def test_launch_count_per_frame(w2x, ctx, shipped, oracle_mod):
    model = shipped["noise2"]
    n = len(model)
    for limit, count in ((16 << 30, 300), (2 << 20, 40)):
        ctx.set_scratch_limit(limit)
        sizes = random_sizes(limit % 97, count, 1, 48)
        frame, _, _, dims = w2x.debug_plan_planes([s[0] for s in sizes], [s[1] for s in sizes], n, 128, limit)
        assert (frame >= 0).all()
        planes = planes_for(oracle_mod, sizes, 5)
        n0 = ctx.launch_count()
        ctx.convert_planes(model, planes)
        assert ctx.launch_count() - n0 == (n + 1) * len(dims)
        if limit == 16 << 30:
            assert len(dims) == 1


@pytest.mark.gpu
def test_argument_errors(w2x, ctx, shipped):
    L = w2x.lib()
    model = shipped["noise2"]
    planes = [np.zeros((8, 8), np.float32) for _ in range(5)]
    outs = [np.zeros((8, 8), np.float32) for _ in range(5)]

    def call(n, ptr_in, ws, hs, strides):
        ip = (C.c_void_p * 5)(*ptr_in)
        op = (C.c_void_p * 5)(*[o.ctypes.data for o in outs])
        st = (C.c_size_t * 5)(*strides)
        r = L.w2x_convert_planes(ctx._h, model._h, n, ip, (C.c_int * 5)(*ws), (C.c_int * 5)(*hs), st, op, st)
        return r, L.w2x_last_error().decode()

    ptrs = [p.ctypes.data for p in planes]
    ok = call(5, ptrs, [8] * 5, [8] * 5, [32] * 5)
    assert ok[0] == 0, ok
    r, msg = call(5, ptrs[:3] + [None] + ptrs[4:], [8] * 5, [8] * 5, [32] * 5)
    assert r == 1 and "plane 3" in msg, msg
    r, msg = call(5, ptrs, [8, 8, 0, 8, 8], [8] * 5, [32] * 5)
    assert r == 1 and "plane 2" in msg, msg
    r, msg = call(5, ptrs, [8] * 5, [8] * 5, [32, 32, 32, 32, 28])
    assert r == 1 and "plane 4" in msg, msg
    r, msg = call(5, ptrs, [8] * 5, [8] * 5, [32, 30, 32, 32, 32])
    assert r == 1 and "plane 1" in msg, msg
    r, msg = call(0, ptrs, [8] * 5, [8] * 5, [32] * 5)
    assert r == 1 and "n_planes" in msg, msg
    with pytest.raises(w2x.W2xError) as e:
        ctx.convert_planes_device(model, [0], [8], [8], [32], [0], [32])
    assert e.value.status == 1 and "plane 0" in e.value.message


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tc", "fp32"])
def test_progress_lines(w2x, shipped, oracle_mod, engine):
    c = w2x.Context(0, engine=w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    try:
        model = shipped["noise2"]
        planes = planes_for(oracle_mod, [(5, 9), (30, 2), (64, 64)], 1)
        lines = []
        c.set_log(lines.append)
        for x in planes:
            c.convert_plane(model, x, block_splitting=False)
        want = list(lines)
        lines.clear()
        c.convert_planes(model, planes)
        assert lines == want and len(want) == 3 * len(model)
    finally:
        c.close()
