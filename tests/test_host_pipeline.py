"""The copy pipeline of the host-buffer entry points.

  * Ordering: a call starts its copies only after the work already queued on the context's stream.  w2x_convert_tiles_async on
    pinned tiles returns while its kernels still read the context's staging buffer; w2x_convert_plane (host copy bands),
    w2x_convert_tiles (copy groups), w2x_convert_planes (several frames) and w2x_convert_chain (a banded last step), called right
    after it on the same context, reuse that buffer without reallocating it.  Both results must equal, bit for bit, the same
    calls made on an idle context -- on the context's own stream and on a torch stream.
  * Argument errors: a NULL output tile or plane is reported with W2X_ERR_ARG before a single launch is queued.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ERR_ARG = 1
T, N_TILES = 512, 64                  # config 5: 64 tiles of 512 x 512, noise2
PLANES_LIMIT = 64 << 20               # packs PLANE_SIZES into several frames


def tiles_async(w2x, ctx, model, tiles, out):
    n, th, tw = tiles.shape
    ip = (C.c_void_p * n)(*[tiles[i].ctypes.data for i in range(n)])
    op = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    L = w2x.lib()
    rc = L.w2x_convert_tiles_async(ctx._h, model._h, ip, op, n, tw, th, tw * 4, tw * 4)
    if rc:
        raise w2x.W2xError(rc, L.w2x_last_error().decode())


@pytest.fixture(scope="module")
def setup(w2x, oracle_models):
    import torch
    models = {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}
    noise2 = models["noise2"]
    rng = np.random.default_rng(7)
    pinned = torch.empty((N_TILES, T, T), dtype=torch.float32).pin_memory()
    pinned_out = torch.empty((N_TILES, T, T), dtype=torch.float32).pin_memory()
    tiles = pinned.numpy()
    tiles[...] = rng.random((N_TILES, T, T), dtype=np.float32)
    plane_sizes = [(int(w), int(h)) for w, h in rng.integers(32, 201, size=(24, 2))]
    _, _, _, dims = w2x.debug_plan_planes([w for w, _ in plane_sizes], [h for _, h in plane_sizes], 7, 128, PLANES_LIMIT)
    assert len(dims) >= 2
    inputs = {
        "plane": rng.random((2048, 2048), dtype=np.float32),                       # 4 host copy bands
        "tiles": rng.random((16, T, T), dtype=np.float32),                         # 4 copy groups
        "planes": [rng.random((h, w), dtype=np.float32) for w, h in plane_sizes],
        "chain": rng.random((1024, 1024), dtype=np.float32),                       # last step 2048 x 2048: 4 bands
    }
    chain = [(models["noise1"], False), (models["scale2.0x"], True)]

    def run(ctx, arm):
        x = inputs[arm]
        if arm == "plane":
            return [ctx.convert_plane(noise2, x)]
        if arm == "tiles":
            return [ctx.convert_tiles(noise2, x)]
        if arm == "planes":
            ctx.set_scratch_limit(PLANES_LIMIT)
            try:
                return ctx.convert_planes(noise2, x)
            finally:
                ctx.set_scratch_limit(0)
        return [ctx.convert_chain(chain, x)]

    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    tiles_async(w2x, ctx, noise2, tiles, pinned_out.numpy())   # sizes the staging for every later call
    ctx.synchronize()
    want_tiles = pinned_out.numpy().copy()
    want = {arm: run(ctx, arm) for arm in inputs}
    yield dict(ctx=ctx, noise2=noise2, tiles=tiles, pinned=pinned, pinned_out=pinned_out, want_tiles=want_tiles, want=want, run=run)
    ctx.close()


@pytest.mark.parametrize("stream", ["own", "torch"])
@pytest.mark.parametrize("arm", ["plane", "tiles", "planes", "chain"])
def test_uploads_wait_for_queued_work(w2x, setup, arm, stream):
    import torch
    ctx = setup["ctx"]
    out = setup["pinned_out"].numpy()
    out.fill(np.nan)
    s = torch.cuda.Stream() if stream == "torch" else None
    if s is not None:
        ctx.set_stream(s.cuda_stream)
    try:
        tiles_async(w2x, ctx, setup["noise2"], setup["tiles"], out)
        got = setup["run"](ctx, arm)
        ctx.synchronize()
    finally:
        ctx.set_stream(0)
    assert np.array_equal(out, setup["want_tiles"]), "tiles"
    assert len(got) == len(setup["want"][arm])
    bad = [k for k, (g, w) in enumerate(zip(got, setup["want"][arm])) if not np.array_equal(g, w)]
    assert not bad, (arm, bad)


def test_bad_arguments_queue_nothing(w2x, setup):
    ctx, L = setup["ctx"], w2x.lib()
    model = setup["noise2"]
    x = np.random.default_rng(8).random((32, 16, 16), dtype=np.float32)
    out = np.empty_like(x)
    ip = (C.c_void_p * 32)(*[x[i].ctypes.data for i in range(32)])
    op = (C.c_void_p * 32)(*[out[i].ctypes.data for i in range(32)])
    op[2] = None
    n0 = ctx.launch_count()
    assert L.w2x_convert_tiles(ctx._h, model._h, ip, op, 4, 16, 16, 64, 64) == ERR_ARG
    assert L.w2x_last_error().decode() == "w2x_convert_tiles: NULL tile 2"
    assert L.w2x_convert_tiles_async(ctx._h, model._h, ip, op, 32, 16, 16, 64, 64) == ERR_ARG
    assert L.w2x_last_error().decode() == "w2x_convert_tiles: NULL tile 2"
    assert model.dims(1)[:2] == (32, 32)
    assert L.w2x_filter_layer(ctx._h, model._h, 1, ip, 32, op, 32, 16, 16, 64, 64) == ERR_ARG
    assert L.w2x_last_error().decode() == "w2x_filter_layer: NULL output plane 2"
    assert ctx.launch_count() == n0
    ctx.synchronize()
