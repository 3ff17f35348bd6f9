"""A context that has used every scratch buffer, stream and event it can own gives all of it back when it is closed.

One round creates a context, runs one small call of every family so that each buffer exists -- the host copy pipeline, the fp32
engine on the literal block walk (the padded plane), tiles, planes, a three-step planes chain with TTA steps (both chain buffers,
the TTA buffers, the frame tables), a single layer, timed calls (recorded spans and pooled events), the debug profile -- opens and
closes a band session with every pair of edge kinds and a slab of three sub-bands, forgets one model, leaves the other cached, and
closes the context.  Free device memory after a round must equal free device memory before it, and two rounds in one process must
produce the same bits.  The number watched is device-wide, as in test_frame_limits and test_tta: a neighbour's job can move it, so
the watched window holds nothing but the round.
"""
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BAND_W, BAND_ROWS = 40, 100


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(oracle_models[n].weights, oracle_models[n].biases) for n in ("noise1", "scale2.0x")}


@pytest.fixture(scope="module")
def data(oracle_mod):
    """every input of a round, and the device tensors of the band session, allocated before any memory is watched"""
    import torch
    plane = lambda w, h, seed: oracle_mod.seeded_plane(w, h, seed, "uniform")   # noqa: E731
    d = {"tall": plane(48, 1040, 1),                    # two row bands of the host copy pipeline
         "split": plane(640, 640, 2),                   # more than 1.5 blocks of 512 x 512: the literal walk cuts it
         "small": plane(45, 33, 3),
         "tiles": np.stack([plane(40, 40, 10 + i) for i in range(8)]),          # two groups of the copy pipeline
         "planes": [plane(w, h, 20 + w) for w, h in ((17, 9), (1, 5), (20, 20), (6, 31))],
         "layer": np.stack([plane(24, 18, 40 + i) for i in range(32)]),
         "band": plane(BAND_W, BAND_ROWS, 5)}
    d["d_band_in"] = torch.from_numpy(d["band"]).cuda()
    d["d_band_out"] = torch.empty_like(d["d_band_in"])
    torch.cuda.synchronize()
    return d


def one_round(w2x, shipped, data):
    """create -> use every buffer -> close; returns every output"""
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    out = {}
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        ctx.debug_tc_profile_enable(True)
        out["tall"] = ctx.convert_plane(scale, data["tall"])
        ctx.set_timing(True)
        out["timed"] = ctx.convert_plane(noise, data["small"])
        assert len(ctx.layer_times(reset=True)) == len(noise)        # the spans' events are pooled now ...
        out["timed again"] = ctx.convert_plane(scale, data["small"])   # ... and these spans are live when the context closes
        ctx.set_timing(False)
        out["tiles"] = ctx.convert_tiles(scale, data["tiles"])
        out["planes"] = np.concatenate([y.ravel() for y in ctx.convert_planes(noise, data["planes"])])
        steps = [(noise, False, True), (scale, True, False), (scale, True, True)]
        out["chain"] = np.concatenate([y.ravel() for y in ctx.convert_planes_chain(steps, data["planes"])])
        out["layer"] = ctx.filter_layer(scale, 1, data["layer"])

        ctx.set_engine(w2x.ENGINE_FP32)
        ctx.set_block_walk(w2x.WALK_BLOCKS)
        assert w2x.requires_splitting(*data["split"].shape[::-1])
        out["fp32 blocks"] = ctx.convert_plane(noise, data["split"])
        ctx.set_block_walk(w2x.WALK_FUSED)
        ctx.set_engine(w2x.ENGINE_TC)

        for up, down in itertools.product((0, 1, 2), repeat=2):
            w2x.Band(ctx, noise, BAND_W, BAND_ROWS, up, down).close()
        band = w2x.Band(ctx, noise, BAND_W, BAND_ROWS, 0, 0)
        try:
            band.load(data["d_band_in"].data_ptr(), BAND_W * 4)
            for k in range(band.steps):
                band.step(k)
            band.finish(data["d_band_out"].data_ptr(), BAND_W * 4)
            ctx.synchronize()
        finally:
            band.close()
        out["band"] = data["d_band_out"].cpu().numpy()
        slab = w2x.Slab(ctx, noise, BAND_W, BAND_ROWS, False, False, n_sub=3)
        try:
            out["slab"] = slab.convert(data["band"], np.empty_like(data["band"]))
        finally:
            slab.close()
        assert np.array_equal(out["band"], out["slab"])

        ctx.forget_model(noise)                                        # the scale model's device copy stays for close()
        ctx.debug_tc_profile_enable(False)
        ctx.debug_tc_profile_enable(True)                              # ... and so does a profile buffer
    finally:
        ctx.close()
    return out


def test_close_returns_all_device_memory(w2x, shipped, data):
    import torch
    one_round(w2x, shipped, data)        # every kernel module is loaded: what the driver keeps for them is not the context's
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    one_round(w2x, shipped, data)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def test_two_rounds_give_the_same_bits(w2x, shipped, data):
    first, second = one_round(w2x, shipped, data), one_round(w2x, shipped, data)
    assert first.keys() == second.keys()
    for name in first:
        assert np.array_equal(first[name], second[name]), name
