"""W2X_PRECISION_F16: the tensor-core engine with one fp16 product per MAC (xh * wh), accumulated in fp32.

This mode keeps the first and last layers in fp32 like the other precisions, and drops the xl * wh and xh * wl
correction products of every inner layer.  It is not held to the 1e-4 gate: its contract is that 8-bit outputs
(rint(255 y), the reference CLI's last step) stay within 1 LSB of the reference's.  It reads and writes the f16x3
records and uses the f16x3 weight image (only the wh half of each stage), so every kernel but the layer kernel runs as
in f16x3.

CPU: an emulator of the mode (fp16(16 x) * fp16(wscale w), wide accumulation, the fp32 epilogue; the first and last
layers repeated in the kernels' own float32 order) against the reference oracle on the three shipped models.  The lattice
emulator (operands [(xh, wh)] only) gives a result different from the f16x3 emulator's on every lattice case, so the
bit-exact GPU tests would catch a stray correction product.
GPU: the layer kernels bit for bit on the lattice (tests/test_tc_exact.py's generator), the shipped models against the
oracle and against the emulator, every entry point against convert_plane, the drop-in CLI and the C interface.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from exact_arith import F32, emulate_first_layer, emulate_last_fused, emulate_last_separate, mul32, readback, tc_activation
from test_tc_exact import (LAYER_SIZES, MODEL_SIZES, NUM_SMS, SHAPES, _grid_models, _mismatch, _tilesets, accumulate,
                           assert_lattice, binary_plane, emulate_filter_layer, emulate_model, lattice_layer, lattice_model,
                           lattice_planes, lattice_report, operands)

ORACLE_TOL_CPU = 1e-3        # emulated worst case over the planes below: see test_emulator_against_the_oracle
ORACLE_TOL_GPU = 1.5e-3      # twice the emulated worst case the mode was chosen on (7.6e-4)
# The kernel and the emulator differ only in how the fp32 sums are accumulated.  One layer's outputs then differ by a few
# fp32 ulps of the sums: on the CPU, the emulator with float32 instead of float64 sums moves them by at most 2.4e-6; on
# the H100 the kernel is 1.7e-6 to 5.7e-6 from the emulator on the shipped models' 32- and 64-wide layers and up to
# 3.4e-5 on their 128 -> 128 layer (1152 products per output, in the tensor cores' own accumulation).  Over a whole model
# such a difference can flip the fp16 rounding of the next layer's input, which this mode, unlike the other two, does not
# correct: on the CPU the same change of sums moves whole-model outputs by 1.9e-4, and the GPU measured 2.4e-4 to 3.9e-4.
LAYER_EMULATOR_TOL = 1e-4
MODEL_EMULATOR_TOL = 8e-4
MODELS = ["scale2.0x", "noise1", "noise2"]


# ---------------------------------------------------------------------------------------------------------------------
# emulators
# ---------------------------------------------------------------------------------------------------------------------
def f16_operands(x16, w):
    """the one factor pair of the mode, [(xh, wh)] as float64, and wscale"""
    pairs, ws = operands(x16, w, False)
    return pairs[:1], ws


def emulate_f16_filter_layer(planes, w, b, exact=True):
    """Context.filter_layer in this mode: planar_to_nhwc (f16x3 records) -> xh * wh -> epilogue -> (hi + lo) / 16"""
    x16 = mul32(np.pad(planes, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16))
    pairs, ws = f16_operands(x16, w)
    return readback(tc_activation(accumulate(pairs, exact), ws, b), False)


def emulate_f16_convert(plane, weights, biases, fused=True, exact=False):
    """Context.convert_plane in this mode, for any 1 -> ... -> 1 model of three layers or more: the first layer
    (first_layer_kernel's float32 order), every inner layer as xh * wh summed exactly (lattice) or in float64 and rounded
    once to float32, the fp32 epilogue, the last layer fused (last_gather) or separate (last_layer_kernel on the records)"""
    n = len(weights)
    a = emulate_first_layer(np.pad(np.asarray(plane, F32), n, mode="edge"), weights[0], biases[0])
    for w, b in zip(weights[1:-1], biases[1:-1]):
        pairs, ws = f16_operands(np.pad(a, ((0, 0), (1, 1), (1, 1))), w)     # the TMA loads zero-fill outside the frame
        a = tc_activation(accumulate(pairs, exact), ws, b)
    if fused:
        return emulate_last_fused(a, weights[-1], biases[-1], n)
    return emulate_last_separate(a, weights[-1], biases[-1], n, False)


def to_u8(y):
    """the reference CLI's last step for a Y plane alone: convertTo(CV_8U, 255)"""
    return np.clip(np.rint(np.asarray(y, np.float64) * 255.0), 0, 255).astype(np.int64)


def adversarial_planes(h, w):
    """binary noise, a checkerboard, 2-pixel stripes and impulses, all in [0, 1]"""
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(5)
    imp = np.zeros((h, w), F32)
    imp[rng.random((h, w)) < 0.02] = 1.0
    return {"binary noise": (rng.random((h, w)) < 0.5).astype(F32), "checkerboard": ((yy + xx) % 2).astype(F32),
            "2-px stripes": ((xx // 2) % 2).astype(F32), "impulses": imp}


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MODELS)
def test_emulator_against_the_oracle(oracle_mod, oracle_models, ncpu, name):
    """The mode's accuracy on the shipped models: white noise and adversarial planes within 1e-3 of the reference, and
    8-bit outputs within 1 LSB, on noise and on a smooth 8-bit plane"""
    om = oracle_models[name]
    planes = {"white noise": oracle_mod.seeded_plane(192, 192, 1, "uniform"), "smooth": oracle_mod.seeded_plane(160, 128, 2, "smooth")}
    planes.update(adversarial_planes(64, 64))
    report = []
    for kind, x in planes.items():
        ref = om.convert(x, n_job=ncpu)
        got = emulate_f16_convert(x, om.weights, om.biases)
        err = float(np.abs(got - ref).max())
        d8 = np.abs(to_u8(got) - to_u8(ref))
        report.append(f"{kind}: max-abs {err:.2e}, 8-bit max {d8.max()}, changed {100 * (d8 > 0).mean():.2f} %")
        assert err <= ORACLE_TOL_CPU, report[-1]
        assert d8.max() <= 1, report[-1]
    print(name, "; ".join(report))


def test_lattice_emulator_tells_a_stray_correction_apart():
    """On the lattice inputs the GPU tests use, xh * wh alone gives a different result from f16x3's three products: a
    correction product left in (or a wrong weight half loaded) cannot pass the bit-exact tests"""
    for cin, cout in SHAPES:
        w, b = lattice_layer(cin, cout, seed=100 * cin + cout)
        x = lattice_planes(cin, LAYER_SIZES[2][1], LAYER_SIZES[2][0], seed=2000 + cin + cout)
        one = emulate_f16_filter_layer(x, w, b)
        assert not np.array_equal(one, emulate_filter_layer(x, w, b, False)), (cin, cout)
        m = lattice_model(cin, cout, seed=10 * cin + cout)
        xp = binary_plane(MODEL_SIZES[3][1], MODEL_SIZES[3][0], seed=3 + cin + cout)
        for fused in (True, False):
            got = emulate_f16_convert(xp, [t[0] for t in m], [t[1] for t in m], fused, exact=True)
            assert not np.array_equal(got, emulate_model(xp, m, False, fused)), (cin, cout, fused)


def test_lattice_emulator_is_the_float_emulator_on_the_lattice():
    """the exact (int64) and the float64 accumulation agree where the lattice makes every sum exact"""
    w, b = lattice_layer(64, 128, seed=9)
    x = lattice_planes(64, 13, 21, seed=10)
    assert np.array_equal(emulate_f16_filter_layer(x, w, b, exact=True), emulate_f16_filter_layer(x, w, b, exact=False))


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def f16_ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    c.set_precision(w2x.PRECISION_F16)
    yield c
    c.close()


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", SHAPES)
def test_single_layer_is_bit_exact(w2x, f16_ctx, cin, cout):
    """tc_conv3x3_kernel<Cin, Cout, FUSE = false, MODE_F16> through filter_layer, at the frame sizes around the tile-set
    and the M-tile, on every SM, one SM and three SMs"""
    w, b = lattice_layer(cin, cout, seed=100 * cin + cout)
    model = w2x.Model.from_arrays([w], [b])
    fails = []
    try:
        for i, (wd, h) in enumerate(LAYER_SIZES):
            x = lattice_planes(cin, h, wd, seed=1000 * i + cin + cout)
            assert_lattice(lattice_report(mul32(np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge"), F32(16)), w, b))
            want = emulate_f16_filter_layer(x, w, b)
            for sms in NUM_SMS:
                f16_ctx.debug_set_num_sms(sms)
                got = f16_ctx.filter_layer(model, 0, x)
                if not np.array_equal(got, want):
                    fails.append(f"{wd}x{h} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        f16_ctx.debug_set_num_sms(0)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("c1,c2", SHAPES)
def test_whole_model_is_bit_exact(w2x, f16_ctx, c1, c2):
    """1 -> C1 -> C2 -> 1 through convert_plane, the last layer fused and separate; the profile counters show that the
    CTAs covered every tile-set once"""
    m = lattice_model(c1, c2, seed=10 * c1 + c2)
    weights, biases = [t[0] for t in m], [t[1] for t in m]
    model = w2x.Model.from_arrays(weights, biases)
    all_sms = torch.cuda.get_device_properties(0).multi_processor_count
    fails = []
    try:
        for i, (wd, h) in enumerate(MODEL_SIZES):
            x = binary_plane(h, wd, seed=i + c1 + c2)
            frame16 = emulate_first_layer(np.pad(x, 3, mode="edge"), *m[0])
            assert_lattice(lattice_report(np.pad(frame16, ((0, 0), (1, 1), (1, 1))), *m[1]))
            n_ts = _tilesets(wd + 6, h + 6)
            for fused in (True, False):
                want = emulate_f16_convert(x, weights, biases, fused, exact=True)
                f16_ctx.debug_set_fuse_last(fused)
                for sms in NUM_SMS:
                    f16_ctx.debug_set_num_sms(sms)
                    f16_ctx.debug_tc_profile_enable(True)              # zero the counters
                    got = f16_ctx.convert_plane(model, x)
                    prof = f16_ctx.debug_tc_profile_read(1)
                    if prof["ctas"] != min(n_ts, sms or all_sms) or round(prof["tilesets"] * prof["ctas"]) != n_ts:
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {prof['ctas']} CTAs x {prof['tilesets']} tile-sets, "
                                     f"want {n_ts} tile-sets")
                    if not np.array_equal(got, want):
                        fails.append(f"{wd}x{h} fused={fused} num_sms={sms}: {_mismatch(got, want)}")
    finally:
        f16_ctx.debug_set_num_sms(0)
        f16_ctx.debug_set_fuse_last(True)
        f16_ctx.debug_tc_profile_enable(False)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_output_does_not_depend_on_the_grid(w2x, f16_ctx, oracle_mod, oracle_models):
    """the shipped models, a chain with every shape as a middle layer (fused and separate) and a 1 -> C1 -> C2 -> 1 model
    per shape, bit-identical at 1, 2, 7 and 64 SMs to the full grid"""
    x = oracle_mod.seeded_plane(200, 150, 9, "uniform")
    fails = []
    try:
        for name, (ws, bs) in _grid_models(oracle_mod, oracle_models).items():
            model = w2x.Model.from_arrays(ws, bs)
            for fused in ((True, False) if name == "chain" else (True,)):
                f16_ctx.debug_set_fuse_last(fused)
                f16_ctx.debug_set_num_sms(0)
                ref = f16_ctx.convert_plane(model, x)
                assert np.isfinite(ref).all(), name
                for sms in (1, 2, 7, 64):
                    f16_ctx.debug_set_num_sms(sms)
                    got = f16_ctx.convert_plane(model, x)
                    if not np.array_equal(got, ref):
                        fails.append(f"{name} fused={fused} num_sms={sms}: {_mismatch(got, ref)}")
    finally:
        f16_ctx.debug_set_num_sms(0)
        f16_ctx.debug_set_fuse_last(True)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_shipped_models_against_oracle_and_emulator(f16_ctx, shipped, oracle_mod, oracle_models, ncpu, name):
    """convert_plane on white noise and a smooth plane: within 1.5e-3 of the reference and within MODEL_EMULATOR_TOL of the
    emulator; 8-bit outputs within 1 LSB"""
    om = oracle_models[name]
    report = []
    for kind, (wd, h) in (("uniform", (200, 150)), ("smooth", (160, 128))):
        x = oracle_mod.seeded_plane(wd, h, 3, kind)
        got = f16_ctx.convert_plane(shipped[name], x)
        ref = om.convert(x, n_job=ncpu)
        em = emulate_f16_convert(x, om.weights, om.biases)
        e_ref, e_em = float(np.abs(got - ref).max()), float(np.abs(got - em).max())
        d8 = np.abs(to_u8(got) - to_u8(ref))
        report.append(f"{kind}: vs oracle {e_ref:.2e}, vs emulator {e_em:.2e}, 8-bit max {d8.max()}, changed {100 * (d8 > 0).mean():.2f} %")
        assert e_ref <= ORACLE_TOL_GPU, report[-1]
        assert e_em <= MODEL_EMULATOR_TOL, report[-1]
        assert d8.max() <= 1, report[-1]
    print(name, "; ".join(report))


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_inner_layers_against_the_emulator(w2x, f16_ctx, oracle_models, name):
    """every inner layer of a shipped model through filter_layer, on ordinary planes with negative values: within 1e-4 of
    the emulator, where a dropped K step, a wrong weight half or a skipped tap moves outputs by far more"""
    om = oracle_models[name]
    rng = np.random.default_rng(11)
    report = []
    for li in range(1, len(om.weights) - 1):
        w, b = om.weights[li], om.biases[li]
        x = (rng.random((w.shape[1], 37, 45)) * 1.5 - 0.3).astype(F32)
        got = f16_ctx.filter_layer(w2x.Model.from_arrays([w], [b]), 0, x)
        err = float(np.abs(got - emulate_f16_filter_layer(x, w, b, exact=False)).max())
        report.append(f"L{li} {err:.2e}")
        assert err <= LAYER_EMULATOR_TOL, report
    print(name, "max-abs vs emulator per layer:", ", ".join(report))


@pytest.mark.gpu
def test_every_entry_point_equals_convert_plane(w2x, f16_ctx, shipped, oracle_mod):
    """host and device buffers, the fused and the literal block walk, scratch-limited bands, convert_band_device,
    convert_tiles (batched and grouped) and caller-exchange Band sessions: bit-identical to convert_plane in this mode"""
    ctx, model = f16_ctx, shipped["noise2"]
    n = len(model)
    W, H = 90, 100
    x = oracle_mod.seeded_plane(W, H, 4, "uniform")
    whole = ctx.convert_plane(model, x)
    fails = []

    def check(what, got, want):
        if not np.array_equal(got, want):
            fails.append(f"{what}: {_mismatch(got, want)}")

    d_in = torch.from_numpy(x).cuda()
    d_out = torch.empty_like(d_in)
    ctx.convert_plane_device(model, d_in.data_ptr(), W, H, W * 4, d_out.data_ptr(), W * 4)
    ctx.synchronize()
    check("device buffers", d_out.cpu().numpy(), whole)
    bw, bh = w2x.get_block_size()
    try:
        w2x.set_block_size(48, 48)
        assert w2x.requires_splitting(W, H)
        for walk in (w2x.WALK_FUSED, w2x.WALK_BLOCKS):
            ctx.set_block_walk(walk)
            check(f"block split walk={walk}", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_block_walk(w2x.WALK_FUSED)
        w2x.set_block_size(bw, bh)
    try:
        for rows in (16, 23):
            ctx.set_scratch_limit(128 * (W + 2 * n) * 4 * (rows + 2 * n))
            check(f"scratch bands of {rows} rows", ctx.convert_plane(model, x), whole)
    finally:
        ctx.set_scratch_limit(0)
    y0, bh_ = 30, 25
    out = torch.empty((bh_, W), device="cuda")
    ctx.convert_band_device(model, d_in[y0 - n:].data_ptr(), W, bh_, n, n, W * 4, out.data_ptr(), W * 4)
    ctx.synchronize()
    check("convert_band_device", out.cpu().numpy(), ctx.convert_plane(model, x[y0 - n:y0 + bh_ + n])[n:n + bh_])
    tiles = np.stack([oracle_mod.seeded_plane(40, 30, 20 + t, "uniform") for t in range(5)])
    want = np.stack([ctx.convert_plane(model, t, block_splitting=False) for t in tiles])
    check("convert_tiles batched", ctx.convert_tiles(model, tiles), want)
    try:
        ctx.set_scratch_limit(128 * (40 + 2 * n) * (30 + 2 * n) * 4 * 2)     # two tiles per pass
        check("convert_tiles grouped", ctx.convert_tiles(model, tiles), want)
    finally:
        ctx.set_scratch_limit(0)
    # Band sessions, the halo rows moved by the caller after every step
    cuts = [0, 7, 30, 61, H]
    bands, outs = [], []
    try:
        for b in range(len(cuts) - 1):
            r0, r1 = cuts[b], cuts[b + 1]
            up, down = b > 0, b < len(cuts) - 2
            band = w2x.Band(ctx, model, W, r1 - r0, up, down)
            bands.append(band)
            band.load(d_in[r0 - (1 if up else 0):].data_ptr(), W * 4)
            outs.append(torch.empty((r1 - r0, W), device="cuda"))

        def dev(ptr, nb):
            return torch.as_tensor(w2x.DevBytes(ptr, nb), device="cuda")

        for k in range(bands[0].steps):
            for band in bands:
                band.step(k)
            halos = [band.halo(k) for band in bands]
            ctx.synchronize()
            for b in range(len(bands) - 1):
                for seg in range(len(halos[b])):
                    _, _, sd, rd, nb = halos[b][seg]
                    su, ru, _, _, _ = halos[b + 1][seg]
                    dev(ru, nb).copy_(dev(sd, nb))
                    dev(rd, nb).copy_(dev(su, nb))
            torch.cuda.synchronize()
        for band, o in zip(bands, outs):
            band.finish(o.data_ptr(), W * 4)
        ctx.synchronize()
        check("band sessions", torch.cat(outs).cpu().numpy(), whole)
    finally:
        for band in bands:
            band.close()
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_bands_slabs_and_multi_across_two_gpus(w2x, shipped, oracle_mod):
    """w2x_band_connect_local + w2x_band_run, w2x_slab_* and w2x_multi_* across two GPUs in this mode: bit-identical to one
    GPU (the same machinery on one GPU is covered by the caller-exchange bands above)"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    model = shipped["noise1"]
    single = w2x.Context(0, engine=w2x.ENGINE_TC)
    single.set_precision(w2x.PRECISION_F16)
    W, H = 170, 150
    x = oracle_mod.seeded_plane(W, H, 31, "uniform")
    whole = single.convert_plane(model, x)
    W2, H2 = 190, 420
    x2 = oracle_mod.seeded_plane(W2, H2, 9, "uniform")
    whole2 = single.convert_plane(model, x2)
    big = oracle_mod.seeded_plane(260, 1700, 5, "uniform")
    want_big = single.convert_plane(model, big)
    single.close()
    ctxs = [w2x.Context(d, engine=w2x.ENGINE_TC) for d in (0, 1)]
    for c in ctxs:
        c.set_precision(w2x.PRECISION_F16)
    try:
        cut = 71
        bands = [w2x.Band(ctxs[0], model, W, cut, False, True), w2x.Band(ctxs[1], model, W, H - cut, True, False)]
        bands[0].connect_local(None, bands[1])
        bands[1].connect_local(bands[0], None)
        d_in = [torch.from_numpy(np.ascontiguousarray(x[:cut])).to("cuda:0"), torch.from_numpy(np.ascontiguousarray(x[cut:])).to("cuda:1")]
        outs = [torch.zeros_like(t) for t in d_in]
        for b in range(2):
            bands[b].run(d_in[b].data_ptr(), W * 4, outs[b].data_ptr(), W * 4)
        for c in ctxs:
            c.synchronize()
        assert np.array_equal(np.concatenate([o.cpu().numpy() for o in outs]), whole)
        for b in bands:
            b.close()
        slabs = [w2x.Slab(ctxs[0], model, W2, H2 // 2, False, True, order=0, n_sub=2),
                 w2x.Slab(ctxs[1], model, W2, H2 - H2 // 2, True, False, order=1, n_sub=3)]
        slabs[0].connect_local(None, slabs[1])
        slabs[1].connect_local(slabs[0], None)
        h_in = torch.from_numpy(x2).pin_memory().numpy()
        h_out = torch.zeros((H2, W2)).pin_memory().numpy()
        slabs[0].convert_async(h_in[:H2 // 2], h_out[:H2 // 2])
        slabs[1].convert_async(h_in[H2 // 2:], h_out[H2 // 2:])
        for sl in slabs:
            sl.synchronize()
        assert np.array_equal(h_out, whole2)
        for sl in slabs:
            sl.close()
    finally:
        for c in ctxs:
            c.close()
    multi = w2x.Multi([0, 1])
    try:
        multi.set_precision(w2x.PRECISION_F16)
        assert np.array_equal(multi.convert_plane(model, big), want_big)
    finally:
        multi.close()


@pytest.fixture(scope="module")
def cli(w2x):
    from test_cli import CLI                              # skips where cv2 is missing, like tests/test_cli.py
    w2x.build()
    assert os.path.exists(CLI)
    return CLI


@pytest.mark.gpu
@pytest.mark.parametrize("mode,level,ratio,name", [("noise_scale", 1, 2.0, "in(noise_scale)(Level1)(x2.000000).png"),
                                                  ("scale", 1, 3.0, "in(scale)(x3.000000).png"),
                                                  ("noise", 2, 2.0, "in(noise)(Level2).png")])
def test_cli_with_the_environment_value(cli, tmp_path, json_models, oracle_models, ncpu, mode, level, ratio, name):
    """the drop-in CLI with W2X_PRECISION=f16 against the reference pipeline: every output byte within 1 LSB and at most
    5 % of them changed"""
    import cv2
    from test_cli import _reference_pipeline, _test_image
    bgr = _test_image(45, 33, 11)
    cv2.imwrite(str(tmp_path / "in.png"), bgr)
    mdir = os.path.dirname(json_models["scale2.0x"])
    r = subprocess.run([cli, "-i", str(tmp_path / "in.png"), "-m", mode, "--noise_level", str(level), "--scale_ratio", str(ratio),
                        "--model_dir", mdir, "-j", "2"], capture_output=True, text=True, env=dict(os.environ, W2X_PRECISION="f16"))
    assert r.returncode == 0, r.stdout + r.stderr
    out = cv2.imread(str(tmp_path / name), cv2.IMREAD_COLOR)
    assert out is not None, os.listdir(tmp_path)
    ref = _reference_pipeline(bgr, mode, level, ratio, oracle_models, ncpu)
    assert out.shape == ref.shape
    diff = np.abs(out.astype(int) - ref.astype(int))
    print(mode, f"8-bit max diff {diff.max()}, changed {100 * (diff > 0).mean():.2f} %")
    assert diff.max() <= 1 and (diff > 0).mean() <= 0.05


@pytest.mark.gpu
def test_interface(w2x, shipped, oracle_mod, monkeypatch):
    monkeypatch.delenv("W2X_PRECISION", raising=False)
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        assert c.get_precision() == w2x.PRECISION_F16_F8X2                   # the default is unchanged
        with pytest.raises(w2x.W2xError) as e:
            c.set_precision(3)
        assert e.value.status == 1                                          # W2X_ERR_ARG
        assert c.get_precision() == w2x.PRECISION_F16_F8X2
        c.set_precision(w2x.PRECISION_F16)
        c.set_timing(True)
        c.convert_plane(shipped["scale2.0x"], oracle_mod.seeded_plane(64, 48, 0, "uniform"))
        names = [t[2] for t in c.layer_times()]
        assert names == ["first_1xN"] + ["wgmma_f16"] * 4 + ["wgmma_f16+last", "last_gather"], names
        c.debug_set_fuse_last(False)
        c.convert_plane(shipped["scale2.0x"], oracle_mod.seeded_plane(64, 48, 0, "uniform"))
        names = [t[2] for t in c.layer_times()]
        assert names == ["first_1xN"] + ["wgmma_f16"] * 5 + ["last_Nx1"], names
    finally:
        c.close()
    monkeypatch.setenv("W2X_PRECISION", "f16")
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    try:
        assert c.get_precision() == w2x.PRECISION_F16 == 2
    finally:
        c.close()
