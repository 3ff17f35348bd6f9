"""w2x_convert_chain / w2x_convert_chain_device: the reference's noise pass and 2x scale iterations (src/main.cpp:82-156) on one
plane in one call, the plane kept on the device between steps and the nearest 2x resize folded into the first layer.

Every step's result is checked bit for bit (np.array_equal) against the per-step loop: convert_plane on the previous result,
resized with np.repeat(np.repeat(y, 2, 0), 2, 1) first for an upscaling step -- in all three precisions, on the shipped and random
1 -> C1 -> C2 -> 1 models, on sizes from 1 x 1 to planes the reference block-splits, through both entry points with strided planes,
on the fp32 engine, the literal block walk and the fuse-off probe, with small scratch limits (bands starting on odd and even 2x
rows), on a plane whose 2x output is taller than one frame, and on a torch stream.  Also: each step against the CPU oracle, launch
counts and kernel names, the progress lines and callbacks, argument errors, W2X_ERR_NOMEM, and the CLI (pixels and stdout).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_gpu_parity import TC_TOL

pytestmark = pytest.mark.gpu

PRECISIONS = [0, 1, 2]   # f16x3, f16+f8x2, f16
ERR_NOMEM = 8
SIZES = [(1, 1), (1, 300), (300, 1), (15, 13), (45, 33), (443, 443), (700, 300)]   # (w, h); 443 x 443 is split once doubled
PATTERNS = ["U", "SU", "UU", "SUU", "US"]
CLI = os.path.join(ROOT, "waifu2x-converter-cpp_b200", "w2x-converter")


def up2(y):
    return np.repeat(np.repeat(y, 2, 0), 2, 1)


def steps_for(pattern, same, scale):
    return [(same, False) if c == "S" else (scale, True) for c in pattern]


def loop(ctx, steps, x, block_splitting=True):
    """the per-step reference: every intermediate plane"""
    outs, y = [], x
    for model, up in steps:
        y = ctx.convert_plane(model, up2(y) if up else y, block_splitting=block_splitting)
        outs.append(y)
    return outs


def plane(oracle_mod, w, h, seed):
    return oracle_mod.seeded_plane(w, h, seed, "uniform")


def random_model(w2x, c1, c2, seed, n_out=1):
    rng = np.random.default_rng(seed)
    ws = [rng.normal(0, 1 / 3, (c1, 1, 3, 3)), rng.normal(0, 1 / np.sqrt(9 * c1), (c2, c1, 3, 3)),
          rng.normal(0, 1 / np.sqrt(9 * c2), (n_out, c2, 3, 3))]
    bs = [rng.normal(0, 0.1, c1), rng.normal(0, 0.1, c2), rng.normal(0, 0.1, n_out)]
    return w2x.Model.from_arrays([w.astype(np.float32) for w in ws], bs)


def device_chain(ctx, steps, x, **kw):
    import torch
    ups = sum(up for _, up in steps)
    h, w = x.shape
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_out = torch.empty((h << ups, w << ups), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.convert_chain_device(steps, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), (w << ups) * 4, **kw)
    ctx.synchronize()
    return d_out.cpu().numpy()


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.fixture(scope="module")
def randoms(w2x):
    return random_model(w2x, 32, 64, 11), random_model(w2x, 128, 32, 12)


@pytest.fixture
def ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.close()


# ---- results, bit for bit ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("models", ["shipped", "random"])
def test_patterns_and_sizes(ctx, shipped, randoms, oracle_mod, precision, models):
    ctx.set_precision(precision)
    same, scale = (shipped["noise1"], shipped["scale2.0x"]) if models == "shipped" else randoms
    for i, (w, h) in enumerate(SIZES):
        x = plane(oracle_mod, w, h, 100 + i)
        for pattern in PATTERNS:
            if models == "random" and (w, h) == (700, 300) and pattern in ("UU", "SUU"):
                continue   # the shipped models cover the largest outputs
            steps = steps_for(pattern, same, scale)
            want = loop(ctx, steps, x)[-1]
            assert np.array_equal(ctx.convert_chain(steps, x), want), (pattern, w, h)
            if (w, h) in ((15, 13), (443, 443)):
                assert np.array_equal(device_chain(ctx, steps, x), want), (pattern, w, h)


def test_both_entries_with_strided_planes(ctx, shipped, oracle_mod):
    import torch
    steps = steps_for("SUU", shipped["noise1"], shipped["scale2.0x"])
    for w, h in ((45, 33), (300, 1), (130, 77)):
        x = plane(oracle_mod, w, h, w + h)
        want = loop(ctx, steps, x)[-1]
        sentinel = np.float32(12345.5)
        buf = np.full((h, w + 5), -7.0, np.float32)
        buf[:, :w] = x
        obuf = np.full((4 * h, 4 * w + 3), sentinel, np.float32)
        ctx.convert_chain(steps, buf[:, :w], out=obuf[:, :4 * w])
        assert np.array_equal(obuf[:, :4 * w], want) and (obuf[:, 4 * w:] == sentinel).all()
        d_in = torch.full((h, w + 3), -7.0, device="cuda")
        d_in[:, :w] = torch.from_numpy(x).cuda()
        d_out = torch.full((4 * h, 4 * w + 9), float(sentinel), device="cuda")
        torch.cuda.synchronize()
        ctx.convert_chain_device(steps, d_in.data_ptr(), w, h, d_in.stride(0) * 4, d_out.data_ptr(), d_out.stride(0) * 4)
        ctx.synchronize()
        got = d_out.cpu().numpy()
        assert np.array_equal(got[:, :4 * w], want) and (got[:, 4 * w:] == sentinel).all()


@pytest.mark.parametrize("case", ["fp32", "walk_blocks", "fuse_off", "no_split"])
def test_other_paths(w2x, shipped, oracle_mod, case):
    c = w2x.Context(0, engine=w2x.ENGINE_FP32 if case == "fp32" else w2x.ENGINE_TC)
    try:
        if case == "walk_blocks":
            c.set_block_walk(w2x.WALK_BLOCKS)
        if case == "fuse_off":
            c.debug_set_fuse_last(0)
        split = case != "no_split"
        for w, h in ((15, 13), (443, 443), (300, 1)):
            x = plane(oracle_mod, w, h, 7 * w + h)
            for pattern in ("SU", "US"):
                steps = steps_for(pattern, shipped["noise1"], shipped["scale2.0x"])
                want = loop(c, steps, x, split)[-1]
                assert np.array_equal(c.convert_chain(steps, x, block_splitting=split), want), (case, pattern, w, h)
                assert np.array_equal(device_chain(c, steps, x, block_splitting=split), want), (case, pattern, w, h)
    finally:
        c.close()


@pytest.mark.parametrize("engine", ["tc", "fp32"])
def test_small_scratch_limits_and_host_bands(w2x, shipped, oracle_mod, engine):
    """bands of the 2x plane that start on odd and on even rows; host copy bands (even starts) of the last step"""
    c = w2x.Context(0, engine=w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    try:
        model = shipped["scale2.0x"]
        x = plane(oracle_mod, 45, 77, 3)
        steps = [(shipped["noise1"], False), (model, True)]
        want = loop(c, steps, x)[-1]
        per_row = 128 * (90 + 14) * 4                 # scratch_band_rows: max channels x padded 2x width x 4 bytes
        for band in (17, 24, 31):
            c.set_scratch_limit(per_row * (band + 14))
            assert np.array_equal(c.convert_chain(steps, x), want), band
            assert np.array_equal(device_chain(c, steps, x), want), band
        c.set_scratch_limit(0)
        for bands in (2, 3, 5, 8):
            c.debug_set_host_bands(bands)
            assert np.array_equal(c.convert_chain(steps, x), want), bands
            assert np.array_equal(c.convert_chain([(model, True)], x), loop(c, [(model, True)], x)[-1]), bands
    finally:
        c.close()


@pytest.mark.parametrize("w", [1, 5])
def test_output_taller_than_one_frame(w2x, ctx, w):
    """2 x 262141 = 524282 output rows: past the 524280 rows a frame may have (test_frame_limits' geometry model)"""
    import torch
    from test_edge_exact import _geometry_model, plane_for
    layers = _geometry_model()
    model = w2x.Model.from_arrays([t[0] for t in layers], [t[1] for t in layers])
    h = 262141
    x = plane_for(h, w, 1 if w == 1 else 2)
    for precision in (0, 1):
        ctx.set_precision(precision)
        d_big = torch.from_numpy(up2(x)).cuda()
        d_want = torch.empty_like(d_big)
        torch.cuda.synchronize()
        ctx.convert_plane_device(model, d_big.data_ptr(), 2 * w, 2 * h, 8 * w, d_want.data_ptr(), 8 * w)
        ctx.synchronize()
        want = d_want.cpu().numpy()
        del d_big, d_want
        assert np.array_equal(device_chain(ctx, [(model, True)], x), want)
        assert np.array_equal(ctx.convert_chain([(model, True)], x), want)


def test_torch_stream(w2x, ctx, shipped, oracle_mod):
    import torch
    steps = steps_for("SU", shipped["noise1"], shipped["scale2.0x"])
    x = plane(oracle_mod, 130, 90, 8)
    want = loop(ctx, steps, x)[-1]
    s = torch.cuda.Stream()
    d_in = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        d_out = torch.empty((180, 260), dtype=torch.float32, device="cuda")
        ctx.set_stream(s.cuda_stream)
        ctx.convert_chain_device(steps, d_in.data_ptr(), 130, 90, 130 * 4, d_out.data_ptr(), 260 * 4)
        got = d_out.cpu()                      # ordered after the chain on the same stream
    s.synchronize()
    ctx.set_stream(0)
    assert np.array_equal(got.numpy(), want)


# ---- accuracy, launches, progress, errors -----------------------------------------------------------------------------------
def test_each_step_against_the_oracle(ctx, shipped, oracle_models, oracle_mod):
    ctx.set_precision(0)   # f16x3, the precision TC_TOL states
    steps = steps_for("SUU", shipped["noise1"], shipped["scale2.0x"])
    names = ["noise1", "scale2.0x", "scale2.0x"]
    x = plane(oracle_mod, 23, 17, 9)
    prev = x
    for k in range(len(steps)):
        got = ctx.convert_chain(steps[:k + 1], x)
        src = up2(prev) if steps[k][1] else prev
        assert np.abs(got - oracle_models[names[k]].convert(src, n_job=4)).max() <= TC_TOL, k
        prev = got


def test_launch_counts_and_kernel_names(w2x, ctx, shipped, oracle_mod):
    import torch
    L = w2x.lib()
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    for w, h, limit in ((45, 33, 0), (443, 443, 0), (45, 77, 128 * 104 * 4 * 31)):
        ctx.set_scratch_limit(limit)
        x = plane(oracle_mod, w, h, 1)
        d_x = torch.from_numpy(x).cuda()
        d_2x = torch.from_numpy(up2(x)).cuda()
        d_o = torch.empty_like(d_2x)
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        ctx.convert_plane_device(scale, d_2x.data_ptr(), 2 * w, 2 * h, 8 * w, d_o.data_ptr(), 8 * w)
        per_plane = ctx.launch_count() - n0
        assert L.w2x_ctx_layer_kernel_name(ctx._h, 0).decode() == "first_1xN"
        n0 = ctx.launch_count()
        ctx.convert_chain_device([(scale, True)], d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), 8 * w)
        assert ctx.launch_count() - n0 == per_plane
        assert L.w2x_ctx_layer_kernel_name(ctx._h, 0).decode() == "first_1xN+up2x"
        n0 = ctx.launch_count()
        ctx.convert_plane_device(noise, d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), w * 4)
        noise_launches = ctx.launch_count() - n0
        n0 = ctx.launch_count()
        ctx.convert_chain_device([(noise, False), (scale, True)], d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), 8 * w)
        assert ctx.launch_count() - n0 == noise_launches + per_plane
        ctx.synchronize()


def expected_lines(w2x, ctx, steps, x, host, block_splitting=True):
    """("step", k) and then the lines the single-plane entry point logs for step k's plane"""
    import torch
    lines = []
    ctx.set_log(lines.append)
    want, y = [], x
    for k, (model, up) in enumerate(steps):
        want.append(("step", k))
        src = up2(y) if up else y
        lines.clear()
        if host:
            y = ctx.convert_plane(model, src, block_splitting=block_splitting)
        else:
            h, w = src.shape
            d_in = torch.from_numpy(np.ascontiguousarray(src)).cuda()
            d_out = torch.empty_like(d_in)
            torch.cuda.synchronize()
            ctx.convert_plane_device(model, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), w * 4, block_splitting)
            ctx.synchronize()
            y = d_out.cpu().numpy()
        want += lines
    return want


@pytest.mark.parametrize("walk", ["fused", "blocks"])
def test_progress_lines_and_callbacks(w2x, ctx, shipped, oracle_mod, walk):
    if walk == "blocks":
        ctx.set_block_walk(w2x.WALK_BLOCKS)
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    for w, h in ((45, 33), (443, 443), (300, 600)):      # plain, block-split once doubled, host copy bands on the last step
        x = plane(oracle_mod, w, h, 2)
        steps = [(noise, False), (scale, True)]
        for host in (True, False):
            want = expected_lines(w2x, ctx, steps, x, host)
            got = []
            ctx.set_log(got.append)
            if host:
                ctx.convert_chain(steps, x, on_step=lambda k: got.append(("step", k)))
            else:
                device_chain(ctx, steps, x, on_step=lambda k: got.append(("step", k)))
            assert got == want, (w, h, host)
            if (w, h) == (443, 443):
                assert any(isinstance(s, str) and s.startswith("start process block") for s in got)
    ctx.set_log(None)


def test_argument_errors_name_the_step(w2x, ctx, shipped):
    L = w2x.lib()
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    bad_out = random_model(w2x, 32, 32, 5, n_out=2)
    x = np.ones((8, 8), np.float32)
    sentinel = np.float32(-3.25)
    out = np.full((32, 32), sentinel, np.float32)

    def call(models, kinds, n=None, in_ptr=x.ctypes.data, width=8, height=8, in_stride=32, out_ptr=out.ctypes.data, out_stride=128):
        n = len(kinds if kinds is not None else models) if n is None else n
        mp = None if models is None else (C.c_void_p * max(len(models), 1))(*[m._h if m is not None else None for m in models])
        kp = None if kinds is None else (C.c_int * max(len(kinds), 1))(*kinds)
        r = L.w2x_convert_chain(ctx._h, n, mp, kp, in_ptr, width, height, in_stride, out_ptr, out_stride, 1, w2x.capi.STEP_FN(), None)
        return r, L.w2x_last_error().decode()

    ok = call([noise, scale, scale], [0, 1, 1])
    assert ok[0] == 0, ok
    out[:] = sentinel
    cases = [
        (call([noise], [0], n=0), "step 0"),
        (call(None, [0, 1]), "step 0"),
        (call([noise, scale], None), "step 0"),
        (call([noise, None, scale], [0, 1, 1]), "step 1"),
        (call([noise, scale, scale], [0, 1, 2]), "step 2"),
        (call([noise, scale, bad_out], [0, 1, 1]), "step 2"),
        (call([scale, scale, scale], [1, 1, 1], width=1 << 29, in_stride=4 << 29), "step 1"),
        (call([noise, scale], [0, 1], in_stride=30), "step 0"),
        (call([noise, scale], [0, 1], in_stride=28), "step 0"),
        (call([noise, scale], [0, 1], in_ptr=None), "step 0"),
        (call([noise, scale, scale], [0, 1, 1], out_stride=126), "step 2"),
        (call([noise, scale, scale], [0, 1, 1], out_stride=124), "step 2"),
        (call([noise, scale, scale], [0, 1, 1], out_ptr=None), "step 2"),
        (call([noise, scale], [0, 1], width=0), "step 0"),
    ]
    for i, ((r, msg), where) in enumerate(cases):
        assert r == 1 and where in msg, (i, r, msg)
        assert (out == sentinel).all(), i
    r, msg = call([noise, scale, scale], [0, 1, 1], in_ptr=out.ctypes.data)   # in and out overlap
    assert r == 1 and "overlap" in msg, msg
    assert (out == sentinel).all()
    with pytest.raises(w2x.W2xError) as e:
        ctx.convert_chain_device([(noise, False), (None, True)], 1 << 20, 8, 8, 32, 1 << 21, 64)
    assert e.value.status == 1 and "step 1" in e.value.message


def act_bytes(om, w, h):
    """one activation frame of a w x h plane converted in one band: the model's widest layer x the padded plane x 4 bytes"""
    n = len(om.weights)
    return max(max(wt.shape[:2]) for wt in om.weights) * (w + 2 * n) * (h + 2 * n) * 4


@pytest.mark.parametrize("case", ["tc", "fp32", "later_step"])
def test_out_of_memory_leaves_nothing_queued(w2x, shipped, oracle_models, oracle_mod, case):
    """W2X_ERR_NOMEM comes before any on_step call, progress line, copy or launch: with the device all but full (both engines, both
    entries), and with room for step 0's activation frames but not for step 1's larger ones (the device entry)"""
    import torch
    c = w2x.Context(0, engine=w2x.ENGINE_FP32 if case == "fp32" else w2x.ENGINE_TC)
    filler = None
    try:
        steps = [(shipped["noise1"], False), (shipped["scale2.0x"], True)]
        c.convert_chain(steps, plane(oracle_mod, 16, 16, 1))      # the models' device copies and small buffers exist
        w = h = 1024 if case == "later_step" else 2048
        x = plane(oracle_mod, w, h, 2)
        out = np.full((2 * h, 2 * w), -3.25, np.float32)
        d_in = torch.from_numpy(x).cuda()
        d_out = torch.full((2 * h, 2 * w), -3.25, device="cuda")
        leave = (w * h + 4 * w * h + w * h) * 4 + (256 << 20)       # the host entry's staging and step 0's output plane
        if case == "later_step":
            step0, step1 = act_bytes(oracle_models["noise1"], w, h), act_bytes(oracle_models["scale2.0x"], 2 * w, 2 * h)
            leave += 2 * step0
            assert step1 > leave - step0, (step0, step1)             # a frame of step 1 does not fit beside one of step 0
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(free - leave, 0), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        lines, calls = [], []
        c.set_log(lines.append)
        n0 = c.launch_count()
        for entry in ["device"] + (["host"] if case != "later_step" else []):
            with pytest.raises(w2x.W2xError) as e:
                if entry == "device":
                    c.convert_chain_device(steps, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), 2 * w * 4, on_step=calls.append)
                else:
                    c.convert_chain(steps, x, out=out, on_step=calls.append)
            assert e.value.status == ERR_NOMEM, (entry, e.value.message)
            assert c.launch_count() == n0 and not calls and not lines, (entry, c.launch_count() - n0, calls, lines[:2])
        c.synchronize()
        del filler
        filler = None
        torch.cuda.empty_cache()
        assert (out == -3.25).all() and (d_out == -3.25).all().item()
        c.convert_chain_device(steps, d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), 2 * w * 4)   # with the memory back, it runs
        c.synchronize()
        assert not (d_out == -3.25).all().item()
    finally:
        c.set_log(None)
        del filler
        torch.cuda.empty_cache()
        c.close()


# ---- the CLI ----------------------------------------------------------------------------------------------------------------
def cli_lines(w2x, mode, ratio, w, h, n=7):
    """the reference's stdout (src/main.cpp:82-192, src/convertRoutine.cpp:67,133-134) for a w x h input"""
    def conv(w, h):
        if not w2x.requires_splitting(w, h):
            return [f"Iteration #{k}..." for k in range(1, n + 1)]
        tab, _, _ = w2x.block_table(w, h, n)
        out = []
        for r, c in tab[:, :2]:
            out += [f"start process block ({c},{r}) ..."] + [f"Iteration #{k}..." for k in range(1, n + 1)]
        return out
    lines = conv(w, h) if "noise" in mode else []
    lines.append("start scaling")
    for i in range(int(np.ceil(np.log2(ratio)))):
        w, h = 2 * w, 2 * h
        lines += [f"#{i + 1} 2x scaling..."] + conv(w, h)
    return lines + ["process successfully done!"]


@pytest.mark.parametrize("mode,ratio,w,h", [("noise_scale", 4.0, 45, 33), ("scale", 3.0, 37, 29)])
def test_cli_matches_the_reference_pipeline(w2x, tmp_path, json_models, oracle_models, ncpu, mode, ratio, w, h):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _reference_pipeline, _test_image
    w2x.build()
    bgr = _test_image(w, h, 11)
    cv2.imwrite(str(tmp_path / "in.png"), bgr)
    r = subprocess.run([CLI, "-i", str(tmp_path / "in.png"), "-o", str(tmp_path / "out.png"), "-m", mode, "--scale_ratio", str(ratio),
                        "--model_dir", os.path.dirname(json_models["scale2.0x"])], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.splitlines() == cli_lines(w2x, mode, ratio, w, h)
    out = cv2.imread(str(tmp_path / "out.png"), cv2.IMREAD_COLOR)
    ref = _reference_pipeline(bgr, mode, 1, ratio, oracle_models, ncpu)
    assert out.shape == ref.shape
    diff = np.abs(out.astype(int) - ref.astype(int))
    assert diff.max() <= 1 and (diff > 0).mean() < 0.01


def test_cli_stdout_on_split_planes(w2x, tmp_path, json_models):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    w, h = 160, 155                                      # x4: the last pass, on 640 x 620, is block-split
    cv2.imwrite(str(tmp_path / "in.png"), _test_image(w, h, 5))
    args = ["-i", str(tmp_path / "in.png"), "-o", str(tmp_path / "out.png"), "-m", "noise_scale", "--scale_ratio", "4",
            "--model_dir", os.path.dirname(json_models["scale2.0x"])]
    r = subprocess.run([CLI, *args], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    want = cli_lines(w2x, "noise_scale", 4.0, w, h)
    assert any(s.startswith("start process block") for s in want)
    assert r.stdout.splitlines() == want
    ref_cli = os.path.join(ROOT, "oracle", "_ref", "waifu2x-reference-cli")
    if os.path.exists(ref_cli):
        args[3] = str(tmp_path / "ref.png")
        ref = subprocess.run([ref_cli, *args], capture_output=True, text=True)
        assert ref.returncode == 0 and r.stdout == ref.stdout


def test_cli_noise_pass_runs_when_the_scale_model_is_missing(w2x, tmp_path, json_models):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    mdir = tmp_path / "models"
    mdir.mkdir()
    os.symlink(json_models["noise1"], mdir / "noise1_model.json")
    cv2.imwrite(str(tmp_path / "in.png"), _test_image(20, 16))
    r = subprocess.run([CLI, "-i", str(tmp_path / "in.png"), "-m", "noise_scale", "--model_dir", str(mdir)], capture_output=True, text=True,
                       cwd=tmp_path)
    assert r.returncode == 255
    assert r.stdout.splitlines() == [f"Iteration #{k}..." for k in range(1, 8)]
    assert "scale2.0x_model.json" in r.stderr
