"""Test-time augmentation: chain steps with W2X_STEP_TTA average a conversion over the plane's 8 flips and transposes.

The contract (include/w2x_b200.h, W2X_STEP_TTA): variant j of X has t = bit 2, fy = bit 1, fx = bit 0 of j; the step's output is
(((O_0 + O_1) + ...) + O_7) * 0.125f in fp32, O_j being convert_plane(block_splitting=0) of V_j(U(P)) carried back through the same
index map.  The GPU tests check that bit for bit against exactly that Python loop (numpy transforms, convert_plane, a float32 sum in
order) on edge and odd sizes, all precisions and both engines, both step kinds, host and device entries with strided planes, mixed
chains, collections where some variants pack and some do not, and planes converted alone in row bands.  Also: progress lines and
launch counts against the plain calls, argument and out-of-memory errors, the CPU oracle, and the CLI's hidden --tta switch.  The CPU
tests check the index maps themselves, that the C++ header stays C++11, and the CLI's flag surface.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

PKG = os.path.join(ROOT, "waifu2x-converter-cpp_b200")
CLI = os.path.join(PKG, "w2x-converter")
PRECISIONS = [0, 1, 2]   # f16x3, f16+f8x2, f16
SIZES = [(1, 1), (1, 17), (17, 1), (37, 29), (29, 37), (256, 256)]   # (w, h)
ERR_ARG, ERR_NOMEM = 1, 8
gpu = pytest.mark.gpu


# ---- the index maps -----------------------------------------------------------------------------------------------------------
def variant(x, j):
    """V_j(x): transpose when bit 2 is set, then flip rows (bit 1) and columns (bit 0)"""
    v = x.T if j & 4 else x
    if j & 2:
        v = v[::-1, :]
    if j & 1:
        v = v[:, ::-1]
    return v


def unvariant(o, j):
    """carries an output of variant j back: out[r][c] = o[y][x] through V_j's index map"""
    if j & 1:
        o = o[:, ::-1]
    if j & 2:
        o = o[::-1, :]
    return o.T if j & 4 else o


def variant_by_formula(x, j):
    """V_j[y][x] = X[r][c], x' = fx ? W'-1-x : x, y' = fy ? H'-1-y : y, (r, c) = t ? (x', y') : (y', x')"""
    h, w = x.shape
    t, fy, fx = j & 4, j & 2, j & 1
    W, H = (h, w) if t else (w, h)
    v = np.empty((H, W), x.dtype)
    for yy in range(H):
        for xx in range(W):
            xp, yp = (W - 1 - xx if fx else xx), (H - 1 - yy if fy else yy)
            r, c = (xp, yp) if t else (yp, xp)
            v[yy, xx] = x[r, c]
    return v


def up2(y):
    return np.repeat(np.repeat(y, 2, 0), 2, 1)


def dense(a):
    """a fresh C-ordered copy: numpy counts a flipped or transposed 1 x n view as contiguous while its row stride stays short"""
    return np.array(a, np.float32, order="C", copy=True)


def mean8(outs):
    acc = outs[0].astype(np.float32)
    for o in outs[1:]:
        acc = (acc + o).astype(np.float32)
    return acc * np.float32(0.125)


def test_variant_maps_form_the_dihedral_group():
    x = np.arange(5 * 3, dtype=np.float32).reshape(5, 3)            # h = 5, w = 3: every map tells its own story
    for j in range(8):
        assert np.array_equal(variant(x, j), variant_by_formula(x, j)), j
        assert np.array_equal(unvariant(variant(x, j), j), x), j
        inverses = [k for k in range(8) if np.array_equal(variant(variant(x, j), k), x)]
        assert len(inverses) == 1, (j, inverses)                     # each map has exactly one inverse among the eight
    assert np.array_equal(variant(x, 0), x)
    images = {variant(x, j).tobytes() + bytes(variant(x, j).shape) for j in range(8)}
    assert len(images) == 8                                          # eight different maps
    for a in range(8):                                               # closed under composition
        for b in range(8):
            ab = variant(variant(x, a), b)
            assert any(np.array_equal(ab, variant(x, k)) for k in range(8)), (a, b)


@pytest.mark.parametrize("w,h", [(3, 5), (4, 6), (1, 7), (6, 1), (1, 1), (8, 3)])
def test_nearest_2x_commutes_with_every_map(w, h):
    x = np.random.default_rng(w * 31 + h).random((h, w), dtype=np.float32)
    for j in range(8):
        assert np.array_equal(variant(up2(x), j), up2(variant(x, j))), j


def test_chain_step_header_stays_cpp11(tmp_path):
    """host/w2xc.hpp with ChainStep::tta compiles as the option-A build compiles it (-std=c++11, through host/dropin), and brace
    initialisation with two or three members still works"""
    src = tmp_path / "c11.cpp"
    src.write_text("""#include "modelHandler.hpp"
#include "convertRoutine.hpp"
int main() {
    std::vector<std::unique_ptr<w2xc::Model>> m;
    std::vector<w2xc::ChainStep> steps;
    steps.push_back({&m, false, true});
    w2xc::ChainStep s = {&m, true, false};
    steps.push_back(s);
    w2xc::ChainStep old = {&m, true};
    return (int)steps.size() + (old.tta ? 1 : 0);
}
""")
    dropin = os.path.join(PKG, "host", "dropin")
    r = subprocess.run(["g++", "-std=c++11", "-fsyntax-only", "-Wall", "-DW2X_CVSHIM_WITH_IMGPROC", "-I", dropin, "-I", os.path.join(PKG, "host"),
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle", "cvshim"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_cli_tta_flag_is_hidden_and_refuses_several_gpus(w2x, tmp_path):
    w2x.build()
    run = lambda *a: subprocess.run([CLI, *a], capture_output=True, text=True, cwd=tmp_path)   # noqa: E731
    help_text = run("--help")
    assert help_text.returncode == 0 and "tta" not in help_text.stdout
    brief = run()
    assert brief.returncode == 1 and "tta" not in brief.stderr
    assert run("-i", "a.png", "--tta", "2").returncode == 1                       # only 0 and 1
    r = run("-i", "missing.png", "--tta", "1", "--gpus", "2")                     # stops before reading the image
    assert r.returncode == 1 and "--tta" in r.stderr and "couldn't read image" not in r.stderr
    assert os.listdir(tmp_path) == []


# ---- the GPU: bit for bit against the Python loop -------------------------------------------------------------------------------
def tta_plane(ctx, model, src):
    """one TTA step on an already resized plane: 8 convert_plane calls and the ordered float32 mean"""
    return mean8([unvariant(ctx.convert_plane(model, dense(variant(src, j)), block_splitting=False), j) for j in range(8)])


def loop(ctx, steps, x):
    """the per-step Python reference; steps are (model, upscale, tta) triples"""
    y = x
    for model, up, tta in steps:
        src = up2(y) if up else y
        y = tta_plane(ctx, model, src) if tta else ctx.convert_plane(model, src, block_splitting=False)
    return y


def plane(oracle_mod, w, h, seed):
    return oracle_mod.seeded_plane(w, h, seed, "uniform")


def device_chain(ctx, steps, x, pad_in=0, pad_out=0, **kw):
    """convert_chain_device with row strides padded by pad_in / pad_out floats"""
    import torch
    ups = sum(1 for s in steps if s[1])
    h, w = x.shape
    d_in = torch.full((h, w + pad_in), -7.0, device="cuda")
    d_in[:, :w] = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_out = torch.full((h << ups, (w << ups) + pad_out), 12345.5, device="cuda")
    torch.cuda.synchronize()
    ctx.convert_chain_device(steps, d_in.data_ptr(), w, h, d_in.stride(0) * 4, d_out.data_ptr(), d_out.stride(0) * 4, **kw)
    ctx.synchronize()
    got = d_out.cpu().numpy()
    assert (got[:, w << ups:] == np.float32(12345.5)).all()
    return got[:, :w << ups]


def device_planes_chain(ctx, steps, planes, on_step=None):
    import torch
    ups = sum(1 for s in steps if s[1])
    d_in = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in planes]
    d_out = [torch.empty((x.shape[0] << ups, x.shape[1] << ups), device="cuda") for x in planes]
    torch.cuda.synchronize()
    ctx.convert_planes_chain_device(steps, [d.data_ptr() for d in d_in], [x.shape[1] for x in planes], [x.shape[0] for x in planes],
                                    [x.shape[1] * 4 for x in planes], [d.data_ptr() for d in d_out],
                                    [(x.shape[1] << ups) * 4 for x in planes], on_step)
    ctx.synchronize()
    return [d.cpu().numpy() for d in d_out]


def assert_all_equal(got, want, what):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if not np.array_equal(g, w)]
    assert len(got) == len(want) and not bad, (what, bad[:10])


@pytest.fixture(scope="module")
def shipped(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.fixture
def ctx(w2x):
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    yield c
    c.set_log(None)
    c.close()


@gpu
@pytest.mark.parametrize("config", ["f16x3", "f16+f8x2", "f16", "fp32"])
def test_sizes_precisions_and_engines(w2x, shipped, oracle_mod, config):
    c = w2x.Context(0, engine=w2x.ENGINE_FP32 if config == "fp32" else w2x.ENGINE_TC)
    try:
        if config != "fp32":
            c.set_precision(["f16x3", "f16+f8x2", "f16"].index(config))
        for i, (w, h) in enumerate(SIZES):
            x = plane(oracle_mod, w, h, 40 + i)
            for steps in ([(shipped["noise1"], False, True)], [(shipped["scale2.0x"], True, True)]):
                if steps[0][1] and (w, h) == (256, 256) and config == "fp32":
                    continue   # the 512 x 512 scale case runs on the tensor-core engine
                want = loop(c, steps, x)
                assert np.array_equal(c.convert_chain(steps, x), want), (config, w, h, steps[0][1])
                assert np.array_equal(device_chain(c, steps, x), want), (config, w, h, steps[0][1])
                got = c.convert_planes_chain(steps, [x])
                assert np.array_equal(got[0], want), (config, w, h, steps[0][1])
                assert np.array_equal(device_planes_chain(c, steps, [x])[0], want), (config, w, h, steps[0][1])
    finally:
        c.close()


@gpu
def test_planes_converted_alone_in_row_bands(w2x, shipped, oracle_mod):
    """a small scratch limit cuts every variant of the 45 x 77 plane (and of its 2x plane) into row bands"""
    for engine in (w2x.ENGINE_TC, w2x.ENGINE_FP32):
        c = w2x.Context(0, engine=engine)
        try:
            x = plane(oracle_mod, 45, 77, 5)
            for steps in ([(shipped["noise1"], False, True)], [(shipped["scale2.0x"], True, True)]):
                c.set_scratch_limit(0)
                want_plain = loop(c, steps, x)
                c.set_scratch_limit(128 * (154 + 14) * 4 * 30)   # ~16 rows per band on the widest variant
                want = loop(c, steps, x)
                assert np.array_equal(want, want_plain)
                assert np.array_equal(c.convert_chain(steps, x), want)
                assert np.array_equal(device_chain(c, steps, x), want)
                assert np.array_equal(c.convert_planes_chain(steps, [x])[0], want)
                assert np.array_equal(device_planes_chain(c, steps, [x])[0], want)
        finally:
            c.close()


@gpu
def test_strided_planes_on_both_entries(ctx, shipped, oracle_mod):
    steps = [(shipped["noise1"], False, True), (shipped["scale2.0x"], True, True)]
    for w, h in ((37, 29), (1, 17), (130, 77)):
        x = plane(oracle_mod, w, h, w + 3 * h)
        want = loop(ctx, steps, x)
        buf = np.full((h, w + 5), -7.0, np.float32)
        buf[:, :w] = x
        sentinel = np.float32(12345.5)
        obuf = np.full((2 * h, 2 * w + 3), sentinel, np.float32)
        ctx.convert_chain(steps, buf[:, :w], out=obuf[:, :2 * w])
        assert np.array_equal(obuf[:, :2 * w], want) and (obuf[:, 2 * w:] == sentinel).all()
        obuf[:] = sentinel
        ctx.convert_planes_chain(steps, [buf[:, :w]], out=[obuf[:, :2 * w]])
        assert np.array_equal(obuf[:, :2 * w], want) and (obuf[:, 2 * w:] == sentinel).all()
        assert np.array_equal(device_chain(ctx, steps, x, pad_in=3, pad_out=9), want)


@gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_chains(ctx, shipped, oracle_mod, precision):
    ctx.set_precision(precision)
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    chains = [[(noise, False, False), (scale, True, True), (scale, True, True)],
              [(noise, False, True), (scale, True, False)],
              [(scale, True, True), (noise, False, False)],
              [(noise, False, True), (noise, False, True)]]
    for i, steps in enumerate(chains):
        for w, h in ((15, 13), (1, 9), (40, 23)):
            x = plane(oracle_mod, w, h, 10 * i + w)
            want = loop(ctx, steps, x)
            assert np.array_equal(ctx.convert_chain(steps, x), want), (i, w, h)
            assert np.array_equal(device_chain(ctx, steps, x), want), (i, w, h)
        planes = [plane(oracle_mod, w, h, 7 * w + h) for w, h in ((15, 13), (1, 9), (40, 23), (9, 1), (33, 2))]
        want = [ctx.convert_chain(steps, x, block_splitting=False) for x in planes]
        assert_all_equal(ctx.convert_planes_chain(steps, planes), want, i)
        assert_all_equal(device_planes_chain(ctx, steps, planes), want, i)


@gpu
def test_collection_where_some_variants_pack_and_some_do_not(ctx, shipped, oracle_mod):
    rng = np.random.default_rng(3)
    sizes = [(37, 29), (29, 37), (1, 17), (17, 1), (200, 90), (90, 200)] + [(int(a), int(b)) for a, b in rng.integers(1, 60, (30, 2))]
    planes = [plane(oracle_mod, w, h, 60 + i) for i, (w, h) in enumerate(sizes)]
    # 4 MB: the padded variants of the small planes pack, those of 200 x 90 (and every 2x variant past ~90 x 90) are converted alone
    ctx.set_scratch_limit(4 << 20)
    for steps in ([(shipped["noise1"], False, True)], [(shipped["scale2.0x"], True, True)],
                  [(shipped["noise1"], False, False), (shipped["scale2.0x"], True, True)]):
        want = [ctx.convert_chain(steps, x, block_splitting=False) for x in planes]
        assert_all_equal(ctx.convert_planes_chain(steps, planes), want, len(steps))
        assert_all_equal(device_planes_chain(ctx, steps, planes), want, len(steps))
        for i in (0, 4, 7):
            assert np.array_equal(want[i], loop(ctx, steps, planes[i])), i


@gpu
def test_progress_lines_and_callbacks_match_the_plain_calls(ctx, shipped, oracle_mod):
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    for w, h in ((45, 33), (300, 600)):       # the second: host copy bands on the plain last step
        x = plane(oracle_mod, w, h, 2)
        for flags in ((True, True), (False, True), (True, False)):
            plain = [(noise, False), (scale, True)]
            tta = [(m, up, f) for (m, up), f in zip(plain, flags)]
            for entry in ("host", "device", "planes_host", "planes_device"):
                lines = {}
                for name, steps in (("plain", plain), ("tta", tta)):
                    got = []
                    ctx.set_log(got.append)
                    cb = lambda k: got.append(("step", k))   # noqa: E731
                    if entry == "host":
                        ctx.convert_chain(steps, x, on_step=cb)
                    elif entry == "device":
                        device_chain(ctx, steps, x, on_step=cb)
                    elif entry == "planes_host":
                        ctx.convert_planes_chain(steps, [x, x[:7, :5]], on_step=cb)
                    else:
                        device_planes_chain(ctx, steps, [x, x[:7, :5]], on_step=cb)
                    lines[name] = got
                assert lines["tta"] == lines["plain"] and len(lines["plain"]) > 2, (w, h, flags, entry)


@gpu
def test_launch_counts(ctx, shipped, oracle_mod):
    import torch
    noise, scale = shipped["noise1"], shipped["scale2.0x"]

    def launches(fn):
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        fn()
        ctx.synchronize()
        return ctx.launch_count() - n0

    for w, h, limit in ((45, 33, 0), (45, 77, 128 * 104 * 4 * 31)):
        ctx.set_scratch_limit(limit)
        x = plane(oracle_mod, w, h, 1)
        d_x = torch.from_numpy(x).cuda()
        d_o = torch.empty((4 * h, 4 * w), device="cuda")
        d_vars = [torch.from_numpy(dense(variant(x, j))).cuda() for j in range(8)]
        plain_noise = sum(launches(lambda v=v: ctx.convert_plane_device(noise, v.data_ptr(), v.shape[1], v.shape[0], v.shape[1] * 4,
                                                                        d_o.data_ptr(), v.shape[1] * 4)) for v in d_vars)
        plain_up = sum(launches(lambda v=v: ctx.convert_chain_device([(scale, True)], v.data_ptr(), v.shape[1], v.shape[0], v.shape[1] * 4,
                                                                     d_o.data_ptr(), v.shape[1] * 8)) for v in d_vars)
        noise_once = launches(lambda: ctx.convert_plane_device(noise, d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), w * 4))
        got = launches(lambda: ctx.convert_chain_device([(noise, False, True)], d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), w * 4))
        assert got == plain_noise + 2, (w, h)
        got = launches(lambda: ctx.convert_chain_device([(scale, True, True)], d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), w * 8))
        assert got == plain_up + 2, (w, h)
        got = launches(lambda: ctx.convert_chain_device([(noise, False), (scale, True, True)], d_x.data_ptr(), w, h, w * 4, d_o.data_ptr(), w * 8))
        assert got == noise_once + plain_up + 2, (w, h)
    ctx.set_scratch_limit(0)
    # a collection: the plain call on the 8n variant planes (packed the same way) + 2
    planes = [plane(oracle_mod, w, h, 9 + w) for w, h in ((37, 29), (1, 17), (60, 8), (13, 13))]
    d_in = [torch.from_numpy(x).cuda() for x in planes]
    d_out = [torch.empty_like(d) for d in d_in]
    vs = [dense(variant(x, j)) for x in planes for j in range(8)]
    d_vs = [torch.from_numpy(v).cuda() for v in vs]
    d_vo = [torch.empty_like(d) for d in d_vs]
    plain = launches(lambda: ctx.convert_planes_device(noise, [d.data_ptr() for d in d_vs], [v.shape[1] for v in vs], [v.shape[0] for v in vs],
                                                       [v.shape[1] * 4 for v in vs], [d.data_ptr() for d in d_vo], [v.shape[1] * 4 for v in vs]))
    got = launches(lambda: ctx.convert_planes_chain_device([(noise, False, True)], [d.data_ptr() for d in d_in], [x.shape[1] for x in planes],
                                                           [x.shape[0] for x in planes], [x.shape[1] * 4 for x in planes],
                                                           [d.data_ptr() for d in d_out], [x.shape[1] * 4 for x in planes]))
    assert got == plain + 2
    assert np.array_equal(d_out[0].cpu().numpy(), mean8([unvariant(d_vo[j].cpu().numpy(), j) for j in range(8)]))


@gpu
def test_argument_errors_name_the_step(w2x, ctx, shipped):
    L = w2x.lib()
    noise, scale = shipped["noise1"], shipped["scale2.0x"]
    x = np.ones((8, 8), np.float32)
    sentinel = np.float32(-3.25)
    out = np.full((32, 32), sentinel, np.float32)
    models = (C.c_void_p * 3)(noise._h, scale._h, scale._h)

    def chain(kinds):
        r = L.w2x_convert_chain(ctx._h, 3, models, (C.c_int * 3)(*kinds), x.ctypes.data, 8, 8, 32, out.ctypes.data, 128, 0,
                                w2x.capi.STEP_FN(), None)
        return r, L.w2x_last_error().decode()

    def planes_chain(kinds):
        r = L.w2x_convert_planes_chain(ctx._h, 3, models, (C.c_int * 3)(*kinds), 1, (C.c_void_p * 1)(x.ctypes.data), (C.c_int * 1)(8),
                                       (C.c_int * 1)(8), (C.c_size_t * 1)(32), (C.c_void_p * 1)(out.ctypes.data), (C.c_size_t * 1)(128),
                                       w2x.capi.STEP_FN(), None)
        return r, L.w2x_last_error().decode()

    for fn in (chain, planes_chain):
        for ok in ([4, 5, 5], [0, 1, 5], [4, 1, 1]):
            assert fn(ok)[0] == 0, (fn.__name__, ok)
        out[:] = sentinel
        for bad in (2, 3, 6, 8, -1):
            for k in range(3):
                kinds = [4, 5, 5]
                kinds[k] = bad
                r, msg = fn(kinds)
                assert r == ERR_ARG and f"step {k}" in msg, (fn.__name__, bad, k, r, msg)
                assert (out == sentinel).all()


@gpu
def test_out_of_memory_leaves_nothing_queued(w2x, shipped, oracle_mod):
    """with the device all but full, a TTA step that cannot reserve its buffers returns W2X_ERR_NOMEM before any launch"""
    import torch
    c = w2x.Context(0, engine=w2x.ENGINE_TC)
    filler = None
    try:
        model = shipped["noise1"]
        c.convert_chain([(model, False, True)], plane(oracle_mod, 16, 16, 1))   # the model's device copy and small buffers exist
        w = h = 2048                                                               # 8 variants + 8 outputs: 256 MB, plus the frames
        d_in = torch.from_numpy(plane(oracle_mod, w, h, 2)).cuda()
        d_out = torch.full((h, w), -3.25, device="cuda")
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(free - (64 << 20), 0), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        n0 = c.launch_count()
        for entry in ("chain", "planes"):
            with pytest.raises(w2x.W2xError) as e:
                if entry == "chain":
                    c.convert_chain_device([(model, False, True)], d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), w * 4)
                else:
                    c.convert_planes_chain_device([(model, False, True)], [d_in.data_ptr()], [w], [h], [w * 4], [d_out.data_ptr()], [w * 4])
            assert e.value.status == ERR_NOMEM, e.value.message
            assert c.launch_count() == n0
        c.synchronize()
        del filler
        filler = None
        torch.cuda.empty_cache()
        assert (d_out == -3.25).all().item()
        # and with the memory back, the same call runs
        c.convert_chain_device([(model, False, True)], d_in.data_ptr(), w, h, w * 4, d_out.data_ptr(), w * 4)
        c.synchronize()
        assert not (d_out == -3.25).all().item()
    finally:
        del filler
        torch.cuda.empty_cache()
        c.close()


@gpu
def test_against_the_oracle(ctx, shipped, oracle_models, oracle_mod):
    ctx.set_precision(0)   # f16x3
    x = plane(oracle_mod, 37, 29, 9)
    for name, up in (("noise1", False), ("scale2.0x", True)):
        src = up2(x) if up else x
        ref = mean8([unvariant(oracle_models[name].convert(dense(variant(src, j)), n_job=4), j) for j in range(8)])
        got = ctx.convert_chain([(shipped[name], up, True)], x)
        assert np.abs(got - ref).max() <= 1e-4, name


# ---- the CLI ------------------------------------------------------------------------------------------------------------------
def _reference_tta_pipeline(bgr, mode, level, ratio, oracle_models, ncpu):
    """src/main.cpp restated with cv2 for the plumbing, every convertWithModels replaced by the oracle's 8-variant mean"""
    import cv2

    def convert(name, y):
        return mean8([unvariant(oracle_models[name].convert(dense(variant(y, j)), n_job=ncpu), j) for j in range(8)])

    image = cv2.cvtColor(bgr.astype(np.float32) * np.float32(1 / 255.0), cv2.COLOR_RGB2YUV)
    if mode in ("noise", "noise_scale"):
        ch = cv2.split(image)
        image = cv2.merge([convert(f"noise{level}", ch[0].copy()), ch[1], ch[2]])
    if mode in ("scale", "noise_scale"):
        it = int(np.ceil(np.log2(ratio)))
        shrink = 0.0 if int(ratio) == 2 ** it else ratio / 2.0 ** it
        for _ in range(it):
            size = (image.shape[1] * 2, image.shape[0] * 2)
            y = cv2.split(cv2.resize(image, size, interpolation=cv2.INTER_NEAREST))[0].copy()
            ch = list(cv2.split(cv2.resize(image, size, interpolation=cv2.INTER_CUBIC)))
            ch[0] = convert("scale2.0x", y)
            image = cv2.merge(ch)
        if shrink != 0.0:
            image = cv2.resize(image, (int(image.shape[1] * shrink), int(image.shape[0] * shrink)), interpolation=cv2.INTER_LINEAR)
    out = cv2.cvtColor(image, cv2.COLOR_YUV2RGB)
    return np.clip(np.rint(out * np.float32(255.0)), 0, 255).astype(np.uint8)


@gpu
@pytest.mark.parametrize("mode,ratio", [("noise", 2.0), ("scale", 2.0), ("noise_scale", 2.0)])
def test_cli_tta_matches_the_reference_pipeline(w2x, tmp_path, json_models, oracle_models, ncpu, mode, ratio):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    bgr = _test_image(45, 33, 11)
    cv2.imwrite(str(tmp_path / "in.png"), bgr)
    mdir = os.path.dirname(json_models["scale2.0x"])
    runs = {}
    for tta in ("0", "1"):
        d = tmp_path / f"tta{tta}"
        d.mkdir()
        args = [CLI, "-i", str(tmp_path / "in.png"), "-o", str(d / "out.png"), "-m", mode, "--scale_ratio", str(ratio), "--model_dir", mdir]
        r = subprocess.run(args + (["--tta", "1"] if tta == "1" else []), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[tta] = (r.stdout, cv2.imread(str(d / "out.png"), cv2.IMREAD_COLOR))
    assert runs["1"][0] == runs["0"][0]
    out = runs["1"][1]
    ref = _reference_tta_pipeline(bgr, mode, 1, ratio, oracle_models, ncpu)
    assert out.shape == ref.shape
    diff = np.abs(out.astype(int) - ref.astype(int))
    assert diff.max() <= 1 and (diff > 0).mean() < 0.01
    assert not np.array_equal(out, runs["0"][1])                       # the switch does change the picture


def test_cli_tta_with_several_gpus_writes_nothing(w2x, tmp_path, json_models):
    cv2 = pytest.importorskip("cv2")
    from test_cli import _test_image
    w2x.build()
    cv2.imwrite(str(tmp_path / "in.png"), _test_image(20, 16))
    for extra, env in ((["--gpus", "2"], {}), ([], {"W2X_GPUS": "2"})):
        r = subprocess.run([CLI, "-i", "in.png", "--tta", "1", "--model_dir", os.path.dirname(json_models["scale2.0x"]), *extra],
                           capture_output=True, text=True, cwd=tmp_path, env=dict(os.environ, **env))
        assert r.returncode == 1 and "--tta" in r.stderr and r.stdout == ""
        assert os.listdir(tmp_path) == ["in.png"]
