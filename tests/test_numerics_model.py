"""Why the tensor-core engine's GPU parity tolerance is what it is: the 3-pass fp16 split scheme,
emulated on the CPU (tests/tc_numerics_model.py), stays within 5e-6 of the fp32 reference
arithmetic on white noise -- 20x inside the 1e-4 gate of BASELINE.json."""
import numpy as np
import pytest

import tc_numerics_model as T


@pytest.mark.parametrize("name", ["scale2.0x", "noise1", "noise2"])
def test_three_pass_fp16_split_is_fp32_faithful(oracle_mod, oracle_models, ncpu, name):
    om = oracle_models[name]
    x = oracle_mod.seeded_plane(72, 64, 2, "uniform")
    ref = om.convert(x, n_job=ncpu)
    emu = T.convert_emulated(x, om.weights, om.biases)
    assert np.abs(emu - ref).max() <= 5e-6


def test_single_pass_fp16_would_fail_the_gate(oracle_mod, oracle_models, ncpu):
    """Control: dropping the two correction passes gives ~1e-3 (SURVEY.md section 7 hard part 1)."""
    import torch
    import torch.nn.functional as F
    om = oracle_models["scale2.0x"]
    x = oracle_mod.seeded_plane(72, 64, 2, "uniform")
    ref = om.convert(x, n_job=ncpu)
    n = len(om)
    a = torch.from_numpy(np.pad(x, n, mode="edge"))[None, None]
    for li in range(n):
        w = torch.from_numpy(om.weights[li])
        if 0 < li < n - 1:
            a, w = a.half().double(), w.half().double()
        v = F.conv2d(a.double(), w.double(), padding=1).float() + torch.from_numpy(om.biases[li].astype(np.float32))[None, :, None, None]
        a = T.leaky(v)
    err = np.abs(a[0, 0, n:-n, n:-n].numpy() - ref).max()
    assert err > 1e-4


def test_fp16_plus_two_e4m3_corrections_is_inside_the_gate(oracle_mod, oracle_models, ncpu):
    """W2X_PRECISION_F16_F8X2: xh*wh in fp16, xl*wh and xh*wl on e4m3 copies (scale exponents F8_A = 10, F8_C = 1).
    Emulated with torch.float8_e4m3fn: ~2e-5 on white noise, 4x inside the 1e-4 gate."""
    import torch
    import torch.nn.functional as F
    A, Cc = 10, 1

    def e4m3(t):
        return t.to(torch.float8_e4m3fn).to(torch.float64)

    worst = 0.0
    for name in ("scale2.0x", "noise1"):
        om = oracle_models[name]
        x = oracle_mod.seeded_plane(96, 80, 4, "uniform")
        ref = om.convert(x, n_job=ncpu)
        n = len(om)
        act = torch.from_numpy(np.pad(x, n, mode="edge"))[None, None]
        act = T.leaky(F.conv2d(F.pad(act, (1, 1, 1, 1), mode="replicate"), torch.from_numpy(om.weights[0])) +
                      torch.from_numpy(om.biases[0].astype(np.float32))[None, :, None, None])
        for li in range(1, n - 1):
            ws = T.wscale_of(om.weights[li])
            w = torch.from_numpy(om.weights[li]) * ws
            wh = w.half().float()
            xs = act * 16.0
            xh = xs.half().float()
            acc = (F.conv2d(xh.double(), wh.double(), padding=1) +
                   F.conv2d(e4m3((xs - xh) * 2.0 ** A), e4m3(wh * 2.0 ** -A), padding=1) +
                   F.conv2d(e4m3(xh * 2.0 ** -Cc), e4m3((w - wh) * 2.0 ** Cc), padding=1))
            act = T.leaky(acc.float() * np.float32(1 / (ws * 16.0)) + torch.from_numpy(om.biases[li].astype(np.float32))[None, :, None, None])
        out = T.leaky(F.conv2d(act, torch.from_numpy(om.weights[-1]), padding=1) + np.float32(om.biases[-1][0]))[0, 0, n:-n, n:-n].numpy()
        worst = max(worst, float(np.abs(out - ref).max()))
    assert worst <= 4e-5, worst


def _f8_emulated(om, x, drop_xl=(), drop_wl=()):
    """the default precision's arithmetic (see the test above) for one plane, wide accumulation; drop_xl / drop_wl: layers
    whose xl*wh / xh*wl correction pass is left out (what-if experiments, not a shipped mode)"""
    import torch
    import torch.nn.functional as F
    A, Cc = 10, 1
    e4m3 = lambda t: t.to(torch.float8_e4m3fn).to(torch.float64)
    n = len(om)
    act = torch.from_numpy(np.pad(x, n, mode="edge"))[None, None]
    act = T.leaky(F.conv2d(F.pad(act, (1, 1, 1, 1), mode="replicate"), torch.from_numpy(om.weights[0])) +
                  torch.from_numpy(om.biases[0].astype(np.float32))[None, :, None, None])
    for li in range(1, n - 1):
        ws = T.wscale_of(om.weights[li])
        w = torch.from_numpy(om.weights[li]) * ws
        wh = w.half().float()
        xs = act * 16.0
        xh = xs.half().float()
        acc = F.conv2d(xh.double(), wh.double(), padding=1)
        if li not in drop_xl:
            acc = acc + F.conv2d(e4m3((xs - xh) * 2.0 ** A), e4m3(wh * 2.0 ** -A), padding=1)
        if li not in drop_wl:
            acc = acc + F.conv2d(e4m3(xh * 2.0 ** -Cc), e4m3((w - wh) * 2.0 ** Cc), padding=1)
        act = T.leaky(acc.float() * np.float32(1 / (ws * 16.0)) + torch.from_numpy(om.biases[li].astype(np.float32))[None, :, None, None])
    return T.leaky(F.conv2d(act, torch.from_numpy(om.weights[-1]), padding=1) + np.float32(om.biases[-1][0]))[0, 0, n:-n, n:-n].numpy()


def test_the_two_pass_equivalents_are_needed_even_on_one_layer(oracle_mod, oracle_models, ncpu):
    """VERDICT r01 item 8 ("dropping xl*wh where the numerics model shows headroom"): it shows none.  Leaving out the xl*wh
    pass on the 128 -> 128 layer alone (51 % of the FLOPs, the only place where it would pay) breaks the 1e-4 gate on white
    noise for every shipped model; leaving out xh*wl there lands at 5e-5 .. 9e-5 -- inside the gate for the noise models,
    without margin for scale2.0x.  The arithmetic stays at 2.0 fp16-pass-equivalents on every tensor-core layer."""
    for name in ("scale2.0x", "noise1", "noise2"):
        om = oracle_models[name]
        x = oracle_mod.seeded_plane(96, 80, 4, "uniform")
        ref = om.convert(x, n_job=ncpu)
        base = float(np.abs(_f8_emulated(om, x) - ref).max())
        no_xl = float(np.abs(_f8_emulated(om, x, drop_xl=(5,)) - ref).max())
        no_wl = float(np.abs(_f8_emulated(om, x, drop_wl=(5,)) - ref).max())
        print(name, f"base {base:.1e}  without xl*wh on L5 {no_xl:.1e}  without xh*wl on L5 {no_wl:.1e}")
        assert base <= 4e-5 and no_xl > 1e-4 and no_wl > 1.5 * base, (name, base, no_xl, no_wl)


@pytest.mark.parametrize("name", ["scale2.0x", "noise1", "noise2"])
def test_default_precision_on_adversarial_planes_stays_inside_the_gate(oracle_mod, oracle_models, ncpu, name):
    """Inputs chosen to excite the network far harder than photographs do -- binary noise, checkerboards, stripes, isolated
    impulses, saturated and out-of-range planes: the emulated default arithmetic stays below 6e-5 (the GPU test's tolerance),
    i.e. the 1e-4 gate holds with margin on every one of them, for all three shipped models."""
    rng = np.random.default_rng(12)
    h, w = 48, 56
    yy, xx = np.mgrid[0:h, 0:w]
    planes = {
        "binary noise": (rng.random((h, w)) > 0.5).astype(np.float32),
        "checkerboard": ((yy + xx) % 2).astype(np.float32),
        "2px stripes": ((xx // 2) % 2).astype(np.float32),
        "impulses": (rng.random((h, w)) > 0.97).astype(np.float32),
        "all ones": np.ones((h, w), np.float32),
        "ramp": (xx / (w - 1)).astype(np.float32),
        "out of range": (rng.random((h, w)) * 3.0 - 1.0).astype(np.float32),     # the path does not clamp (SURVEY 8a)
    }
    om = oracle_models[name]
    worst = {}
    for label, x in planes.items():
        ref = om.convert(x, n_job=ncpu)
        err = float(np.abs(_f8_emulated(om, x) - ref).max())
        scale = max(1.0, float(np.abs(ref).max()))
        worst[label] = err / scale
        assert err <= 6e-5 * scale, (name, label, err)
    print(name, {k: f"{v:.1e}" for k, v in worst.items()})


def test_winograd_f2x2_3x3_in_the_split_arithmetic_would_stay_inside_the_gate(oracle_mod, oracle_models, ncpu):
    """What could come next: the tensor-bound layers are bound by energy, and Winograd F(2x2,3x3) needs
    16/36 of the direct convolution's multiply-adds.  Emulated here with the SAME operand split (fp16 main product + two e4m3
    correction products, fp32 accumulation) applied to the transformed operands V = B^T d B (fp32 transform of the x16
    activations) and U = G g G^T, on the three widest layers: the error against the reference stays where the direct form's
    is (2e-5 on white noise), far inside the 1e-4 gate -- the obstacle is accumulator capacity (16 live accumulator tiles per output
    tile, held in registers by wgmma), not numerics."""
    import torch
    import torch.nn.functional as F
    A, Cc = 10, 1
    e4m3 = lambda t: t.to(torch.float8_e4m3fn).to(torch.float64)
    Bt = torch.tensor([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=torch.float64)
    G = torch.tensor([[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]], dtype=torch.float64)
    At = torch.tensor([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=torch.float64)

    def split_mm(V, U):     # [P, Cin] x [Cout, Cin]^T in the GPU's arithmetic
        Vh, Uh = V.float().half().double(), U.float().half().double()
        return Vh @ Uh.T + e4m3((V - Vh) * 2.0 ** A) @ e4m3(Uh * 2.0 ** -A).T + e4m3(Vh * 2.0 ** -Cc) @ e4m3((U - Uh) * 2.0 ** Cc).T

    def conv_direct(xs, w):
        wh, xh = w.float().half().double(), xs.float().half().double()
        return (F.conv2d(xh, wh, padding=1) + F.conv2d(e4m3((xs - xh) * 2.0 ** A), e4m3(wh * 2.0 ** -A), padding=1) +
                F.conv2d(e4m3(xh * 2.0 ** -Cc), e4m3((w - wh) * 2.0 ** Cc), padding=1))

    def conv_winograd(xs, w):
        _, C, H, W = xs.shape
        Co, th, tw = w.shape[0], (H + 1) // 2, (W + 1) // 2
        tiles = F.pad(xs, (1, 1 + (W % 2), 1, 1 + (H % 2))).unfold(2, 4, 2).unfold(3, 4, 2)          # [1, C, th, tw, 4, 4]
        V = torch.einsum('ij,bcthjk,lk->bcthil', Bt, tiles, Bt).float().double()[0].permute(1, 2, 0, 3, 4).reshape(th * tw, C, 4, 4)
        U = torch.einsum('ij,ocjk,lk->ocil', G, w.double(), G).float().double()
        M = torch.stack([torch.stack([split_mm(V[:, :, i, j], U[:, :, i, j]).float().double() for j in range(4)], -1) for i in range(4)], -2)
        Y = torch.einsum('ij,pojk,lk->poil', At, M, At).float().double()
        return Y.reshape(th, tw, Co, 2, 2).permute(2, 0, 3, 1, 4).reshape(Co, th * 2, tw * 2)[None, :, :H, :W]

    om = oracle_models["scale2.0x"]
    x = oracle_mod.seeded_plane(48, 40, 4, "uniform")
    ref = om.convert(x, n_job=ncpu)
    n = len(om)
    errs = {}
    for label, wino in (("direct", ()), ("winograd on L3-L5", (3, 4, 5))):
        act = torch.from_numpy(np.pad(x, n, mode="edge"))[None, None]
        act = T.leaky(F.conv2d(F.pad(act, (1, 1, 1, 1), mode="replicate"), torch.from_numpy(om.weights[0])) +
                      torch.from_numpy(om.biases[0].astype(np.float32))[None, :, None, None])
        for li in range(1, n - 1):
            ws = T.wscale_of(om.weights[li])
            w, xs = (torch.from_numpy(om.weights[li]) * ws).double(), (act * 16.0).double()
            acc = conv_winograd(xs, w) if li in wino else conv_direct(xs, w)
            act = T.leaky(acc.float() * np.float32(1 / (ws * 16.0)) + torch.from_numpy(om.biases[li].astype(np.float32))[None, :, None, None])
        out = T.leaky(F.conv2d(act, torch.from_numpy(om.weights[-1]), padding=1) + np.float32(om.biases[-1][0]))[0, 0, n:-n, n:-n].numpy()
        errs[label] = float(np.abs(out - ref).max())
    print(errs)
    assert errs["direct"] <= 4e-5 and errs["winograd on L3-L5"] <= 4e-5, errs
