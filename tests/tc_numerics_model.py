"""tc_numerics_model.py -- CPU emulation of the tensor-core engine's arithmetic (test helper only).

Emulates, with torch fp32/fp64 on the CPU, what csrc/kernels_tc.cu computes: activations and
weights split into fp16 hi/lo (activations scaled by 16, weights by a power of two), the three
products xh*wh + xl*wh + xh*wl accumulated in wide precision, fp32 epilogue.  Products of two
fp16 numbers are exact in fp32, so the only thing not modelled is the tensor core's fp32
accumulation order/rounding.  Used to derive and defend the GPU parity tolerance.
"""
import numpy as np
import torch
import torch.nn.functional as F

ACT_SCALE = 16.0


def split16(x):
    hi = x.to(torch.float16)
    lo = (x - hi.to(x.dtype)).to(torch.float16)
    return hi, lo


def wscale_of(w):
    mx = float(np.abs(w).max())
    e = int(np.floor(np.log2(1024.0 / mx))) if mx > 0 else 0
    return float(2.0 ** min(max(e, 0), 14))


def leaky(v):
    return torch.clamp(v, max=0.0) * np.float32(0.1) + torch.clamp(v, min=0.0)


def convert_emulated(plane, weights, biases, acc_dtype=torch.float64):
    """convertWithModels the way the tensor-core engine computes it.  plane: HxW fp32 numpy."""
    n = len(weights)
    x = torch.from_numpy(np.pad(plane.astype(np.float32), n, mode="edge"))[None, None]
    # first layer: fp32 CUDA cores
    w0 = torch.from_numpy(weights[0])
    a = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), w0) + torch.from_numpy(biases[0].astype(np.float32))[None, :, None, None]
    a = leaky(a)
    for li in range(1, n - 1):
        ws = wscale_of(weights[li])
        w = torch.from_numpy(weights[li]) * ws
        wh, wl = split16(w)
        xs = a * ACT_SCALE
        xh, xl = split16(xs)
        xh, xl, wh, wl = (t.to(acc_dtype) for t in (xh, xl, wh, wl))
        acc = F.conv2d(xh, wh, padding=1) + F.conv2d(xl, wh, padding=1) + F.conv2d(xh, wl, padding=1)
        v = acc.to(torch.float32) * np.float32(1.0 / (ws * ACT_SCALE)) + torch.from_numpy(biases[li].astype(np.float32))[None, :, None, None]
        a = leaky(v)
    # last layer reads hi+lo back (fp32 CUDA cores)
    xs = a * ACT_SCALE
    xh, xl = split16(xs)
    a = (xh.float() + xl.float()) / ACT_SCALE
    v = F.conv2d(a, torch.from_numpy(weights[-1]), padding=1) + np.float32(biases[-1][0])
    out = leaky(v)[0, 0]
    return out[n:-n, n:-n].numpy()
