"""Float32, fp16 and e4m3 arithmetic rounded the way the kernels round, and emulators of the kernels whose float32 order is
fully specified (test helper only; tests/test_tc_exact.py and tests/test_edge_exact.py share it).

Every emulator computes with correctly rounded float32 operations in the kernel's own order, so its result is the one bit
pattern the kernel may produce:
  fp32_filter           conv3x3_planar_fp32 (csrc/kernels_fp32.cu), or with contract=False the reference's association
                        without FMA contraction (what oracle/w2x_oracle.c computes)
  emulate_first_layer   first_layer_kernel (csrc/tc_edge_kernels.cuh)
  tc_activation         the wgmma epilogue's scale, bias and leaky-ReLU (csrc/tc_kernel.cuh)
  record_lo, readback   the frame's record encoding and nhwc_to_planar's read-back
  emulate_last_fused    the fused last layer (epilogue_fuse) + last_gather_kernel
  emulate_last_separate last_layer_kernel on the record frame
"""
import numpy as np

F32 = np.float32
F8_A, F8_C = 10, 1                 # xl8 = e4m3(xl * 2^F8_A), xh8 = e4m3(xh * 2^-F8_C)   (csrc/tc_config.cuh)
ACT_SCALE = F32(16)


def f16(x):
    """round to fp16 (nearest, ties to even) and back to float32"""
    return np.asarray(x, F32).astype(np.float16).astype(F32)


def e4m3(x):
    """nearest e4m3fn value (ties to even, saturating at +-448: cvt.rn.satfinite.e4m3), as float64"""
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    _, e = np.frexp(np.maximum(a, 2.0 ** -6))            # a = m 2^e, m in [0.5, 1): the binade's quantum is 2^(e - 4)
    quantum = np.ldexp(1.0, e - 4)
    return np.copysign(np.minimum(np.rint(a / quantum) * quantum, 448.0), x)


def fma32(a, b, c):
    """correctly rounded float32 fmaf(a, b, c): the float64 product is exact, the float64 sum is rounded to odd (TwoSum
    gives its error), and a round-to-odd value with 29 spare bits rounds to the same float32 as the exact sum"""
    a, b, c = (np.asarray(t, F32).astype(np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    s = np.ascontiguousarray(s)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def add32(a, b):
    return (np.asarray(a, F32) + np.asarray(b, F32)).astype(F32)


def mul32(a, b):
    return (np.asarray(a, F32) * np.asarray(b, F32)).astype(F32)


def leaky_tc(v):
    """the tensor-core epilogue's and the first layer's leaky-ReLU: fmaxf(v, 0.1f * v)"""
    return np.maximum(v, mul32(v, F32(0.1)))


def leaky_last(r):
    """last_layer_kernel / last_gather_kernel / conv3x3_planar_fp32: fminf(r, 0) * 0.1f + fmaxf(r, 0)"""
    return add32(mul32(np.minimum(r, F32(0)), F32(0.1)), np.maximum(r, F32(0)))


# ---------------------------------------------------------------------------------------------------------------------
# fp32 CUDA-core engine
# ---------------------------------------------------------------------------------------------------------------------
def fp32_filter(x, w, b, contract=True, chunk=16):
    """Model::filter (same size, replicate border) on planes x [Cin, H, W]: per (o, i) t = w[0] v[0] (one rounded
    multiply), then fmaf over taps 1..8 row-major (contract=False: a rounded multiply and a rounded add per tap, the
    reference's association); acc += t with i ascending; + (float)bias; fminf(v, 0) 0.1f + fmaxf(v, 0)."""
    x = np.asarray(x, F32)
    w = np.asarray(w, F32)
    cout, cin = w.shape[:2]
    h, wd = x.shape[1:]
    p = np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge")
    acc = np.zeros((cout, h, wd), F32)
    for i0 in range(0, cin, chunk):                                   # [Cout, chunk, H, W] at a time
        i1 = min(cin, i0 + chunk)
        t = None
        for k in range(9):
            ky, kx = divmod(k, 3)
            v = p[None, i0:i1, ky:ky + h, kx:kx + wd]
            wk = w[:, i0:i1, ky, kx][:, :, None, None]
            if t is None:
                t = mul32(wk, v)
            elif contract:
                t = fma32(wk, v, t)
            else:
                t = add32(t, mul32(wk, v))
        for i in range(i1 - i0):
            acc = add32(acc, t[:, i])
    return leaky_last(add32(acc, np.asarray(b, np.float64).astype(F32)[:, None, None]))


def fp32_convert(plane, weights, biases):
    """convertWithModels on the fp32 engine: copyMakeBorder(n, replicate), the n layers, crop n"""
    n = len(weights)
    x = np.pad(np.asarray(plane, F32), n, mode="edge")[None]
    for w, b in zip(weights, biases):
        x = fp32_filter(x, w, b)
    return x[0, n:-n, n:-n]


# ---------------------------------------------------------------------------------------------------------------------
# tensor-core engine: the CUDA-core edges and the record encoding
# ---------------------------------------------------------------------------------------------------------------------
def tc_activation(acc32, ws, bias):
    """epilogue: v = leaky(fmaf(acc, 1 / wscale, 16 bias)) -- activations * 16 (ACT_SCALE folded in on the host)"""
    b16 = mul32(np.asarray(bias, np.float64).astype(F32), ACT_SCALE)
    return leaky_tc(fma32(acc32, F32(1.0 / ws), b16[:, None, None]))


def record_lo(v, f8):
    """what the frame's record keeps besides fp16(v), read back as float32: fp16(v - hi) or e4m3((v - hi) 2^10) 2^-10"""
    d = np.asarray(v, F32) - f16(v)                                   # exact
    return (e4m3(d.astype(np.float64) * 2.0 ** F8_A) * 2.0 ** -F8_A).astype(F32) if f8 else f16(d)


def record_xh8(v):
    """the record's xh8 = e4m3(fp16(v) / 2), read back as float64 with the 2^-F8_C taken out"""
    return e4m3(f16(v).astype(np.float64) * 2.0 ** -F8_C) * 2.0 ** F8_C


def readback(v, f8):
    """nhwc_to_planar: (hi + lo) / 16"""
    return mul32(add32(f16(v), record_lo(v, f8)), F32(1.0 / 16))


def emulate_first_layer(frame, w0, b0):
    """first_layer_kernel on a frame (the replicate-padded plane), replicate ring again at the frame edge: per channel
    t = (16 w[0]) v[0], then fmaf over taps 1..8, + 16 b, leaky"""
    p = np.pad(frame, 1, mode="edge")
    h, wd = frame.shape
    w16 = mul32(w0[:, 0], ACT_SCALE)                                  # [C, 3, 3]
    b16 = mul32(np.asarray(b0, np.float64).astype(F32), ACT_SCALE)[:, None, None]
    t = None
    for k in range(9):
        ky, kx = divmod(k, 3)
        v = p[None, ky:ky + h, kx:kx + wd]
        wk = w16[:, ky, kx][:, None, None]
        t = mul32(wk, v) if t is None else fma32(wk, v, t)
    return leaky_tc(add32(t, b16))


def emulate_last_fused(a1, w2, b2, n):
    """epilogue_fuse + last_gather_kernel on the last tensor-core layer's activations a1 ([C, ph, pw], * 16): lane q of a
    quad sums channels 8 jj + 2q, +1 (jj ascending) with weights / 16, two shuffles; then the taps in row-major order"""
    c2, ph, pw = a1.shape
    lw = mul32(np.asarray(w2, F32)[0], F32(1.0 / 16)).reshape(c2, 9)
    part = np.zeros((4, 9, ph, pw), F32)
    for jj in range(c2 // 8):
        ch = 8 * jj + 2 * np.arange(4)
        part = fma32(a1[ch][:, None], lw[ch][:, :, None, None], part)
        part = fma32(a1[ch + 1][:, None], lw[ch + 1][:, :, None, None], part)
    P = add32(add32(part[0], part[1]), add32(part[2], part[3]))       # [9, ph, pw]
    acc = np.zeros((ph - 2 * n, pw - 2 * n), F32)
    for t in range(9):
        ky, kx = divmod(t, 3)
        acc = add32(acc, P[t, n - 1 + ky:ph - n - 1 + ky, n - 1 + kx:pw - n - 1 + kx])
    return leaky_last(add32(acc, F32(b2[0])))


def emulate_last_separate(a1, w2, b2, n, f8):
    """last_layer_kernel: the record read back as (hi + lo) / 16; per group of 8 channels eight partial sums over the taps"""
    c2, ph, pw = a1.shape
    w2 = np.asarray(w2, F32)
    a = mul32(add32(f16(a1), record_lo(a1, f8)), F32(1.0 / 16))
    acc = np.zeros((ph - 2 * n, pw - 2 * n), F32)
    for c8 in range(c2 // 8):
        cs = slice(8 * c8, 8 * c8 + 8)
        t = np.zeros((8,) + acc.shape, F32)
        for ky in range(3):
            for kx in range(3):
                t = fma32(w2[0, cs, ky, kx][:, None, None], a[cs, n - 1 + ky:ph - n - 1 + ky, n - 1 + kx:pw - n - 1 + kx], t)
        for e in range(8):
            acc = add32(acc, t[e])
    return leaky_last(add32(acc, F32(b2[0])))
