"""tc_smem_budget.py -- shared-memory operand traffic of the tensor-core layer kernels, set against their tensor work.

    python tools/tc_smem_budget.py [precision] [--pixels-as-a] [--measure [size]]

Both wgmma operands come from shared memory, which serves about 128 B per clock per SM.  For every layer of the scale2.0x
pass this prints, per 16x16 tile-set (both consumer warpgroups), the operand bytes the wgmmas read, the ideal tensor clocks
(dense H100 rates per SM: 2048 fp16 or 4096 e4m3 multiply-adds per clock) and the operand bytes per tensor clock.  Above
128 B/clk a layer cannot keep its tensor cores busy, whatever else it overlaps.  Computed from the instruction shapes
(Cfg::SWAP in csrc/tc_config.cuh decides the operand roles), not measured.  With --measure (needs the GPU) it adds the
clocks per tile-set the kernels' own counters report (as tools/tc_profile.py), on a size x size plane (default 4096).
--pixels-as-a: the budget with the pixels as the A operand in every layer (the Cout = 64 layers before Cfg::SWAP).
precision: f8 (default: f16 + 2 x e4m3), f16x3 or f16."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMEM_B_PER_CLK = 128
MAC_PER_CLK = {"f16": 2048, "e4m3": 4096}
K_BYTES = 32                              # one K step of either kind: 16 fp16 or 32 e4m3 per row


def wgmmas(prec):
    """the (kind, count) K steps per (tap, 32-channel chunk) of one m64 tile of output rows"""
    return {"f8": [("f16", 2), ("e4m3", 2)], "f16x3": [("f16", 6)], "f16": [("f16", 2)]}[prec]


def budget(cin, cout, prec, fused, pixels_as_a=False):
    """(operand bytes, ideal tensor clocks, swapped) per tile-set"""
    swap = cout == 64 and not fused and not pixels_as_a
    steps = 9 * (cin // 32) * 2            # (tap, chunk) pairs x two consumer warpgroups, 128 pixels each
    byts = clk = 0
    for kind, n in wgmmas(prec):
        if swap:                           # one m64n128: A = 64 weight rows, B = 128 pixels
            per = n * (64 * K_BYTES + 128 * K_BYTES)
        elif kind == "e4m3" and cout > 64:  # two m64 pixel halves, the corrections in 64-column slices
            per = 2 * (cout // 64) * n * (64 * K_BYTES + 64 * K_BYTES)
        else:                              # two m64 pixel halves, N = Cout
            per = 2 * n * (64 * K_BYTES + cout * K_BYTES)
        byts += steps * per
        clk += steps * n * 128 * cout * (K_BYTES if kind == "e4m3" else K_BYTES // 2) / MAC_PER_CLK[kind]
    return byts, clk, swap


def main():
    args = sys.argv[1:]
    measure = "--measure" in args
    pixels_as_a = "--pixels-as-a" in args
    args = [a for a in args if a != "--pixels-as-a"]
    size = 4096
    if measure:
        i = args.index("--measure")
        if i + 1 < len(args) and args[i + 1].isdigit():
            size = int(args.pop(i + 1))
        args.pop(i)
    prec = args[0] if args else "f8"
    from oracle import oracle              # model fixture only
    om = oracle.OracleModel.golden("scale2.0x")
    dims = [(w.shape[1], w.shape[0]) for w in om.weights]
    meas = {}
    if measure:
        import w2x_loader
        w2x = w2x_loader.load()
        m = w2x.Model.from_arrays(om.weights, om.biases)
        ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
        ctx.set_precision({"f16x3": w2x.PRECISION_F16X3, "f8": w2x.PRECISION_F16_F8X2, "f16": w2x.PRECISION_F16}[prec])
        x = oracle.seeded_plane(size, size, 1, "uniform")
        ctx.convert_plane(m, x)
        ctx.debug_tc_profile_enable(True)
        ctx.convert_plane(m, x)
        for li in range(1, len(dims) - 1):
            d = ctx.debug_tc_profile_read(li)
            meas[li] = d["total"] / max(d["tilesets"], 1)
        ctx.close()
    print(f"precision {prec}; per 16x16 tile-set, both consumer warpgroups" + (f"; measured on a {size}x{size} plane" if measure else ""))
    print("layer  shape      roles             operand KB  tensor clk  B/clk   smem clk" + ("  measured clk" if measure else ""))
    for li in range(1, len(dims) - 1):                    # the layers tc_conv3x3_kernel runs; the one before the last is fused
        cin, cout = dims[li]
        fused = li == len(dims) - 2
        byts, clk, swap = budget(cin, cout, prec, fused, pixels_as_a)
        roles = "A=weights B=px" if swap else "A=px B=weights"
        line = (f"L{li}     {cin:3d}->{cout:<3d}{'+1' if fused else '  '}  {roles:16s}  {byts / 1024:10.0f}  {clk:10.0f}  "
                f"{byts / clk:5.0f}  {byts / SMEM_B_PER_CLK:9.0f}")
        if measure:
            line += f"  {meas[li]:12.0f}"
        print(line)


if __name__ == "__main__":
    main()
