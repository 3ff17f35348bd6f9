"""tc_profile.py -- per-role wait/work cycle breakdown of the tensor-core layer kernels.

    mkdir -p build && python tools/tc_profile.py [size] [precision] > build/tc_profile.txt
Uses the kernel's own clock64 counters (w2x_debug_tc_profile_*): for every layer, cycles per
tile-set the first consumer warpgroup spent waiting for staged activations / weight stages, and
what the two producer warps waited for (build/ is git-ignored)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import w2x_loader  # noqa: E402
from oracle import oracle  # noqa: E402  (model fixture only)

w2x = w2x_loader.load()
size = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
om = oracle.OracleModel.golden("scale2.0x")
m = w2x.Model.from_arrays(om.weights, om.biases)
ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
x = oracle.seeded_plane(size, size, 1, "uniform")
mode = int(sys.argv[2]) if len(sys.argv) > 2 else 0      # 0 = f16x3, 1 = f16 + 2 x e4m3 corrections
ctx.set_precision(mode)
ctx.convert_plane(m, x)
ctx.convert_plane(m, x)
ctx.set_timing(True)
ctx.convert_plane(m, x)
clean = ctx.layer_times()
print(f"size {size}x{size} precision {mode}; per-layer ms without counters:", [round(t[0], 3) for t in clean], "sum", round(sum(t[0] for t in clean), 3))
ctx.debug_tc_profile_enable(True)
ctx.convert_plane(m, x)
times = ctx.layer_times()
print(f"per-layer ms with counters:", [round(t[0], 3) for t in times])
print("layer  ms     cyc/tileset  wait_a  wait_b  mma+epilogue | aprod_wait bprod_wait  (cycles per 16x16 tile-set, per-CTA average)")
for li in range(1, 6):
    d = ctx.debug_tc_profile_read(li)
    n = max(d["tilesets"], 1)
    rest = (d["total"] - d["mma_wait_a"] - d["mma_wait_b"]) / n
    print(f"L{li}   {times[li][0]:7.3f} {d['total'] / n:11.0f} {d['mma_wait_a'] / n:7.0f} {d['mma_wait_b'] / n:7.0f} {rest:13.0f} | "
          f"{d['aprod_wait'] / n:10.0f} {d['bprod_wait'] / n:10.0f}   ctas={d['ctas']} tilesets/cta={n:.0f}")
ctx.debug_tc_profile_enable(False)
