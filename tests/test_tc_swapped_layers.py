"""The Cout = 64 tensor-core layers run with the weights as the wgmma A operand and the pixels as B (Cfg::SWAP in
csrc/tc_config.cuh).  The tensor cores' sums do not depend on which operand is A, so these layers give the bits the
pixels-as-A kernel gave.  The operands here are ordinary random values, not exactly representable ones, so a changed order
of additions inside a wgmma or across taps, chunks and corrections would show (tests/test_tc_exact.py cannot see one).

tests/golden/swapped_layers.json holds the SHA-256 of each case's filter_layer output as the pixels-as-A kernel computed it,
written with
    python tests/test_tc_swapped_layers.py --write-golden <repository root of that build> tests/golden/swapped_layers.json
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "swapped_layers.json")
SHAPES = [(32, 64), (64, 64), (128, 64)]
PRECISIONS = ["f16x3", "f16+f8x2", "f16"]
NUM_SMS = (1, 3, 0)                  # 0: every SM
W, H = 40, 30                        # a 42 x 32 frame: 3 x 2 tile-sets


def case_inputs(cin, cout):
    rng = np.random.default_rng(7 * cin + cout)
    w = (rng.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32)
    b = rng.standard_normal(cout) * 0.1
    x = (rng.random((cin, H, W)) * 1.5 - 0.25).astype(np.float32)
    return w, b, x


def run_cases(w2x):
    """{"<cin>x<cout>/<precision>/sms<n>": sha256 of the output}"""
    precs = {"f16x3": w2x.PRECISION_F16X3, "f16+f8x2": w2x.PRECISION_F16_F8X2, "f16": w2x.PRECISION_F16}
    out = {}
    for prec in PRECISIONS:
        ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
        try:
            ctx.set_precision(precs[prec])
            for cin, cout in SHAPES:
                w, b, x = case_inputs(cin, cout)
                model = w2x.Model.from_arrays([w], [b])
                for sms in NUM_SMS:
                    ctx.debug_set_num_sms(sms)
                    y = ctx.filter_layer(model, 0, x)
                    assert np.isfinite(y).all()
                    out[f"{cin}x{cout}/{prec}/sms{sms}"] = hashlib.sha256(np.ascontiguousarray(y, np.float32).tobytes()).hexdigest()
        finally:
            ctx.debug_set_num_sms(0)
            ctx.close()
    return out


@pytest.mark.gpu
def test_cout64_layers_match_the_pixels_as_a_kernel_bit_for_bit(w2x):
    with open(GOLDEN) as f:
        want = json.load(f)
    got = run_cases(w2x)
    assert sorted(got) == sorted(want)
    bad = [k for k in sorted(want) if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(want)} cases differ: {bad}"


if __name__ == "__main__":
    if len(sys.argv) != 4 or sys.argv[1] != "--write-golden":
        sys.exit(__doc__)
    sys.path.insert(0, os.path.abspath(sys.argv[2]))
    import w2x_loader
    with open(sys.argv[3], "w") as f:
        json.dump(run_cases(w2x_loader.load()), f, indent=1, sort_keys=True)
