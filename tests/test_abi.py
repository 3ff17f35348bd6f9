"""The C-ABI library: loads without a GPU, exports every symbol include/w2x_b200.h declares, mirrors
the reference's modelUtility configuration and block arithmetic, and refuses to compute without a
device (no CPU fallback)."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, golden_path, _has_gpu


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "w2x_b200.h")).read()
    return sorted(set(re.findall(r"W2X_API\s+[\w\s\*]+?\b(w2x_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol(w2x):
    declared = _declared_symbols()
    assert len(declared) >= 30
    out = subprocess.check_output(["nm", "-D", "--defined-only", w2x.lib_path()], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    missing = [s for s in declared if s not in exported]
    assert not missing, missing
    from w2x_b200 import capi
    assert sorted(capi.ABI_SYMBOLS) == declared                      # the binding covers the whole header
    L = w2x.lib()
    for s in declared:
        assert getattr(L, s) is not None


def test_library_has_no_oracle_or_torch_dependency(w2x):
    out = subprocess.check_output(["ldd", w2x.lib_path()], text=True)
    assert "oracle" not in out and "torch" not in out and "opencv" not in out.lower()


def test_library_carries_hopper_tensor_and_tma_instructions(w2x):
    """SASS evidence: wgmma f16 -> HGMMA, wgmma e4m3 -> QGMMA, TMA -> UTMALDG / UBLKCP."""
    sass = subprocess.run(["cuobjdump", "-sass", w2x.lib_path()], capture_output=True, text=True)
    if sass.returncode != 0:
        pytest.skip("cuobjdump not available")
    for mnemonic in ("HGMMA", "QGMMA", "UTMALDG", "UBLKCP"):
        assert mnemonic in sass.stdout, mnemonic
    assert "sm_90a" in subprocess.check_output(["cuobjdump", "-lelf", w2x.lib_path()], text=True)


def test_version_and_defaults(w2x):
    assert w2x.version().startswith("1.0.0")
    assert w2x.get_jobs() == 4                      # src/modelHandler.hpp:98
    assert w2x.get_block_size() == (512, 512)       # src/modelHandler.hpp:99


def test_model_utility_setters(w2x):
    try:
        w2x.set_jobs(8)
        assert w2x.get_jobs() == 8
        with pytest.raises(w2x.W2xError):
            w2x.set_jobs(0)                         # setNumberOfJobs(<1) -> false, src/modelHandler.cpp:199-203
        w2x.set_block_size_exp2_square(8)
        assert w2x.get_block_size() == (256, 256)
        w2x.set_block_size(384, 320)
        assert w2x.get_block_size() == (384, 320)
        with pytest.raises(w2x.W2xError):
            w2x.set_block_size(-1, 5)
        with pytest.raises(w2x.W2xError):
            w2x.set_block_size_exp2_square(-1)
    finally:
        w2x.set_jobs(4)
        w2x.set_block_size(512, 512)


def test_block_table_matches_reference_arithmetic(w2x, oracle_mod):
    tabs = json.load(open(golden_path("block_tables.json")))
    for key, t in tabs.items():
        w, h = map(int, key.split("x"))
        tab, sc, sr = w2x.block_table(w, h)
        assert (sc, sr) == (t["split_cols"], t["split_rows"]), key
        assert tab.tolist() == [list(r) for r in t["rows"]], key
        assert w2x.requires_splitting(w, h) == t["require_split"], key
    # threshold of src/convertRoutine.cpp:25-26: 512*512*3/2 = 393216 pixels
    assert not w2x.requires_splitting(512, 768) and w2x.requires_splitting(513, 768)
    # other block sizes agree with the oracle's restatement too
    try:
        w2x.set_block_size(64, 64)
        for (w, h) in ((150, 131), (50, 1), (64, 64), (1000, 51)):
            a, sc, sr = w2x.block_table(w, h)
            b, sc2, sr2 = oracle_mod.block_table(w, h, 64, 64, 7)
            assert (sc, sr) == (sc2, sr2) and np.array_equal(a, b)
    finally:
        w2x.set_block_size(512, 512)


@pytest.mark.skipif(_has_gpu(), reason="this is the no-GPU behaviour check")
def test_no_device_means_error_not_fallback(w2x):
    with pytest.raises(w2x.W2xError) as ei:
        w2x.Context(0)
    assert ei.value.status == 6 and "no CPU fallback" in ei.value.message
