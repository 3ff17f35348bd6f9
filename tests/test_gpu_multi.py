"""Multi-GPU machinery of the product (csrc/engine_band.cu) on ONE device -- every mechanism is the same code the
multi-GPU runs use, only the "neighbour" lives on the same GPU (separate contexts / streams / processes):

  * w2x_convert_tiles: a batch of independent planes as one stacked frame is bit-identical to plane-by-plane calls
    (the reference's block loop, src/convertRoutine.cpp:114-165; BASELINE config 5);
  * w2x_band_connect_local + w2x_band_run: row bands with the per-layer halo exchange done INSIDE the library through
    peer-mapped frames (one exchange kernel per layer: rows, flag, wait) reproduce the whole-plane bits;
  * w2x_multi_*: the one-process N-context driver (both in tools/multi_selftest.py, which also runs on N GPUs);
  * w2x_band_export / w2x_band_connect: the same between PROCESSES over CUDA IPC.
These are one fixed configuration per mechanism; test_band_exchange.py covers the shapes, precisions and edges (thin
bands, odd frame widths, slab sub-band layouts, bench.py's slab export / connect path, the multi plan cache) bit for bit.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def models(w2x, oracle_models):
    return {n: w2x.Model.from_arrays(om.weights, om.biases) for n, om in oracle_models.items()}


@pytest.mark.parametrize("engine,precision", [("tc", 1), ("tc", 0), ("fp32", 1)])
def test_batched_tiles_equal_plane_by_plane(w2x, models, oracle_mod, engine, precision):
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC if engine == "tc" else w2x.ENGINE_FP32)
    ctx.set_precision(precision)
    try:
        tiles = np.stack([oracle_mod.seeded_plane(96, 80, 100 + t, "uniform") for t in range(5)])
        batch = ctx.convert_tiles(models["noise2"], tiles)
        for t in range(5):
            assert np.array_equal(batch[t], ctx.convert_plane(models["noise2"], tiles[t], block_splitting=False)), t
        # a scratch limit smaller than the batch: processed in groups, same bits
        ctx.set_scratch_limit(128 * (96 + 14) * (80 + 14) * 4 * 2)
        assert np.array_equal(ctx.convert_tiles(models["noise2"], tiles), batch)
        # eight tiles and more run as copy-pipelined groups (uploads / layers / downloads overlap): same bits per tile, twice in a row
        many = np.stack([oracle_mod.seeded_plane(64, 48, 300 + t, "uniform") for t in range(11)])
        ctx.set_scratch_limit(1 << 34)
        piped = ctx.convert_tiles(models["noise2"], many)
        for t in range(11):
            assert np.array_equal(piped[t], ctx.convert_plane(models["noise2"], many[t], block_splitting=False)), t
        assert np.array_equal(ctx.convert_tiles(models["noise2"], many), piped)
    finally:
        ctx.close()


def test_peer_exchange_and_multi_driver_selftest():
    """tools/multi_selftest.py: three band sessions wired through peer memory (w2x_band_connect_local + w2x_band_run, both
    precisions, three passes each) and the one-process driver (w2x_multi_convert_plane / _tiles) reproduce the single-GPU
    bits.  Runs in its own process: on one device the bands' exchange kernels must run concurrently, which needs
    CUDA_DEVICE_MAX_CONNECTIONS >= the number of streams before CUDA initialises (see the tool's header)."""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "multi_selftest.py"), "3"], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "multi selftest ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("world,precision", [(2, 1), (3, 0)])
def test_ipc_ranks_in_separate_processes(w2x, models, oracle_mod, tmp_path, world, precision):
    W, H = 200, 190
    x = oracle_mod.seeded_plane(W, H, 77, "uniform")
    ctx = w2x.Context(0, engine=w2x.ENGINE_TC)
    ctx.set_precision(precision)
    whole = ctx.convert_plane(models["noise2"], x)
    ctx.close()
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tools", "ipc_band_worker.py"), str(r), str(world), str(tmp_path), str(W), str(H),
                               "noise2", str(precision)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(world)]
    logs = [p.communicate(timeout=300)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), logs
    got = np.concatenate([np.load(tmp_path / f"out_{r}.npy") for r in range(world)])
    assert np.array_equal(got, whole)
