"""CPU models of the row-strip design for the narrow layers (csrc/tc_strip_plan.h, model.cpp pack_tc_layer_strip), no GPU needed:

  1. the issuer / epilogue schedule -- units, strips, the descending ring of TMEM accumulator blocks, the wrap split,
     block acquisition and completion -- replayed literally (same index arithmetic as the kernel) with real numbers:
     every output row must receive exactly W(ky=0)*x[y-1] + W(ky=1)*x[y] + W(ky=2)*x[y+1] (rows outside the frame are
     zero), be drained after its last contribution and before its block is reused;
  2. the shared-memory addressing of RECORD frames (one 128-byte record per pixel per 32 channels, SWIZZLE_128B): tap
     column kx of a staged 130-pixel row is the descriptor start offset kx*128 (SBO = 1024), the fp16 K steps / xh8 /
     xl8 slices are its 32-byte quarters; and the staging tiles the epilogue and the first layer build are exactly what
     the TMA stores read;
  3. the packed weight image (model.cpp pack_tc_layer_strip): a K-major descriptor at row offset ky*Cout of stage
     (chunk, kx) reads W[o][c*32+k][ky][kx] (scaled, split) for GEMM row ky*Cout + o.
"""
import numpy as np
import pytest


def blk_of(n, NB):
    return NB - 1 - (n % NB)


def replay(Hp, seg_rows, NB, n_ctas, ncols=1, epi_sets=2, strips=None):
    """Replays the kernel's issuer loop for every CTA; returns {(col, y): [(r, ky), ...]} in accumulation order.
    Asserts the block protocol on the way (a block is never written before it was handed back, never drained twice).
    `strips`, if a list, receives one tuple per strip: (cta, u, col, y0, j, ky_lo, b0, cnt0, cnt1, acq_n, acq_cnt, com_n, com_cnt)."""
    n_units = ncols * ((Hp + seg_rows - 1) // seg_rows)
    got = {}
    for cta in range(n_ctas):
        owner = [None] * NB            # which (unit, row) currently lives in each block
        nrow = 0
        for u in range(cta, n_units, n_ctas):
            seg, col = divmod(u, ncols)
            y0 = seg * seg_rows
            y1 = min(y0 + seg_rows, Hp)
            rows = y1 - y0
            r_first, r_last = max(y0 - 1, 0), min(y1, Hp - 1)
            next_new = next_done = 0
            for r in range(r_first, r_last + 1):
                ky_lo, ky_hi = max(0, r + 2 - y1), min(2, r + 1 - y0)
                assert ky_lo <= ky_hi
                i_top = r + 1 - ky_lo - y0
                acq = (nrow + next_new, i_top + 1 - next_new)
                while next_new <= i_top:
                    n = nrow + next_new
                    b = blk_of(n, NB)
                    assert owner[b] is None, "block reused before it was drained"
                    owner[b] = (u, next_new)
                    got[(col, y0 + next_new)] = []
                    next_new += 1
                b0 = blk_of(nrow + i_top, NB)
                nky = ky_hi - ky_lo + 1
                cnt0 = min(nky, NB - b0)
                cnt1 = nky - cnt0
                runs = [(b0, ky_lo, cnt0)] + ([(0, ky_lo + cnt0, cnt1)] if cnt1 else [])
                for (bstart, ky_start, cnt) in runs:
                    for j in range(cnt):              # N-block j of this MMA = B rows [(ky_start+j)*Cout, ...) -> TMEM block bstart+j
                        b, ky = bstart + j, ky_start + j
                        assert b < NB
                        i = r + 1 - ky - y0
                        assert owner[b] == (u, i), (owner[b], u, i)
                        got[(col, y0 + i)].append((r, ky))
                i_done = rows - 1 if r == r_last else r - 1 - y0
                if strips is not None:
                    strips.append((cta, u, col, y0, r - (y0 - 1), ky_lo, b0, cnt0, cnt1, acq[0], acq[1],
                                   nrow + next_done, max(0, i_done + 1 - next_done)))
                while next_done <= i_done:
                    b = blk_of(nrow + next_done, NB)
                    assert owner[b] == (u, next_done)
                    owner[b] = None                    # committed -> epilogue drains + zeroes -> free
                    next_done += 1
            assert next_new == rows and next_done == rows
            nrow += rows
    return got


@pytest.mark.parametrize("Hp,seg_rows,NB", [(15, 32, 8), (15, 32, 16), (3, 32, 8), (33, 32, 8), (64, 32, 16), (100, 7, 8),
                                             (100, 2, 8), (41, 1, 8), (530, 32, 16), (17, 16, 8)])
def test_schedule_gives_every_row_its_three_taps_in_order(Hp, seg_rows, NB):
    for n_ctas in (1, 3):
        got = replay(Hp, seg_rows, NB, n_ctas, ncols=2)
        assert len(got) == 2 * Hp
        for (col, y), contrib in got.items():
            want = [(r, ky) for ky, r in ((0, y - 1), (1, y), (2, y + 1)) if 0 <= r < Hp]
            assert contrib == want, (y, contrib, want)     # same taps, same order, whatever the unit geometry


def test_kernel_plan_arithmetic_is_the_replayed_schedule(tmp_path):
    """csrc/tc_strip_plan.h -- the closed-form per-strip plan the kernel's software-pipelined issuer computes one strip ahead --
    compiled with g++ and compared, strip by strip, with the literal replay above (taps, blocks, wrap split, the rows whose
    blocks are acquired before and handed to the epilogue after the strip)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "strip_plan_dump")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "waifu2x-converter-cpp_b200", "csrc"),
                           os.path.join(root, "tests", "cpp", "strip_plan_dump.cpp"), "-o", exe])
    for (Hp, seg_rows, NB) in [(15, 32, 8), (15, 32, 16), (3, 32, 8), (1, 32, 8), (2, 1, 8), (33, 32, 8), (64, 32, 16), (100, 7, 8),
                               (100, 2, 8), (41, 1, 8), (530, 32, 16), (17, 16, 8), (4110, 32, 8)]:
        for n_ctas in (1, 3, 7):
            want = []
            replay(Hp, seg_rows, NB, n_ctas, ncols=2, strips=want)
            out = subprocess.check_output([exe, str(Hp), str(seg_rows), str(NB), str(n_ctas), "2"], text=True)
            got = [tuple(int(v) for v in line.split()) for line in out.splitlines()]
            assert got == want, (Hp, seg_rows, NB, n_ctas)


def swz(a, rowb):
    return a ^ (((a >> 7) & (rowb // 16 - 1)) << 4)


def test_tap_columns_and_record_quarters_are_start_offsets_into_one_staged_row():
    """RECORD frames: TMA (SWIZZLE_128B) writes pixel px, byte b of its 128-byte record at swz(base + px*128 + b); a K-major
    descriptor with start S and SBO = 1024 reads GEMM row m, byte b at swz(S + (m//8)*1024 + (m%8)*128 + b).  With
    S = base + kx*128 + 32*q row m must be quarter q (fp16 K step 0 / 1, xh8, xl8) of pixel m + kx of the staged row."""
    BOXW, rowb = 130, 128
    rng = np.random.default_rng(7)
    row = rng.integers(0, 256, size=(BOXW, rowb), dtype=np.uint8)
    base = 3 * 1024                                   # slots are aligned to the swizzle period
    smem = np.zeros(32 * 1024, np.uint8)
    for px in range(BOXW):
        for b in range(rowb):
            smem[swz(base + px * rowb + b, rowb)] = row[px, b]
    for kx in range(3):
        for q in range(4):
            start = base + kx * rowb + 32 * q
            for m in range(128):
                for b in (0, 7, 16, 31):
                    a = swz(start + (m // 8) * 1024 + (m % 8) * rowb + b, rowb)
                    assert smem[a] == row[m + kx, 32 * q + b]


def test_record_staging_tiles_are_the_tma_store_images():
    """epilogue_store32_rec: lane = pixel, 16-byte unit u of its record at tile + lane*128 + ((u ^ (lane & 7)) << 4);
    first_layer_kernel<REC>: row r = threadIdx.x, fp16 unit c8, e4m3 8-byte halves at units 4 + c8/2 (xh8) and 6 + c8/2 (xl8).
    The TMA store (SWIZZLE_128B, box rows of 128 B) reads row r, byte b from swz(tile + r*128 + b)."""
    rng = np.random.default_rng(8)
    tile = 5 * 1024
    smem = np.zeros(64 * 1024, np.uint8)
    rec = rng.integers(0, 256, size=(32, 128), dtype=np.uint8)
    for lane in range(32):
        for u in range(8):
            a = tile + lane * 128 + ((u ^ (lane & 7)) << 4)
            smem[a:a + 16] = rec[lane, 16 * u:16 * u + 16]
    for lane in range(32):
        for b in range(128):
            assert smem[swz(tile + lane * 128 + b, 128)] == rec[lane, b]
    rec = rng.integers(0, 256, size=(256, 128), dtype=np.uint8)
    smem[:] = 0
    for r in range(256):
        for c8 in range(4):
            a = tile + r * 128 + ((c8 ^ (r & 7)) << 4)
            smem[a:a + 16] = rec[r, 16 * c8:16 * c8 + 16]
            for plane, unit0 in ((0, 4), (1, 6)):                       # xh8 bytes [64, 96), xl8 bytes [96, 128)
                a8 = tile + r * 128 + (((unit0 + (c8 >> 1)) ^ (r & 7)) << 4) + (c8 & 1) * 8
                smem[a8:a8 + 8] = rec[r, 64 + 32 * plane + 8 * c8:64 + 32 * plane + 8 * c8 + 8]
    for r in range(256):
        for b in range(128):
            assert smem[swz(tile + r * 128 + b, 128)] == rec[r, b]


def _f16(bits):
    return np.frombuffer(np.asarray(bits, np.uint16).tobytes(), np.float16).astype(np.float32)


def _e4m3(byte):
    b = int(byte)
    s, e, m = b >> 7, (b >> 3) & 15, b & 7
    v = (m / 8.0) * 2.0 ** -6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7)
    return -v if s else v


@pytest.mark.parametrize("layer", [1, 2, 3])
def test_strip_weight_image(w2x, oracle_models, layer):
    om = oracle_models["scale2.0x"]
    m = w2x.Model.from_arrays(om.weights, om.biases)
    n_in, n_out, _ = m.dims(layer)
    _, _, _, wscale = m.debug_tc_pack(layer)
    w = om.weights[layer].astype(np.float32) * np.float32(wscale)
    nrows, stage = 3 * n_out, 3 * n_out * 128
    img16, img8 = m.debug_tc_strip(layer, 0), m.debug_tc_strip(layer, 1)
    assert img16.size == img8.size == (n_in // 32) * 3 * stage
    rng = np.random.default_rng(layer)
    for _ in range(400):
        c, kx, ky = int(rng.integers(n_in // 32)), int(rng.integers(3)), int(rng.integers(3))
        o, k = int(rng.integers(n_out)), int(rng.integers(32))
        want = w[o, c * 32 + k, ky, kx]
        wh = np.float32(np.float16(want))
        sb = (c * 3 + kx) * stage
        # what a SWIZZLE_64B K-major descriptor starting at row ky*n_out reads for GEMM row o, K element k
        a16 = swz(sb + (ky * n_out + o) * 64 + 2 * k, 64)
        for img in (img16, img8):
            assert _f16(img[a16:a16 + 2].view(np.uint16))[0] == wh
        al = swz(sb + nrows * 64 + (ky * n_out + o) * 64 + 2 * k, 64)
        assert _f16(img16[al:al + 2].view(np.uint16))[0] == np.float32(np.float16(want - wh))
        a8 = swz(sb + nrows * 64 + (ky * n_out + o) * 32 + k, 32)
        b8 = swz(sb + nrows * 96 + (ky * n_out + o) * 32 + k, 32)
        # e4m3 copies: wh8 = e4m3(wh * 2^-10), wl8 = e4m3((w - wh) * 2^1): within half an e4m3 ulp (3 mantissa bits)
        for byte, val in ((img8[a8], wh * 2.0 ** -10), (img8[b8], (want - wh) * 2.0)):
            got = _e4m3(byte)
            assert abs(got - val) <= max(abs(val) * 2.0 ** -4, 2.0 ** -10), (got, val)
    assert m.debug_tc_strip(4, 1) is None and m.debug_tc_strip(5, 0) is None      # the 128-wide layers keep the tile kernels
