"""Index arithmetic of the 16x16-tile tensor-core kernel, checked on the CPU against a byte-level model of what the
hardware units do with shared memory:

  * TMA (SWIZZLE_128B) writes byte b of box row e at  swz(box_base + e*128 + b);
  * a wgmma K-major shared-memory descriptor (start S, stride-byte-offset SBO) reads GEMM row r, byte b of its 32-byte K slice at
    swz(S + (r // 8) * SBO + (r % 8) * 128 + b),

with swz(a) = a ^ (((a >> 7) & 7) << 4) applied to the shared-memory ADDRESS (CUTLASS: Swizzle<3,4,3> o smem_ptr).
Activations are RECORD frames: one 128-byte record per pixel per 32-channel block = {xh fp16 x32 | xh8 x32 | xl8 x32}.
The test proves that the descriptor offsets used in csrc/tc_kernel.cuh
((ky*18 + 8j + kx)*128 + 32*q, SBO = 18*128) address exactly the 3x3-shifted windows, and the four record quarters, of
the ONE staged 18x18 box -- i.e. that no per-tap reload is needed."""
import numpy as np

HALO = 18


def swz(a, rowb=128):
    return a ^ (((a >> 7) & (rowb // 16 - 1)) << 4)


def test_tap_windows_and_record_quarters_come_from_one_staged_box():
    rng = np.random.default_rng(7)
    box = rng.integers(0, 256, size=(HALO, HALO, 128), dtype=np.uint8)      # [hy][hx][128 B record] as TMA delivers it
    base = 7 * 1024                                                          # slots are 1024-byte aligned
    smem = np.zeros(64 * 1024, np.uint8)
    for hy in range(HALO):
        for hx in range(HALO):
            for b in range(128):
                smem[swz(base + (hy * HALO + hx) * 128 + b)] = box[hy, hx, b]
    sbo = HALO * 128
    for ky in range(3):
        for kx in range(3):
            for j in range(2):
                for q in range(4):                                           # fp16 K step 0 / 1, xh8, xl8
                    start = base + (ky * HALO + 8 * j + kx) * 128 + 32 * q
                    for r in range(128):
                        oy, ox = r // 8, r % 8
                        for b in (0, 5, 16, 31):
                            a = swz(start + (r // 8) * sbo + (r % 8) * 128 + b)
                            assert smem[a] == box[oy + ky, 8 * j + ox + kx, 32 * q + b]


def test_descriptor_fields_fit():
    # 14-bit fields in 16-byte units: addresses < 256 KiB, SBO 18*128 = 2304
    assert (227 * 1024) >> 4 < (1 << 14) and (HALO * 128) >> 4 < (1 << 14)


def test_tile_kernel_store_box_is_the_staging_tile():
    """epilogue_store32_rec in the tile kernels: lane = pixel of the warp's 8x4 block (lane = y*8 + x), staged as row `lane`
    of a [32][128 B] SWIZZLE_128B tile; the TMA store box {128 B, 1 block, 8 px, 4 rows} enumerates x fastest, then y --
    the same order."""
    rng = np.random.default_rng(8)
    tile = 9 * 1024
    smem = np.zeros(32 * 1024, np.uint8)
    rec = rng.integers(0, 256, size=(32, 128), dtype=np.uint8)
    for lane in range(32):
        for u in range(8):                                  # the kernel's sts128 addresses
            a = tile + lane * 128 + ((u ^ (lane & 7)) << 4)
            smem[a:a + 16] = rec[lane, 16 * u:16 * u + 16]
    for lane in range(32):
        for b in range(128):                                # what the TMA unit reads for box row `lane`
            assert smem[swz(tile + lane * 128 + b)] == rec[lane, b]
