// tc_config.cuh -- per-layer compile-time configuration (shared-memory map, stages), kernel parameters, profile record
// Part of the tensor-core engine's single translation unit: included by kernels_tc.cu inside namespace w2x::tc, in this order:
//   tc_ptx.cuh, tc_wgmma.cuh, tc_config.cuh, tc_kernel.cuh, tc_edge_kernels.cuh
// (pure code organisation: the generated SASS is the same as with one file).

// ================================================================================================
// Per-layer configuration
// ================================================================================================
// Activations are RECORD frames (kernels.h): [Hp][Wp][C/32][128 B], one 128-byte record per pixel per 32-channel block =
// {xh fp16 x32 | xh8 e4m3 x32 | xl8 e4m3 x32} (F8) or {hi fp16 x32 | lo fp16 x32}.  One staged box = the 18x18-pixel halo
// region of ONE 32-channel block: 324 rows of 128 B, SWIZZLE_128B; the fp16 K steps / xh8 / xl8 (or lo) slices of a pixel
// are the 32-byte quarters of its row (+0, +2, +4, +6 sixteen-byte units in the descriptor start address).
//
// F8 = false: three f16 products xh*wh + xl*wh + xh*wl ("f16x3").
// F8 = true : xh*wh in f16, the two correction products in e4m3 on e4m3 copies
//             xl8*wh8 + xh8*wl8 (K = 32 per wgmma at twice the rate: 2.0 instead of 3.0 pass-equivalents).
// F8 = false with TcParams::xh_only ("f16", W2X_PRECISION_F16): xh*wh alone (1.0 pass-equivalent, not fp32-faithful) on the
//             same f16x3 records and weight image, of which only the wh half of each stage is loaded.  A runtime flag, not
//             a template parameter: the f16x3 kernels run it, choosing the loop once per tile-set.
// Rec::BF16 ("bf16x3", W2X_PRECISION_BF16X3): f16x3 with bf16 hi/lo records and weights, Cfg<..., F8 = false>'s layout.
constexpr int F8_A = 10, F8_C = 1;   // xl8 = e4m3((x16 - xh) * 2^F8_A), xh8 = e4m3(xh * 2^-F8_C); must match w2x_internal.h

template <int CIN, int COUT, bool FUSE = false, bool F8 = false>
struct Cfg {
    // ---- A operand (activations): one TMA box per (tile-set, 32-channel block) ----
    static constexpr int KC = 32;                       // channels per activation chunk
    static constexpr int NCHUNK = CIN / KC;
    static constexpr int ROWB = 128;                    // bytes per pixel per chunk (one record = the swizzle span)
    static constexpr int A_TX = HALO * HALO * ROWB;     // bytes the TMA load of one slot delivers
    static constexpr int A_SLOT = (A_TX + 1023) / 1024 * 1024;
    static constexpr int A_SLOTS = 2;
    // ---- B operand (weights): one stage per (32-channel block, tap), rows of 64 B (fp16, SWIZZLE_64B) ----
    //   f16x3: [wh (Cout rows) | wl (Cout rows)]        F8: [wh (Cout rows of 64 B) | wh8 | wl8 (Cout rows of 32 B, SWIZZLE_32B)]
    static constexpr int B_ROWB = KC * 2;
    static constexpr int B_BLOCK = COUT * B_ROWB;
    static constexpr int B_STAGE = 2 * B_BLOCK;
    static constexpr int STAGES_PER_TILESET = NCHUNK * 9;
    // ---- operand roles (see tc_kernel.cuh) ----
    //   SWAP = false: A = an m64 half of the M-tile's pixels, B = the Cout weight rows (N = Cout)
    //   SWAP = true : A = the 64 weight rows (M = Cout), B = all 128 pixels of the M-tile (N = 128).  The stage image and the
    //                 record boxes are read as they are; only the descriptors change.  Cout = 64 only: a 32-row A would
    //                 leave half of every m64 wgmma empty, and at Cout = 128 two m64 channel halves would need 128
    //                 accumulators plus two 64-register correction buffers per thread.  The fused last layer keeps
    //                 SWAP = false (epilogue_fuse sums a pixel's channels across the lanes of a quad).
    static constexpr bool SWAP = COUT == 64 && !FUSE;
    // ---- shared memory map: [A slots][B stages][store staging][barriers (1 KB)][bias | last-layer weights] ----
    static constexpr int BAR_BYTES = 1024;
    static constexpr int PRM_BYTES = 4 * COUT * (FUSE ? 10 : 1);             // the epilogue indexes them per lane: shared, not parameter space
    // one 32-channel record block of an M-tile (128 px); SWAP: both blocks, each written by the two warps holding its channels
    static constexpr int STG_WG = (SWAP ? 2 : 1) * 128 * 128;
    static constexpr int STG_BYTES = FUSE ? 0 : 2 * STG_WG;
    static constexpr int SMEM_MAX = 227 * 1024;
    static constexpr int NB_FIT = (SMEM_MAX - 1024 - BAR_BYTES - PRM_BYTES - STG_BYTES - A_SLOTS * A_SLOT) / B_STAGE;
    // Narrow layers: ALL weight stages of a tile-set fit -> loaded once per CTA and kept (no ring traffic, no stage barriers
    // after the first tile-set).
    static constexpr bool RESIDENT = STAGES_PER_TILESET <= NB_FIT && STAGES_PER_TILESET <= 24;
    static constexpr int NB = RESIDENT ? STAGES_PER_TILESET : (NB_FIT > 8 ? 8 : NB_FIT);
    static constexpr int SMEM_BYTES = 1024 + A_SLOTS * A_SLOT + NB * B_STAGE + STG_BYTES + BAR_BYTES + PRM_BYTES;
    static_assert(NB >= 3, "need at least three weight stages");
    static_assert((4 + 2 * NB) * 8 <= BAR_BYTES, "barrier area overflow");
    static_assert(SMEM_BYTES <= SMEM_MAX, "shared memory");
    static_assert(B_STAGE % 1024 == 0 && A_SLOT % 1024 == 0, "swizzle pattern alignment");
    static_assert(CIN % KC == 0 && COUT % 32 == 0 && COUT <= 128, "shape");
};

// warps: 0 A producer | 1 B producer | 2, 3 idle | 4-7 consumer warpgroup of M-tile 0 | 8-11 consumer warpgroup of M-tile 1
constexpr int NUM_THREADS = 12 * 32;

struct TcParams {
    const uint16_t *wpack;   // [chunk][tap] stages (see Cfg::B_STAGE), pre-swizzled (see model.cpp)
    float bias[128];         // [COUT] (float)bias * ACT_SCALE, by value
    int Wp, Hp;
    int out_y0, out_rows;    // only frame rows [out_y0, out_y0 + out_rows) are stored (row-band sessions keep the halo rows their neighbours write)
    int tiles_x, n_tilesets;
    float out_scale;         // 1 / wscale  (accumulator -> ACT_SCALE * conv)
    unsigned long long *prof;   // optional [gridDim.x][16] cycle counters (see PROF_* below), nullptr = off
    // fused last layer (FUSE kernels only): this layer's activations never reach HBM; instead each pixel's
    // nine tap partials P[t] = sum_c act[c] * w_last[c][t] are written ([Hp][Wp][12] fp32, 3 pad words).
    float *partial;             // nullptr = not fused
    float last_w[9 * 128];      // [9][COUT] tap-major, by value
    int xh_only;                // F8 = false kernels: 1 = the xh*wh product alone (W2X_PRECISION_F16), 0 = f16x3
};

// per-CTA profile record (cycles, accumulated over launches)
enum { PROF_TOTAL = 0, PROF_MMA_WAIT_ACC, PROF_MMA_WAIT_A, PROF_MMA_WAIT_B, PROF_APROD_WAIT, PROF_BPROD_WAIT,
       PROF_EPI_WAIT, PROF_EPI_WORK, PROF_TILESETS, PROF_N = 16 };

__device__ __forceinline__ void mbar_wait_prof(uint32_t bar, uint32_t parity, bool on, unsigned long long &acc) {
    if (on) {
        long long t0 = clock64();
        mbar_wait(bar, parity);
        acc += (unsigned long long)(clock64() - t0);
    } else {
        mbar_wait(bar, parity);
    }
}
