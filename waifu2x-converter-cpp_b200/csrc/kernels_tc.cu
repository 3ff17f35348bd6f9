// kernels_tc.cu -- the tensor-core engine (W2X_ENGINE_TC): sm_90a (Hopper wgmma + TMA).
//
// What it computes (reference src/modelHandler.cpp:134-152 for all output planes of a layer at
// once): out[o](y,x) = leaky( sum_i sum_{ky,kx} W[o][i][ky][kx] * in[i](y+ky-1, x+kx-1) + bias[o] ).
//
// How: implicit GEMM, D[pixel][o] += A[pixel][(tap,i)] * B[(tap,i)][o], on the Hopper tensor cores
// (wgmma.mma_async, fp32 accumulators in registers).  fp32 fidelity comes from a 2-term split of
// both operands (x = xh + xl, w = wh + wl, h = the fp16 rounding) and three accumulated products
// xh*wh + xl*wh + xh*wl (the dropped xl*wl term is ~2^-22 relative); SURVEY.md section 7 shows a
// single fp16/tf32 pass misses the 1e-4 gate by 10x.  Three arithmetic modes (template flag F8, TcParams::xh_only):
//   f16x3      all three products as f16 wgmmas on fp16 hi/lo planes
//   f16+f8x2   xh*wh as f16; the two correction products as e4m3 wgmmas on e4m3 copies of the
//              operands (K = 32 per instruction, twice the rate) -- the default, 2.0 instead of 3.0 passes
//   f16        xh*wh alone, by the f16x3 kernels on the f16x3 frames and weights: 1.0 pass, not
//              fp32-faithful (8-bit outputs within 1 LSB); chosen by the caller, never by default
//
// Data layout in HBM: every activation is an NHWC "frame" of 4 bytes per element holding value*ACT_SCALE,
// [hi fp16][lo fp16] or [xh fp16][xh8 e4m3][xl8 e4m3] planes of [Hp][Wp][C]; all layers of one pass share
// the frame size (the padded plane), reads outside the frame are zero-filled by TMA, so each layer is a
// same-size convolution whose polluted ring grows by one pixel per layer and is cropped at the end -- the
// same argument that makes the reference's per-layer BORDER_REPLICATE harmless (SURVEY.md section 8a).
//
// Per CTA (persistent, 1 per SM, 12 warps):
//   warp 0      A producer   one TMA box {KC ch, 18, 18} per (tile-set, channel chunk): the 16x16 output
//                            region plus a 1-pixel ring, staged ONCE and addressed nine times (the 3x3 taps
//                            are wgmma-descriptor start-address offsets into it)
//   warp 1      B producer   pre-swizzled (32-channel, tap) weight stages: a cp.async.bulk ring, or resident
//                            for the narrow layers
//   warps 4-11  consumers    two warpgroups, one per M-tile (8 wide x 16 tall pixels = two m64 wgmmas), N = Cout,
//                            K = 16 (fp16) / 32 (e4m3) per instruction; each drains its own accumulators: scale,
//                            +bias, leaky-ReLU -> either the frame's records, staged in the TMA swizzle pattern and
//                            TMA-stored, or (FUSE) the last layer's nine tap partials
//
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <cstdio>
#include <type_traits>

#include "kernels.h"
#include "w2x_b200.h"

namespace w2x {
namespace tc {

#include "tc_ptx.cuh"
#include "tc_wgmma.cuh"
#include "tc_config.cuh"
#include "tc_kernel.cuh"
#include "tc_edge_kernels.cuh"

// ================================================================================================
// Host side
// ================================================================================================
bool layer_supported(int cin, int cout) {
    auto ok = [](int c) { return c == 32 || c == 64 || c == 128; };
    return ok(cin) && ok(cout);
}

template <int CIN, int COUT, bool FUSE, bool F8>
static cudaError_t set_attr1() {
    return cudaFuncSetAttribute(tc_conv3x3_kernel<CIN, COUT, FUSE, F8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                Cfg<CIN, COUT, FUSE, F8>::SMEM_BYTES);
}
template <int CIN, int COUT>
static cudaError_t set_attr() {
    cudaError_t e;
    if ((e = set_attr1<CIN, COUT, false, false>()) != cudaSuccess) return e;
    if ((e = set_attr1<CIN, COUT, true, false>()) != cudaSuccess) return e;
    if ((e = set_attr1<CIN, COUT, false, true>()) != cudaSuccess) return e;
    return set_attr1<CIN, COUT, true, true>();
}

#define W2X_TC_SHAPES(X) \
    X(32, 32) X(32, 64) X(32, 128) X(64, 32) X(64, 64) X(64, 128) X(128, 32) X(128, 64) X(128, 128)

size_t layer_smem_bytes(int cin, int cout) {
#define X(ci, co) \
    if (cin == ci && cout == co) return Cfg<ci, co, true, false>::SMEM_BYTES;
    W2X_TC_SHAPES(X)
#undef X
    return 0;
}

cudaError_t init_kernels() {
    cudaError_t e;
#define X(ci, co) \
    if ((e = set_attr<ci, co>()) != cudaSuccess) return e;
    W2X_TC_SHAPES(X)
#undef X
    return cudaSuccess;
}

template <int CIN, int COUT, bool FUSE, bool F8>
static cudaError_t launch_k(const CUtensorMap *tmap, const CUtensorMap *omap, const TcParams &p, int grid, cudaStream_t s) {
    tc_conv3x3_kernel<CIN, COUT, FUSE, F8><<<grid, NUM_THREADS, Cfg<CIN, COUT, FUSE, F8>::SMEM_BYTES, s>>>(*tmap, *omap, p);
    return cudaGetLastError();
}

template <int CIN, int COUT>
static cudaError_t launch_one(const CUtensorMap *tmap, const CUtensorMap *omap, const TcParams &p, int num_sms, bool f8, cudaStream_t s) {
    int grid = p.n_tilesets < num_sms ? p.n_tilesets : num_sms;
    if (f8) return p.partial ? launch_k<CIN, COUT, true, true>(tmap, omap, p, grid, s) : launch_k<CIN, COUT, false, true>(tmap, omap, p, grid, s);
    return p.partial ? launch_k<CIN, COUT, true, false>(tmap, omap, p, grid, s) : launch_k<CIN, COUT, false, false>(tmap, omap, p, grid, s);
}

static int make_rec_map(CUtensorMap *map, const void *base, int C, int Wp, int Hp, int box_w, int box_h, int y0, int rows);

cudaError_t launch_tc_layer(const __half *in, const void *wpack, const float *bias, __half *out, int cin,
                            int cout, int pw, int ph, float out_scale, int mode, int num_sms, cudaStream_t s,
                            unsigned long long *prof, const float *last_w, float *partial, int out_y0, int out_rows) {
    if (out_rows < 0) { out_y0 = 0; out_rows = ph; }
    CUtensorMap tmap_in;
    if (make_rec_map(&tmap_in, in, cin, pw, ph, HALO, HALO, 0, ph)) return cudaErrorInvalidValue;
    TcParams p;
    p.wpack = reinterpret_cast<const uint16_t *>(wpack);
    // ACT_SCALE (a power of two) is folded into the epilogue's affine step: leaky(16 v) = 16 leaky(v) exactly, so the
    // kernel produces the frame's x16 values without a separate multiply; the fused last layer gets weights / 16.
    for (int i = 0; i < cout; i++) p.bias[i] = bias[i] * ACT_SCALE;      // HOST pointer
    p.Wp = pw;
    p.Hp = ph;
    p.out_y0 = out_y0;
    p.out_rows = out_rows;
    p.tiles_x = (pw + REGION - 1) / REGION;
    p.n_tilesets = p.tiles_x * ((out_rows + REGION - 1) / REGION);   // tile-sets tile the store window (TMA store coordinates stay non-negative)
    p.out_scale = out_scale * ACT_SCALE;
    p.xh_only = mode == W2X_PRECISION_F16 ? 1 : 0;
    p.prof = prof;
    p.partial = partial;
    if (partial) {
        if (!last_w) return cudaErrorInvalidValue;
        for (int i = 0; i < 9 * cout; i++) p.last_w[i] = last_w[i] * (1.0f / ACT_SCALE);      // HOST pointer: [9][cout]
    }
    // the epilogue's TMA stores: one 8x16-pixel box of records (an M-tile) per 32-channel block (fused layers store no frame)
    CUtensorMap omap;
    if (partial) omap = tmap_in;
    else if (make_rec_map(&omap, out, cout, pw, ph, 8, 16, out_y0, out_rows)) return cudaErrorInvalidValue;
#define X(ci, co) \
    if (cin == ci && cout == co) return launch_one<ci, co>(&tmap_in, &omap, p, num_sms, mode == W2X_PRECISION_F16_F8X2, s);
    W2X_TC_SHAPES(X)
#undef X
    return cudaErrorInvalidValue;
}

template <int COUT>
static cudaError_t launch_first_c(const FirstSource &src, int pw, int ph, const float *wgt, const float *bias, __half *out, cudaStream_t s, int f8,
                                  int out_y0, int out_rows) {
    static_assert(FIRST_TILE_BYTES + 1024 <= 48 * 1024, "the first layer's staging tile stays under the default dynamic shared memory limit");
    FirstParams<COUT> prm;                                    // HOST pointers -> kernel parameters; ACT_SCALE folded in (exact: a power of two)
    for (int p = 0; p < COUT / 2; p++) {
        for (int k = 0; k < 9; k++) prm.w[p * 9 + k] = make_float2(wgt[(2 * p) * 9 + k] * ACT_SCALE, wgt[(2 * p + 1) * 9 + k] * ACT_SCALE);
        prm.b[p] = make_float2(bias[2 * p] * ACT_SCALE, bias[2 * p + 1] * ACT_SCALE);
    }
    FirstSrc fs{src.in, src.stride_floats, src.w, src.h, src.pad_x, src.pad_top, src.rows_above, src.rows_below};
    CUtensorMap omap;
    dim3 grid((pw + 31) / 32, (out_rows + 7) / 8);   // blocks tile the store window
    if (grid.y > 65535) return cudaErrorInvalidConfiguration;
    if (make_rec_map(&omap, out, COUT, pw, ph, 32, 8, out_y0, out_rows)) return cudaErrorInvalidValue;
    if (f8) first_layer_kernel<COUT, true><<<grid, 256, FIRST_TILE_BYTES + 1024, s>>>(fs, pw, ph, out_y0, omap, prm);
    else first_layer_kernel<COUT, false><<<grid, 256, FIRST_TILE_BYTES + 1024, s>>>(fs, pw, ph, out_y0, omap, prm);
    return cudaGetLastError();
}

cudaError_t launch_first(const FirstSource &src, int pw, int ph, const float *wgt, const float *bias, int cout, __half *out, cudaStream_t s, int f8,
                         int out_y0, int out_rows) {
    if (out_rows < 0) { out_y0 = 0; out_rows = ph; }
    switch (cout) {
        case 32: return launch_first_c<32>(src, pw, ph, wgt, bias, out, s, f8, out_y0, out_rows);
        case 64: return launch_first_c<64>(src, pw, ph, wgt, bias, out, s, f8, out_y0, out_rows);
        case 128: return launch_first_c<128>(src, pw, ph, wgt, bias, out, s, f8, out_y0, out_rows);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_last(const __half *in, int cin, int pw, int ph, const float *wgt, float bias, int crop, float *dst,
                        long dst_stride_floats, cudaStream_t s, int f8) {
    const int ow = pw - 2 * crop, oh = ph - 2 * crop;
    if (ow < 1 || oh < 1 || crop < 1) return cudaErrorInvalidValue;
    dim3 grid((ow + 31) / 32, (oh + 7) / 8);
    if (grid.y > 65535) return cudaErrorInvalidConfiguration;
#define W2X_LAST(C)                                                                                              \
    case C:                                                                                                          \
        if (f8) last_layer_kernel<C, true><<<grid, 256, 0, s>>>(in, pw, ph, wgt, bias, crop, dst, dst_stride_floats);    \
        else last_layer_kernel<C, false><<<grid, 256, 0, s>>>(in, pw, ph, wgt, bias, crop, dst, dst_stride_floats);      \
        break;
    switch (cin) {
        W2X_LAST(32) W2X_LAST(64) W2X_LAST(128)
        default: return cudaErrorInvalidValue;
    }
#undef W2X_LAST
    return cudaGetLastError();
}

cudaError_t launch_last_gather(const float *partial, int pw, int ph, float bias, int crop, float *dst,
                               long dst_stride_floats, cudaStream_t s) {
    return launch_last_gather_xy(partial, pw, ph, bias, crop, crop, crop, dst, dst_stride_floats, s);
}

cudaError_t launch_last_gather_xy(const float *partial, int pw, int ph, float bias, int crop_x, int crop_top,
                                  int crop_bottom, float *dst, long dst_stride_floats, cudaStream_t s) {
    const int ow = pw - 2 * crop_x, oh = ph - crop_top - crop_bottom;
    if (ow < 1 || oh < 1 || crop_x < 1 || crop_top < 1 || crop_bottom < 1) return cudaErrorInvalidValue;
    dim3 grid((ow + 31) / 32, (oh + 7) / 8);
    if (grid.y > 65535) return cudaErrorInvalidConfiguration;
    last_gather_kernel<<<grid, 256, 0, s>>>(partial, pw, ph, bias, crop_x, crop_top, crop_bottom, dst, dst_stride_floats);
    return cudaGetLastError();
}

cudaError_t launch_pack_planes(const PlaneRect *rect, const int *shelf_y0, const int *shelf_first, int n_shelf, int pad, int fw,
                               int fh, float *frame, cudaStream_t s) {
    if (n_shelf < 1 || fw < 1 || fh < 1) return cudaErrorInvalidValue;
    dim3 grid((fw + 31) / 32, (fh + 7) / 8);
    if (grid.y > 65535) return cudaErrorInvalidConfiguration;
    pack_planes_kernel<<<grid, 256, 0, s>>>(rect, shelf_y0, shelf_first, n_shelf, pad, fw, fh, frame);
    return cudaGetLastError();
}

cudaError_t launch_gather_planes(const float *partial, int fw, const PlaneRect *rect, int n_rect, int n_blocks, float bias, int pad,
                                 cudaStream_t s) {
    if (n_rect < 1 || n_blocks < 1 || pad < 1) return cudaErrorInvalidValue;
    gather_planes_kernel<<<n_blocks, 256, 0, s>>>(partial, fw, rect, n_rect, bias, pad);
    return cudaGetLastError();
}

cudaError_t launch_planar_to_nhwc(const float *in, int C, int w, int h, __half *out, cudaStream_t s, int f8) {
    long total = (long)(w + 2) * (h + 2) * C;
    planar_to_nhwc_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, C, w, h, out, f8);
    return cudaGetLastError();
}

cudaError_t launch_nhwc_to_planar(const __half *in, int C, int w, int h, float *out, cudaStream_t s, int f8) {
    long total = (long)w * h * C;
    nhwc_to_planar_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, C, w, h, out, f8);
    return cudaGetLastError();
}

// ---- TMA descriptor ----------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

// RECORD frame [Hp][Wp][C/32][128 B] (kernels.h) as a byte tensor {128, C/32, Wp, rows}, box {128, 1, box_w, box_h},
// SWIZZLE_128B; only frame rows [y0, y0 + rows) are part of the map (row coordinate 0 = frame row y0).
static int make_rec_map(CUtensorMap *map, const void *base, int C, int Wp, int Hp, int box_w, int box_h, int y0, int rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc || rows < 1 || y0 < 0 || y0 + rows > Hp || C % 32) return -1;
    cuuint64_t dims[4] = {128, (cuuint64_t)(C / 32), (cuuint64_t)Wp, (cuuint64_t)rows};
    cuuint64_t strides[3] = {128, (cuuint64_t)C * 4, (cuuint64_t)Wp * C * 4};
    cuuint32_t box[4] = {128, 1, (cuuint32_t)box_w, (cuuint32_t)box_h};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<char *>(reinterpret_cast<const char *>(base)) + (size_t)y0 * Wp * C * 4, dims, strides,
                     box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

}  // namespace tc
}  // namespace w2x
