// kernels.h -- launchers of every kernel in the library (device code lives in the .cu files).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "w2x_b200.h"

namespace w2x {

// The padded input frame of a conversion, pw x ph pixels, read by the first layer (tc::launch_first) or materialised by launch_pad:
// cv::copyMakeBorder(BORDER_REPLICATE) (src/convertRoutine.cpp:35,96) of a w x h plane, where the plane may have real rows and
// columns beyond it (row bands, windows).  Frame pixel (fy, fx) is the plane's pixel
//     (clamp(fy - pad_top, -rows_above, h - 1 + rows_below), clamp(fx - pad_x, -cols_left, w - 1 + cols_right))
// of `in` (row stride stride_floats), whose pixel (0, 0) it points at.  pad_x and pad_top are the left and top pads; the right and
// bottom ones are pw - w - pad_x and ph - h - pad_top.
// up2x: the plane is the nearest-neighbour 2x resize of `in` (cv::resize INTER_NEAREST to exactly twice the size,
// src/main.cpp:135-139), never materialised: the pixel (y, x) above is in[y >> 1][x >> 1] (>> floors, also above and to the left).
// Every count is then in 2x rows and columns, and row 0 and column 0 of the plane are the first copies of in's row 0 and column 0: a
// window or band that starts on an odd 2x row (column) widens by one, its h (w) one larger and pad_top and rows_above (pad_x and
// cols_left) one smaller.
struct FrameSource {
    const float *in;
    long stride_floats;
    int w, h, pad_x, pad_top, rows_above, rows_below;
    bool up2x = false;
    int cols_left = 0, cols_right = 0;

    // A pw x ph region (row stride `stride` floats) that already is a padded frame.
    static FrameSource padded(const float *p, long stride, int pw, int ph) { return FrameSource{p, stride, pw, ph, 0, 0, 0, 0}; }
    // The frame of rows [r, r + rows + 2 pad) of this one.  When this frame has pad rows above the plane it converts, that is the frame
    // of the plane's rows [r, r + rows) with pad rows above and below, the plane's other rows being real rows beyond them.  An up2x
    // band starting on an odd 2x row widens by one.
    FrameSource band(int r, int rows, int pad) const {
        const int v0 = r + pad - pad_top, p = up2x ? v0 & 1 : 0, o = v0 - p;    // plane rows: v0 the band's first, o its row 0 (even with up2x)
        FrameSource b = *this;
        b.in = in + (long)(up2x ? o >> 1 : o) * stride_floats;
        b.h = rows + p;
        b.pad_top = pad - p;
        b.rows_above = rows_above + o;
        b.rows_below = h + rows_below - v0 - rows;
        return b;
    }
};

#ifdef __CUDACC__
// One axis of FrameSource's mapping: frame coordinate f -> the row (column) of `in` it reads.  The one definition of the clamp:
// the first layer's loads and the padding kernel both call it.
template <bool UP2X>
__device__ __forceinline__ int frame_src(int f, int pad, int len, int before, int after) {
    const int v = min(max(f - pad, -before), len - 1 + after);
    return UP2X ? v >> 1 : v;
}
#endif

// ---- kernels_fp32.cu --------------------------------------------------------------------------
// The frame of src, pw x ph, dense.  Only frame rows [out_y0, out_y0 + out_rows) are written (-1: the whole frame), as in
// tc::launch_first; a row-band session leaves its halo rows to the neighbours that write them.
cudaError_t launch_pad(const FrameSource &src, int pw, int ph, float *out, cudaStream_t s, int out_y0 = 0, int out_rows = -1);
// Peer-memory halo exchange (engine_band.cu): ONE kernel copies up to 8 row segments into the neighbour GPUs' frames,
// publishes `value` in their flag words once every byte is visible system-wide, then waits until the neighbours have
// published the same value here.  Flag values only grow, so nothing is ever reset.
struct HaloXArgs {
    int n;                       // segments
    const char *src[8];
    char *dst[8];
    size_t bytes;                // per segment (multiple of 4)
    unsigned *counter;           // block-completion counter in this GPU's memory (self-resetting)
    unsigned *peer_flag[2];      // where to publish (nullptr = no neighbour on that side)
    const unsigned *my_flag[2];  // what to wait for
    unsigned value;
};
cudaError_t launch_halo_exchange(const HaloXArgs &a, cudaStream_t s);
cudaError_t launch_crop(const float *in, int w, int h, int pad, float *out, long out_stride_floats, cudaStream_t s);
cudaError_t launch_copy2d(const float *in, long in_stride_floats, float *out, long out_stride_floats, int w, int h,
                          cudaStream_t s);
cudaError_t launch_conv3x3_fp32(const float *in, float *out, const float *wgt, const float *bias, int Cin, int Cout,
                                int W, int H, cudaStream_t s);
// Test-time augmentation (chain steps with W2X_STEP_TTA), both engines.  Variant j = 0..7 of a w x h plane X, with t = bit 2,
// fy = bit 1 and fx = bit 0 of j, is W' x H' = (t ? h : w) x (t ? w : h) and V_j[y][x] = X[r][c], x' = fx ? W'-1-x : x,
// y' = fy ? H'-1-y : y, (r, c) = t ? (x', y') : (y', x').  A DEVICE table of TtaPlane lists the planes of one call; each kernel
// tiles every plane into 32 x 32 tiles, plane i owning tiles [blk0_i, blk0_i + ceil(w/32) * ceil(h/32)).
struct TtaPlane {
    const float *src;    // tta_variants: the plane X, row stride src_stride floats
    float *var[8];       // variant j (tta_variants) or its conversion (tta_mean), dense and W' wide, on the GPU that converts it
                         // (a peer address when that is not the launching GPU)
    float *dst;          // tta_mean: the output plane, row stride dst_stride floats
    long src_stride, dst_stride;
    int w, h;            // X's size (tta_variants) or the output's (tta_mean)
    int blk0;
};
// V_0 .. V_7 of every plane of the table.  One launch of n_tiles blocks.
cudaError_t launch_tta_variants(const TtaPlane *tab, int n_planes, int n_tiles, cudaStream_t s);
// dst[r][c] = (((O_0 + O_1) + O_2) + ... + O_7) * 0.125f in fp32, O_j = the variant output j at the pixel V_j maps (r, c) to.  One
// launch of n_tiles blocks.
cudaError_t launch_tta_mean(const TtaPlane *tab, int n_planes, int n_tiles, cudaStream_t s);

// ---- kernels_tc.cu ----------------------------------------------------------------------------
namespace tc {
constexpr int REGION = 16;          // a tile-set covers REGION x REGION output pixels (two 8x16 M-tiles)
constexpr int HALO = REGION + 2;    // staged input footprint per side
constexpr float ACT_SCALE = 16.0f;  // activations are stored as hi/lo records of (value * ACT_SCALE)

// The record format of the activation frames between layers (RECORD frames, see launch_tc_layer): 128 bytes per pixel per
// 32-channel block, 4 bytes per element, in every format.
enum class Rec : int {
    F16 = 0,    // {hi fp16 x32 | lo fp16 x32}                 W2X_PRECISION_F16X3, W2X_PRECISION_F16
    F8 = 1,     // {xh fp16 x32 | xh8 e4m3 x32 | xl8 e4m3 x32}  W2X_PRECISION_F16_F8X2
    BF16 = 2,   // {hi bf16 x32 | lo bf16 x32}                 W2X_PRECISION_BF16X3
};
// The one place a precision (W2X_PRECISION_*) decides the record format.
inline Rec rec_format(int precision) {
    return precision == W2X_PRECISION_F16_F8X2 ? Rec::F8 : precision == W2X_PRECISION_BF16X3 ? Rec::BF16 : Rec::F16;
}

// Activation frame between layers: 4 bytes per element (RECORD frame, see launch_tc_layer).
inline size_t act_bytes(int C, int Wp, int Hp) { return (size_t)Hp * Wp * C * 4; }

bool layer_supported(int cin, int cout);
size_t layer_smem_bytes(int cin, int cout);
// One-time per process: raise the dynamic shared memory limit of every instantiation.
cudaError_t init_kernels();

// First layer (Cin = 1): same-size 3x3 correlation with BORDER_REPLICATE (src/modelHandler.cpp:141-142) on src's frame of pw x ph,
// whose padding is folded into the loads (FrameSource::padded() reads an already padded region).  -> RECORD frame.
// `wgt` ([C][9]) and `bias` ((float)bias) are HOST pointers: they travel as kernel parameters.
cudaError_t launch_first(const FrameSource &src, int pw, int ph, const float *wgt /*[C][9]*/, const float *bias, int cout, __half *out,
                         cudaStream_t s, Rec rec, int out_y0 = 0, int out_rows = -1);
// Tensor-core (wgmma) layer: in/out NHWC frames (pw x ph); the tensor maps are built inside.
// `bias` is a HOST pointer to the layer's (float)bias values (they travel as kernel parameters).
// mode = W2X_PRECISION_*, records rec_format(mode): F16X3 (0) and F16 (2): Rec::F16 frames, wpack = TcPack::bytes (F16 reads
// only its wh halves);  F16_F8X2 (1): Rec::F8 frames, wpack = TcPack::bytes8;  BF16X3 (4): Rec::BF16 frames,
// wpack = TcPack::bytes_bf16.
cudaError_t launch_tc_layer(const __half *in, const void *wpack, const float *bias, __half *out,
                            int cin, int cout, int pw, int ph, float out_scale, int mode, int num_sms,
                            cudaStream_t s, unsigned long long *prof = nullptr, const float *last_w = nullptr,
                            float *partial = nullptr, int out_y0 = 0, int out_rows = -1);
// Frames: every activation between layers is a RECORD frame [Hp][Wp][C/32][128 B] -- one 128-byte record per pixel per
// 32-channel block in the format Rec: 4 bytes per element, one TMA box row per record (SWIZZLE_128B).
// out_y0 / out_rows (both launchers): only frame rows [out_y0, out_y0 + out_rows) are stored (-1 = the whole frame); a
// row-band session keeps its halo rows out of the window because its neighbours write them.
// Fused last layer: launch_tc_layer(..., last_w = HOST pointer to [9][cout] fp32 tap-major, partial = [ph][pw][12] fp32) makes the
// tensor-core layer emit per-pixel tap partials instead of activations; launch_last_gather sums the 3x3
// neighbourhood of partials, adds the bias, applies the leaky-ReLU and writes the fp32 plane cropped by crop_x columns left and
// right, crop_top rows above and crop_bottom rows below.
cudaError_t launch_last_gather(const float *partial, int pw, int ph, float bias, int crop_x, int crop_top, int crop_bottom, float *dst,
                               long dst_stride_floats, cudaStream_t s);
inline size_t partial_bytes(int Wp, int Hp) { return (size_t)Hp * Wp * 12 * sizeof(float); }
// Packed frames: independent planes (or windows) side by side in one frame, each inside its own padded rectangle of
// (w + 2 pad) x (h + 2 pad) pixels (pad = the model's layer count).  A DEVICE table of PlaneRect lists them by shelf: ascending y0,
// then ascending x0; rectangles sharing a y0 form a shelf, shelf_y0[s] is its row and rect[shelf_first[s] .. shelf_first[s + 1]) its
// rectangles.
struct PlaneRect {
    FrameSource src;     // the rectangle's frame (pack): (w + 2 pad) x (h + 2 pad), its pads pad (less a window's phase), with the
                         // window's real rows and columns beyond it as context; a whole plane's has none
    float *dst;          // its interior output, row stride dst_stride floats (gather)
    long dst_stride;
    int w, h;            // output window size (the interior)
    int x0, y0;          // top-left corner of its padded rectangle in the frame
    int blk0;            // first gather block: plane i owns blocks [blk0_i, blk0_i + ceil(w/32) * ceil(h/8))
};
// The frame's padded fp32 image (fw x fh, dense): every rectangle's FrameSource inside it, 0 elsewhere.  One launch.
// up2x: every rectangle's FrameSource is up2x (pixel (y, x) of its plane = in[y >> 1][x >> 1]).
cudaError_t launch_pack_planes(const PlaneRect *rect, const int *shelf_y0, const int *shelf_first, int n_shelf, int pad, int fw,
                               int fh, bool up2x, float *frame, cudaStream_t s);
// The fused last layer's output for every plane of the frame, from its tap partials ([fh][fw][12]).  One launch of n_blocks.
cudaError_t launch_gather_planes(const float *partial, int fw, const PlaneRect *rect, int n_rect, int n_blocks, float bias, int pad,
                                 cudaStream_t s);
constexpr int PROF_WORDS = 16;      // per-CTA profile record (see tc_config.cuh PROF_*)
constexpr int PROF_MAX_CTAS = 256;
// Last layer (Cout = 1): RECORD frame -> fp32 plane, interior only: out(y,x) for
// y in [crop, ph-crop), x in [crop, pw-crop) is written to dst[(y-crop)*stride + (x-crop)].
cudaError_t launch_last(const __half *in, int cin, int pw, int ph, const float *wgt /*[C][9]*/, float bias,
                        int crop, float *dst, long dst_stride_floats, cudaStream_t s, Rec rec);
// planar fp32 [C][h][w] -> RECORD frame (h+2) x (w+2), replicate ring of 1 (for w2x_filter_layer)
cudaError_t launch_planar_to_nhwc(const float *in, int C, int w, int h, __half *out, cudaStream_t s, Rec rec);
// RECORD frame (h+2) x (w+2) -> planar fp32 [C][h][w] (interior)
cudaError_t launch_nhwc_to_planar(const __half *in, int C, int w, int h, float *out, cudaStream_t s, Rec rec);

}  // namespace tc

}  // namespace w2x
