// w2x_internal.h -- shared declarations of the library's translation units (not installed).
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "w2x_b200.h"

namespace w2x {

// ---- error plumbing -------------------------------------------------------------------------
int fail(int code, const char *fmt, ...) __attribute__((format(printf, 2, 3)));

// ---- model ----------------------------------------------------------------------------------
// One reference `Model` (src/modelHandler.hpp:24-45): nInputPlanes, nOutputPlanes, kernelSize,
// weights[o*nIn+i] = 3x3 fp32, biases[o] fp64.
struct Layer {
    int n_in = 0, n_out = 0, k = 3;
    std::vector<float> w;    // [n_out][n_in][3][3]
    std::vector<double> b;   // [n_out]
};

// Packed operands of one layer for the tensor-core path (built once per model, host side):
//   bytes = [activation chunk c][tap t][32-channel block kb][part hi|lo][n_out rows x 64 bytes], every
//   block an exact shared memory image: K-major rows of 32 fp16 channels, 16-byte units XOR-swizzled
//   (SWIZZLE_64B).  hi = fp16(w * wscale), lo = fp16(w * wscale - hi).
struct TcPack {
    int kc = 0, n_chunk = 0, kblocks = 0, row_bytes = 0;
    float wscale = 1.0f;          // power of two
    std::vector<uint16_t> bytes;  // fp16 bit patterns
    // "f8" flavour (fp16 main product + two e4m3 correction products): per (chunk, tap, 32-channel block)
    //   [wh fp16: n_out rows x 64 B, SWIZZLE_64B][wh8 = e4m3(wh * 2^-F8_A): n_out rows x 32 B, SWIZZLE_32B]
    //   [wl8 = e4m3((w*wscale - wh) * 2^F8_C): n_out rows x 32 B, SWIZZLE_32B]
    std::vector<uint8_t> bytes8;
    // Row-strip design images, built only on request by w2x_debug_tc_strip (Cin, Cout <= 64 only, else empty): [chunk][kx] stages with ky-major rows, see model.cpp
    // pack_tc_layer_strip.  strip = f16x3 flavour [wh | wl], strip8 = f8 flavour [wh | wh8 | wl8].
    std::vector<uint8_t> strip, strip8;
};
// Scale exponents of the e4m3 correction operands: activations store xl8 = e4m3((x16 - xh) * 2^F8_A) and
// xh8 = e4m3(xh * 2^-F8_C); the weight side carries the inverse so both correction products land on the
// main product's scale (x16 * w * wscale).  Chosen by CPU emulation (tests/test_numerics_model.py).
constexpr int F8_A = 10, F8_C = 1;

}  // namespace w2x

struct w2x_model {
    std::vector<w2x::Layer> layers;
    std::vector<w2x::TcPack> tc;   // per layer; empty pack when the layer is not tensor-core-eligible
    bool tc_eligible = false;      // 1->32 ... ->1 chain with every inner layer in {32,64,128}
    uint64_t uid = 0;              // identity for per-context device caches
};

namespace w2x {
// model.cpp
int parse_model_json(const char *path, w2x_model **out);
int finalize_model(w2x_model *m);   // validation + tensor-core packing
uint16_t f32_to_f16_rn(float f);    // round-to-nearest-even, subnormals kept
float f16_to_f32(uint16_t h);
uint8_t f32_to_e4m3_rn(float f);    // OCP e4m3 (max 448, no inf), round-to-nearest-even, saturating (cvt.rn.satfinite.e4m3x2.f32)

// The most rows a frame (a padded plane, band or packed frame that one layer pass covers) may have: the first layer, the
// separate last layer, the gathers and the pack tile it in 8-row blocks on grid.y, which is at most 65535.
constexpr long MAX_FRAME_ROWS = 8L * 65535;

// geometry.cpp
struct Config { int n_job = 4, block_w = 512, block_h = 512; };
Config &config();
int block_table(int w, int h, int bw, int bh, int n_model, int *table, int capacity, int *sc, int *sr);
// Places the padded rectangles (w + 2 n_layers) x (h + 2 n_layers) of n independent planes side by side into frames of at most
// scratch_limit / (max_channels * 4) pixels and MAX_FRAME_ROWS rows.  frame[i] = the plane's frame, or -1 when its rectangle fits no
// frame (the caller converts it alone); (x0[i], y0[i]) = the rectangle's top-left corner.  Returns the frame count; fw / fh
// receive the frame sizes.
int plan_planes(int n, const int *widths, const int *heights, int n_layers, int max_channels, size_t scratch_limit, int *frame,
                int *x0, int *y0, std::vector<int> *fw, std::vector<int> *fh);
}  // namespace w2x
