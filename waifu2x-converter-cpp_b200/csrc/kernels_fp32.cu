// kernels_fp32.cu -- the fp32 CUDA-core engine (W2X_ENGINE_FP32) and the plane plumbing kernels.
//
// conv3x3_planar_fp32 is Model::filterWorker (reference src/modelHandler.cpp:117-159) as ONE fused
// kernel per layer: planar fp32 planes in, planar fp32 planes out, same size, BORDER_REPLICATE.
// The arithmetic keeps the reference's association: for every (output plane o, input plane i) the
// 9-tap correlation is summed on its own (taps row-major, as cv::filter2D does, :141-142), then
// added to the running plane sum with i ascending (cv::add, :144); bias is added as a float
// (:147) and the leaky-ReLU is max(v,0) + 0.1f*min(v,0) (:148-152).  Only FMA contraction inside
// the 9-tap sum differs from a non-FMA CPU build (<= 1 ulp per tap sum).
//
// Roofline: CUDA-core FFMA.  32 output planes x (9 FFMA + 1 FADD) per input plane per pixel.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "kernels.h"

namespace w2x {

// Every kernel here tiles its plane in row blocks on grid.y, which is at most 65535: a launch covers min(row blocks, 65535) of
// them and each block also takes the row blocks gridDim.y, 2 gridDim.y, ... further down, so a plane of any height runs.
constexpr unsigned MAX_GRID_Y = 65535;
__device__ __forceinline__ int row_blocks(int rows, unsigned block_rows) { return (int)((rows + block_rows - 1) / block_rows); }

// ---- cv::copyMakeBorder(BORDER_REPLICATE) (src/convertRoutine.cpp:35,96) ----------------------
// rows_above/rows_below > 0 mean real neighbour rows exist there (row-band mode): the source
// pointer addresses band row 0 and may be read at rows [-rows_above, h + rows_below); likewise cols_left/cols_right for
// columns (windows).  pad_x is the left pad, pad_right the right one.
__global__ void pad_replicate_kernel(const float *__restrict__ in, int w, int h, long in_stride,
                                     int pad_x, int pad_top, int pad_bottom, int rows_above, int rows_below,
                                     float *__restrict__ out, int skip_top, int skip_bottom, int pad_right, int cols_left,
                                     int cols_right) {
    const int W = w + pad_x + pad_right, H = h + pad_top + pad_bottom;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const int sx = min(max(x - pad_x, -cols_left), w - 1 + cols_right);
    for (int by = blockIdx.y; by < row_blocks(H, blockDim.y); by += gridDim.y) {
        const int y = by * blockDim.y + threadIdx.y;
        if (y >= H - skip_bottom || y < skip_top) continue;
        const int sy = min(max(y - pad_top, -rows_above), h - 1 + rows_below);
        out[(long)y * W + x] = in[(long)sy * in_stride + sx];
    }
}

// The same padding of the nearest-neighbour 2x resize of `in` (cv::resize INTER_NEAREST to exactly twice the size,
// src/main.cpp:135-139, whose pixel (y, x) is in[y >> 1][x >> 1]): w2 x h2 are the 2x plane's (or band's) size, the rows count
// in 2x rows, and the band starts on an even 2x row, so that its first row is the first copy of in's row 0.  The left and top pads
// may be smaller than pad (a window starting on an odd 2x column / row), and cols_left / cols_right count real 2x columns.
__global__ void pad_upsample2x_kernel(const float *__restrict__ in, int w2, int h2, long in_stride, int pad, int rows_above,
                                      int rows_below, float *__restrict__ out, int pad_left, int pad_top, int cols_left,
                                      int cols_right) {
    const int W = w2 + pad_left + pad, H = h2 + pad_top + pad;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const int sx = min(max(x - pad_left, -cols_left), w2 - 1 + cols_right) >> 1;   // arithmetic shift: floor, also left of the window
    for (int by = blockIdx.y; by < row_blocks(H, blockDim.y); by += gridDim.y) {
        const int y = by * blockDim.y + threadIdx.y;
        if (y >= H) continue;
        const int sy = min(max(y - pad_top, -rows_above), h2 - 1 + rows_below) >> 1;   // arithmetic shift: floor, also above the band
        out[(long)y * W + x] = in[(long)sy * in_stride + sx];
    }
}

// The band-frame form of pad_upsample2x_kernel (pad_replicate_kernel's frame, read through the resize): separate top / bottom pads
// and frame rows left to a neighbour GPU.  A thread owns 4 frame columns of one 2x row PAIR (2q, 2q + 1): clamping either row to
// [-rows_above, h2 - 1 + rows_below] and halving gives the same source row (a clamp bound inside the pair pulls the other row onto
// its partner), so the at most 3 source floats behind the 4 columns are read once, through the read-only path, and stored to both
// rows -- as one 16-byte store each when VEC (frame rows of a multiple of 4 floats in a 16-byte aligned frame).
template <bool VEC>
__global__ void __launch_bounds__(256) pad_upsample2x_xy_kernel(const float *__restrict__ in, int w2, int h2, long in_stride, int pad_x,
                                                                int pad_top, int pad_bottom, int rows_above, int rows_below,
                                                                float *__restrict__ out, int skip_top, int skip_bottom, int pad_right,
                                                                int cols_left, int cols_right) {
    const int W = w2 + pad_x + pad_right, H = h2 + pad_top + pad_bottom;
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x0 >= W) return;
    const int q0 = -((pad_top + 1) >> 1);                  // the pair holding frame row 0 (2x row -pad_top)
    const int pairs = ((h2 + pad_bottom - 1) >> 1) - q0 + 1;
    int sx[4];
#pragma unroll
    for (int j = 0; j < 4; j++) sx[j] = min(max(x0 + j - pad_x, -cols_left), w2 - 1 + cols_right) >> 1;
    for (int by = blockIdx.y; by < row_blocks(pairs, blockDim.y); by += gridDim.y) {
        const int p = by * blockDim.y + threadIdx.y;
        if (p >= pairs) continue;
        const int y = 2 * (q0 + p);                        // the pair's first 2x row; frame rows y + pad_top and y + pad_top + 1
        const int fy = y + pad_top;
        const bool st0 = fy >= skip_top && fy < H - skip_bottom, st1 = fy + 1 >= skip_top && fy + 1 < H - skip_bottom;
        if (!st0 && !st1) continue;
        const int sy = min(max(y, -rows_above), h2 - 1 + rows_below) >> 1;   // arithmetic shift: floor, also above the band
        const float *row = in + (long)sy * in_stride;
        float v[4];
        v[0] = __ldg(row + sx[0]);
#pragma unroll
        for (int j = 1; j < 4; j++) v[j] = sx[j] == sx[j - 1] ? v[j - 1] : __ldg(row + sx[j]);
        float *o = out + (long)fy * W + x0;
        if (VEC) {
            const float4 v4 = make_float4(v[0], v[1], v[2], v[3]);
            if (st0) *reinterpret_cast<float4 *>(o) = v4;
            if (st1) *reinterpret_cast<float4 *>(o + W) = v4;
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (x0 + j >= W) break;
                if (st0) o[j] = v[j];
                if (st1) o[W + j] = v[j];
            }
        }
    }
}

// crop [pad, pad+h) x [pad, pad+w) of a dense (h+2pad) x (w+2pad) plane (src/convertRoutine.cpp:40-46)
__global__ void crop_kernel(const float *__restrict__ in, int w, int h, int pad,
                            float *__restrict__ out, long out_stride) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    for (int by = blockIdx.y; by < row_blocks(h, blockDim.y); by += gridDim.y) {
        const int y = by * blockDim.y + threadIdx.y;
        if (y < h) out[(long)y * out_stride + x] = in[(long)(y + pad) * (w + 2 * pad) + x + pad];
    }
}

// 2-D strided copy (block ROI extraction / stitching, src/convertRoutine.cpp:116-131, :143-161)
__global__ void copy2d_kernel(const float *__restrict__ in, long in_stride, float *__restrict__ out,
                              long out_stride, int w, int h) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    for (int by = blockIdx.y; by < row_blocks(h, blockDim.y); by += gridDim.y) {
        const int y = by * blockDim.y + threadIdx.y;
        if (y < h) out[(long)y * out_stride + x] = in[(long)y * in_stride + x];
    }
}

// ---- test-time augmentation: the 8 flips / transposes of a plane and the mean of their conversions ---------------------------
// One block of 32 x 8 threads per 32 x 32 tile; both kernels stage the tile in shared memory so that the transposed variants
// (t = 1) are read and written along rows too.  The row pitch of 33 floats keeps the column walks free of bank conflicts.
constexpr int TTA_TILE = 32;

__device__ __forceinline__ int tta_plane_of(const TtaPlane *__restrict__ tab, int n_planes, int b) {
    int p = 0, p1 = n_planes - 1;                // the plane owning tile b
    while (p < p1) {
        const int mid = (p + p1 + 1) >> 1;
        if (__ldg(&tab[mid].blk0) <= b) p = mid;
        else p1 = mid - 1;
    }
    return p;
}

// Tile (r0, c0) of X: pixel (r, c) goes to V_j[fy ? h-1-r : r][fx ? w-1-c : c] (t = 0, w wide) or V_j[fy ? w-1-c : c][fx ? h-1-r : r]
// (t = 1, h wide); a warp writes 32 consecutive columns of one variant row either way.
__global__ void __launch_bounds__(256) tta_variants_kernel(const TtaPlane *__restrict__ tab, int n_planes) {
    __shared__ float s[TTA_TILE][TTA_TILE + 1];
    const TtaPlane R = tab[tta_plane_of(tab, n_planes, (int)blockIdx.x)];
    const int lb = (int)blockIdx.x - R.blk0, tiles_x = (R.w + TTA_TILE - 1) / TTA_TILE;
    const int r0 = lb / tiles_x * TTA_TILE, c0 = lb % tiles_x * TTA_TILE;
    const int l = threadIdx.x & 31, q0 = threadIdx.x >> 5;
    for (int q = q0; q < TTA_TILE; q += 8)
        if (r0 + q < R.h && c0 + l < R.w) s[q][l] = __ldg(R.src + (long)(r0 + q) * R.src_stride + c0 + l);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const bool t = j & 4, fy = j & 2, fx = j & 1;
        float *V = R.var[j];
        for (int q = q0; q < TTA_TILE; q += 8) {
            if (!t) {
                const int r = r0 + q, c = c0 + l;
                if (r < R.h && c < R.w) V[(size_t)(fy ? R.h - 1 - r : r) * R.w + (fx ? R.w - 1 - c : c)] = s[q][l];
            } else {
                const int r = r0 + l, c = c0 + q;
                if (r < R.h && c < R.w) V[(size_t)(fy ? R.w - 1 - c : c) * R.h + (fx ? R.h - 1 - r : r)] = s[l][q];
            }
        }
    }
}

// Tile (r0, c0) of the output: all 8 variant outputs' values for it are staged (each read along variant rows), then every pixel sums
// them in the order j = 0..7 with round-to-nearest adds and scales by 0.125f (exact: a power of two).
__global__ void __launch_bounds__(256) tta_mean_kernel(const TtaPlane *__restrict__ tab, int n_planes) {
    __shared__ float s[8][TTA_TILE][TTA_TILE + 1];
    const TtaPlane R = tab[tta_plane_of(tab, n_planes, (int)blockIdx.x)];
    const int lb = (int)blockIdx.x - R.blk0, tiles_x = (R.w + TTA_TILE - 1) / TTA_TILE;
    const int r0 = lb / tiles_x * TTA_TILE, c0 = lb % tiles_x * TTA_TILE;
    const int l = threadIdx.x & 31, q0 = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const bool t = j & 4, fy = j & 2, fx = j & 1;
        const float *O = R.var[j];
        for (int q = q0; q < TTA_TILE; q += 8) {
            if (!t) {
                const int r = r0 + q, c = c0 + l;
                if (r < R.h && c < R.w) s[j][q][l] = __ldg(O + (size_t)(fy ? R.h - 1 - r : r) * R.w + (fx ? R.w - 1 - c : c));
            } else {
                const int r = r0 + l, c = c0 + q;
                if (r < R.h && c < R.w) s[j][l][q] = __ldg(O + (size_t)(fy ? R.w - 1 - c : c) * R.h + (fx ? R.h - 1 - r : r));
            }
        }
    }
    __syncthreads();
    for (int q = q0; q < TTA_TILE; q += 8) {
        const int r = r0 + q, c = c0 + l;
        if (r >= R.h || c >= R.w) continue;
        float acc = s[0][q][l];
#pragma unroll
        for (int j = 1; j < 8; j++) acc = __fadd_rn(acc, s[j][q][l]);
        R.dst[(long)r * R.dst_stride + c] = __fmul_rn(acc, 0.125f);
    }
}

// ---- the fp32 layer kernel --------------------------------------------------------------------
constexpr int TX = 32, TY = 8;   // pixels per block (one per thread)
constexpr int CK = 8;            // input planes staged per step

template <int CT>  // output planes per block
__global__ void __launch_bounds__(TX *TY)
conv3x3_planar_fp32(const float *__restrict__ in, float *__restrict__ out,
                    const float *__restrict__ wgt,   // [Cout][Cin][3][3]
                    const float *__restrict__ bias,  // [Cout], already (float)bias
                    int Cin, int Cout, int W, int H) {
    __shared__ float s_in[CK][TY + 2][TX + 2];
    __shared__ __align__(16) float s_w[CK][9][CT];

    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int x0 = blockIdx.x * TX;
    const int co0 = blockIdx.z * CT;
    const long plane = (long)W * H;

    for (int by = blockIdx.y; by < row_blocks(H, TY); by += gridDim.y) {   // block-uniform: the __syncthreads below stay legal
        const int y0 = by * TY;
        float acc[CT];
#pragma unroll
        for (int i = 0; i < CT; i++) acc[i] = 0.f;

        for (int c0 = 0; c0 < Cin; c0 += CK) {
            const int nck = min(CK, Cin - c0);
            // stage the input tile (+1 halo, replicate at the plane border)
            for (int idx = threadIdx.x; idx < nck * (TY + 2) * (TX + 2); idx += TX * TY) {
                int ck = idx / ((TY + 2) * (TX + 2));
                int r = idx % ((TY + 2) * (TX + 2));
                int yy = r / (TX + 2), xx = r % (TX + 2);
                int gy = min(max(y0 + yy - 1, 0), H - 1);
                int gx = min(max(x0 + xx - 1, 0), W - 1);
                s_in[ck][yy][xx] = __ldg(in + plane * (c0 + ck) + (long)gy * W + gx);
            }
            // stage the weights transposed to [ck][tap][co]
            for (int idx = threadIdx.x; idx < nck * 9 * CT; idx += TX * TY) {
                int co = idx / (nck * 9);
                int r = idx % (nck * 9);
                int ck = r / 9, t = r % 9;
                float v = 0.f;
                if (co0 + co < Cout) v = __ldg(wgt + ((long)(co0 + co) * Cin + c0 + ck) * 9 + t);
                s_w[ck][t][co] = v;
            }
            __syncthreads();
            for (int ck = 0; ck < nck; ck++) {
                float v[9];
#pragma unroll
                for (int ky = 0; ky < 3; ky++)
#pragma unroll
                    for (int kx = 0; kx < 3; kx++) v[ky * 3 + kx] = s_in[ck][ty + ky][tx + kx];
                if constexpr (CT % 4 == 0) {
#pragma unroll
                    for (int c4 = 0; c4 < CT / 4; c4++) {
                        float4 t4 = *reinterpret_cast<const float4 *>(&s_w[ck][0][c4 * 4]);
                        float t0 = t4.x * v[0], t1 = t4.y * v[0], t2 = t4.z * v[0], t3 = t4.w * v[0];
#pragma unroll
                        for (int t = 1; t < 9; t++) {
                            float4 w4 = *reinterpret_cast<const float4 *>(&s_w[ck][t][c4 * 4]);
                            t0 = fmaf(w4.x, v[t], t0);
                            t1 = fmaf(w4.y, v[t], t1);
                            t2 = fmaf(w4.z, v[t], t2);
                            t3 = fmaf(w4.w, v[t], t3);
                        }
                        acc[c4 * 4 + 0] += t0;
                        acc[c4 * 4 + 1] += t1;
                        acc[c4 * 4 + 2] += t2;
                        acc[c4 * 4 + 3] += t3;
                    }
                } else {
#pragma unroll
                    for (int co = 0; co < CT; co++) {
                        float t0 = s_w[ck][0][co] * v[0];
#pragma unroll
                        for (int t = 1; t < 9; t++) t0 = fmaf(s_w[ck][t][co], v[t], t0);
                        acc[co] += t0;
                    }
                }
            }
            __syncthreads();
        }
        const int x = x0 + tx, y = y0 + ty;
        if (x < W && y < H) {
#pragma unroll
            for (int co = 0; co < CT; co++) {
                if (co0 + co < Cout) {
                    float v = acc[co] + __ldg(bias + co0 + co);
                    float pos = fmaxf(v, 0.f), neg = fminf(v, 0.f);
                    out[plane * (co0 + co) + (long)y * W + x] = neg * 0.1f + pos;
                }
            }
        }
    }
}

// ---- launchers --------------------------------------------------------------------------------
static inline dim3 grid2d(int w, int h, dim3 b) { return dim3((w + b.x - 1) / b.x, std::min<unsigned>((h + b.y - 1) / b.y, MAX_GRID_Y)); }

cudaError_t launch_pad_replicate(const float *in, int w, int h, long in_stride_floats, int pad,
                                 int rows_above, int rows_below, float *out, cudaStream_t s, int cols_left, int cols_right) {
    return launch_pad_replicate_xy(in, w, h, in_stride_floats, pad, pad, pad, rows_above, rows_below, out, s, 0, 0, cols_left, cols_right);
}

cudaError_t launch_pad_replicate_xy(const float *in, int w, int h, long in_stride_floats, int pad_x, int pad_top,
                                    int pad_bottom, int rows_above, int rows_below, float *out, cudaStream_t s,
                                    int skip_top, int skip_bottom, int cols_left, int cols_right, int pad_right) {
    if (pad_right < 0) pad_right = pad_x;
    dim3 b(32, 8);
    pad_replicate_kernel<<<grid2d(w + pad_x + pad_right, h + pad_top + pad_bottom, b), b, 0, s>>>(
        in, w, h, in_stride_floats, pad_x, pad_top, pad_bottom, rows_above, rows_below, out, skip_top, skip_bottom, pad_right,
        cols_left, cols_right);
    return cudaGetLastError();
}

cudaError_t launch_pad_upsample2x(const float *in, int w2, int h2, long in_stride_floats, int pad, int rows_above, int rows_below,
                                  float *out, cudaStream_t s, int cols_left, int cols_right, int pad_left, int pad_top) {
    if (pad_left < 0) pad_left = pad;
    if (pad_top < 0) pad_top = pad;
    dim3 b(32, 8);
    pad_upsample2x_kernel<<<grid2d(w2 + pad_left + pad, h2 + pad_top + pad, b), b, 0, s>>>(in, w2, h2, in_stride_floats, pad, rows_above,
                                                                                          rows_below, out, pad_left, pad_top, cols_left,
                                                                                          cols_right);
    return cudaGetLastError();
}

// A row band's padded 2x input frame, materialised.  Folding the resize into the band's first-layer loads (the first_1xN+up2x form
// of the one-GPU chain) is deliberately not done: the frame is 4 bytes per pixel beside 512 bytes per pixel of activations, and the
// fold would need the halo exchange to deliver half-resolution rows into a side buffer instead of a row of the frame.
cudaError_t launch_pad_upsample2x_xy(const float *in, int w2, int h2, long in_stride_floats, int pad_x, int pad_top, int pad_bottom,
                                     int rows_above, int rows_below, float *out, cudaStream_t s, int skip_top, int skip_bottom,
                                     int cols_left, int cols_right, int pad_right) {
    if (pad_right < 0) pad_right = pad_x;
    const int W = w2 + pad_x + pad_right, pairs = ((h2 + pad_bottom - 1) >> 1) + ((pad_top + 1) >> 1) + 1;
    dim3 b(32, 8);
    const dim3 g = grid2d((W + 3) / 4, pairs, b);
    if (W % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0)
        pad_upsample2x_xy_kernel<true><<<g, b, 0, s>>>(in, w2, h2, in_stride_floats, pad_x, pad_top, pad_bottom, rows_above, rows_below, out,
                                                       skip_top, skip_bottom, pad_right, cols_left, cols_right);
    else
        pad_upsample2x_xy_kernel<false><<<g, b, 0, s>>>(in, w2, h2, in_stride_floats, pad_x, pad_top, pad_bottom, rows_above, rows_below, out,
                                                        skip_top, skip_bottom, pad_right, cols_left, cols_right);
    return cudaGetLastError();
}

// ---- peer-memory halo exchange (row-band sessions on neighbouring GPUs) -----------------------------------------------
// The rows go straight into the neighbour's frame over NVLink (peer-mapped memory: cudaDeviceEnablePeerAccess inside one
// process, CUDA IPC between processes).  Ordering is by flag words in the RECEIVER's memory; values only grow, so a flag
// is never reset and a late reader cannot miss an update.  A protocol bug must not hang the GPU: the spin gives up with
// __trap() after ~4 s.
__device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void spin_until(const unsigned *flag, unsigned value) {
    if (!flag) return;
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(flag) - value) < 0) {
        __nanosleep(100);
        if (clock64() - t0 > 8000000000LL) __trap();
    }
}

__global__ void __launch_bounds__(256) halo_exchange_kernel(const HaloXArgs a) {
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
    for (int sg = 0; sg < a.n; sg++) {
        if (a.bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(a.src[sg]) | reinterpret_cast<uintptr_t>(a.dst[sg])) % 16 == 0) {
            const uint4 *src = reinterpret_cast<const uint4 *>(a.src[sg]);
            uint4 *dst = reinterpret_cast<uint4 *>(a.dst[sg]);
            for (size_t i = tid; i < a.bytes / 16; i += nthr) dst[i] = src[i];
        } else {
            const unsigned *src = reinterpret_cast<const unsigned *>(a.src[sg]);
            unsigned *dst = reinterpret_cast<unsigned *>(a.dst[sg]);
            for (size_t i = tid; i < a.bytes / 4; i += nthr) dst[i] = src[i];
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned done = atomicAdd(a.counter, 1u) + 1u;
        if (done == gridDim.x) {                       // the last block: every row of this GPU is visible system-wide
            *a.counter = 0;
            __threadfence_system();
            if (a.peer_flag[0]) st_release_sys(a.peer_flag[0], a.value);
            if (a.peer_flag[1]) st_release_sys(a.peer_flag[1], a.value);
            spin_until(a.my_flag[0], a.value);         // ... and the neighbours' rows are here
            spin_until(a.my_flag[1], a.value);
        }
    }
}

cudaError_t launch_halo_exchange(const HaloXArgs &a, cudaStream_t s) {
    if (a.n < 0 || a.n > 8 || a.bytes % 4 || !a.counter) return cudaErrorInvalidValue;
    const int blocks = a.n == 0 ? 1 : (int)std::min<size_t>(16, (a.bytes * (size_t)a.n / 16 + 255) / 256 + 1);
    halo_exchange_kernel<<<blocks, 256, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_crop(const float *in, int w, int h, int pad, float *out, long out_stride_floats, cudaStream_t s) {
    dim3 b(32, 8);
    crop_kernel<<<grid2d(w, h, b), b, 0, s>>>(in, w, h, pad, out, out_stride_floats);
    return cudaGetLastError();
}

cudaError_t launch_copy2d(const float *in, long in_stride_floats, float *out, long out_stride_floats, int w, int h,
                          cudaStream_t s) {
    dim3 b(32, 8);
    copy2d_kernel<<<grid2d(w, h, b), b, 0, s>>>(in, in_stride_floats, out, out_stride_floats, w, h);
    return cudaGetLastError();
}

cudaError_t launch_tta_variants(const TtaPlane *tab, int n_planes, int n_tiles, cudaStream_t s) {
    if (n_planes < 1 || n_tiles < 1) return cudaErrorInvalidValue;
    tta_variants_kernel<<<n_tiles, 256, 0, s>>>(tab, n_planes);
    return cudaGetLastError();
}

cudaError_t launch_tta_mean(const TtaPlane *tab, int n_planes, int n_tiles, cudaStream_t s) {
    if (n_planes < 1 || n_tiles < 1) return cudaErrorInvalidValue;
    tta_mean_kernel<<<n_tiles, 256, 0, s>>>(tab, n_planes);
    return cudaGetLastError();
}

cudaError_t launch_conv3x3_fp32(const float *in, float *out, const float *wgt, const float *bias, int Cin, int Cout,
                                int W, int H, cudaStream_t s) {
    dim3 grid((W + TX - 1) / TX, std::min<unsigned>((H + TY - 1) / TY, MAX_GRID_Y), 1);
    if (Cout > 16) {
        grid.z = (Cout + 31) / 32;
        conv3x3_planar_fp32<32><<<grid, TX * TY, 0, s>>>(in, out, wgt, bias, Cin, Cout, W, H);
    } else if (Cout > 1) {
        grid.z = (Cout + 3) / 4;
        conv3x3_planar_fp32<4><<<grid, TX * TY, 0, s>>>(in, out, wgt, bias, Cin, Cout, W, H);
    } else {
        grid.z = 1;
        conv3x3_planar_fp32<1><<<grid, TX * TY, 0, s>>>(in, out, wgt, bias, Cin, Cout, W, H);
    }
    return cudaGetLastError();
}

}  // namespace w2x
