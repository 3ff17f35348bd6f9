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

// ---- cv::copyMakeBorder(BORDER_REPLICATE) (src/convertRoutine.cpp:35,96): a FrameSource's frame, materialised ----------------
// A thread owns 4 columns of the two frame rows of a PAIR of plane rows (2q, 2q + 1), and writes those of frame rows [y_lo, y_hi).
// Each row reads the source row its clamp gives; when both read the same one, it is read once and stored twice.  With UP2X that is
// always so (a clamp bound inside the pair pulls the other row onto its partner), and the at most 3 source floats behind 4 adjacent
// columns are read once too.  VEC (frame rows of a multiple of 4 floats in a 16-byte aligned frame): the 4 columns are adjacent and
// leave as one 16-byte store per row; else they are 32 apart, so that each store of a warp covers 32 adjacent columns.
template <bool UP2X, bool VEC>
__global__ void __launch_bounds__(256) pad_kernel(const FrameSource src, int pw, float *__restrict__ out, int q0, int pairs, int y_lo,
                                                  int y_hi) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int x[4], sx[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        x[j] = VEC ? 4 * t + j : 4 * (t & ~31) + (t & 31) + 32 * j;
        sx[j] = frame_src<UP2X>(x[j], src.pad_x, src.w, src.cols_left, src.cols_right);
    }
    if (x[0] >= pw) return;
    for (int by = blockIdx.y; by < row_blocks(pairs, blockDim.y); by += gridDim.y) {
        const int p = by * blockDim.y + threadIdx.y;
        if (p >= pairs) continue;
        const float *row = nullptr;
        float v[4];
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int fy = 2 * (q0 + p) + i + src.pad_top;
            if (fy < y_lo || fy >= y_hi) continue;
            const float *r = src.in + (long)frame_src<UP2X>(fy, src.pad_top, src.h, src.rows_above, src.rows_below) * src.stride_floats;
            if (r != row) {
                row = r;
                v[0] = __ldg(row + sx[0]);
#pragma unroll
                for (int j = 1; j < 4; j++) v[j] = sx[j] == sx[j - 1] ? v[j - 1] : __ldg(row + sx[j]);
            }
            float *o = out + (long)fy * pw;
            if (VEC) {
                *reinterpret_cast<float4 *>(o + x[0]) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (x[j] < pw) o[x[j]] = v[j];
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

// A row band's padded 2x input frame is materialised here too.  Folding the resize into the band's first-layer loads (the
// first_1xN+up2x form of the one-GPU chain) is deliberately not done: the frame is 4 bytes per pixel beside 512 bytes per pixel of
// activations, and the fold would need the halo exchange to deliver half-resolution rows into a side buffer instead of a row of the
// frame.
cudaError_t launch_pad(const FrameSource &src, int pw, int ph, float *out, cudaStream_t s, int out_y0, int out_rows) {
    if (out_rows < 0) { out_y0 = 0; out_rows = ph; }
    if (out_y0 < 0 || out_rows < 1 || out_y0 + out_rows > ph) return cudaErrorInvalidValue;
    // the pairs of plane rows (2q, 2q + 1) behind the window: q0 .. q1
    const int q0 = (out_y0 - src.pad_top) >> 1, q1 = (out_y0 + out_rows - 1 - src.pad_top) >> 1;
    const dim3 b(32, 8), g = grid2d((pw + 3) / 4, q1 - q0 + 1, b);
    const bool vec = pw % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
    auto go = [&](void (*kernel)(const FrameSource, int, float *, int, int, int, int)) {
        kernel<<<g, b, 0, s>>>(src, pw, out, q0, q1 - q0 + 1, out_y0, out_y0 + out_rows);
    };
    if (src.up2x) go(vec ? pad_kernel<true, true> : pad_kernel<true, false>);
    else go(vec ? pad_kernel<false, true> : pad_kernel<false, false>);
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
