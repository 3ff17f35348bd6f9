// engine_internal.h -- the GPU context, the row-band session and the helpers shared by engine.cu (plane driver, C ABI) and
// engine_band.cu (row-band sessions, peer-memory halo exchange, the one-process multi-GPU driver).  Not installed.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges cost a few nanoseconds when no tool is attached
#include <unistd.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "kernels.h"
#include "w2x_internal.h"

namespace w2x {
namespace eng {

// One cudaMalloc block and its owner: freed by the destructor, move-only.  It only ever grows, and a grow keeps no contents.  The
// device that allocated it must be current whenever it grows or goes (DeviceGuard in the caller).
struct DevMem {
    void *p = nullptr;
    size_t bytes = 0;
    DevMem() = default;
    DevMem(DevMem &&o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevMem &operator=(DevMem &&o) noexcept {   // o takes this block away and frees it when it goes
        std::swap(p, o.p);
        std::swap(bytes, o.bytes);
        return *this;
    }
    ~DevMem() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
    // At least `need` bytes: nothing happens when they are there; else the old block is freed first (cudaFree also orders the free
    // after the kernels that still read it) and a failed cudaMalloc leaves the buffer empty and no sticky error behind.
    cudaError_t grow(size_t need) {
        if (bytes >= need) return cudaSuccess;
        release();
        cudaError_t e = cudaMalloc(&p, need);
        if (e == cudaSuccess) bytes = need;
        else cudaGetLastError();
        return e;
    }
    int reserve(size_t need) {   // grow() for scratch: running out of device memory is W2X_ERR_NOMEM
        cudaError_t e = grow(need);
        if (e != cudaSuccess) return fail(W2X_ERR_NOMEM, "cudaMalloc of %zu bytes failed (%s)", need, cudaGetErrorString(e));
        return W2X_OK;
    }
};
template <class T>
struct DevBuf : DevMem {
    T *get() const { return static_cast<T *>(p); }
};

struct DevModel {                       // device-resident copy of one model
    std::vector<DevBuf<float>> w;       // per layer [Cout][Cin][9] fp32
    std::vector<DevBuf<float>> b;       // per layer [Cout] fp32  ((float)bias, src/modelHandler.cpp:147)
    std::vector<std::vector<float>> b_host;   // the same on the host (the tensor-core kernels take them as kernel parameters)
    std::vector<DevBuf<uint16_t>> pack; // per layer tensor-core operand image (empty if not eligible)
    std::vector<DevBuf<uint8_t>> pack8; // same for the "f8" flavour (fp16 main product + e4m3 corrections)
    std::vector<DevBuf<uint16_t>> pack_bf16;   // same for bf16x3: uploaded when the context first converts in that precision
    std::vector<float> out_scale;       // 1 / (wscale * ACT_SCALE)
    std::vector<float> last_w_t;        // HOST: last layer's weights transposed to [9][Cin] (fused last layer, passed as kernel parameters)
    int band_sessions = 0;              // live w2x_band sessions that launch with these copies (w2x_ctx_forget_model refuses while > 0)
};

struct TimedSpan { int layer; cudaEvent_t e0, e1; };

}  // namespace eng
}  // namespace w2x

struct w2x_ctx {
    int device = 0;
    int num_sms = 0;
    int cc_major = 0, cc_minor = 0;
    int engine = W2X_ENGINE_AUTO;
    int walk = W2X_WALK_FUSED;
    bool fuse_last = true;             // fold the N->1 last layer into the preceding tensor-core layer's epilogue
    int precision = W2X_PRECISION_F16_F8X2;   // default; W2X_PRECISION=f16x3|f16 in the environment or w2x_ctx_set_precision() selects another scheme
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t switch_ev = nullptr;   // w2x_ctx_set_stream: recorded on the old stream, waited for by the new one
    size_t scratch_limit = (size_t)16 << 30;
    w2x_log_fn log = nullptr;
    void *log_user = nullptr;
    uint64_t launches = 0;
    bool timing = false;
    std::vector<w2x::eng::TimedSpan> spans;
    std::vector<cudaEvent_t> event_pool;
    std::vector<std::string> layer_kernel;
    std::map<uint64_t, w2x::eng::DevModel> models;
    // scratch
    w2x::eng::DevBuf<void> buf[2];
    w2x::eng::DevBuf<float> pad_buf;
    w2x::eng::DevBuf<float> io_buf[2];      // device staging for the host-buffer entry points
    w2x::eng::DevBuf<float> chain_buf[2];   // the planes between the steps of w2x_convert_chain*
    w2x::eng::DevBuf<float> tta_buf[2];     // a W2X_STEP_TTA step's 8 variants per plane (0) and their conversions (1)
    cudaEvent_t tta_ev[2] = {};             // w2x_multi_convert_planes_chain: after a TTA step's variants kernel (0), after its units (1)
    bool tc_ready = false;
    cudaStream_t copy_in = nullptr, copy_out = nullptr;   // host<->device copies of run_host_groups overlap the compute stream
    cudaEvent_t ev_in[8] = {}, ev_done[8] = {};
    int host_bands = 0;                                   // 0 = automatic (up to 4 bands of >= 512 rows), 1 = no pipelining
    w2x::eng::DevBuf<char> plan_buf;                      // device tables of the packed frames (w2x_convert_planes, w2x_convert_tiles)
    cudaEvent_t plan_ev = nullptr;                        // recorded after the last kernel that reads plan_buf
    bool plan_ev_live = false;
    w2x::eng::DevBuf<unsigned long long> prof_buf;   // [16 layers][PROF_MAX_CTAS][PROF_WORDS], debug profile

    // The streams and events (those w2x_ctx_create got as far as creating); the buffers and the models free themselves after this
    // body.  The caller has made `device` current and keeps it so until the delete returns (w2x_ctx_destroy).
    ~w2x_ctx() {
        auto drop = [](cudaEvent_t e) { if (e) cudaEventDestroy(e); };
        drop(plan_ev);
        drop(switch_ev);
        drop(tta_ev[0]);
        drop(tta_ev[1]);
        for (auto &s : spans) { drop(s.e0); drop(s.e1); }
        for (auto e : event_pool) drop(e);
        for (int i = 0; i < 8; i++) { drop(ev_in[i]); drop(ev_done[i]); }
        if (copy_in) cudaStreamDestroy(copy_in);
        if (copy_out) cudaStreamDestroy(copy_out);
        if (own_stream) cudaStreamDestroy(own_stream);
    }
};

// One rank's rows of a plane (w2x_band_*): every intermediate activation keeps only the band's rows plus one halo row per
// neighbour side; the halo rows are written by the neighbours (peer memory) or by the caller (w2x_band_halo segments).
struct w2x_band {
    w2x_ctx *ctx = nullptr;
    const w2x_model *model = nullptr;
    w2x::eng::DevModel *dm = nullptr;   // set together with its band_sessions count
    int width = 0, rows = 0, n = 0;
    bool up = false, down = false; // a neighbour GPU owns the rows above / below: one halo row, exchanged after every layer
    bool ov_up = false, ov_down = false;   // the n rows above / below are REAL input rows supplied with the band (recomputed overlap, no exchange)
    int pt = 0, pb = 0;            // frame rows above / below the band: 1 (neighbour halo) or n (image border: replicated; overlap: real rows)
    int pw = 0, hf = 0;            // frame width / height
    int win_y0 = 0, win_rows = 0;  // the store window of the input load and every step: all frame rows but the neighbours' halo rows
    w2x::eng::DevBuf<float> pad;   // padded fp32 input frame
    w2x::eng::DevBuf<__half> act[2];
    size_t act_bytes = 0;
    int cur = 0;                   // act[cur] holds the output of the last queued step
    int last_step = -1;
    // peer-memory exchange (w2x_band_connect* / w2x_band_exchange)
    w2x::eng::DevBuf<unsigned> flags;   // [0] "rows from the up neighbour have landed", [1] same from down, [4] block counter
    unsigned seq = 0;              // exchanges issued so far: the value the next one publishes / waits for is seq + 1
    struct Peer {
        float *pad = nullptr;
        char *act[2] = {nullptr, nullptr};
        unsigned *flags = nullptr;
        int hf = 0;
        bool ipc = false;          // mapped with cudaIpcOpenMemHandle (closed with the session); else the neighbour's own pointers
    } peer[2];                     // 0 = up, 1 = down

    // Unmaps the neighbours' memory before the session's own buffers go (after this body), and gives the model's device copies
    // back to w2x_ctx_forget_model.  The caller has made the context's device current (w2x_band_create, w2x_band_destroy).
    ~w2x_band() {
        for (auto &p : peer) {
            if (!p.ipc) continue;
            for (void *q : {(void *)p.pad, (void *)p.act[0], (void *)p.act[1], (void *)p.flags})
                if (q) cudaIpcCloseMemHandle(q);
        }
        if (dm) dm->band_sessions--;
    }
};

namespace w2x {
namespace eng {

#define CU_CHECK(expr)                                                                              \
    do {                                                                                            \
        cudaError_t e__ = (expr);                                                                   \
        if (e__ != cudaSuccess)                                                                     \
            return fail(W2X_ERR_CUDA, "CUDA error %s at %s:%d (%s)", cudaGetErrorName(e__), __FILE__, __LINE__, \
                        cudaGetErrorString(e__));                                                   \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// ---- helpers defined in engine.cu --------------------------------------------------------------------------------------
int max_channels(const w2x_model *m);   // the widest activation of the model, in channels
int get_dev_model(w2x_ctx *ctx, const w2x_model *m, DevModel **out);
cudaEvent_t take_event(w2x_ctx *ctx);
void note_kernel(w2x_ctx *ctx, int layer, const char *name);
int ensure_tc(w2x_ctx *ctx);
int check_ctx(w2x_ctx *ctx);
int pick_engine(w2x_ctx *ctx, const w2x_model *m);
// Whether the tensor-core engine can run the model in the precision: its shape, and inner weights the precision's operand images
// hold (finite and below 65520 for the fp16 images, finite for bf16x3).
inline bool tc_eligible(const w2x_model *m, int precision) {
    return precision == W2X_PRECISION_BF16X3 ? m->tc_eligible_bf16 : m->tc_eligible;
}
// The bf16x3 operand images of every tensor-core layer on the context's device (once per model and context).
int upload_pack_bf16(w2x_ctx *ctx, const w2x_model *m, DevModel *dm);
void emit_reference_progress(w2x_ctx *ctx, int w, int h, int n_layers, bool split);   // the reference's stdout lines of one convertWithModels call
// The lines of one plane of w x h through w2x_convert_plane (host) / w2x_convert_plane_device: a step of w2x_convert_chain*
void emit_plane_progress(w2x_ctx *ctx, const w2x_model *m, int w, int h, int block_splitting, bool host);
// Every argument of w2x_convert_chain (HOST planes), before anything is printed, allocated or queued: W2X_ERR_ARG /
// W2X_ERR_UNSUPPORTED naming `fn` and the step.
int check_chain_host(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, const float *in, int width,
                     int height, size_t in_stride_bytes, const float *out, size_t out_stride_bytes, int block_splitting);
// One tensor-core layer `li` on frames of pw x ph: in -> out (or, fused with the last layer, -> per-pixel tap partials in `out`).
// Only frame rows [out_y0, out_y0 + out_rows) are stored (out_rows < 0: the whole frame).
int launch_layer_tc(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int li, const __half *in, __half *out, int pw, int ph,
                    bool fused, bool profile, int out_y0 = 0, int out_rows = -1);

// w2x_multi_convert_planes_chain on the contexts of a w2x_multi (engine.cu): `fn` names the entry point in messages.
int multi_planes_chain(const char *fn, const std::vector<w2x_ctx *> &ctxs, int n_steps, const w2x_model *const *models, const int *kinds,
                       int n_planes, const float *const *in, const int *widths, const int *heights, const size_t *in_strides,
                       float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user);
// w2x_multi_convert_chain_regions on the contexts of a w2x_multi (engine.cu): `fn` names the entry point in messages.
int multi_regions(const char *fn, const std::vector<w2x_ctx *> &ctxs, int n_steps, const w2x_model *const *models, const int *kinds,
                  int n_windows, const int *widths, const int *heights, const int *windows, const float *const *src,
                  const size_t *src_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user);

int tiles_enqueue_compute(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles, int width, int height, size_t in_stride_bytes, size_t out_stride_bytes);
int tiles_enqueue_download(w2x_ctx *ctx, float *const *out_tiles, int n_tiles, int width, int height, size_t out_stride_bytes);

// pinned view of a caller buffer for the duration of one call (pageable memory makes every async copy a staged, blocking one)
struct HostPin {
    void *p = nullptr;
    HostPin(const void *ptr, size_t bytes) {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, ptr) == cudaSuccess && at.type != cudaMemoryTypeUnregistered) return;   // already pinned (w2x_host_alloc, cudaHostAlloc, ...)
        cudaGetLastError();
        if (bytes >= ((size_t)4 << 20) && cudaHostRegister(const_cast<void *>(ptr), bytes, cudaHostRegisterPortable) == cudaSuccess) p = const_cast<void *>(ptr);
        else cudaGetLastError();
    }
    HostPin(const HostPin &) = delete;
    HostPin &operator=(const HostPin &) = delete;
    ~HostPin() {
        if (p) cudaHostUnregister(p);
    }
};

// Pinned views of many caller ranges for one call.  The ranges may overlap or share pages (windows whose sources are strided views
// of one plane, outputs that are strided views of one array), and cudaHostRegister refuses a range that shares a page with a
// registered one.  So the ranges not already pinned are rounded out to whole pages and merged, and each merged interval is one
// HostPin (4 MiB and more).  Every page of an interval belongs to one of the ranges, so all of it is mapped.  A range is {first
// byte, bytes from the first to the last byte}.
struct HostRange { const void *p; size_t span; };
struct HostPins {
    std::vector<std::unique_ptr<HostPin>> pins;
    explicit HostPins(const std::vector<HostRange> &ranges) {
        const uintptr_t page = (uintptr_t)sysconf(_SC_PAGESIZE);
        std::vector<std::pair<uintptr_t, uintptr_t>> iv;
        for (const HostRange &r : ranges) {
            cudaPointerAttributes at{};
            if (cudaPointerGetAttributes(&at, r.p) == cudaSuccess && at.type != cudaMemoryTypeUnregistered) continue;
            cudaGetLastError();
            const uintptr_t a = reinterpret_cast<uintptr_t>(r.p);
            iv.push_back({a / page * page, (a + r.span + page - 1) / page * page});
        }
        std::sort(iv.begin(), iv.end());
        for (size_t i = 0; i < iv.size();) {
            const uintptr_t a = iv[i].first;
            uintptr_t b = iv[i].second;
            for (i++; i < iv.size() && iv[i].first <= b; i++) b = std::max(b, iv[i].second);
            pins.push_back(std::make_unique<HostPin>(reinterpret_cast<const void *>(a), (size_t)(b - a)));
        }
    }
};

struct NvtxRange {    // a named range on the calling thread's timeline (nsys / ncu --nvtx), e.g. "w2x L3", "w2x halo exchange"
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

struct LayerTimer {   // brackets one layer launch with an NVTX range, and with events when timing is on
    w2x_ctx *ctx;
    TimedSpan span{};
    bool on;
    LayerTimer(w2x_ctx *c, int layer) : ctx(c), on(c->timing) {
        char name[24];
        snprintf(name, sizeof name, "w2x L%d", layer);
        nvtxRangePushA(name);
        if (on) {
            span.layer = layer;
            span.e0 = take_event(c);
            span.e1 = take_event(c);
            cudaEventRecord(span.e0, c->stream);
        }
    }
    ~LayerTimer() {
        if (on) {
            cudaEventRecord(span.e1, ctx->stream);
            ctx->spans.push_back(span);
        }
        nvtxRangePop();
    }
};

}  // namespace eng
}  // namespace w2x
