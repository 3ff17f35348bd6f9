// engine.cu -- GPU context, plane driver and the compute half of the C ABI.
//
// The plane driver re-creates w2xc::convertWithModels (reference src/convertRoutine.cpp:21-51),
// convertWithModelsBasic (:53-82) and convertWithModelsBlockSplit (:84-169) on top of the layer
// kernels: replicate-pad by nModel, run the layers, crop nModel.  A plane the reference would
// block-split is by default processed whole (every output pixel still sees exactly the operands
// and the operation order it sees inside its reference block, so the result is bit-identical);
// W2X_WALK_BLOCKS walks the reference's blocks literally.
//
// There is no CPU fallback anywhere in this file: without an sm_90 device every compute entry
// point fails with W2X_ERR_NO_DEVICE.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "engine_internal.h"

using namespace w2x;

namespace w2x {
namespace eng {

int ensure(void **p, size_t *have, size_t need) {
    if (*have >= need) return W2X_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *have = 0;
    cudaError_t e = cudaMalloc(p, need);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(W2X_ERR_NOMEM, "cudaMalloc of %zu bytes failed (%s)", need, cudaGetErrorString(e));
    }
    *have = need;
    return W2X_OK;
}

int get_dev_model(w2x_ctx *ctx, const w2x_model *m, DevModel **out) {
    auto it = ctx->models.find(m->uid);
    if (it != ctx->models.end()) {
        *out = &it->second;
        return W2X_OK;
    }
    DevModel dm;
    const size_t n = m->layers.size();
    dm.w.assign(n, nullptr);
    dm.b.assign(n, nullptr);
    dm.pack.assign(n, nullptr);
    dm.pack8.assign(n, nullptr);
    dm.out_scale.assign(n, 1.f);
    for (size_t i = 0; i < n; i++) {
        const Layer &L = m->layers[i];
        CU_CHECK(cudaMalloc(&dm.w[i], L.w.size() * sizeof(float)));
        CU_CHECK(cudaMemcpyAsync(dm.w[i], L.w.data(), L.w.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        std::vector<float> bf(L.b.size());
        for (size_t k = 0; k < bf.size(); k++) bf[k] = static_cast<float>(L.b[k]);
        dm.b_host.push_back(bf);
        CU_CHECK(cudaMalloc(&dm.b[i], bf.size() * sizeof(float)));
        CU_CHECK(cudaMemcpyAsync(dm.b[i], bf.data(), bf.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        CU_CHECK(cudaStreamSynchronize(ctx->stream));   // bf goes out of scope
        const TcPack &P = m->tc[i];
        if (!P.bytes.empty()) {
            CU_CHECK(cudaMalloc(&dm.pack[i], P.bytes.size() * 2));
            CU_CHECK(cudaMemcpyAsync(dm.pack[i], P.bytes.data(), P.bytes.size() * 2, cudaMemcpyHostToDevice, ctx->stream));
            dm.out_scale[i] = 1.0f / (P.wscale * tc::ACT_SCALE);
            CU_CHECK(cudaMalloc(&dm.pack8[i], P.bytes8.size()));
            CU_CHECK(cudaMemcpyAsync(dm.pack8[i], P.bytes8.data(), P.bytes8.size(), cudaMemcpyHostToDevice, ctx->stream));
        }
    }
    if (m->tc_eligible) {
        const Layer &L = m->layers.back();                // n_out == 1: w is [1][Cin][9]
        dm.last_w_t.assign((size_t)9 * L.n_in, 0.f);
        for (int c = 0; c < L.n_in; c++)
            for (int t = 0; t < 9; t++) dm.last_w_t[(size_t)t * L.n_in + c] = L.w[(size_t)c * 9 + t];
    }
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    auto res = ctx->models.emplace(m->uid, std::move(dm));
    *out = &res.first->second;
    return W2X_OK;
}

cudaEvent_t take_event(w2x_ctx *ctx) {
    if (!ctx->event_pool.empty()) {
        cudaEvent_t e = ctx->event_pool.back();
        ctx->event_pool.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

void note_kernel(w2x_ctx *ctx, int layer, const char *name) {
    if ((int)ctx->layer_kernel.size() <= layer) ctx->layer_kernel.resize((size_t)layer + 1);
    ctx->layer_kernel[(size_t)layer] = name;
}

void logf(w2x_ctx *ctx, const char *fmt, int a, int b = 0) {
    if (!ctx->log || ctx->log_muted) return;
    char line[128];
    snprintf(line, sizeof line, fmt, a, b);
    ctx->log(line, ctx->log_user);
}

// The progress lines the reference prints for one convertWithModels call (src/convertRoutine.cpp:67,133-134): per block
// "start process block (c,r) ..." + one "Iteration #k..." per layer when the plane is split, else just the iterations.
// The fused walk and the copy pipeline process the plane in other units, so they emit the reference's sequence up front.
void emit_reference_progress(w2x_ctx *ctx, int w, int h, int n_layers, bool split) {
    if (!ctx->log) return;
    int nb = 1;
    std::vector<int> tab;
    if (split) {
        const Config &cfg = config();
        nb = block_table(w, h, cfg.block_w, cfg.block_h, n_layers, nullptr, 0, nullptr, nullptr);
        if (nb < 1) return;
        tab.resize((size_t)nb * 8);
        block_table(w, h, cfg.block_w, cfg.block_h, n_layers, tab.data(), nb, nullptr, nullptr);
    }
    for (int i = 0; i < nb; i++) {
        if (split) logf(ctx, "start process block (%d,%d) ...", tab[(size_t)i * 8 + 1], tab[(size_t)i * 8]);
        for (int k = 1; k <= n_layers; k++) logf(ctx, "Iteration #%d...", k);
    }
}

struct LogMute {   // silences the per-launch lines while a caller that already emitted the reference's sequence runs the layers
    w2x_ctx *ctx;
    bool prev;
    explicit LogMute(w2x_ctx *c, bool on) : ctx(c), prev(c->log_muted) { if (on) c->log_muted = true; }
    ~LogMute() { ctx->log_muted = prev; }
};

int pick_engine(w2x_ctx *ctx, const w2x_model *m) {
    int e = ctx->engine;
    if (e == W2X_ENGINE_AUTO) e = m->tc_eligible ? W2X_ENGINE_TC : W2X_ENGINE_FP32;
    if (e == W2X_ENGINE_TC && !m->tc_eligible) {
        fail(W2X_ERR_UNSUPPORTED, "tensor-core engine needs a 1->{32,64,128}...->1 layer chain");
        return -1;
    }
    return e;
}

int ensure_tc(w2x_ctx *ctx) {
    if (ctx->tc_ready) return W2X_OK;
    CU_CHECK(tc::init_kernels());
    ctx->tc_ready = true;
    return W2X_OK;
}

// One tensor-core layer `li` on frames of pw x ph: in -> out (or, fused with the last layer, -> per-pixel tap partials in `out`).
int launch_layer_tc(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int li, const __half *in, __half *out, int pw, int ph,
                    bool fused, bool profile, int out_y0, int out_rows) {
    if (out_rows < 0) { out_y0 = 0; out_rows = ph; }
    const Layer &L = m->layers[(size_t)li];
    const int f8 = ctx->precision == W2X_PRECISION_F16_F8X2 ? 1 : 0;
    {
        LayerTimer t(ctx, li);
        CU_CHECK(tc::launch_tc_layer(in, f8 ? (const void *)dm->pack8[(size_t)li] : (const void *)dm->pack[(size_t)li],
                                     dm->b_host[(size_t)li].data(), out, L.n_in, L.n_out, pw, ph, dm->out_scale[(size_t)li], ctx->precision,
                                     ctx->num_sms, ctx->stream,
                                     profile && ctx->prof_buf ? ctx->prof_buf + (size_t)li * tc::PROF_MAX_CTAS * tc::PROF_WORDS : nullptr,
                                     fused ? dm->last_w_t.data() : nullptr, fused ? reinterpret_cast<float *>(out) : nullptr, out_y0, out_rows));
    }
    static const char *const names[3][2] = {{"wgmma_f16x3", "wgmma_f16x3+last"}, {"wgmma_f16+f8x2", "wgmma_f16+f8x2+last"}, {"wgmma_f16", "wgmma_f16+last"}};
    note_kernel(ctx, li, names[ctx->precision][fused ? 1 : 0]);
    ctx->launches++;
    return W2X_OK;
}

// ---- convertWithModelsBasic on an already padded ROI ------------------------------------------
// src: pw x ph fp32 region (row stride src_stride floats) that already contains the n-pixel ring.
// dst: receives the (pw-2n) x (ph-2n) interior.
// packed (tensor-core engine with the fused last layer only): src is a packed frame of pw x ph holding many padded planes (see
// tc::PlaneRect); the layers run ONCE on it -- the seams pollute only the rings that are cropped anyway -- and one gather writes
// every plane's interior to its own destination; dst / dst_stride are then unused.
// direct (tensor-core engine, one plane): the first layer reads the UNPADDED plane it describes and folds the replicate padding into
// its loads; src / src_stride are then unused.
struct PackedGather { const tc::PlaneRect *rect; int n_rect, n_blocks; };
int run_basic(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int engine, const float *src, long src_stride, int pw,
              int ph, float *dst, long dst_stride, const PackedGather *packed = nullptr, const tc::FirstSource *direct = nullptr) {
    const int n = (int)m->layers.size();
    if (pw - 2 * n < 1 || ph - 2 * n < 1) return fail(W2X_ERR_ARG, "plane smaller than the model's receptive ring");
    int maxc = 1;
    for (auto &L : m->layers) maxc = std::max(maxc, std::max(L.n_in, L.n_out));
    if (engine == W2X_ENGINE_FP32) {
        const size_t need = (size_t)maxc * pw * ph * sizeof(float);
        for (int i = 0; i < 2; i++) {
            int rc = ensure(&ctx->buf[i], &ctx->buf_bytes[i], need);
            if (rc) return rc;
        }
        float *cur = static_cast<float *>(ctx->buf[0]), *nxt = static_cast<float *>(ctx->buf[1]);
        CU_CHECK(launch_copy2d(src, src_stride, cur, pw, pw, ph, ctx->stream));   // ROI -> dense plane
        ctx->launches++;
        for (int li = 0; li < n; li++) {
            const Layer &L = m->layers[(size_t)li];
            logf(ctx, "Iteration #%d...", li + 1);                                 // src/convertRoutine.cpp:67
            {
                LayerTimer t(ctx, li);
                CU_CHECK(launch_conv3x3_fp32(cur, nxt, dm->w[(size_t)li], dm->b[(size_t)li], L.n_in, L.n_out, pw, ph,
                                             ctx->stream));
            }
            note_kernel(ctx, li, "fp32_direct");
            ctx->launches++;
            std::swap(cur, nxt);
        }
        CU_CHECK(launch_crop(cur, pw - 2 * n, ph - 2 * n, n, dst, dst_stride, ctx->stream));
        ctx->launches++;
        return W2X_OK;
    }
    // ---- tensor-core engine ----
    const int f8 = ctx->precision == W2X_PRECISION_F16_F8X2 ? 1 : 0;
    int rc = ensure_tc(ctx);
    if (rc) return rc;
    const size_t need = tc::act_bytes(maxc, pw, ph);
    for (int i = 0; i < 2; i++) {
        rc = ensure(&ctx->buf[i], &ctx->buf_bytes[i], need);
        if (rc) return rc;
    }
    __half *cur = static_cast<__half *>(ctx->buf[0]), *nxt = static_cast<__half *>(ctx->buf[1]);
    {
        const Layer &L = m->layers[0];
        logf(ctx, "Iteration #%d...", 1);
        LayerTimer t(ctx, 0);
        const tc::FirstSource padded{src, src_stride, pw, ph, 0, 0, 0, 0};
        CU_CHECK(tc::launch_first(direct ? *direct : padded, pw, ph, L.w.data(), dm->b_host[0].data(), L.n_out, cur, ctx->stream, f8));
        note_kernel(ctx, 0, "first_1xN");
        ctx->launches++;
    }
    const bool fuse = ctx->fuse_last && n >= 3 && !dm->last_w_t.empty();
    for (int li = 1; li + 1 < n; li++) {
        logf(ctx, "Iteration #%d...", li + 1);
        rc = launch_layer_tc(ctx, m, dm, li, cur, nxt, pw, ph, fuse && li == n - 2, true);
        if (rc) return rc;
        std::swap(cur, nxt);
    }
    {
        const Layer &L = m->layers[(size_t)n - 1];
        logf(ctx, "Iteration #%d...", n);
        LayerTimer t(ctx, n - 1);
        if (fuse) {
            if (packed)
                CU_CHECK(tc::launch_gather_planes(reinterpret_cast<const float *>(cur), pw, packed->rect, packed->n_rect, packed->n_blocks,
                                                  static_cast<float>(L.b[0]), n, ctx->stream));
            else
                CU_CHECK(tc::launch_last_gather(reinterpret_cast<const float *>(cur), pw, ph, static_cast<float>(L.b[0]), n, dst, dst_stride, ctx->stream));
            note_kernel(ctx, n - 1, "last_gather");
        } else {
            if (packed) return fail(W2X_ERR_UNSUPPORTED, "packed frames need the fused last layer");
            CU_CHECK(tc::launch_last(cur, L.n_in, pw, ph, dm->w[(size_t)n - 1], static_cast<float>(L.b[0]), n, dst,
                                     dst_stride, ctx->stream, f8));
            note_kernel(ctx, n - 1, "last_Nx1");
        }
        ctx->launches++;
    }
    return W2X_OK;
}

// Whole plane (or row band) already available as a padded plane: cut it into horizontal bands that
// respect the scratch limit, each band re-reads n rows of context above and below.
// direct_in != nullptr (tensor-core engine): no padded plane exists; the first layer reads d_in (rows_above / rows_below real rows
// beyond the plane) with the padding folded into its loads.
int max_channels(const w2x_model *m) {
    int maxc = 1;
    for (auto &L : m->layers) maxc = std::max(maxc, std::max(L.n_in, L.n_out));
    return maxc;
}

// rows per band of run_padded_plane for a plane w wide: the band's frame (band + 2n rows) fits the scratch limit and has at most
// MAX_FRAME_ROWS rows
int scratch_band_rows(const w2x_ctx *ctx, const w2x_model *m, int w, int h) {
    const int n = (int)m->layers.size();
    const size_t per_row = (size_t)max_channels(m) * (w + 2 * n) * 4;   // both engines: 4 bytes per activation element
    long max_rows = std::min((long)(ctx->scratch_limit / per_row), MAX_FRAME_ROWS) - 2 * n;
    if (max_rows < 16) max_rows = 16;
    return (int)std::min<long>(h, max_rows);
}

int run_padded_plane(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int engine, const float *padp, int w, int h,
                     float *dst, long dst_stride, const float *direct_in = nullptr, long in_stride = 0, int rows_above = 0, int rows_below = 0) {
    const int n = (int)m->layers.size();
    const int pw = w + 2 * n;
    const int band = scratch_band_rows(ctx, m, w, h);
    for (int y0 = 0; y0 < h; y0 += band) {
        const int bh = std::min(band, h - y0);
        int rc;
        if (direct_in) {
            const tc::FirstSource fs{direct_in + (long)y0 * in_stride, in_stride, w, bh, n, n, std::min(n, y0 + rows_above), std::min(n, h - y0 - bh + rows_below)};
            rc = run_basic(ctx, m, dm, engine, nullptr, 0, pw, bh + 2 * n, dst + (long)y0 * dst_stride, dst_stride, nullptr, &fs);
        } else {
            rc = run_basic(ctx, m, dm, engine, padp + (long)y0 * pw, pw, pw, bh + 2 * n, dst + (long)y0 * dst_stride, dst_stride);
        }
        if (rc) return rc;
    }
    return W2X_OK;
}

int check_ctx(w2x_ctx *ctx) {
    if (!ctx) return fail(W2X_ERR_ARG, "NULL context");
    return W2X_OK;
}

int convert_device(w2x_ctx *ctx, const w2x_model *m, const float *d_in, int w, int h, size_t in_stride_bytes,
                   int rows_above, int rows_below, float *d_out, size_t out_stride_bytes, int block_splitting) {
    if (!m || !d_in || !d_out || w < 1 || h < 1) return fail(W2X_ERR_ARG, "w2x_convert_plane: bad argument");
    if (in_stride_bytes % 4 || out_stride_bytes % 4 || in_stride_bytes < (size_t)w * 4 || out_stride_bytes < (size_t)w * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: row strides must be multiples of 4 bytes and >= width*4");
    if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: model must map 1 plane to 1 plane");
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convertWithModels");
    const int engine = pick_engine(ctx, m);
    if (engine < 0) return W2X_ERR_UNSUPPORTED;
    DevModel *dm = nullptr;
    int rc = get_dev_model(ctx, m, &dm);
    if (rc) return rc;
    const int n = (int)m->layers.size();
    const int pw = w + 2 * n, ph = h + 2 * n;
    const long ostride = (long)(out_stride_bytes / 4);
    const bool split = block_splitting && w2x_requires_splitting(w, h);
    if (engine == W2X_ENGINE_TC && !(split && ctx->walk == W2X_WALK_BLOCKS)) {
        // cv::copyMakeBorder (src/convertRoutine.cpp:35, :96) is folded into the first layer's loads: no padded copy of the plane
        if (split && !ctx->log_muted) emit_reference_progress(ctx, w, h, n, true);
        LogMute mute(ctx, split);
        return run_padded_plane(ctx, m, dm, engine, nullptr, w, h, d_out, ostride, d_in, (long)(in_stride_bytes / 4), rows_above, rows_below);
    }
    rc = ensure(reinterpret_cast<void **>(&ctx->pad_buf), &ctx->pad_bytes, (size_t)pw * ph * sizeof(float));
    if (rc) return rc;
    // cv::copyMakeBorder(in, temp, n, n, n, n, BORDER_REPLICATE)   (src/convertRoutine.cpp:35, :96)
    CU_CHECK(launch_pad_replicate(d_in, w, h, (long)(in_stride_bytes / 4), n, std::min(rows_above, n),
                                  std::min(rows_below, n), ctx->pad_buf, ctx->stream));
    ctx->launches++;
    if (split && ctx->walk == W2X_WALK_BLOCKS) {
        // the literal block walk of convertWithModelsBlockSplit (src/convertRoutine.cpp:114-165)
        const Config &cfg = config();
        int nb = block_table(w, h, cfg.block_w, cfg.block_h, n, nullptr, 0, nullptr, nullptr);
        if (nb < 0) return fail(W2X_ERR_ARG, "block size too small for a %d-layer model", n);
        std::vector<int> tab((size_t)nb * 8);
        block_table(w, h, cfg.block_w, cfg.block_h, n, tab.data(), nb, nullptr, nullptr);
        for (int i = 0; i < nb; i++) {
            const int *t = &tab[(size_t)i * 8];
            logf(ctx, "start process block (%d,%d) ...", t[1], t[0]);              // :133-134 prints (c,r)
            const int bw_i = t[5] - t[4], bh_i = t[3] - t[2];
            if (t[6] + bh_i - 2 * n > h || t[7] + bw_i - 2 * n > w)
                return fail(W2X_ERR_ARG, "block (%d,%d) does not fit the output plane (non-square block size?)", t[1], t[0]);
            rc = run_basic(ctx, m, dm, engine, ctx->pad_buf + (long)t[2] * pw + t[4], pw, bw_i, bh_i,
                           d_out + (long)t[6] * ostride + t[7], ostride);
            if (rc) return rc;
        }
        return W2X_OK;
    }
    if (split && !ctx->log_muted) emit_reference_progress(ctx, w, h, n, true);     // fused walk: the reference's per-block lines, up front
    LogMute mute(ctx, split);
    return run_padded_plane(ctx, m, dm, engine, ctx->pad_buf, w, h, d_out, ostride);
}

}  // namespace eng
}  // namespace w2x

using namespace w2x::eng;

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int w2x_ctx_create(int device, w2x_ctx **out_ctx) {
    if (!out_ctx) return fail(W2X_ERR_ARG, "w2x_ctx_create: NULL out pointer");
    *out_ctx = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        return fail(W2X_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= count) return fail(W2X_ERR_ARG, "w2x_ctx_create: device %d out of range [0,%d)", device, count);
    cudaDeviceProp prop;
    CU_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(W2X_ERR_NO_DEVICE, "device %d (%s) is sm_%d%d; this build carries sm_90a code only", device,
                    prop.name, prop.major, prop.minor);
    auto ctx = std::make_unique<w2x_ctx>();
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->cc_major = prop.major;
    ctx->cc_minor = prop.minor;
    DeviceGuard g(device);
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    if (const char *pe = std::getenv("W2X_PRECISION")) {
        if (!std::strcmp(pe, "f16x3")) ctx->precision = W2X_PRECISION_F16X3;
        else if (!std::strcmp(pe, "f16+f8x2") || !std::strcmp(pe, "f8")) ctx->precision = W2X_PRECISION_F16_F8X2;
        else if (!std::strcmp(pe, "f16")) ctx->precision = W2X_PRECISION_F16;
    }
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking));
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking));
    for (int i = 0; i < 8; i++) {
        CU_CHECK(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
        CU_CHECK(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
    }
    CU_CHECK(cudaEventCreateWithFlags(&ctx->plan_ev, cudaEventDisableTiming));
    *out_ctx = ctx.release();
    return W2X_OK;
}

static void free_dev_model(DevModel &dm) {
    for (auto p : dm.w) cudaFree(p);
    for (auto p : dm.b) cudaFree(p);
    for (auto p : dm.pack) cudaFree(p);
    for (auto p : dm.pack8) cudaFree(p);
}

// Drops the context's device copies of a model (weights, packed operands); call it before w2x_model_free in a long-lived
// context that cycles through many models.  The next conversion with the same model uploads it again.
int w2x_ctx_forget_model(w2x_ctx *ctx, const w2x_model *model) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model) return fail(W2X_ERR_ARG, "w2x_ctx_forget_model: NULL model");
    auto it = ctx->models.find(model->uid);
    if (it == ctx->models.end()) return W2X_OK;
    DeviceGuard g(ctx->device);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    free_dev_model(it->second);
    ctx->models.erase(it);
    return W2X_OK;
}

void w2x_ctx_destroy(w2x_ctx *ctx) {
    if (!ctx) return;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &kv : ctx->models) free_dev_model(kv.second);
    for (int i = 0; i < 2; i++) {
        cudaFree(ctx->buf[i]);
        cudaFree(ctx->io_buf[i]);
    }
    cudaFree(ctx->pad_buf);
    cudaFree(ctx->plan_buf);
    cudaFree(ctx->prof_buf);
    if (ctx->plan_ev) cudaEventDestroy(ctx->plan_ev);
    for (auto &s : ctx->spans) { cudaEventDestroy(s.e0); cudaEventDestroy(s.e1); }
    for (auto e : ctx->event_pool) cudaEventDestroy(e);
    for (int i = 0; i < 8; i++) {
        if (ctx->ev_in[i]) cudaEventDestroy(ctx->ev_in[i]);
        if (ctx->ev_done[i]) cudaEventDestroy(ctx->ev_done[i]);
    }
    if (ctx->copy_in) cudaStreamDestroy(ctx->copy_in);
    if (ctx->copy_out) cudaStreamDestroy(ctx->copy_out);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

int w2x_ctx_set_engine(w2x_ctx *ctx, int engine) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (engine < W2X_ENGINE_AUTO || engine > W2X_ENGINE_TC) return fail(W2X_ERR_ARG, "unknown engine %d", engine);
    ctx->engine = engine;
    return W2X_OK;
}
int w2x_ctx_get_engine(const w2x_ctx *ctx) { return ctx ? ctx->engine : -1; }

int w2x_ctx_set_precision(w2x_ctx *ctx, int precision) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (precision != W2X_PRECISION_F16X3 && precision != W2X_PRECISION_F16_F8X2 && precision != W2X_PRECISION_F16) return fail(W2X_ERR_ARG, "unknown precision mode %d", precision);
    ctx->precision = precision;
    return W2X_OK;
}
int w2x_ctx_get_precision(const w2x_ctx *ctx) { return ctx ? ctx->precision : -1; }

int w2x_ctx_set_stream(w2x_ctx *ctx, void *cuda_stream) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
    return W2X_OK;
}

int w2x_ctx_synchronize(w2x_ctx *ctx) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    DeviceGuard g(ctx->device);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}

int w2x_ctx_set_log(w2x_ctx *ctx, w2x_log_fn fn, void *user) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->log = fn;
    ctx->log_user = user;
    return W2X_OK;
}

int w2x_ctx_set_block_walk(w2x_ctx *ctx, int mode) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (mode != W2X_WALK_FUSED && mode != W2X_WALK_BLOCKS) return fail(W2X_ERR_ARG, "unknown block walk mode %d", mode);
    ctx->walk = mode;
    return W2X_OK;
}

int w2x_ctx_set_scratch_limit(w2x_ctx *ctx, size_t bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->scratch_limit = bytes ? bytes : (size_t)16 << 30;
    return W2X_OK;
}

// Probe hooks (not part of the stable ABI): per-role wait/work cycle counters of the tensor-core layer kernels.
W2X_API int w2x_debug_tc_profile_enable(w2x_ctx *ctx, int on) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    DeviceGuard g(ctx->device);
    const size_t bytes = (size_t)16 * tc::PROF_MAX_CTAS * tc::PROF_WORDS * sizeof(unsigned long long);
    if (on) {
        if (!ctx->prof_buf) CU_CHECK(cudaMalloc(&ctx->prof_buf, bytes));
        CU_CHECK(cudaMemsetAsync(ctx->prof_buf, 0, bytes, ctx->stream));
    } else if (ctx->prof_buf) {
        CU_CHECK(cudaStreamSynchronize(ctx->stream));
        cudaFree(ctx->prof_buf);
        ctx->prof_buf = nullptr;
    }
    return W2X_OK;
}
// out[PROF_WORDS]: counters of `layer` summed over CTAs; *n_ctas = CTAs that ran.
W2X_API int w2x_debug_tc_profile_read(w2x_ctx *ctx, int layer, unsigned long long *out, int *n_ctas) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!ctx->prof_buf || layer < 0 || layer >= 16 || !out) return fail(W2X_ERR_ARG, "profile not enabled or bad layer");
    DeviceGuard g(ctx->device);
    std::vector<unsigned long long> h((size_t)tc::PROF_MAX_CTAS * tc::PROF_WORDS);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    CU_CHECK(cudaMemcpy(h.data(), ctx->prof_buf + (size_t)layer * h.size(), h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    int n = 0;
    for (int w = 0; w < tc::PROF_WORDS; w++) out[w] = 0;
    for (int c = 0; c < tc::PROF_MAX_CTAS; c++) {
        if (h[(size_t)c * tc::PROF_WORDS] == 0) continue;
        n++;
        for (int w = 0; w < tc::PROF_WORDS; w++) out[w] += h[(size_t)c * tc::PROF_WORDS + w];
    }
    if (n_ctas) *n_ctas = n;
    return W2X_OK;
}

// Probe switch (not part of the stable ABI): number of SMs the persistent tensor-core kernels of this context occupy (0 = all).
W2X_API int w2x_debug_set_num_sms(w2x_ctx *ctx, int n) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    cudaDeviceProp prop;
    CU_CHECK(cudaGetDeviceProperties(&prop, ctx->device));
    ctx->num_sms = n > 0 && n < prop.multiProcessorCount ? n : prop.multiProcessorCount;
    return W2X_OK;
}

// Probe switch (not part of the stable ABI): number of host-copy pipeline bands of w2x_convert_plane (0 auto, 1 off).
W2X_API int w2x_debug_set_host_bands(w2x_ctx *ctx, int bands) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->host_bands = bands < 0 ? 0 : bands;
    return W2X_OK;
}

// Probe switch (not part of the stable ABI): 1 = fold the last layer into the preceding tensor-core layer (default), 0 = separate kernel.
W2X_API int w2x_debug_set_fuse_last(w2x_ctx *ctx, int on) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->fuse_last = on != 0;
    return W2X_OK;
}

int w2x_convert_plane_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, int width, int height,
                             size_t in_stride_bytes, float *d_out, size_t out_stride_bytes, int block_splitting) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    return convert_device(ctx, model, d_in, width, height, in_stride_bytes, 0, 0, d_out, out_stride_bytes, block_splitting);
}

int w2x_convert_band_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, int width, int band_height,
                            int rows_above, int rows_below, size_t in_stride_bytes, float *d_out, size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (rows_above < 0 || rows_below < 0) return fail(W2X_ERR_ARG, "w2x_convert_band_device: negative halo");
    if (model && ((rows_above && rows_above < (int)model->layers.size()) || (rows_below && rows_below < (int)model->layers.size())))
        return fail(W2X_ERR_ARG, "w2x_convert_band_device: a halo must be 0 (image border) or >= the layer count (%zu)",
                    model->layers.size());
    if (!d_in) return fail(W2X_ERR_ARG, "w2x_convert_band_device: NULL input");
    const float *band0 = d_in + (size_t)rows_above * (in_stride_bytes / 4);
    return convert_device(ctx, model, band0, width, band_height, in_stride_bytes, rows_above, rows_below, d_out,
                          out_stride_bytes, 0);
}

int w2x_convert_plane(w2x_ctx *ctx, const w2x_model *model, const float *in, int width, int height, size_t in_stride_bytes,
                      float *out, size_t out_stride_bytes, int block_splitting) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!in || !out || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_convert_plane: bad argument");
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: row stride smaller than a row");
    DeviceGuard g(ctx->device);
    const size_t bytes = (size_t)width * height * sizeof(float);
    for (int i = 0; i < 2; i++) {
        int rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[i]), &ctx->io_bytes[i], bytes);
        if (rc) return rc;
    }
    // Large planes are cut into row bands so that the upload of band i+1 and the download of band i-1 overlap the
    // layers of band i (copy engines + compute run concurrently); each band re-reads n real rows of context from its
    // neighbours, which keeps the result bit-identical to the single-pass path.
    const int n_model = model ? (int)model->layers.size() : 0;
    int nb = ctx->host_bands > 0 ? ctx->host_bands : std::min(4, height / 512);
    const bool literal_walk = block_splitting && ctx->walk == W2X_WALK_BLOCKS && w2x_requires_splitting(width, height);
    if (nb > 8) nb = 8;
    if (nb < 2 || literal_walk || !model || height / nb < 2 * n_model) {
        CU_CHECK(cudaMemcpy2DAsync(ctx->io_buf[0], (size_t)width * 4, in, in_stride_bytes, (size_t)width * 4, (size_t)height,
                                   cudaMemcpyHostToDevice, ctx->stream));
        int rc = convert_device(ctx, model, ctx->io_buf[0], width, height, (size_t)width * 4, 0, 0, ctx->io_buf[1],
                                (size_t)width * 4, block_splitting);
        if (rc) return rc;
        CU_CHECK(cudaMemcpy2DAsync(out, out_stride_bytes, ctx->io_buf[1], (size_t)width * 4, (size_t)width * 4, (size_t)height,
                                   cudaMemcpyDeviceToHost, ctx->stream));
        CU_CHECK(cudaStreamSynchronize(ctx->stream));
        return W2X_OK;
    }
    // the copy pipeline cuts the plane its own way: the reference's progress lines for this plane go out first
    emit_reference_progress(ctx, width, height, n_model, block_splitting && w2x_requires_splitting(width, height));
    LogMute mute(ctx, true);
    std::vector<int> r0((size_t)nb + 1);
    for (int i = 0; i <= nb; i++) r0[(size_t)i] = (int)((long)height * i / nb);
    for (int i = 0; i < nb; i++) {
        // upload i carries band i plus the n rows of context band i needs from band i+1, so that band i waits for ITS upload only
        const int y = i == 0 ? 0 : r0[(size_t)i] + n_model, y_end = i + 1 < nb ? r0[(size_t)i + 1] + n_model : height;
        CU_CHECK(cudaMemcpy2DAsync(ctx->io_buf[0] + (size_t)y * width, (size_t)width * 4, reinterpret_cast<const char *>(in) + (size_t)y * in_stride_bytes,
                                   in_stride_bytes, (size_t)width * 4, (size_t)(y_end - y), cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(ctx->ev_in[i], ctx->copy_in));
    }
    for (int i = 0; i < nb; i++) {
        const int y = r0[(size_t)i], rows = r0[(size_t)i + 1] - y;
        CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[i], 0));
        const int above = i > 0 ? n_model : 0, below = i + 1 < nb ? n_model : 0;
        int rc = convert_device(ctx, model, ctx->io_buf[0] + (size_t)y * width, width, rows, (size_t)width * 4, above, below,
                                ctx->io_buf[1] + (size_t)y * width, (size_t)width * 4, 0);
        if (rc) {   // uploads / downloads already queued still touch the caller's buffers and the staging: drain them first
            cudaStreamSynchronize(ctx->copy_in);
            cudaStreamSynchronize(ctx->stream);
            cudaStreamSynchronize(ctx->copy_out);
            return rc;
        }
        CU_CHECK(cudaEventRecord(ctx->ev_done[i], ctx->stream));
        CU_CHECK(cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[i], 0));
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(out) + (size_t)y * out_stride_bytes, out_stride_bytes, ctx->io_buf[1] + (size_t)y * width,
                                   (size_t)width * 4, (size_t)width * 4, (size_t)rows, cudaMemcpyDeviceToHost, ctx->copy_out));
    }
    CU_CHECK(cudaStreamSynchronize(ctx->copy_out));
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}

int w2x_filter_layer_device(w2x_ctx *ctx, const w2x_model *model, int layer, const float *d_in, float *d_out, int width,
                            int height) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || layer < 0 || layer >= (int)model->layers.size() || !d_in || !d_out || width < 1 || height < 1)
        return fail(W2X_ERR_ARG, "w2x_filter_layer: bad argument");
    DeviceGuard g(ctx->device);
    DevModel *dm = nullptr;
    int rc = get_dev_model(ctx, model, &dm);
    if (rc) return rc;
    const Layer &L = model->layers[(size_t)layer];
    int engine = ctx->engine == W2X_ENGINE_AUTO ? W2X_ENGINE_FP32 : ctx->engine;
    if (engine == W2X_ENGINE_TC) {
        if (!tc::layer_supported(L.n_in, L.n_out))
            return fail(W2X_ERR_UNSUPPORTED, "tensor-core engine does not support a %d->%d layer", L.n_in, L.n_out);
        rc = ensure_tc(ctx);
        if (rc) return rc;
        // Model::filter semantics (same size, BORDER_REPLICATE): stage a frame with a replicated ring
        // of one pixel, run the same-size tensor-core layer on it, return the interior.
        const int pw = width + 2, ph = height + 2;
        rc = ensure(&ctx->buf[0], &ctx->buf_bytes[0], tc::act_bytes(L.n_in, pw, ph));
        if (rc) return rc;
        rc = ensure(&ctx->buf[1], &ctx->buf_bytes[1], tc::act_bytes(L.n_out, pw, ph));
        if (rc) return rc;
        __half *fin = static_cast<__half *>(ctx->buf[0]), *fout = static_cast<__half *>(ctx->buf[1]);
        const int f8 = ctx->precision == W2X_PRECISION_F16_F8X2 ? 1 : 0;
        CU_CHECK(tc::launch_planar_to_nhwc(d_in, L.n_in, width, height, fin, ctx->stream, f8));
        rc = launch_layer_tc(ctx, model, dm, layer, fin, fout, pw, ph, false, false);
        if (rc) return rc;
        CU_CHECK(tc::launch_nhwc_to_planar(fout, L.n_out, width, height, d_out, ctx->stream, f8));
        ctx->launches += 2;
        return W2X_OK;
    }
    {
        LayerTimer t(ctx, layer);
        CU_CHECK(launch_conv3x3_fp32(d_in, d_out, dm->w[(size_t)layer], dm->b[(size_t)layer], L.n_in, L.n_out, width, height,
                                     ctx->stream));
    }
    note_kernel(ctx, layer, "fp32_direct");
    ctx->launches++;
    return W2X_OK;
}

int w2x_filter_layer(w2x_ctx *ctx, const w2x_model *model, int layer, const float *const *in_planes, int n_in_planes,
                     float *const *out_planes, int n_out_planes, int width, int height, size_t in_stride_bytes,
                     size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || layer < 0 || layer >= (int)model->layers.size() || !in_planes || !out_planes || width < 1 || height < 1)
        return fail(W2X_ERR_ARG, "w2x_filter_layer: bad argument");
    const Layer &L = model->layers[(size_t)layer];
    if (n_in_planes != L.n_in)   // src/modelHandler.cpp:29-35
        return fail(W2X_ERR_ARG, "Error : Model-filter : \nnumber of input planes mismatch.\n%d,%d", n_in_planes, L.n_in);
    if (n_out_planes != L.n_out)
        return fail(W2X_ERR_ARG, "w2x_filter_layer: %d output planes supplied, layer produces %d", n_out_planes, L.n_out);
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4)
        return fail(W2X_ERR_ARG, "w2x_filter_layer: row stride smaller than a row");
    DeviceGuard g(ctx->device);
    const size_t plane = (size_t)width * height * sizeof(float);
    int rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[0]), &ctx->io_bytes[0], plane * (size_t)L.n_in);
    if (rc) return rc;
    rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[1]), &ctx->io_bytes[1], plane * (size_t)L.n_out);
    if (rc) return rc;
    for (int i = 0; i < L.n_in; i++) {
        if (!in_planes[i]) return fail(W2X_ERR_ARG, "w2x_filter_layer: NULL input plane %d", i);
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(ctx->io_buf[0]) + plane * (size_t)i, (size_t)width * 4, in_planes[i],
                                   in_stride_bytes, (size_t)width * 4, (size_t)height, cudaMemcpyHostToDevice, ctx->stream));
    }
    rc = w2x_filter_layer_device(ctx, model, layer, ctx->io_buf[0], ctx->io_buf[1], width, height);
    if (rc) return rc;
    for (int i = 0; i < L.n_out; i++) {
        if (!out_planes[i]) return fail(W2X_ERR_ARG, "w2x_filter_layer: NULL output plane %d", i);
        CU_CHECK(cudaMemcpy2DAsync(out_planes[i], out_stride_bytes, reinterpret_cast<char *>(ctx->io_buf[1]) + plane * (size_t)i,
                                   (size_t)width * 4, (size_t)width * 4, (size_t)height, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}

// Page-locked host memory for planes: copies from / to it are truly asynchronous and run at the link rate (the reference's
// cv::Mat data is pageable; host/w2xc.hpp's Plane allocates through this).  Falls back to malloc without a device.
void *w2x_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (bytes == 0) bytes = 1;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) == cudaSuccess) return p;
    cudaGetLastError();
    return nullptr;
}
void w2x_host_free(void *p) {
    if (p && cudaFreeHost(p) != cudaSuccess) cudaGetLastError();
}

int w2x_ctx_launch_count(const w2x_ctx *ctx, uint64_t *n_launches) {
    if (!ctx || !n_launches) return fail(W2X_ERR_ARG, "w2x_ctx_launch_count: NULL argument");
    *n_launches = ctx->launches;
    return W2X_OK;
}

int w2x_ctx_set_timing(w2x_ctx *ctx, int enabled) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    ctx->timing = enabled != 0;
    return W2X_OK;
}

int w2x_ctx_layer_times(w2x_ctx *ctx, int max_layers, float *ms, int *launches, int *n_layers_out, int reset) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (max_layers < 0 || (max_layers > 0 && (!ms || !launches))) return fail(W2X_ERR_ARG, "w2x_ctx_layer_times: bad argument");
    DeviceGuard g(ctx->device);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < max_layers; i++) { ms[i] = 0.f; launches[i] = 0; }
    int top = 0;
    for (auto &s : ctx->spans) {
        float t = 0.f;
        cudaEventElapsedTime(&t, s.e0, s.e1);
        if (s.layer >= 0 && s.layer < max_layers) { ms[s.layer] += t; launches[s.layer]++; }
        top = std::max(top, s.layer + 1);
    }
    if (n_layers_out) *n_layers_out = top;
    if (reset) {
        for (auto &s : ctx->spans) { ctx->event_pool.push_back(s.e0); ctx->event_pool.push_back(s.e1); }
        ctx->spans.clear();
    }
    return W2X_OK;
}

const char *w2x_ctx_layer_kernel_name(const w2x_ctx *ctx, int layer) {
    if (!ctx || layer < 0 || layer >= (int)ctx->layer_kernel.size()) return "";
    return ctx->layer_kernel[(size_t)layer].c_str();
}

}  // extern "C"

// ---- packed frames: independent planes side by side, every layer one launch per frame ----------------------------------------
namespace {
// Whether a conversion packs planes into frames: the tensor-core engine with the fused last layer (the gather writes each plane's
// interior).  Every other case converts plane by plane.
bool packs_frames(const w2x_ctx *ctx, const w2x_model *m, const DevModel *dm, int engine) {
    return engine == W2X_ENGINE_TC && ctx->fuse_last && m->layers.size() >= 3 && !dm->last_w_t.empty();
}

struct FramePlan {                  // one packed frame: its size and its planes (any order; upload_frames sorts them)
    int fw = 0, fh = 0;
    std::vector<tc::PlaneRect> rect;
};
struct FrameDev {                   // the same frame with its table in ctx->plan_buf
    int fw, fh, n_rect, n_shelf, n_blocks;
    const tc::PlaneRect *rect;
    const int *shelf_y0, *shelf_first;
};

// Puts each frame's rectangles in shelf order, numbers their gather blocks and uploads all tables in ONE copy on the context's
// stream.  The copy waits for the kernels of an earlier call that still read the buffer (plan_ev), and its source is pageable
// memory, so it is staged before cudaMemcpyAsync returns and the host vectors may go at once.
int upload_frames(w2x_ctx *ctx, std::vector<FramePlan> &frames, std::vector<FrameDev> *out) {
    auto align = [](size_t b) { return (b + 15) & ~(size_t)15; };
    std::vector<char> blob;
    std::vector<size_t> off_rect, off_shelf;
    out->assign(frames.size(), FrameDev{});
    for (size_t f = 0; f < frames.size(); f++) {
        auto &R = frames[f].rect;
        std::sort(R.begin(), R.end(), [](const tc::PlaneRect &a, const tc::PlaneRect &b) { return a.y0 != b.y0 ? a.y0 < b.y0 : a.x0 < b.x0; });
        std::vector<int> sy, sf;
        int blk = 0;
        for (size_t i = 0; i < R.size(); i++) {
            if (i == 0 || R[i].y0 != R[i - 1].y0) {
                sy.push_back(R[i].y0);
                sf.push_back((int)i);
            }
            R[i].blk0 = blk;
            blk += ((R[i].w + 31) / 32) * ((R[i].h + 7) / 8);
        }
        sf.push_back((int)R.size());
        FrameDev &d = (*out)[f];
        d.fw = frames[f].fw;
        d.fh = frames[f].fh;
        d.n_rect = (int)R.size();
        d.n_shelf = (int)sy.size();
        d.n_blocks = blk;
        off_rect.push_back(align(blob.size()));
        blob.resize(off_rect.back() + R.size() * sizeof(tc::PlaneRect));
        std::memcpy(blob.data() + off_rect.back(), R.data(), R.size() * sizeof(tc::PlaneRect));
        off_shelf.push_back(align(blob.size()));
        blob.resize(off_shelf.back() + (sy.size() + sf.size()) * sizeof(int));
        std::memcpy(blob.data() + off_shelf.back(), sy.data(), sy.size() * sizeof(int));
        std::memcpy(blob.data() + off_shelf.back() + sy.size() * sizeof(int), sf.data(), sf.size() * sizeof(int));
    }
    if (ctx->plan_ev_live) CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->plan_ev, 0));
    int rc = ensure(&ctx->plan_buf, &ctx->plan_bytes, blob.size());
    if (rc) return rc;
    CU_CHECK(cudaMemcpyAsync(ctx->plan_buf, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
    const char *base = static_cast<const char *>(ctx->plan_buf);
    for (size_t f = 0; f < frames.size(); f++) {
        FrameDev &d = (*out)[f];
        d.rect = reinterpret_cast<const tc::PlaneRect *>(base + off_rect[f]);
        d.shelf_y0 = reinterpret_cast<const int *>(base + off_shelf[f]);
        d.shelf_first = d.shelf_y0 + d.n_shelf;
    }
    return W2X_OK;
}

// Sizes the scratch for the largest frame once, so that no buffer is reallocated between frames.
int reserve_frames(w2x_ctx *ctx, const w2x_model *m, const std::vector<FrameDev> &frames) {
    size_t px = 0;
    for (auto &f : frames) px = std::max(px, (size_t)f.fw * f.fh);
    int rc = ensure(reinterpret_cast<void **>(&ctx->pad_buf), &ctx->pad_bytes, px * sizeof(float));
    for (int i = 0; i < 2 && !rc; i++) rc = ensure(&ctx->buf[i], &ctx->buf_bytes[i], px * (size_t)max_channels(m) * 4);
    return rc;
}

// One packed frame: the pack, the layers on the whole frame, the gather -- n + 1 launches whatever the number of planes.
int run_packed_frame(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, const FrameDev &f) {
    const int n = (int)m->layers.size();
    int rc = ensure(reinterpret_cast<void **>(&ctx->pad_buf), &ctx->pad_bytes, (size_t)f.fw * f.fh * sizeof(float));
    if (rc) return rc;
    CU_CHECK(tc::launch_pack_planes(f.rect, f.shelf_y0, f.shelf_first, f.n_shelf, n, f.fw, f.fh, ctx->pad_buf, ctx->stream));
    ctx->launches++;
    const PackedGather g{f.rect, f.n_rect, f.n_blocks};
    return run_basic(ctx, m, dm, W2X_ENGINE_TC, ctx->pad_buf, f.fw, f.fw, f.fh, nullptr, 0, &g);
}

int run_packed_frames(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, std::vector<FramePlan> &frames) {
    std::vector<FrameDev> fd;
    int rc = upload_frames(ctx, frames, &fd);
    if (!rc) rc = reserve_frames(ctx, m, fd);
    for (size_t f = 0; f < fd.size() && !rc; f++) rc = run_packed_frame(ctx, m, dm, fd[f]);
    if (rc) return rc;
    CU_CHECK(cudaEventRecord(ctx->plan_ev, ctx->stream));
    ctx->plan_ev_live = true;
    return W2X_OK;
}

// ---- independent planes of one shape, one pass (the reference's block loop, src/convertRoutine.cpp:114-165) ------------------
int convert_tiles_dev(w2x_ctx *ctx, const w2x_model *m, const float *d_in, float *d_out, int n_tiles, int w, int h) {
    if (!m || !d_in || !d_out || n_tiles < 1 || w < 1 || h < 1) return fail(W2X_ERR_ARG, "w2x_convert_tiles: bad argument");
    if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1) return fail(W2X_ERR_ARG, "w2x_convert_tiles: model must map 1 plane to 1 plane");
    DeviceGuard g(ctx->device);
    const int engine = pick_engine(ctx, m);
    if (engine < 0) return W2X_ERR_UNSUPPORTED;
    DevModel *dm = nullptr;
    int rc = get_dev_model(ctx, m, &dm);
    if (rc) return rc;
    const int n = (int)m->layers.size();
    const int pw = w + 2 * n, ph = h + 2 * n;
    if (packs_frames(ctx, m, dm, engine)) {
        // tiles per frame: what the scratch limit (one frame of maxc channels, 4 bytes per element) and MAX_FRAME_ROWS allow; the
        // tiles of a frame are stacked vertically, each padded like cv::copyMakeBorder (src/convertRoutine.cpp:35) by the pack
        const size_t per_tile = (size_t)max_channels(m) * pw * ph * 4;
        const size_t fit = std::min(ctx->scratch_limit / per_tile, (size_t)(MAX_FRAME_ROWS / ph));
        const int group = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_tiles, fit));
        std::vector<FramePlan> frames;
        for (int t0 = 0; t0 < n_tiles; t0 += group) {
            FramePlan f;
            f.fw = pw;
            f.fh = std::min(group, n_tiles - t0) * ph;
            for (int t = 0; t0 + t < n_tiles && t < group; t++) {
                const size_t off = (size_t)(t0 + t) * w * h;
                f.rect.push_back(tc::PlaneRect{d_in + off, d_out + off, w, w, w, h, 0, t * ph, 0});
            }
            frames.push_back(std::move(f));
        }
        return run_packed_frames(ctx, m, dm, frames);
    }
    rc = ensure(reinterpret_cast<void **>(&ctx->pad_buf), &ctx->pad_bytes, (size_t)pw * ph * sizeof(float));
    if (rc) return rc;
    for (int t = 0; t < n_tiles; t++) {   // cv::copyMakeBorder per tile (src/convertRoutine.cpp:35)
        CU_CHECK(launch_pad_replicate(d_in + (size_t)t * w * h, w, h, w, n, 0, 0, ctx->pad_buf, ctx->stream));
        ctx->launches++;
        rc = run_basic(ctx, m, dm, engine, ctx->pad_buf, pw, pw, ph, d_out + (size_t)t * w * h, w);
        if (rc) return rc;
    }
    return W2X_OK;
}

// ---- independent planes of any sizes (w2x_convert_planes*) ------------------------------------------------------------------
int check_planes(const char *fn, const w2x_model *m, int n_planes, const float *const *in, const int *widths, const int *heights,
                 const size_t *in_strides, float *const *out, const size_t *out_strides) {
    if (!m) return fail(W2X_ERR_ARG, "%s: NULL model", fn);
    if (n_planes < 1) return fail(W2X_ERR_ARG, "%s: n_planes is %d, at least 1 plane is needed", fn, n_planes);
    if (!in || !widths || !heights || !in_strides || !out || !out_strides) return fail(W2X_ERR_ARG, "%s: NULL array argument", fn);
    for (int i = 0; i < n_planes; i++) {
        if (!in[i] || !out[i]) return fail(W2X_ERR_ARG, "%s: plane %d: NULL %s pointer", fn, i, in[i] ? "output" : "input");
        if (widths[i] < 1 || heights[i] < 1) return fail(W2X_ERR_ARG, "%s: plane %d: size %d x %d", fn, i, widths[i], heights[i]);
        if (in_strides[i] % 4 || out_strides[i] % 4 || in_strides[i] < (size_t)widths[i] * 4 || out_strides[i] < (size_t)widths[i] * 4)
            return fail(W2X_ERR_ARG, "%s: plane %d: row strides must be multiples of 4 bytes and >= width*4", fn, i);
    }
    if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1) return fail(W2X_ERR_ARG, "%s: model must map 1 plane to 1 plane", fn);
    return W2X_OK;
}

// The progress lines of the whole call, plane by plane in order, as the single-plane entry point (w2x_convert_plane with
// host = true, else w2x_convert_plane_device) would log them with block_splitting = 0: one "Iteration #k..." per layer, per
// scratch band of a plane too large to pack (the host entry point's copy pipeline logs a plane it cuts once).
void emit_planes_progress(w2x_ctx *ctx, const w2x_model *m, int n_planes, const int *widths, const int *heights, const int *frame, bool host) {
    if (!ctx->log || ctx->log_muted) return;
    const int n = (int)m->layers.size();
    for (int i = 0; i < n_planes; i++) {
        int passes = 1;
        if (frame[i] < 0) {
            const int h = heights[i];
            const int nb = std::min(8, ctx->host_bands > 0 ? ctx->host_bands : std::min(4, h / 512));
            if (!(host && nb >= 2 && h / nb >= 2 * n)) {
                const int band = scratch_band_rows(ctx, m, widths[i], h);
                passes = (h + band - 1) / band;
            }
        }
        for (int p = 0; p < passes; p++)
            for (int k = 1; k <= n; k++) logf(ctx, "Iteration #%d...", k);
    }
}

struct PlanesPlan {
    std::vector<int> frame, x0, y0, fw, fh;
    int n_frames = 0;
};
void plan_for(const w2x_ctx *ctx, const w2x_model *m, int n_planes, const int *widths, const int *heights, PlanesPlan *p) {
    p->frame.resize((size_t)n_planes);
    p->x0.resize((size_t)n_planes);
    p->y0.resize((size_t)n_planes);
    p->n_frames = plan_planes(n_planes, widths, heights, (int)m->layers.size(), max_channels(m), ctx->scratch_limit, p->frame.data(),
                              p->x0.data(), p->y0.data(), &p->fw, &p->fh);
}
std::vector<FramePlan> frames_for(const PlanesPlan &p) {
    std::vector<FramePlan> frames((size_t)p.n_frames);
    for (int f = 0; f < p.n_frames; f++) {
        frames[(size_t)f].fw = p.fw[(size_t)f];
        frames[(size_t)f].fh = p.fh[(size_t)f];
    }
    return frames;
}

int convert_planes_dev(w2x_ctx *ctx, const w2x_model *m, int n_planes, const float *const *d_in, const int *widths, const int *heights,
                       const size_t *in_strides, float *const *d_out, const size_t *out_strides) {
    int rc = check_planes("w2x_convert_planes_device", m, n_planes, d_in, widths, heights, in_strides, d_out, out_strides);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    const int engine = pick_engine(ctx, m);
    if (engine < 0) return W2X_ERR_UNSUPPORTED;
    DevModel *dm = nullptr;
    rc = get_dev_model(ctx, m, &dm);
    if (rc) return rc;
    if (!packs_frames(ctx, m, dm, engine)) {
        for (int i = 0; i < n_planes && !rc; i++)
            rc = convert_device(ctx, m, d_in[i], widths[i], heights[i], in_strides[i], 0, 0, d_out[i], out_strides[i], 0);
        return rc;
    }
    PlanesPlan p;
    plan_for(ctx, m, n_planes, widths, heights, &p);
    emit_planes_progress(ctx, m, n_planes, widths, heights, p.frame.data(), false);
    LogMute mute(ctx, true);
    std::vector<FramePlan> frames = frames_for(p);
    for (int i = 0; i < n_planes; i++)
        if (p.frame[(size_t)i] >= 0)
            frames[(size_t)p.frame[(size_t)i]].rect.push_back(tc::PlaneRect{d_in[i], d_out[i], (long)(in_strides[i] / 4), (long)(out_strides[i] / 4),
                                                                            widths[i], heights[i], p.x0[(size_t)i], p.y0[(size_t)i], 0});
    if (!frames.empty()) rc = run_packed_frames(ctx, m, dm, frames);
    for (int i = 0; i < n_planes && !rc; i++)   // too large to pack: the single-plane path, which fills the GPU by itself
        if (p.frame[(size_t)i] < 0)
            rc = convert_device(ctx, m, d_in[i], widths[i], heights[i], in_strides[i], 0, 0, d_out[i], out_strides[i], 0);
    return rc;
}

// Host planes, packed: dense device staging (plane i at the same offset in io_buf[0] and io_buf[1]); the uploads of later frames
// and the downloads of earlier ones overlap the layers of the current one, as in w2x_convert_tiles.  A group is a frame or one
// plane too large to pack.  Up to 8 uploads are queued ahead (ev_in / ev_done are 8 deep).
int planes_host_pipeline(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int n_planes, const float *const *in, const int *widths,
                         const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides) {
    PlanesPlan p;
    plan_for(ctx, m, n_planes, widths, heights, &p);
    emit_planes_progress(ctx, m, n_planes, widths, heights, p.frame.data(), true);
    LogMute mute(ctx, true);
    std::vector<size_t> off((size_t)n_planes + 1, 0);
    for (int i = 0; i < n_planes; i++) off[(size_t)i + 1] = off[(size_t)i] + (size_t)widths[i] * heights[i];
    for (int i = 0; i < 2; i++) {
        int rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[i]), &ctx->io_bytes[i], off.back() * sizeof(float));
        if (rc) return rc;
    }
    std::vector<FramePlan> frames = frames_for(p);
    std::vector<std::vector<int>> groups(frames.size());
    for (int i = 0; i < n_planes; i++) {
        const int f = p.frame[(size_t)i];
        if (f < 0) continue;
        frames[(size_t)f].rect.push_back(tc::PlaneRect{ctx->io_buf[0] + off[(size_t)i], ctx->io_buf[1] + off[(size_t)i], widths[i], widths[i],
                                                       widths[i], heights[i], p.x0[(size_t)i], p.y0[(size_t)i], 0});
        groups[(size_t)f].push_back(i);
    }
    for (int i = 0; i < n_planes; i++)
        if (p.frame[(size_t)i] < 0) groups.push_back({i});
    std::vector<FrameDev> fd;
    int rc = 0;
    if (!frames.empty()) {
        rc = upload_frames(ctx, frames, &fd);
        if (!rc) rc = reserve_frames(ctx, m, fd);
        if (rc) return rc;
    }
    const int n_groups = (int)groups.size();
    auto upload = [&](int gi) -> int {
        for (int i : groups[(size_t)gi])
            CU_CHECK(cudaMemcpy2DAsync(ctx->io_buf[0] + off[(size_t)i], (size_t)widths[i] * 4, in[i], in_strides[i], (size_t)widths[i] * 4,
                                       (size_t)heights[i], cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(ctx->ev_in[gi % 8], ctx->copy_in));
        return W2X_OK;
    };
    for (int gi = 0; gi < std::min(8, n_groups) && !rc; gi++) rc = upload(gi);
    for (int gi = 0; gi < n_groups && !rc; gi++) {
        CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[gi % 8], 0));
        if (gi < (int)fd.size()) {
            rc = run_packed_frame(ctx, m, dm, fd[(size_t)gi]);
        } else {
            const int i = groups[(size_t)gi][0];
            rc = convert_device(ctx, m, ctx->io_buf[0] + off[(size_t)i], widths[i], heights[i], (size_t)widths[i] * 4, 0, 0,
                                ctx->io_buf[1] + off[(size_t)i], (size_t)widths[i] * 4, 0);
        }
        if (rc) break;
        if (gi + 1 == (int)fd.size()) {   // the last kernel reading the frame tables is queued
            CU_CHECK(cudaEventRecord(ctx->plan_ev, ctx->stream));
            ctx->plan_ev_live = true;
        }
        CU_CHECK(cudaEventRecord(ctx->ev_done[gi % 8], ctx->stream));
        CU_CHECK(cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[gi % 8], 0));
        for (int i : groups[(size_t)gi])
            CU_CHECK(cudaMemcpy2DAsync(out[i], out_strides[i], ctx->io_buf[1] + off[(size_t)i], (size_t)widths[i] * 4, (size_t)widths[i] * 4,
                                       (size_t)heights[i], cudaMemcpyDeviceToHost, ctx->copy_out));
        if (gi + 8 < n_groups) rc = upload(gi + 8);   // its event's previous record has been waited for above
    }
    if (rc) return rc;
    CU_CHECK(cudaStreamSynchronize(ctx->copy_out));
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}
}  // namespace

namespace w2x {
namespace eng {
// phase 1: uploads + the batched pass (results stay in the context's staging buffer); phase 2: downloads.  Split so that a
// multi-GPU driver can queue phase 1 everywhere before a download into pageable memory blocks its thread.
int tiles_enqueue_compute(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, int n_tiles, int width, int height, size_t in_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!in_tiles || n_tiles < 1 || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_convert_tiles: bad argument");
    if (in_stride_bytes < (size_t)width * 4) return fail(W2X_ERR_ARG, "w2x_convert_tiles: row stride smaller than a row");
    DeviceGuard g(ctx->device);
    const size_t tile_bytes = (size_t)width * height * sizeof(float);
    for (int i = 0; i < 2; i++) {
        int rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[i]), &ctx->io_bytes[i], tile_bytes * (size_t)n_tiles);
        if (rc) return rc;
    }
    for (int t = 0; t < n_tiles; t++) {
        if (!in_tiles[t]) return fail(W2X_ERR_ARG, "w2x_convert_tiles: NULL tile %d", t);
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(ctx->io_buf[0]) + tile_bytes * (size_t)t, (size_t)width * 4, in_tiles[t], in_stride_bytes,
                                   (size_t)width * 4, (size_t)height, cudaMemcpyHostToDevice, ctx->stream));
    }
    return convert_tiles_dev(ctx, model, ctx->io_buf[0], ctx->io_buf[1], n_tiles, width, height);
}

int tiles_enqueue_download(w2x_ctx *ctx, float *const *out_tiles, int n_tiles, int width, int height, size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!out_tiles || out_stride_bytes < (size_t)width * 4) return fail(W2X_ERR_ARG, "w2x_convert_tiles: bad output argument");
    DeviceGuard g(ctx->device);
    const size_t tile_bytes = (size_t)width * height * sizeof(float);
    for (int t = 0; t < n_tiles; t++) {
        if (!out_tiles[t]) return fail(W2X_ERR_ARG, "w2x_convert_tiles: NULL tile %d", t);
        CU_CHECK(cudaMemcpy2DAsync(out_tiles[t], out_stride_bytes, reinterpret_cast<char *>(ctx->io_buf[1]) + tile_bytes * (size_t)t, (size_t)width * 4,
                                   (size_t)width * 4, (size_t)height, cudaMemcpyDeviceToHost, ctx->stream));
    }
    return W2X_OK;
}
}  // namespace eng
}  // namespace w2x

extern "C" {

int w2x_convert_tiles_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, float *d_out, int n_tiles, int width, int height) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    return convert_tiles_dev(ctx, model, d_in, d_out, n_tiles, width, height);
}

int w2x_convert_tiles_async(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles,
                            int width, int height, size_t in_stride_bytes, size_t out_stride_bytes) {
    int rc = tiles_enqueue_compute(ctx, model, in_tiles, n_tiles, width, height, in_stride_bytes);
    if (rc) return rc;
    return tiles_enqueue_download(ctx, out_tiles, n_tiles, width, height, out_stride_bytes);
}

int w2x_convert_tiles(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles,
                      int width, int height, size_t in_stride_bytes, size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    // Larger batches run as up to four groups: the uploads of group g+1 and the downloads of group g-1 overlap the layers of
    // group g (copy engines + compute), as the row bands of w2x_convert_plane do.  Tiles are independent, so the grouping
    // does not change a bit of any of them.
    const int groups = n_tiles >= 8 ? std::min(4, n_tiles / 4) : 1;
    if (groups < 2) {
        int rc = w2x_convert_tiles_async(ctx, model, in_tiles, out_tiles, n_tiles, width, height, in_stride_bytes, out_stride_bytes);
        int rc2 = w2x_ctx_synchronize(ctx);
        return rc ? rc : rc2;
    }
    if (!in_tiles || !out_tiles || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_convert_tiles: bad argument");
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_tiles: row stride smaller than a row");
    for (int t = 0; t < n_tiles; t++)
        if (!in_tiles[t] || !out_tiles[t]) return fail(W2X_ERR_ARG, "w2x_convert_tiles: NULL tile %d", t);
    DeviceGuard g(ctx->device);
    const size_t tile_px = (size_t)width * height, tile_bytes = tile_px * sizeof(float);
    for (int i = 0; i < 2; i++) {
        int rc = ensure(reinterpret_cast<void **>(&ctx->io_buf[i]), &ctx->io_bytes[i], tile_bytes * (size_t)n_tiles);
        if (rc) return rc;
    }
    auto first = [&](int gi) { return (int)((long)n_tiles * gi / groups); };
    for (int gi = 0; gi < groups; gi++) {
        for (int t = first(gi); t < first(gi + 1); t++)
            CU_CHECK(cudaMemcpy2DAsync(ctx->io_buf[0] + tile_px * (size_t)t, (size_t)width * 4, in_tiles[t], in_stride_bytes, (size_t)width * 4,
                                       (size_t)height, cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(ctx->ev_in[gi], ctx->copy_in));
    }
    for (int gi = 0; gi < groups; gi++) {
        const int t0 = first(gi), nt = first(gi + 1) - t0;
        CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[gi], 0));
        int rc = convert_tiles_dev(ctx, model, ctx->io_buf[0] + tile_px * (size_t)t0, ctx->io_buf[1] + tile_px * (size_t)t0, nt, width, height);
        if (rc) {   // copies already queued still touch the caller's buffers and the staging: drain them first
            cudaStreamSynchronize(ctx->copy_in);
            cudaStreamSynchronize(ctx->stream);
            cudaStreamSynchronize(ctx->copy_out);
            return rc;
        }
        CU_CHECK(cudaEventRecord(ctx->ev_done[gi], ctx->stream));
        CU_CHECK(cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[gi], 0));
        for (int t = t0; t < t0 + nt; t++)
            CU_CHECK(cudaMemcpy2DAsync(out_tiles[t], out_stride_bytes, ctx->io_buf[1] + tile_px * (size_t)t, (size_t)width * 4, (size_t)width * 4,
                                       (size_t)height, cudaMemcpyDeviceToHost, ctx->copy_out));
    }
    CU_CHECK(cudaStreamSynchronize(ctx->copy_out));
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}

int w2x_convert_planes_device(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *d_in, const int *widths,
                              const int *heights, const size_t *in_strides, float *const *d_out, const size_t *out_strides) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    return convert_planes_dev(ctx, model, n_planes, d_in, widths, heights, in_strides, d_out, out_strides);
}

int w2x_convert_planes(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *in, const int *widths,
                       const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    int rc = check_planes("w2x_convert_planes", model, n_planes, in, widths, heights, in_strides, out, out_strides);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    const int engine = pick_engine(ctx, model);
    if (engine < 0) return W2X_ERR_UNSUPPORTED;
    DevModel *dm = nullptr;
    rc = get_dev_model(ctx, model, &dm);
    if (rc) return rc;
    if (!packs_frames(ctx, model, dm, engine)) {
        for (int i = 0; i < n_planes && !rc; i++)
            rc = w2x_convert_plane(ctx, model, in[i], widths[i], heights[i], in_strides[i], out[i], out_strides[i], 0);
        return rc;
    }
    rc = planes_host_pipeline(ctx, model, dm, n_planes, in, widths, heights, in_strides, out, out_strides);
    if (rc) {   // copies already queued still touch the caller's buffers and the staging: drain them first
        cudaStreamSynchronize(ctx->copy_in);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->copy_out);
    }
    return rc;
}

}  // extern "C"
