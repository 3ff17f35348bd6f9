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
#include <climits>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "engine_internal.h"

using namespace w2x;

namespace w2x {
namespace eng {

int max_channels(const w2x_model *m) {
    int maxc = 1;
    for (auto &L : m->layers) maxc = std::max(maxc, std::max(L.n_in, L.n_out));
    return maxc;
}

// The two staging buffers of a host-buffer entry point: its inputs in io_buf[0], its outputs in io_buf[1].
int reserve_io(w2x_ctx *ctx, size_t in_bytes, size_t out_bytes) {
    int rc = ctx->io_buf[0].reserve(in_bytes);
    return rc ? rc : ctx->io_buf[1].reserve(out_bytes);
}

int get_dev_model(w2x_ctx *ctx, const w2x_model *m, DevModel **out) {
    auto it = ctx->models.find(m->uid);
    if (it != ctx->models.end()) {
        *out = &it->second;
        return W2X_OK;
    }
    DevModel dm;
    const size_t n = m->layers.size();
    dm.w.resize(n);
    dm.b.resize(n);
    dm.pack.resize(n);
    dm.pack8.resize(n);
    dm.pack_bf16.resize(n);
    dm.out_scale.assign(n, 1.f);
    for (size_t i = 0; i < n; i++) {
        const Layer &L = m->layers[i];
        CU_CHECK(dm.w[i].grow(L.w.size() * sizeof(float)));
        CU_CHECK(cudaMemcpyAsync(dm.w[i].get(), L.w.data(), L.w.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        std::vector<float> bf(L.b.size());
        for (size_t k = 0; k < bf.size(); k++) bf[k] = static_cast<float>(L.b[k]);
        dm.b_host.push_back(bf);
        CU_CHECK(dm.b[i].grow(bf.size() * sizeof(float)));
        CU_CHECK(cudaMemcpyAsync(dm.b[i].get(), bf.data(), bf.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        CU_CHECK(cudaStreamSynchronize(ctx->stream));   // bf goes out of scope
        const TcPack &P = m->tc[i];
        if (!P.bytes.empty()) {
            CU_CHECK(dm.pack[i].grow(P.bytes.size() * 2));
            CU_CHECK(cudaMemcpyAsync(dm.pack[i].get(), P.bytes.data(), P.bytes.size() * 2, cudaMemcpyHostToDevice, ctx->stream));
            dm.out_scale[i] = 1.0f / (P.wscale * tc::ACT_SCALE);
            CU_CHECK(dm.pack8[i].grow(P.bytes8.size()));
            CU_CHECK(cudaMemcpyAsync(dm.pack8[i].get(), P.bytes8.data(), P.bytes8.size(), cudaMemcpyHostToDevice, ctx->stream));
        }
    }
    if (m->tc_eligible || m->tc_eligible_bf16) {
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

int upload_pack_bf16(w2x_ctx *ctx, const w2x_model *m, DevModel *dm) {
    for (size_t i = 0; i < m->layers.size(); i++) {
        const std::vector<uint16_t> &v = m->tc[i].bytes_bf16;
        if (v.empty() || dm->pack_bf16[i].get()) continue;
        CU_CHECK(dm->pack_bf16[i].grow(v.size() * 2));
        CU_CHECK(cudaMemcpyAsync(dm->pack_bf16[i].get(), v.data(), v.size() * 2, cudaMemcpyHostToDevice, ctx->stream));
    }
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
    char line[128];
    snprintf(line, sizeof line, fmt, a, b);
    ctx->log(line, ctx->log_user);
}

// The reference's blocks of a w x h plane for an n-layer model, 8 ints each (block_table); empty when the block size is too small.
std::vector<int> blocks_of(int w, int h, int n) {
    const Config &cfg = config();
    const int nb = block_table(w, h, cfg.block_w, cfg.block_h, n, nullptr, 0, nullptr, nullptr);
    std::vector<int> tab((size_t)std::max(nb, 0) * 8);
    if (nb > 0) block_table(w, h, cfg.block_w, cfg.block_h, n, tab.data(), nb, nullptr, nullptr);
    return tab;
}

// The progress lines the reference prints for one convertWithModels call (src/convertRoutine.cpp:67,133-134): per block
// "start process block (c,r) ..." + one "Iteration #k..." per layer when the plane is split, else just the iterations.
void emit_reference_progress(w2x_ctx *ctx, int w, int h, int n_layers, bool split) {
    if (!ctx->log) return;
    const std::vector<int> tab = split ? blocks_of(w, h, n_layers) : std::vector<int>(8);   // unsplit: one block without a line
    for (size_t i = 0; i < tab.size(); i += 8) {
        if (split) logf(ctx, "start process block (%d,%d) ...", tab[i + 1], tab[i]);
        for (int k = 1; k <= n_layers; k++) logf(ctx, "Iteration #%d...", k);
    }
}

int pick_engine(w2x_ctx *ctx, const w2x_model *m) {
    int e = ctx->engine;
    const bool ok = tc_eligible(m, ctx->precision);
    if (e == W2X_ENGINE_AUTO) e = ok ? W2X_ENGINE_TC : W2X_ENGINE_FP32;
    if (e == W2X_ENGINE_TC && !ok) {
        fail(W2X_ERR_UNSUPPORTED, ctx->precision == W2X_PRECISION_BF16X3
                                      ? "tensor-core engine needs a 1->{32,64,128}...->1 layer chain with finite inner weights"
                                      : "tensor-core engine needs a 1->{32,64,128}...->1 layer chain with finite inner weights below 65520");
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
    const tc::Rec rec = tc::rec_format(ctx->precision);
    if (rec == tc::Rec::BF16 && !dm->pack_bf16[(size_t)li].get()) {
        const int rc = upload_pack_bf16(ctx, m, dm);
        if (rc) return rc;
    }
    const void *wpack = rec == tc::Rec::F8     ? (const void *)dm->pack8[(size_t)li].get()
                        : rec == tc::Rec::BF16 ? (const void *)dm->pack_bf16[(size_t)li].get()
                                               : (const void *)dm->pack[(size_t)li].get();
    const float out_scale = rec == tc::Rec::BF16 ? 1.0f / tc::ACT_SCALE : dm->out_scale[(size_t)li];   // bf16x3 packs at wscale 1
    {
        LayerTimer t(ctx, li);
        CU_CHECK(tc::launch_tc_layer(in, wpack, dm->b_host[(size_t)li].data(), out, L.n_in, L.n_out, pw, ph, out_scale, ctx->precision,
                                     ctx->num_sms, ctx->stream,
                                     profile && ctx->prof_buf.get() ? ctx->prof_buf.get() + (size_t)li * tc::PROF_MAX_CTAS * tc::PROF_WORDS : nullptr,
                                     fused ? dm->last_w_t.data() : nullptr, fused ? reinterpret_cast<float *>(out) : nullptr, out_y0, out_rows));
    }
    static const char *const names[5][2] = {{"wgmma_f16x3", "wgmma_f16x3+last"}, {"wgmma_f16+f8x2", "wgmma_f16+f8x2+last"}, {"wgmma_f16", "wgmma_f16+last"},
                                            {nullptr, nullptr}, {"wgmma_bf16x3", "wgmma_bf16x3+last"}};
    note_kernel(ctx, li, names[ctx->precision][fused ? 1 : 0]);
    ctx->launches++;
    return W2X_OK;
}

// ---- convertWithModelsBasic on a pw x ph frame ------------------------------------------------
// src: what the first layer reads: a padded region (FrameSource::padded()), or (tensor-core engine only) an unpadded plane with the
// replicate padding folded into the loads.  The fp32 engine copies src.in / src.stride_floats, which is then always a padded region.
// dst: receives the (pw-2n) x (ph-2n) interior.
// packed (tensor-core engine with the fused last layer only): src is a packed frame of pw x ph holding many padded planes (see
// tc::PlaneRect); the layers run ONCE on it -- the seams pollute only the rings that are cropped anyway -- and one gather writes
// every plane's interior to its own destination; dst / dst_stride are then unused.
struct PackedGather { const tc::PlaneRect *rect; int n_rect, n_blocks; };
int run_basic(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, int engine, const FrameSource &src, int pw, int ph, float *dst,
              long dst_stride, const PackedGather *packed = nullptr) {
    const int n = (int)m->layers.size();
    if (pw - 2 * n < 1 || ph - 2 * n < 1) return fail(W2X_ERR_ARG, "plane smaller than the model's receptive ring");
    const int maxc = max_channels(m);
    if (engine == W2X_ENGINE_FP32) {
        const size_t need = (size_t)maxc * pw * ph * sizeof(float);
        for (int i = 0; i < 2; i++) {
            int rc = ctx->buf[i].reserve(need);
            if (rc) return rc;
        }
        float *cur = static_cast<float *>(ctx->buf[0].get()), *nxt = static_cast<float *>(ctx->buf[1].get());
        CU_CHECK(launch_copy2d(src.in, src.stride_floats, cur, pw, pw, ph, ctx->stream));   // ROI -> dense plane
        ctx->launches++;
        for (int li = 0; li < n; li++) {
            const Layer &L = m->layers[(size_t)li];
            {
                LayerTimer t(ctx, li);
                CU_CHECK(launch_conv3x3_fp32(cur, nxt, dm->w[(size_t)li].get(), dm->b[(size_t)li].get(), L.n_in, L.n_out, pw, ph,
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
    const tc::Rec rec = tc::rec_format(ctx->precision);
    int rc = ensure_tc(ctx);
    if (rc) return rc;
    const size_t need = tc::act_bytes(maxc, pw, ph);
    for (int i = 0; i < 2; i++) {
        rc = ctx->buf[i].reserve(need);
        if (rc) return rc;
    }
    __half *cur = static_cast<__half *>(ctx->buf[0].get()), *nxt = static_cast<__half *>(ctx->buf[1].get());
    {
        const Layer &L = m->layers[0];
        LayerTimer t(ctx, 0);
        CU_CHECK(tc::launch_first(src, pw, ph, L.w.data(), dm->b_host[0].data(), L.n_out, cur, ctx->stream, rec));
        note_kernel(ctx, 0, src.up2x ? "first_1xN+up2x" : "first_1xN");
        ctx->launches++;
    }
    const bool fuse = ctx->fuse_last && n >= 3 && !dm->last_w_t.empty();
    for (int li = 1; li + 1 < n; li++) {
        rc = launch_layer_tc(ctx, m, dm, li, cur, nxt, pw, ph, fuse && li == n - 2, true);
        if (rc) return rc;
        std::swap(cur, nxt);
    }
    {
        const Layer &L = m->layers[(size_t)n - 1];
        LayerTimer t(ctx, n - 1);
        if (fuse) {
            if (packed)
                CU_CHECK(tc::launch_gather_planes(reinterpret_cast<const float *>(cur), pw, packed->rect, packed->n_rect, packed->n_blocks,
                                                  static_cast<float>(L.b[0]), n, ctx->stream));
            else
                CU_CHECK(tc::launch_last_gather(reinterpret_cast<const float *>(cur), pw, ph, static_cast<float>(L.b[0]), n, n, n, dst, dst_stride,
                                                ctx->stream));
            note_kernel(ctx, n - 1, "last_gather");
        } else {
            if (packed) return fail(W2X_ERR_UNSUPPORTED, "packed frames need the fused last layer");
            CU_CHECK(tc::launch_last(cur, L.n_in, pw, ph, dm->w[(size_t)n - 1].get(), static_cast<float>(L.b[0]), n, dst,
                                     dst_stride, ctx->stream, rec));
            note_kernel(ctx, n - 1, "last_Nx1");
        }
        ctx->launches++;
    }
    return W2X_OK;
}

// rows per scratch band of convert_device for a plane w wide: the band's frame (band + 2n rows) fits the scratch limit and has at
// most MAX_FRAME_ROWS rows
int scratch_band_rows(const w2x_ctx *ctx, const w2x_model *m, int w, int h) {
    const int n = (int)m->layers.size();
    const size_t per_row = (size_t)max_channels(m) * (w + 2 * n) * 4;   // both engines: 4 bytes per activation element
    long max_rows = std::min((long)(ctx->scratch_limit / per_row), MAX_FRAME_ROWS) - 2 * n;
    if (max_rows < 16) max_rows = 16;
    return (int)std::min<long>(h, max_rows);
}

int check_ctx(w2x_ctx *ctx) {
    if (!ctx) return fail(W2X_ERR_ARG, "NULL context");
    return W2X_OK;
}

// Whether a plane conversion walks the reference's blocks literally (convertWithModelsBlockSplit, src/convertRoutine.cpp:114-165).
bool literal_walk(const w2x_ctx *ctx, int w, int h, int block_splitting) {
    return block_splitting && ctx->walk == W2X_WALK_BLOCKS && w2x_requires_splitting(w, h);
}

// Row bands of a host plane's copy pipeline (chain_host) for a plane of width x height (1 = no pipeline: one upload, one pass,
// one download).  The literal block walk keeps its own order, and a band needs 2n rows of its own.
int host_copy_bands(const w2x_ctx *ctx, int n_model, int width, int height, int block_splitting) {
    int nb = ctx->host_bands > 0 ? ctx->host_bands : std::min(4, height / 512);
    if (nb > 8) nb = 8;
    if (nb < 2 || literal_walk(ctx, width, height, block_splitting) || height / nb < 2 * n_model) return 1;
    return nb;
}

// One group of a host-buffer call's copy pipeline: its uploads, the work that reads them (queued on the context's stream), and its
// downloads.  Each copy is one cudaMemcpy2DAsync.
struct HostGroup {
    struct Copy { void *dst; size_t dst_pitch; const void *src; size_t src_pitch, row_bytes, rows; };
    std::vector<Copy> up;
    std::function<int()> compute;
    std::vector<Copy> down;
};

// Queues the groups in order (start, then queue(g1) for successive ends g1; several contexts' pipes may be interleaved so), then
// finish() returns once every download has landed.  One group runs on the context's stream alone.  With more, uploads go on copy_in
// up to 8 groups ahead (ev_in / ev_done are 8 deep) and downloads on copy_out, so that the uploads of later groups and the downloads
// of earlier ones overlap the compute of the current one.  The first upload waits for the work already queued on the context's
// stream, which may still read the staging buffers.  On an error every stream is drained before returning: queued copies still touch
// the caller's buffers and the staging.
struct HostPipe {
    w2x_ctx *ctx;
    const std::vector<HostGroup> &groups;
    int next = 0;

    static cudaError_t copy(const HostGroup::Copy &c, cudaMemcpyKind kind, cudaStream_t s) {
        return cudaMemcpy2DAsync(c.dst, c.dst_pitch, c.src, c.src_pitch, c.row_bytes, c.rows, kind, s);
    }
    int ng() const { return (int)groups.size(); }
    int upload(int gi) {
        if (groups[(size_t)gi].up.empty()) return W2X_OK;
        for (auto &c : groups[(size_t)gi].up) CU_CHECK(copy(c, cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(ctx->ev_in[gi % 8], ctx->copy_in));
        return W2X_OK;
    }
    int start() {
        if (ng() <= 1) return W2X_OK;
        DeviceGuard g(ctx->device);
        CU_CHECK(cudaEventRecord(ctx->ev_done[0], ctx->stream));   // not recorded again before group 0's compute is queued
        CU_CHECK(cudaStreamWaitEvent(ctx->copy_in, ctx->ev_done[0], 0));
        int rc = W2X_OK;
        for (int gi = 0; gi < std::min(8, ng()) && !rc; gi++) rc = upload(gi);
        return rc;
    }
    int queue(int g1) {   // groups [next, g1)
        DeviceGuard g(ctx->device);
        for (; next < g1; next++) {
            const HostGroup &G = groups[(size_t)next];
            if (ng() == 1) {
                for (auto &c : G.up) CU_CHECK(copy(c, cudaMemcpyHostToDevice, ctx->stream));
                int rc = G.compute();
                if (rc) return rc;
                for (auto &c : G.down) CU_CHECK(copy(c, cudaMemcpyDeviceToHost, ctx->stream));
                continue;
            }
            const int gi = next;
            if (!G.up.empty()) CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[gi % 8], 0));
            int rc = G.compute();
            if (rc) return rc;
            CU_CHECK(cudaEventRecord(ctx->ev_done[gi % 8], ctx->stream));
            CU_CHECK(cudaStreamWaitEvent(ctx->copy_out, ctx->ev_done[gi % 8], 0));
            for (auto &c : G.down) CU_CHECK(copy(c, cudaMemcpyDeviceToHost, ctx->copy_out));
            if (gi + 8 < ng()) {   // ev_in[gi % 8]'s previous record has been waited for above
                rc = upload(gi + 8);
                if (rc) return rc;
            }
        }
        return W2X_OK;
    }
    int finish(int rc) {
        DeviceGuard g(ctx->device);
        if (rc) {
            cudaStreamSynchronize(ctx->copy_in);
            cudaStreamSynchronize(ctx->stream);
            cudaStreamSynchronize(ctx->copy_out);
            return rc;
        }
        if (ng() > 1) CU_CHECK(cudaStreamSynchronize(ctx->copy_out));
        CU_CHECK(cudaStreamSynchronize(ctx->stream));
        return W2X_OK;
    }
};

int run_host_groups(w2x_ctx *ctx, const std::vector<HostGroup> &groups) {
    HostPipe p{ctx, groups};
    int rc = p.start();
    if (!rc) rc = p.queue(p.ng());
    return p.finish(rc);
}

// The literal walk needs every block inside the plane; block_table places columns by the block height, as the reference does, so
// a non-square block size can put one past the plane's edge.
int check_blocks(const w2x_ctx *ctx, int n, int w, int h, int block_splitting) {
    if (!literal_walk(ctx, w, h, block_splitting)) return W2X_OK;
    const std::vector<int> tab = blocks_of(w, h, n);
    if (tab.empty()) return fail(W2X_ERR_ARG, "block size too small for a %d-layer model", n);
    for (size_t i = 0; i < tab.size(); i += 8) {
        const int *t = &tab[i];
        if (t[6] + (t[3] - t[2]) - 2 * n > h || t[7] + (t[5] - t[4]) - 2 * n > w)
            return fail(W2X_ERR_ARG, "block (%d,%d) does not fit the output plane (non-square block size?)", t[1], t[0]);
    }
    return W2X_OK;
}

// Every argument of a plane conversion on device buffers, before anything is printed or queued.
int check_plane(w2x_ctx *ctx, const w2x_model *m, const float *d_in, int w, int h, size_t in_stride_bytes, const float *d_out,
                size_t out_stride_bytes, int block_splitting) {
    if (!m || !d_in || !d_out || w < 1 || h < 1) return fail(W2X_ERR_ARG, "w2x_convert_plane: bad argument");
    if (in_stride_bytes % 4 || out_stride_bytes % 4 || in_stride_bytes < (size_t)w * 4 || out_stride_bytes < (size_t)w * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: row strides must be multiples of 4 bytes and >= width*4");
    if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: model must map 1 plane to 1 plane");
    if (pick_engine(ctx, m) < 0) return W2X_ERR_UNSUPPORTED;
    return check_blocks(ctx, (int)m->layers.size(), w, h, block_splitting);
}

// The progress lines of one convertWithModels-equivalent plane of w x h (host: through w2x_convert_plane's copy pipeline).  A
// plane the reference splits gets the reference's block sequence, whichever walk runs it; any other the layers' lines once when
// the copy pipeline cuts it into bands, else once per scratch band of convert_device.
void emit_plane_progress(w2x_ctx *ctx, const w2x_model *m, int w, int h, int block_splitting, bool host) {
    if (!ctx->log) return;
    const int n = (int)m->layers.size();
    if (block_splitting && w2x_requires_splitting(w, h)) return emit_reference_progress(ctx, w, h, n, true);
    const int band = scratch_band_rows(ctx, m, w, h);
    const int passes = host && host_copy_bands(ctx, n, w, h, 0) > 1 ? 1 : (h + band - 1) / band;
    for (int p = 0; p < passes; p++) emit_reference_progress(ctx, w, h, n, false);
}

// The scratch of a convert_device call on a w x h plane, reserved: the two activation frames of its largest scratch band (on the
// literal walk, of its largest reference block), the padded plane unless the first layer reads the plane directly, and the
// tensor-core kernels.  An upscaling call's plane is its 2x size; the resize changes none of it.
int reserve_convert(w2x_ctx *ctx, const w2x_model *m, int engine, int w, int h, int block_splitting) {
    const int n = (int)m->layers.size(), maxc = max_channels(m), pw = w + 2 * n;
    const bool literal = literal_walk(ctx, w, h, block_splitting);
    size_t act = 0;   // both engines: 4 bytes per activation element
    if (literal) {
        const std::vector<int> tab = blocks_of(w, h, n);
        for (size_t i = 0; i < tab.size(); i += 8) act = std::max(act, tc::act_bytes(maxc, tab[i + 5] - tab[i + 4], tab[i + 3] - tab[i + 2]));
    } else {
        act = tc::act_bytes(maxc, pw, scratch_band_rows(ctx, m, w, h) + 2 * n);
    }
    int rc = engine == W2X_ENGINE_TC ? ensure_tc(ctx) : W2X_OK;
    for (int i = 0; i < 2 && !rc; i++) rc = ctx->buf[i].reserve(act);
    if (!rc && (engine != W2X_ENGINE_TC || literal)) rc = ctx->pad_buf.reserve((size_t)pw * (h + 2 * n) * sizeof(float));
    return rc;
}

// Where a plane (or a window of one) comes from and goes to (row strides in bytes), and the real neighbours its source holds
// beyond it: rows above and below, columns left and right (all 0 for a whole plane).  up2x (an upscaling step): the counts are in
// 2x pixels, src points at the source pixel holding the window's first row and column, and phase_y / phase_x = 1 when those are
// that pixel's second copies (a window starting on an odd 2x row / column).
struct PlaneIO {
    const float *src; size_t src_stride; float *dst; size_t dst_stride;
    int above = 0, below = 0, left = 0, right = 0, phase_x = 0, phase_y = 0;
};

// The frame a model of n layers converts for the w x h window of p: cv::copyMakeBorder(BORDER_REPLICATE) by n
// (src/convertRoutine.cpp:35, :96) at the plane's own border, up to n real neighbour rows and columns elsewhere.  The one
// description of a window's frame: convert_device's first layer or padding kernel reads it, and a packed frame's rectangle holds it.
FrameSource window_frame(const PlaneIO &p, int w, int h, int n, bool up2x) {
    const int px = up2x ? p.phase_x : 0, py = up2x ? p.phase_y : 0;
    return FrameSource{p.src, (long)(p.src_stride / 4), w + px, h + py, n - px, n - py, std::min(p.above, n) - py, std::min(p.below, n), up2x,
                       std::min(p.left, n) - px, std::min(p.right, n)};
}

// convertWithModels on checked device buffers (rows_above / rows_below: real neighbour rows available around the band;
// cols_left / cols_right: real neighbour columns left and right of it, for a window).  up2x: the plane converted is the
// nearest-neighbour 2x resize of d_in, never materialised; w x h is its (2x) size, and the counts and phases are PlaneIO's.
int convert_device(w2x_ctx *ctx, const w2x_model *m, const float *d_in, int w, int h, size_t in_stride_bytes,
                   int rows_above, int rows_below, float *d_out, size_t out_stride_bytes, int block_splitting, bool up2x = false,
                   int cols_left = 0, int cols_right = 0, int phase_x = 0, int phase_y = 0) {
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convertWithModels");
    const int engine = pick_engine(ctx, m);
    DevModel *dm = nullptr;
    int rc = get_dev_model(ctx, m, &dm);
    if (!rc) rc = reserve_convert(ctx, m, engine, w, h, block_splitting);
    if (rc) return rc;
    const int n = (int)m->layers.size();
    const int pw = w + 2 * n;
    const long ostride = (long)(out_stride_bytes / 4);
    const bool literal = literal_walk(ctx, w, h, block_splitting);
    // cv::copyMakeBorder(in, temp, n, n, n, n, BORDER_REPLICATE)   (src/convertRoutine.cpp:35, :96): the plane's frame.  The
    // tensor-core engine folds it into the first layer's loads and reads d_in directly, except on the literal walk, whose blocks
    // are regions of the padded plane.
    const FrameSource plane = window_frame(PlaneIO{d_in, in_stride_bytes, d_out, out_stride_bytes, rows_above, rows_below, cols_left, cols_right,
                                                   phase_x, phase_y},
                                           w, h, n, up2x);
    const bool direct = engine == W2X_ENGINE_TC && !literal;
    float *pad = direct ? nullptr : ctx->pad_buf.get();
    if (!direct) {
        CU_CHECK(launch_pad(plane, pw, h + 2 * n, pad, ctx->stream));
        ctx->launches++;
    }
    if (literal) {   // check_blocks has seen every block fit
        const std::vector<int> tab = blocks_of(w, h, n);
        for (size_t i = 0; i < tab.size(); i += 8) {
            const int *t = &tab[i];
            rc = run_basic(ctx, m, dm, engine, FrameSource::padded(pad + (long)t[2] * pw + t[4], pw, t[5] - t[4], t[3] - t[2]), t[5] - t[4],
                           t[3] - t[2], d_out + (long)t[6] * ostride + t[7], ostride);
            if (rc) return rc;
        }
        return W2X_OK;
    }
    // horizontal bands that respect the scratch limit, each re-reading n rows of context above and below
    const int band = scratch_band_rows(ctx, m, w, h);
    for (int y0 = 0; y0 < h; y0 += band) {
        const int bh = std::min(band, h - y0);
        const FrameSource src = direct ? plane.band(y0, bh, n) : FrameSource::padded(pad + (long)y0 * pw, pw, pw, bh + 2 * n);
        rc = run_basic(ctx, m, dm, engine, src, pw, bh + 2 * n, d_out + (long)y0 * ostride, ostride);
        if (rc) return rc;
    }
    return W2X_OK;
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
    DeviceGuard g(device);   // before the context: it is still current when an early return destroys what has been created
    auto ctx = std::make_unique<w2x_ctx>();
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->cc_major = prop.major;
    ctx->cc_minor = prop.minor;
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    if (const char *pe = std::getenv("W2X_PRECISION")) {
        if (!std::strcmp(pe, "f16x3")) ctx->precision = W2X_PRECISION_F16X3;
        else if (!std::strcmp(pe, "f16+f8x2") || !std::strcmp(pe, "f8")) ctx->precision = W2X_PRECISION_F16_F8X2;
        else if (!std::strcmp(pe, "f16")) ctx->precision = W2X_PRECISION_F16;
        else if (!std::strcmp(pe, "bf16x3")) ctx->precision = W2X_PRECISION_BF16X3;
    }
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking));
    CU_CHECK(cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking));
    for (int i = 0; i < 8; i++) {
        CU_CHECK(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
        CU_CHECK(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
    }
    CU_CHECK(cudaEventCreateWithFlags(&ctx->plan_ev, cudaEventDisableTiming));
    CU_CHECK(cudaEventCreateWithFlags(&ctx->switch_ev, cudaEventDisableTiming));
    for (auto &e : ctx->tta_ev) CU_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    *out_ctx = ctx.release();
    return W2X_OK;
}

// Drops the context's device copies of a model (weights, packed operands); call it before w2x_model_free in a long-lived
// context that cycles through many models.  The next conversion with the same model uploads it again.  Refused while band
// sessions (w2x_band_*, the sub-bands of w2x_slab_*, the cached plan of w2x_multi_*) hold the copies: their passes launch
// with them, and a pass cannot upload them again without stalling the neighbours that wait in the exchange kernel.
int w2x_ctx_forget_model(w2x_ctx *ctx, const w2x_model *model) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model) return fail(W2X_ERR_ARG, "w2x_ctx_forget_model: NULL model");
    auto it = ctx->models.find(model->uid);
    if (it == ctx->models.end()) return W2X_OK;
    if (it->second.band_sessions > 0)
        return fail(W2X_ERR_ARG, "w2x_ctx_forget_model: %d band session(s) on this context still use the model; destroy them first",
                    it->second.band_sessions);
    DeviceGuard g(ctx->device);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->models.erase(it);
    return W2X_OK;
}

void w2x_ctx_destroy(w2x_ctx *ctx) {
    if (!ctx) return;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
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
    if (precision != W2X_PRECISION_F16X3 && precision != W2X_PRECISION_F16_F8X2 && precision != W2X_PRECISION_F16 &&
        precision != W2X_PRECISION_BF16X3)
        return fail(W2X_ERR_ARG, "unknown precision mode %d", precision);
    ctx->precision = precision;
    return W2X_OK;
}
int w2x_ctx_get_precision(const w2x_ctx *ctx) { return ctx ? ctx->precision : -1; }

// Every call on the context shares its scratch, and only the order of one stream keeps two calls apart.  So a switch makes the new
// stream wait for everything queued on the old one: the calls after it never overlap the calls before it, and whatever waits for the
// current stream (w2x_ctx_synchronize, w2x_ctx_layer_times, w2x_ctx_forget_model, w2x_ctx_destroy, the first upload of
// run_host_groups) waits for those too.
int w2x_ctx_set_stream(w2x_ctx *ctx, void *cuda_stream) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
    if (s == ctx->stream) return W2X_OK;
    DeviceGuard g(ctx->device);
    CU_CHECK(cudaEventRecord(ctx->switch_ev, ctx->stream));
    CU_CHECK(cudaStreamWaitEvent(s, ctx->switch_ev, 0));
    ctx->stream = s;
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
        CU_CHECK(ctx->prof_buf.grow(bytes));
        CU_CHECK(cudaMemsetAsync(ctx->prof_buf.get(), 0, bytes, ctx->stream));
    } else if (ctx->prof_buf.get()) {
        CU_CHECK(cudaStreamSynchronize(ctx->stream));
        ctx->prof_buf.release();
    }
    return W2X_OK;
}
// out[PROF_WORDS]: counters of `layer` summed over CTAs; *n_ctas = CTAs that ran.
W2X_API int w2x_debug_tc_profile_read(w2x_ctx *ctx, int layer, unsigned long long *out, int *n_ctas) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!ctx->prof_buf.get() || layer < 0 || layer >= 16 || !out) return fail(W2X_ERR_ARG, "profile not enabled or bad layer");
    DeviceGuard g(ctx->device);
    std::vector<unsigned long long> h((size_t)tc::PROF_MAX_CTAS * tc::PROF_WORDS);
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    CU_CHECK(cudaMemcpy(h.data(), ctx->prof_buf.get() + (size_t)layer * h.size(), h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
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

int w2x_convert_band_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, int width, int band_height,
                            int rows_above, int rows_below, size_t in_stride_bytes, float *d_out, size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (rows_above < 0 || rows_below < 0) return fail(W2X_ERR_ARG, "w2x_convert_band_device: negative halo");
    if (model && ((rows_above && rows_above < (int)model->layers.size()) || (rows_below && rows_below < (int)model->layers.size())))
        return fail(W2X_ERR_ARG, "w2x_convert_band_device: a halo must be 0 (image border) or >= the layer count (%zu)",
                    model->layers.size());
    if (!d_in) return fail(W2X_ERR_ARG, "w2x_convert_band_device: NULL input");
    const float *band0 = d_in + (size_t)rows_above * (in_stride_bytes / 4);
    int rc = check_plane(ctx, model, band0, width, band_height, in_stride_bytes, d_out, out_stride_bytes, 0);
    if (rc) return rc;
    emit_plane_progress(ctx, model, width, band_height, 0, false);
    return convert_device(ctx, model, band0, width, band_height, in_stride_bytes, rows_above, rows_below, d_out,
                          out_stride_bytes, 0);
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
        const tc::Rec rec = tc::rec_format(ctx->precision);
        if (rec == tc::Rec::BF16 ? model->tc[(size_t)layer].bytes_bf16.empty() : model->tc[(size_t)layer].bytes.empty())
            return fail(W2X_ERR_UNSUPPORTED, rec == tc::Rec::BF16 ? "tensor-core engine needs finite layer weights"
                                                                  : "tensor-core engine needs finite layer weights below 65520 in magnitude");
        rc = ensure_tc(ctx);
        if (rc) return rc;
        // Model::filter semantics (same size, BORDER_REPLICATE): stage a frame with a replicated ring
        // of one pixel, run the same-size tensor-core layer on it, return the interior.
        const int pw = width + 2, ph = height + 2;
        rc = ctx->buf[0].reserve(tc::act_bytes(L.n_in, pw, ph));
        if (rc) return rc;
        rc = ctx->buf[1].reserve(tc::act_bytes(L.n_out, pw, ph));
        if (rc) return rc;
        __half *fin = static_cast<__half *>(ctx->buf[0].get()), *fout = static_cast<__half *>(ctx->buf[1].get());
        CU_CHECK(tc::launch_planar_to_nhwc(d_in, L.n_in, width, height, fin, ctx->stream, rec));
        rc = launch_layer_tc(ctx, model, dm, layer, fin, fout, pw, ph, false, false);
        if (rc) return rc;
        CU_CHECK(tc::launch_nhwc_to_planar(fout, L.n_out, width, height, d_out, ctx->stream, rec));
        ctx->launches += 2;
        return W2X_OK;
    }
    {
        LayerTimer t(ctx, layer);
        CU_CHECK(launch_conv3x3_fp32(d_in, d_out, dm->w[(size_t)layer].get(), dm->b[(size_t)layer].get(), L.n_in, L.n_out, width, height,
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
    for (int i = 0; i < L.n_in; i++)
        if (!in_planes[i]) return fail(W2X_ERR_ARG, "w2x_filter_layer: NULL input plane %d", i);
    for (int i = 0; i < L.n_out; i++)
        if (!out_planes[i]) return fail(W2X_ERR_ARG, "w2x_filter_layer: NULL output plane %d", i);
    DeviceGuard g(ctx->device);
    const size_t plane = (size_t)width * height, row = (size_t)width * 4;
    int rc = reserve_io(ctx, plane * sizeof(float) * (size_t)L.n_in, plane * sizeof(float) * (size_t)L.n_out);
    if (rc) return rc;
    float *din = ctx->io_buf[0].get(), *dout = ctx->io_buf[1].get();
    std::vector<HostGroup> groups(1);
    for (int i = 0; i < L.n_in; i++) groups[0].up.push_back({din + plane * (size_t)i, row, in_planes[i], in_stride_bytes, row, (size_t)height});
    groups[0].compute = [=] { return w2x_filter_layer_device(ctx, model, layer, din, dout, width, height); };
    for (int i = 0; i < L.n_out; i++) groups[0].down.push_back({out_planes[i], out_stride_bytes, dout + plane * (size_t)i, row, row, (size_t)height});
    return run_host_groups(ctx, groups);
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
        CU_CHECK(cudaEventElapsedTime(&t, s.e0, s.e1));
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

// The device tables of a call's frames, then those of its TTA kernels, as one blob for plan_buf.
struct Tables {
    std::vector<char> blob;
    std::vector<size_t> off_rect, off_shelf;
    size_t off_tta = 0;
    size_t bytes(size_t n_tta) const { return off_tta + n_tta * sizeof(TtaPlane); }
};

// Puts each frame's rectangles in shelf order, numbers their gather blocks and lays their tables out in t (*out gets the sizes).
void frame_tables(std::vector<FramePlan> &frames, std::vector<FrameDev> *out, Tables *t) {
    auto align = [](size_t b) { return (b + 15) & ~(size_t)15; };
    std::vector<char> &blob = t->blob;
    std::vector<size_t> &off_rect = t->off_rect, &off_shelf = t->off_shelf;
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
    t->off_tta = align(blob.size());
}

// Uploads t's frame tables and `tta` (the tables of the TTA kernels, at *tta_dev) in ONE copy on the context's stream, into plan_buf
// as reserved for them.  The copy waits for the kernels of an earlier call that still read the buffer (plan_ev), and its source is
// pageable memory, so it is staged before cudaMemcpyAsync returns and the host vectors may go at once.
int upload_tables(w2x_ctx *ctx, Tables &t, std::vector<FrameDev> *out, const std::vector<TtaPlane> &tta = {}, const TtaPlane **tta_dev = nullptr) {
    std::vector<char> &blob = t.blob;
    blob.resize(t.bytes(tta.size()));
    if (!tta.empty()) std::memcpy(blob.data() + t.off_tta, tta.data(), tta.size() * sizeof(TtaPlane));
    if (ctx->plan_ev_live) CU_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->plan_ev, 0));
    const char *base = ctx->plan_buf.get();
    CU_CHECK(cudaMemcpyAsync(ctx->plan_buf.get(), blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (tta_dev) *tta_dev = reinterpret_cast<const TtaPlane *>(base + t.off_tta);
    for (size_t f = 0; f < out->size(); f++) {
        FrameDev &d = (*out)[f];
        d.rect = reinterpret_cast<const tc::PlaneRect *>(base + t.off_rect[f]);
        d.shelf_y0 = reinterpret_cast<const int *>(base + t.off_shelf[f]);
        d.shelf_first = d.shelf_y0 + d.n_shelf;
    }
    return W2X_OK;
}

int upload_frames(w2x_ctx *ctx, std::vector<FramePlan> &frames, std::vector<FrameDev> *out) {
    Tables t;
    frame_tables(frames, out, &t);
    int rc = ctx->plan_buf.reserve(t.bytes(0));
    return rc ? rc : upload_tables(ctx, t, out);
}

// Sizes the scratch for the largest of frames [f0, f1) of a model of maxc channels once, so that no buffer is reallocated between
// frames.
int reserve_frames(w2x_ctx *ctx, const std::vector<FramePlan> &frames, size_t f0, size_t f1, int maxc) {
    size_t px = 0;
    for (size_t f = f0; f < f1; f++) px = std::max(px, (size_t)frames[f].fw * frames[f].fh);
    int rc = ctx->pad_buf.reserve(px * sizeof(float));
    for (int i = 0; i < 2 && !rc; i++) rc = ctx->buf[i].reserve(px * (size_t)maxc * 4);
    return rc;
}

// One packed frame: the pack, the layers on the whole frame, the gather -- n + 1 launches whatever the number of planes.  up2x: the
// frame's planes are the nearest-neighbour 2x resizes of their sources (tc::launch_pack_planes).
int run_packed_frame(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, const FrameDev &f, bool up2x = false) {
    const int n = (int)m->layers.size();
    int rc = ctx->pad_buf.reserve((size_t)f.fw * f.fh * sizeof(float));
    if (rc) return rc;
    CU_CHECK(tc::launch_pack_planes(f.rect, f.shelf_y0, f.shelf_first, f.n_shelf, n, f.fw, f.fh, up2x, ctx->pad_buf.get(), ctx->stream));
    ctx->launches++;
    const PackedGather g{f.rect, f.n_rect, f.n_blocks};
    return run_basic(ctx, m, dm, W2X_ENGINE_TC, FrameSource::padded(ctx->pad_buf.get(), f.fw, f.fw, f.fh), f.fw, f.fh, nullptr, 0, &g);
}

int run_packed_frames(w2x_ctx *ctx, const w2x_model *m, DevModel *dm, std::vector<FramePlan> &frames) {
    std::vector<FrameDev> fd;
    int rc = reserve_frames(ctx, frames, 0, frames.size(), max_channels(m));
    if (!rc) rc = upload_frames(ctx, frames, &fd);
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
    const bool packed = packs_frames(ctx, m, dm, engine);
    // tiles per frame (1 unpacked): what the scratch limit (one frame of maxc channels, 4 bytes per element) and MAX_FRAME_ROWS allow;
    // the tiles of a frame are stacked vertically, each padded like cv::copyMakeBorder (src/convertRoutine.cpp:35) by the pack
    const size_t per_tile = (size_t)max_channels(m) * pw * ph * 4;
    const size_t fit = std::min(ctx->scratch_limit / per_tile, (size_t)(MAX_FRAME_ROWS / ph));
    const int group = packed ? (int)std::max<size_t>(1, std::min<size_t>((size_t)n_tiles, fit)) : 1;
    for (int t0 = 0; t0 < n_tiles; t0 += group) emit_reference_progress(ctx, w, h, n, false);   // the layers run once per frame
    if (packed) {
        std::vector<FramePlan> frames;
        for (int t0 = 0; t0 < n_tiles; t0 += group) {
            FramePlan f;
            f.fw = pw;
            f.fh = std::min(group, n_tiles - t0) * ph;
            for (int t = 0; t0 + t < n_tiles && t < group; t++) {
                const size_t off = (size_t)(t0 + t) * w * h;
                f.rect.push_back(tc::PlaneRect{window_frame(PlaneIO{d_in + off, (size_t)w * 4, d_out + off, (size_t)w * 4}, w, h, n, false),
                                               d_out + off, w, w, h, 0, t * ph, 0});
            }
            frames.push_back(std::move(f));
        }
        return run_packed_frames(ctx, m, dm, frames);
    }
    rc = ctx->pad_buf.reserve((size_t)pw * ph * sizeof(float));
    if (rc) return rc;
    for (int t = 0; t < n_tiles; t++) {   // cv::copyMakeBorder per tile (src/convertRoutine.cpp:35)
        CU_CHECK(launch_pad(FrameSource{d_in + (size_t)t * w * h, w, w, h, n, n, 0, 0}, pw, ph, ctx->pad_buf.get(), ctx->stream));
        ctx->launches++;
        rc = run_basic(ctx, m, dm, engine, FrameSource::padded(ctx->pad_buf.get(), pw, pw, ph), pw, ph, d_out + (size_t)t * w * h, w);
        if (rc) return rc;
    }
    return W2X_OK;
}

// ---- independent planes of any sizes (w2x_convert_planes*), also through a chain of steps (w2x_convert_planes_chain*) ---------
// The plane arrays: plane i is widths[i] x heights[i] at in[i] and comes out (widths[i] << u) x (heights[i] << u) at out[i], u being
// the number of 2x steps; row strides in bytes.
int check_plane_arrays(const char *fn, int n_planes, const float *const *in, const int *widths, const int *heights, const size_t *in_strides,
                       float *const *out, const size_t *out_strides, int u) {
    if (n_planes < 1) return fail(W2X_ERR_ARG, "%s: n_planes is %d, at least 1 plane is needed", fn, n_planes);
    if (!in || !widths || !heights || !in_strides || !out || !out_strides) return fail(W2X_ERR_ARG, "%s: NULL array argument", fn);
    for (int i = 0; i < n_planes; i++) {
        if (!in[i] || !out[i]) return fail(W2X_ERR_ARG, "%s: plane %d: NULL %s pointer", fn, i, in[i] ? "output" : "input");
        if (widths[i] < 1 || heights[i] < 1) return fail(W2X_ERR_ARG, "%s: plane %d: size %d x %d", fn, i, widths[i], heights[i]);
        if (u > 30 || ((long)widths[i] << u) > INT_MAX || ((long)heights[i] << u) > INT_MAX)
            return fail(W2X_ERR_ARG, "%s: plane %d: %d x %d after %d 2x steps overflows int", fn, i, widths[i], heights[i], u);
        const size_t out_row = ((size_t)widths[i] << u) * 4;
        if (in_strides[i] % 4 || out_strides[i] % 4 || in_strides[i] < (size_t)widths[i] * 4 || out_strides[i] < out_row)
            return fail(W2X_ERR_ARG, "%s: plane %d: row strides must be multiples of 4 bytes and >= width*4", fn, i);
    }
    return W2X_OK;
}

int check_planes(const char *fn, const w2x_model *m, int n_planes, const float *const *in, const int *widths, const int *heights,
                 const size_t *in_strides, float *const *out, const size_t *out_strides) {
    if (!m) return fail(W2X_ERR_ARG, "%s: NULL model", fn);
    int rc = check_plane_arrays(fn, n_planes, in, widths, heights, in_strides, out, out_strides, 0);
    if (rc) return rc;
    if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1) return fail(W2X_ERR_ARG, "%s: model must map 1 plane to 1 plane", fn);
    return W2X_OK;
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

// One step of a chain (w2x_convert_chain*, w2x_convert_planes*): every plane through one model, after the nearest 2x resize when
// `up`.  A single-plane chain is a collection of one plane.  A step converts a window of each plane: the whole plane, except in the
// region calls (w2x_convert_chain_region*, w2x_convert_chain_regions*), which have no TTA step.  Each plane's PlaneIO carries the
// context around its window, which its frame (window_frame) reads, converted alone or packed.
struct Step {
    const w2x_model *m;
    bool up;
    bool tta = false;                   // W2X_STEP_TTA: the model runs on the 8 variants of every plane, the mean is the output
    std::vector<int> w, h;              // the step's output sizes: of each plane's output window
    std::vector<int> x0, y0;            // where each output window starts on the step's output plane
    std::vector<Rect> in;               // each plane's input window on the step's input plane: what its source holds
    DevModel *dm = nullptr;
    bool packed = false;                // packs_frames: frames plus planes too large to pack, else every plane alone
    PlanesPlan plan;                    // packed: each converted plane's frame (-1: converted alone) and place
    size_t f0 = 0;                      // packed: index of its frame 0 in the call's frame table
    std::vector<PlaneIO> io;            // each plane's source and destination at this step
    // tta: the variant planes the model converts on this context -- vof lists them as 8 i + j, variant j of plane i in the call's
    // numbering; every one of the 8n on one context -- their outputs vw x vh, with their sources in ctx->tta_buf[0] and outputs in
    // ctx->tta_buf[1], and the tables of the variants and the mean kernel of the planes (w, h) the context owns (tiles: their blocks)
    std::vector<int> vof, vw, vh;
    std::vector<PlaneIO> vio;
    const TtaPlane *vtab = nullptr, *mtab = nullptr;
    int vtiles = 0, mtiles = 0;
    // the planes the model converts
    const std::vector<int> &cw() const { return tta ? vw : w; }
    const std::vector<int> &ch() const { return tta ? vh : h; }
    const std::vector<PlaneIO> &cio() const { return tta ? vio : io; }
};

// The steps of checked arguments, each with its output size per plane (and, for a TTA step, per variant).
std::vector<Step> step_table(int n_steps, const w2x_model *const *models, const int *kinds, int n_planes, const int *widths, const int *heights) {
    std::vector<int> w(widths, widths + n_planes), h(heights, heights + n_planes);
    std::vector<Step> steps((size_t)n_steps);
    for (int k = 0; k < n_steps; k++) {
        Step &s = steps[(size_t)k];
        s.m = models[k];
        s.up = (kinds[k] & W2X_STEP_UPSCALE2X) != 0;
        s.tta = (kinds[k] & W2X_STEP_TTA) != 0;
        for (int i = 0; i < n_planes; i++) s.in.push_back(Rect{0, 0, w[(size_t)i], h[(size_t)i]});
        if (s.up)
            for (int i = 0; i < n_planes; i++) w[(size_t)i] *= 2, h[(size_t)i] *= 2;
        s.w = w;
        s.h = h;
        s.x0 = s.y0 = std::vector<int>((size_t)n_planes, 0);
        for (int i = 0; i < n_planes && s.tta; i++)
            for (int j = 0; j < 8; j++) {
                s.vof.push_back(8 * i + j);
                s.vw.push_back(j & 4 ? h[(size_t)i] : w[(size_t)i]);
                s.vh.push_back(j & 4 ? w[(size_t)i] : h[(size_t)i]);
            }
    }
    return steps;
}

std::vector<Step> one_step(const w2x_model *m, int n_planes, const int *widths, const int *heights) {
    const int same = W2X_STEP_SAME;
    return step_table(1, &m, &same, n_planes, widths, heights);
}

// Every argument of a chain call, before anything is printed, allocated or queued, in this order: the step arrays (W2X_ERR_ARG
// naming the step); the caller's planes, by check_planes(number of 2x steps); each step's engine (W2X_ERR_UNSUPPORTED naming the
// step) and, with block_splitting, its literal walk on every plane (W2X_ERR_ARG naming the step).  Then *steps is the step table.
int check_steps(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes, const int *widths,
                const int *heights, int block_splitting, const std::function<int(int)> &check_planes, std::vector<Step> *steps) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (n_steps < 1) return fail(W2X_ERR_ARG, "%s: n_steps is %d: at least one step (step 0) is needed", fn, n_steps);
    if (!models) return fail(W2X_ERR_ARG, "%s: step 0: NULL models array", fn);
    if (!kinds) return fail(W2X_ERR_ARG, "%s: step 0: NULL kinds array", fn);
    int u = 0;
    for (int k = 0; k < n_steps; k++) {
        const w2x_model *m = models[k];
        if (!m) return fail(W2X_ERR_ARG, "%s: step %d: NULL model", fn, k);
        if (kinds[k] & ~(W2X_STEP_UPSCALE2X | W2X_STEP_TTA))
            return fail(W2X_ERR_ARG, "%s: step %d: kind %d is neither W2X_STEP_SAME (0) nor W2X_STEP_UPSCALE2X (1), each optionally | W2X_STEP_TTA (4)",
                        fn, k, kinds[k]);
        if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1)
            return fail(W2X_ERR_ARG, "%s: step %d: model must map 1 plane to 1 plane", fn, k);
        if (kinds[k] & W2X_STEP_UPSCALE2X) u++;
    }
    int rc = check_planes(u);
    if (rc) return rc;
    *steps = step_table(n_steps, models, kinds, n_planes, widths, heights);
    for (int k = 0; k < n_steps; k++) {   // engine choice (the tensor-core engine needs a 1->{32,64,128}...->1 chain), literal walk
        const Step &s = (*steps)[(size_t)k];
        rc = pick_engine(ctx, s.m) < 0 ? W2X_ERR_UNSUPPORTED : W2X_OK;
        for (size_t i = 0; i < s.cw().size() && !rc; i++) rc = check_blocks(ctx, (int)s.m->layers.size(), s.cw()[i], s.ch()[i], block_splitting);
        if (rc) {
            const std::string why = w2x_last_error();
            return fail(rc, "%s: step %d: %s", fn, k, why.c_str());
        }
    }
    return W2X_OK;
}

// Every argument of w2x_convert_planes_chain*: the steps, and the planes by check_plane_arrays (W2X_ERR_ARG naming the plane).
int check_planes_chain(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                       const float *const *in, const int *widths, const int *heights, const size_t *in_strides, float *const *out,
                       const size_t *out_strides, std::vector<Step> *steps) {
    return check_steps(fn, ctx, n_steps, models, kinds, n_planes, widths, heights, 0, [&](int u) {
        return check_plane_arrays(fn, n_planes, in, widths, heights, in_strides, out, out_strides, u);
    }, steps);
}

// What one context does in a call: the steps on the planes it owns (own: their numbers in the call; Step::w, h and io are theirs), of
// a TTA step the variants it converts (Step::vof), where its planes come from and go to (ends), and its frame tables (fd).  A call on
// one context has one part owning every plane and converting every variant.
struct Part {
    w2x_ctx *ctx;
    std::vector<int> own;
    std::vector<Step> steps;
    std::vector<PlaneIO> ends;
    std::vector<FrameDev> fd;
    std::vector<FramePlan> frames;   // prepare_parts' working state
    Tables tables;
    size_t n_tta = 0;
    int band_rows = 0;               // > 0: the last step's one plane is converted in row bands of at most this many rows (chain_host)
};

// Part p's steps: the call's steps on its planes, a TTA step's variants restricted to vof[k] (8 i + j each, ascending).
std::vector<Step> part_steps(const std::vector<Step> &all, const std::vector<int> &own, const std::vector<std::vector<int>> &vof) {
    std::vector<Step> steps(all.size());
    for (size_t k = 0; k < all.size(); k++) {
        const Step &a = all[k];
        Step &s = steps[k];
        s.m = a.m;
        s.up = a.up;
        s.tta = a.tta;
        for (int i : own) {
            s.w.push_back(a.w[(size_t)i]);
            s.h.push_back(a.h[(size_t)i]);
            s.x0.push_back(a.x0[(size_t)i]);
            s.y0.push_back(a.y0[(size_t)i]);
            s.in.push_back(a.in[(size_t)i]);
        }
        for (int v : vof[k]) {
            s.vof.push_back(v);
            s.vw.push_back(a.vw[(size_t)v]);
            s.vh.push_back(a.vh[(size_t)v]);
        }
    }
    return steps;
}

// The first half of prepare_parts on one part: every device buffer and the model copies, where each plane and variant lives.  Its
// planes come from and go to: step 0 reads ends[i].src, the last step writes ends[i].dst, step k < last writes its outputs (output
// windows) densely into chain_buf[k & 1]; a TTA step's variants (an upscaling step's are those of its half-resolution sources: the
// nearest 2x resize commutes with every flip and transpose) lie dense in tta_buf[0] in vof order, their outputs dense in tta_buf[1].
// With `pack`, each step that packs_frames allows is planned into frames on its OUTPUT sizes, so that a plane may pack at one step and
// be converted alone after a 2x step (without, every plane is converted alone); a TTA step's frames are planned on the variants it
// converts.  Every plane or variant converted alone gets the scratch of its convert_device call (reserve_convert, with the call's
// block_splitting), so that the call's own reservations find it there.
int reserve_part(Part &P, bool pack, int block_splitting) {
    w2x_ctx *ctx = P.ctx;
    DeviceGuard g(ctx->device);
    std::vector<Step> &steps = P.steps;
    const size_t n_planes = P.own.size(), last = steps.size() - 1;
    size_t need[2] = {0, 0}, tta_need[2] = {0, 0};
    for (size_t k = 0; k <= last; k++) {
        const Step &s = steps[k];
        size_t px = 0, vin = 0, vout = 0;
        for (size_t i = 0; i < n_planes; i++) px += (size_t)s.w[i] * s.h[i];
        for (size_t v = 0; v < s.vw.size(); v++) {
            vout += (size_t)s.vw[v] * s.vh[v];
            vin += (size_t)s.vw[v] * s.vh[v] / (s.up ? 4 : 1);
        }
        if (k < last) need[k & 1] = std::max(need[k & 1], px * sizeof(float));
        tta_need[0] = std::max(tta_need[0], vin * sizeof(float));
        tta_need[1] = std::max(tta_need[1], vout * sizeof(float));
    }
    for (int i = 0; i < 2; i++) {
        if (!need[i]) continue;
        int rc = ctx->chain_buf[i].reserve(need[i]);
        if (rc) return rc;
    }
    for (int i = 0; i < 2; i++) {
        if (!tta_need[i]) continue;
        int rc = ctx->tta_buf[i].reserve(tta_need[i]);
        if (rc) return rc;
    }
    P.frames.clear();
    P.n_tta = 0;
    for (size_t k = 0; k <= last; k++) {
        Step &s = steps[k];
        int rc = get_dev_model(ctx, s.m, &s.dm);
        if (rc) return rc;
        const int engine = pick_engine(ctx, s.m), u = s.up ? 2 : 1;
        s.packed = pack && !s.cw().empty() && packs_frames(ctx, s.m, s.dm, engine);
        s.io.resize(n_planes);
        size_t off = 0;
        for (size_t i = 0; i < n_planes; i++) {
            // the source holds the input window, and the output window starts at its source pixel (o.y0 / u, o.x0 / u)
            const Rect &in = s.in[i];
            const Rect o{s.x0[i], s.y0[i], s.w[i], s.h[i]};
            PlaneIO &p = s.io[i];
            const char *src = reinterpret_cast<const char *>(k == 0 ? P.ends[i].src : steps[k - 1].io[i].dst);
            p.src_stride = k == 0 ? P.ends[i].src_stride : steps[k - 1].io[i].dst_stride;
            p.src = reinterpret_cast<const float *>(src + (size_t)(o.y0 / u - in.y0) * p.src_stride) + (o.x0 / u - in.x0);
            p.dst = k == last ? P.ends[i].dst : ctx->chain_buf[k & 1].get() + off;
            p.dst_stride = k == last ? P.ends[i].dst_stride : (size_t)s.w[i] * sizeof(float);
            p.above = o.y0 - u * in.y0, p.below = u * in.y1() - o.y1();
            p.left = o.x0 - u * in.x0, p.right = u * in.x1() - o.x1();
            p.phase_x = o.x0 % u, p.phase_y = o.y0 % u;
            off += (size_t)s.w[i] * s.h[i];
        }
        if (s.tta) {
            s.vio.resize(s.vof.size());
            size_t in_off = 0, out_off = 0;
            for (size_t v = 0; v < s.vof.size(); v++) {
                const int sw = s.up ? s.vw[v] / 2 : s.vw[v], sh = s.up ? s.vh[v] / 2 : s.vh[v];
                s.vio[v] = PlaneIO{ctx->tta_buf[0].get() + in_off, (size_t)sw * sizeof(float), ctx->tta_buf[1].get() + out_off,
                                   (size_t)s.vw[v] * sizeof(float)};
                in_off += (size_t)sw * sh;
                out_off += (size_t)s.vw[v] * s.vh[v];
            }
            P.n_tta += 2 * n_planes;   // the variants and the mean kernel's rows of the planes it owns
        }
        const std::vector<int> &cw = s.cw(), &ch = s.ch();
        const std::vector<PlaneIO> &cio = s.cio();
        if (s.packed) {
            plan_for(ctx, s.m, (int)cw.size(), cw.data(), ch.data(), &s.plan);
            s.f0 = P.frames.size();
            for (FramePlan &f : frames_for(s.plan)) P.frames.push_back(std::move(f));
            for (size_t i = 0; i < cw.size(); i++) {
                const int f = s.plan.frame[i];
                if (f >= 0)
                    P.frames[s.f0 + (size_t)f].rect.push_back(tc::PlaneRect{window_frame(cio[i], cw[i], ch[i], (int)s.m->layers.size(), s.up),
                                                                            cio[i].dst, (long)(cio[i].dst_stride / 4), cw[i], ch[i],
                                                                            s.plan.x0[i], s.plan.y0[i], 0});
            }
            rc = reserve_frames(ctx, P.frames, s.f0, P.frames.size(), max_channels(s.m));
            if (rc) return rc;
        }
        for (size_t i = 0; i < cw.size(); i++) {   // the planes converted alone; band_rows: chain_host's copy bands of the last step
            if (s.packed && s.plan.frame[i] >= 0) continue;
            rc = reserve_convert(ctx, s.m, engine, cw[i], k == last && P.band_rows ? P.band_rows : ch[i], block_splitting);
            if (rc) return rc;
        }
    }
    P.tables = Tables();
    frame_tables(P.frames, &P.fd, &P.tables);
    if (P.frames.empty() && !P.n_tta) return W2X_OK;
    return ctx->plan_buf.reserve(P.tables.bytes(P.n_tta));
}

// Everything before the first line, on_step call or launch of a call, on every part: first every buffer of every part, convert_device's
// scratch included (reserve_part), so that W2X_ERR_NOMEM leaves nothing queued on any context; then on each part ONE upload of every step's frame tables and TTA kernel tables, so that no
// step waits for the host.  A TTA step's variants kernel on the part owning plane i writes variant j wherever the part converting it
// keeps it, and the mean kernel reads its output there.
int prepare_parts(std::vector<Part> &parts, bool pack, int block_splitting) {
    for (Part &P : parts)
        if (int rc = reserve_part(P, pack, block_splitting)) return rc;
    const size_t n_steps = parts[0].steps.size();
    std::vector<std::vector<const PlaneIO *>> var_at(n_steps);   // [k][8 i + j]: where variant j of plane i lives at TTA step k
    for (const Part &P : parts)
        for (size_t k = 0; k < n_steps; k++) {
            const Step &s = P.steps[k];
            for (size_t v = 0; v < s.vof.size(); v++) {
                if (var_at[k].size() <= (size_t)s.vof[v]) var_at[k].resize((size_t)s.vof[v] + 1);
                var_at[k][(size_t)s.vof[v]] = &s.vio[v];
            }
        }
    auto tiles = [](int w, int h) { return ((w + 31) / 32) * ((h + 31) / 32); };
    for (Part &P : parts) {
        if (P.frames.empty() && !P.n_tta) continue;
        DeviceGuard g(P.ctx->device);
        std::vector<TtaPlane> tta;
        std::vector<size_t> tab0(n_steps);   // a TTA step's variants table at tta[tab0], its mean table right after it
        for (size_t k = 0; k < n_steps; k++) {
            Step &s = P.steps[k];
            if (!s.tta) continue;
            tab0[k] = tta.size();
            for (size_t i = 0; i < P.own.size(); i++) {   // the variants kernel: plane -> its 8 variants
                const int sw = s.up ? s.w[i] / 2 : s.w[i], sh = s.up ? s.h[i] / 2 : s.h[i];
                TtaPlane t{s.io[i].src, {}, nullptr, (long)(s.io[i].src_stride / 4), 0, sw, sh, s.vtiles};
                for (int j = 0; j < 8; j++) t.var[j] = const_cast<float *>(var_at[k][(size_t)(8 * P.own[i] + j)]->src);
                tta.push_back(t);
                s.vtiles += tiles(sw, sh);
            }
            for (size_t i = 0; i < P.own.size(); i++) {   // the mean kernel: 8 variant outputs -> the step's output
                TtaPlane t{nullptr, {}, s.io[i].dst, 0, (long)(s.io[i].dst_stride / 4), s.w[i], s.h[i], s.mtiles};
                for (int j = 0; j < 8; j++) t.var[j] = var_at[k][(size_t)(8 * P.own[i] + j)]->dst;
                tta.push_back(t);
                s.mtiles += tiles(s.w[i], s.h[i]);
            }
        }
        const TtaPlane *tab = nullptr;
        int rc = upload_tables(P.ctx, P.tables, &P.fd, tta, &tab);
        if (rc) return rc;
        for (size_t k = 0; k < n_steps; k++)
            if (P.steps[k].tta) {
                P.steps[k].vtab = tab + tab0[k];
                P.steps[k].mtab = tab + tab0[k] + P.own.size();
            }
    }
    return W2X_OK;
}

// The one-context call: one part owning every plane (its ends still to be set).
Part one_part(w2x_ctx *ctx, std::vector<Step> &steps) {
    Part P{ctx, std::vector<int>(steps[0].w.size()), std::move(steps), {}, {}, {}, {}, 0};
    for (size_t i = 0; i < P.own.size(); i++) P.own[i] = (int)i;
    return P;
}

// A unit of work of one step: one packed frame (n + 1 launches for all its planes), or one plane converted alone by convert_device
// (too large to pack, or a step that does not pack).  A step's units: its frames, then its other planes, each in order.  The planes
// are the ones the model converts: a TTA step's variants.
struct PlanesUnit { int frame; std::vector<int> planes; };
std::vector<PlanesUnit> units_of(const Step &s) {
    std::vector<PlanesUnit> units;
    const int n_planes = (int)s.cw().size();
    if (s.packed) {
        units.resize((size_t)s.plan.n_frames);
        for (int f = 0; f < s.plan.n_frames; f++) units[(size_t)f].frame = f;
        for (int i = 0; i < n_planes; i++)
            if (s.plan.frame[(size_t)i] >= 0) units[(size_t)s.plan.frame[(size_t)i]].planes.push_back(i);
    }
    for (int i = 0; i < n_planes; i++)
        if (!s.packed || s.plan.frame[(size_t)i] < 0) units.push_back(PlanesUnit{-1, {i}});
    return units;
}

int run_unit(w2x_ctx *ctx, const Step &s, const std::vector<FrameDev> &fd, const PlanesUnit &u, int block_splitting) {
    if (u.frame < 0) {
        const size_t i = (size_t)u.planes[0];
        const PlaneIO &p = s.cio()[i];
        return convert_device(ctx, s.m, p.src, s.cw()[i], s.ch()[i], p.src_stride, p.above, p.below, p.dst, p.dst_stride, block_splitting,
                              s.up, p.left, p.right, p.phase_x, p.phase_y);
    }
    const size_t f = s.f0 + (size_t)u.frame;
    int rc = run_packed_frame(ctx, s.m, s.dm, fd[f], s.up);
    if (rc || f + 1 < fd.size()) return rc;
    CU_CHECK(cudaEventRecord(ctx->plan_ev, ctx->stream));   // the last kernel reading the frame tables is queued
    ctx->plan_ev_live = true;
    return W2X_OK;
}

// The three launches of a TTA step around its units, on the context's stream: the variants kernel of the planes the context owns,
// the units of the variants it converts, the mean kernel of its planes (which reads the tables last).
int tta_variants(w2x_ctx *ctx, const Step &s) {
    CU_CHECK(launch_tta_variants(s.vtab, (int)s.w.size(), s.vtiles, ctx->stream));
    ctx->launches++;
    return W2X_OK;
}

int run_units(w2x_ctx *ctx, const Step &s, const std::vector<FrameDev> &fd, int block_splitting) {
    for (const PlanesUnit &u : units_of(s))
        if (int rc = run_unit(ctx, s, fd, u, block_splitting)) return rc;
    return W2X_OK;
}

int tta_mean(w2x_ctx *ctx, const Step &s) {
    CU_CHECK(launch_tta_mean(s.mtab, (int)s.w.size(), s.mtiles, ctx->stream));
    ctx->launches++;
    CU_CHECK(cudaEventRecord(ctx->plan_ev, ctx->stream));
    ctx->plan_ev_live = true;
    return W2X_OK;
}

// The launches of one prepared step, after its progress lines: its units, for a TTA step between the variants kernel and the mean
// kernel.
int run_step(w2x_ctx *ctx, const Step &s, const std::vector<FrameDev> &fd, int block_splitting) {
    int rc = s.tta ? tta_variants(ctx, s) : W2X_OK;
    if (!rc) rc = run_units(ctx, s, fd, block_splitting);
    if (!rc && s.tta) rc = tta_mean(ctx, s);
    return rc;
}

// on_step(k), then the step's (resized) planes' lines, plane by plane, as the single-plane entry point prints them.  A packed
// plane's padded rectangle fits the scratch limit and MAX_FRAME_ROWS (plan_planes), so it is one scratch band: its lines come once.
void begin_step(w2x_ctx *ctx, const std::vector<Step> &steps, size_t k, int block_splitting, w2x_step_fn on_step, void *user, bool host) {
    if (on_step) on_step((int)k, user);
    const Step &s = steps[k];
    for (size_t i = 0; i < s.w.size(); i++) emit_plane_progress(ctx, s.m, s.w[i], s.h[i], block_splitting, host);
}

// Steps [k0, k1) of prepared steps, in order on the context's stream.
int run_steps(w2x_ctx *ctx, const std::vector<Step> &steps, const std::vector<FrameDev> &fd, size_t k0, size_t k1, int block_splitting,
              w2x_step_fn on_step, void *user, bool host) {
    for (size_t k = k0; k < k1; k++) {
        begin_step(ctx, steps, k, block_splitting, on_step, user, host);
        if (int rc = run_step(ctx, steps[k], fd, block_splitting)) return rc;
    }
    return W2X_OK;
}

// Device planes, checked: the steps in order on the context's stream (pack: see reserve_part).
int planes_device(w2x_ctx *ctx, std::vector<Step> &steps, const float *const *d_in, const size_t *in_strides, float *const *d_out,
                  const size_t *out_strides, bool pack, int block_splitting, w2x_step_fn on_step, void *user) {
    std::vector<Part> parts{one_part(ctx, steps)};
    Part &P = parts[0];
    P.ends.resize(P.own.size());
    for (size_t i = 0; i < P.ends.size(); i++) P.ends[i] = PlaneIO{d_in[i], in_strides[i], d_out[i], out_strides[i]};
    int rc = prepare_parts(parts, pack, block_splitting);
    if (rc) return rc;
    return run_steps(ctx, P.steps, P.fd, 0, P.steps.size(), block_splitting, on_step, user, false);
}

// Host planes, checked, on parts (one per context) of the call's step table `all`, staged densely on each part's context, inputs in
// io_buf[0] and outputs in io_buf[1], and ONE run of a copy pipeline per part.  Each unit of step 0 is a group carrying its planes'
// uploads, each step between the first and the last one compute-only group, each unit of the last step a group carrying its planes'
// downloads: uploads overlap the first step and downloads the last.  A TTA step is three groups: the variants kernel (carrying the
// uploads at step 0), the units of the variants, the mean kernel (carrying the downloads at the last step).  Every part's groups are
// queued before any part is waited for, phase by phase (a plain step is one phase, a TTA step three), and on_step(k) and step k's lines
// (through `log`) come before its first phase.  Between parts, the units of a TTA step wait for every other part's variants kernel
// (tta_ev[0]) and a mean kernel for every other part's units (tta_ev[1]): every record is queued before the waits that name it.
// host_lines: each step logs its planes' lines as the host entry points do (emit_plane_progress), else as the device ones.
int planes_host(w2x_ctx *log, const std::vector<Step> &all, std::vector<Part> &parts, const float *const *in, const int *widths,
                const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user,
                bool host_lines = true) {
    const size_t np = parts.size(), last = all.size() - 1;
    std::vector<std::vector<size_t>> in_off(np), out_off(np);
    for (size_t p = 0; p < np; p++) {
        Part &P = parts[p];
        const Step &L = P.steps.back();
        const size_t n = P.own.size();
        in_off[p].assign(n + 1, 0);
        out_off[p].assign(n + 1, 0);
        for (size_t i = 0; i < n; i++) {
            const int g = P.own[i];
            in_off[p][i + 1] = in_off[p][i] + (size_t)widths[g] * heights[g];
            out_off[p][i + 1] = out_off[p][i] + (size_t)L.w[i] * L.h[i];
        }
        DeviceGuard dg(P.ctx->device);
        int rc = reserve_io(P.ctx, in_off[p].back() * sizeof(float), out_off[p].back() * sizeof(float));
        if (rc) return rc;
        P.ends.resize(n);
        for (size_t i = 0; i < n; i++)
            P.ends[i] = PlaneIO{P.ctx->io_buf[0].get() + in_off[p][i], (size_t)widths[P.own[i]] * 4, P.ctx->io_buf[1].get() + out_off[p][i], (size_t)L.w[i] * 4};
    }
    int rc = prepare_parts(parts, true, 0);
    if (rc) return rc;
    std::vector<std::vector<HostGroup>> groups(np);
    std::vector<std::vector<int>> upto(np);   // [part][phase]: how many of the part's groups are queued by the end of the phase
    for (size_t p = 0; p < np; p++) {
        Part &P = parts[p];
        w2x_ctx *ctx = P.ctx;
        std::vector<HostGroup> &G = groups[p];
        auto copies = [&, p](HostGroup &g, const std::vector<int> &planes, bool up, bool down) {
            const Step &L = P.steps.back();
            for (int i : planes) {
                const int gi = P.own[(size_t)i];
                const size_t row = (size_t)widths[gi] * 4, out_row = (size_t)L.w[(size_t)i] * 4;
                if (up) g.up.push_back({P.ctx->io_buf[0].get() + in_off[p][(size_t)i], row, in[gi], in_strides[gi], row, (size_t)heights[gi]});
                if (down)
                    g.down.push_back({out[gi], out_strides[gi], P.ctx->io_buf[1].get() + out_off[p][(size_t)i], out_row, out_row, (size_t)L.h[(size_t)i]});
            }
        };
        std::vector<int> mine(P.own.size());
        for (size_t i = 0; i < mine.size(); i++) mine[i] = (int)i;
        auto add = [&](HostGroup &&g) { G.push_back(std::move(g)); };
        for (size_t k = 0; k <= last; k++) {
            const Step &s = P.steps[k];
            if (s.tta) {
                if (!mine.empty()) {
                    HostGroup g;
                    copies(g, mine, k == 0, false);
                    g.compute = [ctx, &s] {
                        int rc = tta_variants(ctx, s);
                        if (!rc) CU_CHECK(cudaEventRecord(ctx->tta_ev[0], ctx->stream));
                        return rc;
                    };
                    add(std::move(g));
                }
                upto[p].push_back((int)G.size());
                if (!s.vof.empty()) {
                    HostGroup g;
                    g.compute = [&parts, &P, &s, k] {
                        for (const Part &Q : parts)
                            if (&Q != &P && !Q.own.empty()) CU_CHECK(cudaStreamWaitEvent(P.ctx->stream, Q.ctx->tta_ev[0], 0));
                        int rc = run_units(P.ctx, s, P.fd, 0);
                        if (!rc) CU_CHECK(cudaEventRecord(P.ctx->tta_ev[1], P.ctx->stream));
                        return rc;
                    };
                    add(std::move(g));
                }
                upto[p].push_back((int)G.size());
                if (!mine.empty()) {
                    HostGroup g;
                    copies(g, mine, false, k == last);
                    g.compute = [&parts, &P, &s, k] {
                        for (const Part &Q : parts)
                            if (&Q != &P && !Q.steps[k].vof.empty()) CU_CHECK(cudaStreamWaitEvent(P.ctx->stream, Q.ctx->tta_ev[1], 0));
                        return tta_mean(P.ctx, s);
                    };
                    add(std::move(g));
                }
            } else if (k > 0 && k < last) {
                if (!mine.empty()) {
                    HostGroup g;
                    g.compute = [&P, &s] { return run_step(P.ctx, s, P.fd, 0); };
                    add(std::move(g));
                }
            } else {
                for (const PlanesUnit &u : units_of(s)) {
                    HostGroup g;
                    copies(g, u.planes, k == 0, k == last);
                    g.compute = [&P, &s, u] { return run_unit(P.ctx, s, P.fd, u, 0); };
                    add(std::move(g));
                }
            }
            upto[p].push_back((int)G.size());
        }
    }
    std::vector<HostPipe> pipes;
    for (size_t p = 0; p < np; p++) pipes.push_back(HostPipe{parts[p].ctx, groups[p]});
    for (size_t p = 0; p < np && !rc; p++) rc = pipes[p].start();
    for (size_t k = 0, ph = 0; k <= last && !rc; k++) {
        begin_step(log, all, k, 0, on_step, user, host_lines);
        for (int t = 0; t < (all[k].tta ? 3 : 1) && !rc; t++, ph++)
            for (size_t p = 0; p < np && !rc; p++) rc = pipes[p].queue(upto[p][ph]);
    }
    for (HostPipe &pp : pipes) {
        const int r2 = pp.finish(rc);
        if (!rc) rc = r2;
    }
    return rc;
}

// The one-context host call.
int planes_host(w2x_ctx *ctx, std::vector<Step> &steps, const float *const *in, const int *widths, const int *heights,
                const size_t *in_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user,
                bool host_lines = true) {
    std::vector<Part> parts{one_part(ctx, steps)};
    return planes_host(ctx, parts[0].steps, parts, in, widths, heights, in_strides, out, out_strides, on_step, user, host_lines);
}

// ---- a collection across the GPUs of a w2x_multi (w2x_multi_convert_planes*) ----------------------------------------------------
// The work of a model per output pixel: 9 Cin Cout multiply-adds summed over its layers.
long long macs_per_pixel(const w2x_model *m) {
    long long s = 0;
    for (const Layer &L : m->layers) s += 9LL * L.n_in * L.n_out;
    return s;
}

// The placement of w2x_multi_convert_planes_chain on n_dev GPUs (include/w2x_b200.h): returns nd, the GPUs used, with owner[i] in
// [0, nd) and the planned work per GPU in load[0 .. nd).  A plane's plain steps run on its owner and variant j of its TTA steps on
// (owner + j) mod nd; planes are placed greedily in decreasing order of total work (ties: the lower index), each on the owner that
// keeps the largest load after it smallest (ties: the owner with the smaller load before it, then the lower index).
int plan_multi(int n_dev, const std::vector<Step> &steps, std::vector<int> *owner, std::vector<long long> *load) {
    const size_t n = steps[0].w.size();
    bool tta = false;
    for (const Step &s : steps) tta = tta || s.tta;
    const int nd = (int)std::min<long long>(n_dev, (tta ? 8LL : 1LL) * (long long)n);
    std::vector<long long> plain(n, 0), var(n, 0);   // a plane's work on its owner, and per variant of its TTA steps
    for (const Step &s : steps) {
        const long long macs = macs_per_pixel(s.m);
        for (size_t i = 0; i < n; i++) (s.tta ? var : plain)[i] += (long long)s.w[i] * s.h[i] * macs;
    }
    std::vector<int> order(n);
    for (size_t i = 0; i < n; i++) order[i] = (int)i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return plain[(size_t)a] + 8 * var[(size_t)a] > plain[(size_t)b] + 8 * var[(size_t)b]; });
    owner->assign(n, 0);
    load->assign((size_t)nd, 0);
    std::vector<long long> &L = *load, with(L);
    for (int i : order) {
        int best = -1;
        long long best_max = 0;
        for (int o = 0; o < nd; o++) {
            with = L;
            with[(size_t)o] += plain[(size_t)i];
            for (int j = 0; j < 8 && tta; j++) with[(size_t)((o + j) % nd)] += var[(size_t)i];
            const long long mx = *std::max_element(with.begin(), with.end());
            if (best < 0 || mx < best_max || (mx == best_max && L[(size_t)o] < L[(size_t)best])) {
                best = o;
                best_max = mx;
            }
        }
        (*owner)[(size_t)i] = best;
        L[(size_t)best] += plain[(size_t)i];
        for (int j = 0; j < 8 && tta; j++) L[(size_t)((best + j) % nd)] += var[(size_t)i];
    }
    return nd;
}
}  // namespace

namespace w2x {
namespace eng {
int multi_planes_chain(const char *fn, const std::vector<w2x_ctx *> &ctxs, int n_steps, const w2x_model *const *models, const int *kinds,
                       int n_planes, const float *const *in, const int *widths, const int *heights, const size_t *in_strides,
                       float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user) {
    w2x_ctx *ctx0 = ctxs[0];
    std::vector<Step> all;
    int rc = check_planes_chain(fn, ctx0, n_steps, models, kinds, n_planes, in, widths, heights, in_strides, out, out_strides, &all);
    if (rc) return rc;
    std::vector<int> owner;
    std::vector<long long> load;
    const int nd = plan_multi((int)ctxs.size(), all, &owner, &load);
    if (nd == 1) return w2x_convert_planes_chain(ctx0, n_steps, models, kinds, n_planes, in, widths, heights, in_strides, out, out_strides, on_step, user);
    bool tta = false;
    for (const Step &s : all) tta = tta || s.tta;
    for (int a = 0; a < nd && tta; a++)   // a TTA step's kernels on one GPU store to and load from the others' buffers
        for (int b = 0; b < nd; b++) {
            const int da = ctxs[(size_t)a]->device, db = ctxs[(size_t)b]->device;
            if (da == db) continue;
            int can = 0;
            CU_CHECK(cudaDeviceCanAccessPeer(&can, da, db));
            if (!can) return fail(W2X_ERR_UNSUPPORTED, "%s: device %d cannot map the memory of device %d (no peer access)", fn, da, db);
            DeviceGuard g(da);
            cudaError_t e = cudaDeviceEnablePeerAccess(db, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU_CHECK(e);
            cudaGetLastError();
        }
    std::vector<Part> parts((size_t)nd);
    for (int i = 0; i < n_planes; i++) parts[(size_t)owner[(size_t)i]].own.push_back(i);
    for (int d = 0; d < nd; d++) {
        Part &P = parts[(size_t)d];
        P.ctx = ctxs[(size_t)d];
        P.ctx->precision = ctx0->precision;
        P.ctx->engine = ctx0->engine;
        std::vector<std::vector<int>> vof(all.size());
        for (size_t k = 0; k < all.size(); k++)
            for (int i = 0; i < n_planes && all[k].tta; i++)
                for (int j = 0; j < 8; j++)
                    if ((owner[(size_t)i] + j) % nd == d) vof[k].push_back(8 * i + j);
        P.steps = part_steps(all, P.own, vof);
    }
    NvtxRange nvtx("w2x multi convert planes chain");
    const Step &L = all.back();
    std::vector<std::unique_ptr<HostPin>> pins;
    for (int i = 0; i < n_planes; i++) {
        pins.push_back(std::make_unique<HostPin>(in[i], in_strides[i] * (size_t)(heights[i] - 1) + (size_t)widths[i] * 4));
        pins.push_back(std::make_unique<HostPin>(out[i], out_strides[i] * (size_t)(L.h[(size_t)i] - 1) + (size_t)L.w[(size_t)i] * 4));
    }
    return planes_host(ctx0, all, parts, in, widths, heights, in_strides, out, out_strides, on_step, user);
}
}  // namespace eng
}  // namespace w2x

extern "C" {
// Test hook (not part of the stable ABI): the placement of w2x_multi_convert_planes_chain on n_devices GPUs, without a device.  owner
// gets every plane's GPU, load (n_devices entries) the planned work per GPU used.  Returns the number of GPUs used, or -W2X_ERR_ARG.
W2X_API int w2x_debug_plan_multi_planes(int n_devices, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                                        const int *widths, const int *heights, int *owner, long long *load) {
    if (n_devices < 1 || n_steps < 1 || !models || !kinds || n_planes < 1 || !widths || !heights || !owner || !load)
        return -fail(W2X_ERR_ARG, "w2x_debug_plan_multi_planes: bad argument");
    for (int k = 0; k < n_steps; k++)
        if (!models[k] || kinds[k] & ~(W2X_STEP_UPSCALE2X | W2X_STEP_TTA)) return -fail(W2X_ERR_ARG, "w2x_debug_plan_multi_planes: step %d", k);
    for (int i = 0; i < n_planes; i++)
        if (widths[i] < 1 || heights[i] < 1) return -fail(W2X_ERR_ARG, "w2x_debug_plan_multi_planes: plane %d has no pixels", i);
    std::vector<int> own;
    std::vector<long long> ld;
    const int nd = plan_multi(n_devices, step_table(n_steps, models, kinds, n_planes, widths, heights), &own, &ld);
    std::copy(own.begin(), own.end(), owner);
    std::copy(ld.begin(), ld.end(), load);
    return nd;
}
}  // extern "C"

namespace w2x {
namespace eng {
// The host tiles of w2x_convert_tiles*, all checked before anything is queued.
int check_tiles(w2x_ctx *ctx, const float *const *in_tiles, float *const *out_tiles, int n_tiles, int width, int height, size_t in_stride_bytes,
                size_t out_stride_bytes) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!in_tiles || !out_tiles || n_tiles < 1 || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_convert_tiles: bad argument");
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_tiles: row stride smaller than a row");
    for (int t = 0; t < n_tiles; t++)
        if (!in_tiles[t] || !out_tiles[t]) return fail(W2X_ERR_ARG, "w2x_convert_tiles: NULL tile %d", t);
    return W2X_OK;
}

// phase 1: uploads + the batched pass (results stay in the context's staging buffer); phase 2: downloads.  Split so that a
// multi-GPU driver can queue phase 1 everywhere before a download into pageable memory blocks its thread.  Phase 1 checks the
// tiles of both phases.
int tiles_enqueue_compute(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles, int width,
                          int height, size_t in_stride_bytes, size_t out_stride_bytes) {
    int rc = check_tiles(ctx, in_tiles, out_tiles, n_tiles, width, height, in_stride_bytes, out_stride_bytes);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    const size_t tile_bytes = (size_t)width * height * sizeof(float);
    rc = reserve_io(ctx, tile_bytes * (size_t)n_tiles, tile_bytes * (size_t)n_tiles);
    if (rc) return rc;
    for (int t = 0; t < n_tiles; t++)
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(ctx->io_buf[0].get()) + tile_bytes * (size_t)t, (size_t)width * 4, in_tiles[t], in_stride_bytes,
                                   (size_t)width * 4, (size_t)height, cudaMemcpyHostToDevice, ctx->stream));
    return convert_tiles_dev(ctx, model, ctx->io_buf[0].get(), ctx->io_buf[1].get(), n_tiles, width, height);
}

int tiles_enqueue_download(w2x_ctx *ctx, float *const *out_tiles, int n_tiles, int width, int height, size_t out_stride_bytes) {
    DeviceGuard g(ctx->device);
    const size_t tile_bytes = (size_t)width * height * sizeof(float);
    for (int t = 0; t < n_tiles; t++)
        CU_CHECK(cudaMemcpy2DAsync(out_tiles[t], out_stride_bytes, reinterpret_cast<char *>(ctx->io_buf[1].get()) + tile_bytes * (size_t)t, (size_t)width * 4,
                                   (size_t)width * 4, (size_t)height, cudaMemcpyDeviceToHost, ctx->stream));
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
    int rc = tiles_enqueue_compute(ctx, model, in_tiles, out_tiles, n_tiles, width, height, in_stride_bytes, out_stride_bytes);
    if (rc) return rc;
    return tiles_enqueue_download(ctx, out_tiles, n_tiles, width, height, out_stride_bytes);
}

int w2x_convert_tiles(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles,
                      int width, int height, size_t in_stride_bytes, size_t out_stride_bytes) {
    int rc = check_tiles(ctx, in_tiles, out_tiles, n_tiles, width, height, in_stride_bytes, out_stride_bytes);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    const size_t tile_px = (size_t)width * height, row = (size_t)width * 4;
    rc = reserve_io(ctx, tile_px * sizeof(float) * (size_t)n_tiles, tile_px * sizeof(float) * (size_t)n_tiles);
    if (rc) return rc;
    float *din = ctx->io_buf[0].get(), *dout = ctx->io_buf[1].get();
    // Larger batches run as up to four groups: the uploads of group g+1 and the downloads of group g-1 overlap the layers of
    // group g (copy engines + compute), as the row bands of w2x_convert_plane do.  Tiles are independent, so the grouping
    // does not change a bit of any of them.
    const int ng = n_tiles >= 8 ? std::min(4, n_tiles / 4) : 1;
    std::vector<HostGroup> groups((size_t)ng);
    for (int gi = 0; gi < ng; gi++) {
        const int t0 = (int)((long)n_tiles * gi / ng), t1 = (int)((long)n_tiles * (gi + 1) / ng);
        for (int t = t0; t < t1; t++) {
            groups[(size_t)gi].up.push_back({din + tile_px * (size_t)t, row, in_tiles[t], in_stride_bytes, row, (size_t)height});
            groups[(size_t)gi].down.push_back({out_tiles[t], out_stride_bytes, dout + tile_px * (size_t)t, row, row, (size_t)height});
        }
        groups[(size_t)gi].compute = [=] {
            return convert_tiles_dev(ctx, model, din + tile_px * (size_t)t0, dout + tile_px * (size_t)t0, t1 - t0, width, height);
        };
    }
    return run_host_groups(ctx, groups);
}

int w2x_convert_planes_device(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *d_in, const int *widths,
                              const int *heights, const size_t *in_strides, float *const *d_out, const size_t *out_strides) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    int rc = check_planes("w2x_convert_planes_device", model, n_planes, d_in, widths, heights, in_strides, d_out, out_strides);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    if (pick_engine(ctx, model) < 0) return W2X_ERR_UNSUPPORTED;
    std::vector<Step> steps = one_step(model, n_planes, widths, heights);
    return planes_device(ctx, steps, d_in, in_strides, d_out, out_strides, true, 0, nullptr, nullptr);
}

int w2x_convert_planes(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *in, const int *widths,
                       const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    int rc = check_planes("w2x_convert_planes", model, n_planes, in, widths, heights, in_strides, out, out_strides);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    if (pick_engine(ctx, model) < 0) return W2X_ERR_UNSUPPORTED;
    std::vector<Step> steps = one_step(model, n_planes, widths, heights);
    return planes_host(ctx, steps, in, widths, heights, in_strides, out, out_strides, nullptr, nullptr);
}

int w2x_convert_planes_chain_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                                    const float *const *d_in, const int *widths, const int *heights, const size_t *in_strides,
                                    float *const *d_out, const size_t *out_strides, w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_planes_chain("w2x_convert_planes_chain_device", ctx, n_steps, models, kinds, n_planes, d_in, widths, heights, in_strides,
                                d_out, out_strides, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert planes chain");
    return planes_device(ctx, steps, d_in, in_strides, d_out, out_strides, true, 0, on_step, user);
}

int w2x_convert_planes_chain(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                             const float *const *in, const int *widths, const int *heights, const size_t *in_strides, float *const *out,
                             const size_t *out_strides, w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_planes_chain("w2x_convert_planes_chain", ctx, n_steps, models, kinds, n_planes, in, widths, heights, in_strides, out,
                                out_strides, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert planes chain");
    return planes_host(ctx, steps, in, widths, heights, in_strides, out, out_strides, on_step, user);
}

}  // extern "C"

// ---- chains of conversions on one plane (w2x_convert_chain*) ---------------------------------------------------------------
// The reference's main loop (src/main.cpp:82-156) runs the Y plane through the noise model (:96) and then through k scale
// iterations, each a nearest-neighbour 2x resize (:132-140) followed by the scale model (:148).  The Y plane after a step depends
// only on the Y plane before it, so the whole sequence stays on the device: intermediate planes live in ctx->chain_buf, and an
// upscaling step reads its half-resolution source through the first layer (or the padding kernel) instead of a 2x plane.
// The steps run as those of w2x_convert_planes_chain* on a collection of one plane that never packs into a frame: each step is one
// convert_device call with the caller's block_splitting.
namespace {
// Every argument of w2x_convert_chain*: the steps, then the plane, W2X_ERR_ARG naming the step it concerns.
int check_chain(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, const void *in, int width,
                int height, size_t in_stride_bytes, const void *out, size_t out_stride_bytes, int block_splitting, bool host,
                std::vector<Step> *steps) {
    return check_steps(fn, ctx, n_steps, models, kinds, 1, &width, &height, block_splitting, [&](int) -> int {
        if (width < 1 || height < 1) return fail(W2X_ERR_ARG, "%s: step 0: input size %d x %d", fn, width, height);
        if (!in) return fail(W2X_ERR_ARG, "%s: step 0: NULL input plane", fn);
        if (in_stride_bytes % 4 || in_stride_bytes < (size_t)width * 4)
            return fail(W2X_ERR_ARG, "%s: step 0: the input row stride must be a multiple of 4 bytes and >= width*4", fn);
        long w = width, h = height;
        for (int k = 0; k < n_steps; k++)
            if (kinds[k] & W2X_STEP_UPSCALE2X) {
                w *= 2;
                h *= 2;
                if (w > INT_MAX || h > INT_MAX) return fail(W2X_ERR_ARG, "%s: step %d: the output size %ld x %ld overflows int", fn, k, w, h);
            }
        const int last = n_steps - 1;
        if (!out) return fail(W2X_ERR_ARG, "%s: step %d: NULL output plane", fn, last);
        if (out_stride_bytes % 4 || out_stride_bytes < (size_t)w * 4)
            return fail(W2X_ERR_ARG, "%s: step %d: the output row stride must be a multiple of 4 bytes and >= width*4 (%ld)", fn, last, w * 4);
        if (host) {   // device planes may alias in ways the host cannot see; host planes are checked
            const char *i0 = static_cast<const char *>(in), *i1 = i0 + (size_t)(height - 1) * in_stride_bytes + (size_t)width * 4;
            const char *o0 = static_cast<const char *>(out), *o1 = o0 + (size_t)(h - 1) * out_stride_bytes + (size_t)w * 4;
            if (i0 < o1 && o0 < i1) return fail(W2X_ERR_ARG, "%s: step %d: the output plane overlaps the input plane", fn, last);
        }
        return W2X_OK;
    }, steps);
}

// Host plane, staged densely in io_buf[0] (input) and io_buf[1] (output).  The last step runs as groups of the copy pipeline: the
// row bands of host_copy_bands when it cuts the plane, so that the download of band i overlaps the layers of band i + 1, else one.
// An upscaling step's bands start on even 2x rows (the source row of a band's first row is then whole).  When the last step is
// step 0, group i also uploads the input rows that band i is the first to read, so that uploads overlap the layers as well;
// otherwise one upload and steps 0 ... n - 2 go first on the context's stream.  A TTA last step is one group: its download waits for
// the mean kernel.
int chain_host(w2x_ctx *ctx, std::vector<Step> &table, const float *in, int width, int height, size_t in_stride_bytes, float *out,
               size_t out_stride_bytes, int block_splitting, w2x_step_fn on_step, void *user) {
    std::vector<Part> parts{one_part(ctx, table)};
    std::vector<Step> &steps = parts[0].steps;
    std::vector<FrameDev> &fd = parts[0].fd;
    const size_t last = steps.size() - 1;
    const w2x_model *m = steps[last].m;
    const bool up = steps[last].up, band_uploads = last == 0 && !steps[last].tta;
    const int n = (int)m->layers.size(), w = steps[last].w[0], h = steps[last].h[0];
    const int nb = steps[last].tta ? 1 : host_copy_bands(ctx, n, w, h, block_splitting);
    auto band_y = [&](int i) { return (int)((long)h * i / nb) & (up ? ~1 : ~0); };
    for (int i = 0; i < nb && nb > 1; i++) parts[0].band_rows = std::max(parts[0].band_rows, band_y(i + 1) - band_y(i));
    const size_t in_dense = (size_t)width * 4;
    int rc = reserve_io(ctx, (size_t)width * height * sizeof(float), (size_t)w * h * sizeof(float));
    parts[0].ends = {PlaneIO{ctx->io_buf[0].get(), in_dense, ctx->io_buf[1].get(), (size_t)w * 4}};
    if (!rc) rc = prepare_parts(parts, false, block_splitting);
    if (rc) return rc;
    if (!band_uploads)
        CU_CHECK(cudaMemcpy2DAsync(ctx->io_buf[0].get(), in_dense, in, in_stride_bytes, in_dense, (size_t)height, cudaMemcpyHostToDevice, ctx->stream));
    rc = run_steps(ctx, steps, fd, 0, last, block_splitting, on_step, user, true);
    if (rc) {   // the upload may still read the caller's plane
        cudaStreamSynchronize(ctx->stream);
        return rc;
    }
    const PlaneIO io = steps[last].io[0];
    begin_step(ctx, steps, last, block_splitting, on_step, user, true);
    if (steps[last].tta) {   // the download follows the mean kernel, which needs every variant's whole output
        std::vector<HostGroup> one(1);
        one[0].compute = [&] { return run_step(ctx, steps[last], fd, block_splitting); };
        one[0].down = {{out, out_stride_bytes, io.dst, io.dst_stride, io.dst_stride, (size_t)h}};
        return run_host_groups(ctx, one);
    }
    // band_uploads: upload i carries input rows [u(i), u(i + 1)); band i reads source rows up to (band_y(i + 1) + n - 1) >> up, its n
    // rows of context below included, so that it waits for its own upload only
    auto u = [&](int i) { return i == 0 ? 0 : i == nb ? height : std::min(height, ((band_y(i) + n - 1) >> (up ? 1 : 0)) + 1); };
    std::vector<HostGroup> groups((size_t)nb);
    for (int i = 0; i < nb; i++) {
        const int y = band_y(i), rows = band_y(i + 1) - y;
        const float *band_src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(io.src) + (size_t)(up ? y / 2 : y) * io.src_stride);
        float *band_dst = io.dst + (size_t)y * w;
        if (band_uploads)
            groups[(size_t)i].up = {{ctx->io_buf[0].get() + (size_t)u(i) * width, in_dense, reinterpret_cast<const char *>(in) + (size_t)u(i) * in_stride_bytes,
                                     in_stride_bytes, in_dense, (size_t)(u(i + 1) - u(i))}};
        groups[(size_t)i].compute = [=] {
            return convert_device(ctx, m, band_src, w, rows, io.src_stride, i > 0 ? n : 0, i + 1 < nb ? n : 0, band_dst, io.dst_stride,
                                  nb > 1 ? 0 : block_splitting, up);
        };
        groups[(size_t)i].down = {{reinterpret_cast<char *>(out) + (size_t)y * out_stride_bytes, out_stride_bytes, band_dst, io.dst_stride,
                                   io.dst_stride, (size_t)rows}};
    }
    return run_host_groups(ctx, groups);
}
}  // namespace

namespace w2x {
namespace eng {
int check_chain_host(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, const float *in, int width,
                     int height, size_t in_stride_bytes, const float *out, size_t out_stride_bytes, int block_splitting) {
    std::vector<Step> steps;
    return check_chain(fn, ctx, n_steps, models, kinds, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting, true, &steps);
}
}  // namespace eng
}  // namespace w2x

extern "C" {

// The plane entry points: a one-step W2X_STEP_SAME w2x_convert_chain_device / w2x_convert_chain behind their own argument checks.
int w2x_convert_plane_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, int width, int height,
                             size_t in_stride_bytes, float *d_out, size_t out_stride_bytes, int block_splitting) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    int rc = check_plane(ctx, model, d_in, width, height, in_stride_bytes, d_out, out_stride_bytes, block_splitting);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    std::vector<Step> steps = one_step(model, 1, &width, &height);
    return planes_device(ctx, steps, &d_in, &in_stride_bytes, &d_out, &out_stride_bytes, false, block_splitting, nullptr, nullptr);
}

int w2x_convert_plane(w2x_ctx *ctx, const w2x_model *model, const float *in, int width, int height, size_t in_stride_bytes,
                      float *out, size_t out_stride_bytes, int block_splitting) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || !in || !out || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_convert_plane: bad argument");
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4)
        return fail(W2X_ERR_ARG, "w2x_convert_plane: row stride smaller than a row");
    const size_t row = (size_t)width * 4;
    int rc = check_plane(ctx, model, in, width, height, row, out, row, block_splitting);   // the rest, on the dense staged planes
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    std::vector<Step> steps = one_step(model, 1, &width, &height);
    return chain_host(ctx, steps, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting, nullptr, nullptr);
}

int w2x_convert_chain_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, const float *d_in, int width,
                             int height, size_t in_stride_bytes, float *d_out, size_t out_stride_bytes, int block_splitting,
                             w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_chain("w2x_convert_chain_device", ctx, n_steps, models, kinds, d_in, width, height, in_stride_bytes, d_out, out_stride_bytes,
                         block_splitting, false, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain");
    return planes_device(ctx, steps, &d_in, &in_stride_bytes, &d_out, &out_stride_bytes, false, block_splitting, on_step, user);
}

int w2x_convert_chain(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, const float *in, int width, int height,
                      size_t in_stride_bytes, float *out, size_t out_stride_bytes, int block_splitting, w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_chain("w2x_convert_chain", ctx, n_steps, models, kinds, in, width, height, in_stride_bytes, out, out_stride_bytes,
                         block_splitting, true, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain");
    return chain_host(ctx, steps, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting, on_step, user);
}

}  // extern "C"

// ---- windows of a chain's output (w2x_convert_chain_region*, w2x_convert_chain_regions*) ----------------------------------------
// The steps of w2x_convert_planes_chain* on a collection of windows, step k converting each window's output window wins[k + 1] from
// its input window wins[k]: the source rectangle at step 0, else the previous step's output window, dense in chain_buf[(k - 1) & 1].
// A window is a plane of its own, with the real neighbours its input window holds beyond it as row and column context, so that
// only the plane's own border is replicated: converted alone by convert_device, or packed into a frame whose rectangle holds the
// same frame (window_frame).  No step has TTA, and every buffer is reserved by prepare_parts before the first launch, as for the
// other step-table calls.
namespace {
// The step table of the windows from the step table of their source rectangles: step k converts window i's output window
// wins[i][k + 1] from its input window wins[i][k] (region_windows).
void set_region_windows(std::vector<Step> &steps, const std::vector<std::vector<Rect>> &wins) {
    for (size_t k = 0; k < steps.size(); k++) {
        Step &t = steps[k];
        for (size_t i = 0; i < wins.size(); i++) {
            const Rect &w = wins[i][k + 1];
            t.w[i] = w.w, t.h[i] = w.h, t.x0[i] = w.x0, t.y0[i] = w.y0;
            t.in[i] = wins[i][k];
        }
    }
}

// Every argument of a region call on n_windows windows, before anything is printed, allocated or queued: the steps (no TTA) by
// region_windows, then each window by region_windows and its buffers, then each step's engine by check_steps.  numbered: the
// messages of a window's checks name it ("window i: ..."); the one-window call's do not.  Then *steps is the step table of the
// windows: step k converts window i's output window from its input window.
int check_regions(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows,
                  const int *widths, const int *heights, const int *windows, const void *const *src, const size_t *src_strides,
                  const void *const *out, const size_t *out_strides, bool numbered, std::vector<Step> *steps) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (numbered) {
        if (n_windows < 1) return fail(W2X_ERR_ARG, "%s: n_windows is %d, at least 1 window is needed", fn, n_windows);
        if (!widths || !heights || !windows || !src || !src_strides || !out || !out_strides) return fail(W2X_ERR_ARG, "%s: NULL array argument", fn);
        // the steps alone: every window's checks begin with them, and a 1 x 1 window of a 1 x 1 plane passes every other one
        const int unit[4] = {0, 0, 1, 1};
        std::vector<Rect> wins;
        if (int rc = region_windows(fn, n_steps, models, kinds, 1, 1, unit, &wins)) return rc;
    }
    std::vector<std::vector<Rect>> wins((size_t)n_windows);
    std::vector<int> sw((size_t)n_windows), sh((size_t)n_windows);
    for (int i = 0; i < n_windows; i++) {
        const std::string name = numbered ? std::string(fn) + ": window " + std::to_string(i) : std::string(fn);
        const char *wn = name.c_str();
        int rc = region_windows(wn, n_steps, models, kinds, widths[i], heights[i], windows + 4 * i, &wins[(size_t)i]);
        if (rc) return rc;
        const Rect &s = wins[(size_t)i].front(), &o = wins[(size_t)i].back();
        if (!src[i]) return fail(W2X_ERR_ARG, "%s: NULL source", wn);
        if (src_strides[i] % 4 || src_strides[i] < (size_t)s.w * 4)
            return fail(W2X_ERR_ARG, "%s: the source row stride must be a multiple of 4 bytes and >= the source rectangle's row (%d bytes)",
                        wn, s.w * 4);
        if (!out[i]) return fail(W2X_ERR_ARG, "%s: NULL output", wn);
        if (out_strides[i] % 4 || out_strides[i] < (size_t)o.w * 4)
            return fail(W2X_ERR_ARG, "%s: the output row stride must be a multiple of 4 bytes and >= the window's row (%d bytes)", wn,
                        o.w * 4);
        sw[(size_t)i] = s.w;
        sh[(size_t)i] = s.h;
    }
    int rc = check_steps(fn, ctx, n_steps, models, kinds, n_windows, sw.data(), sh.data(), 0, [](int) { return W2X_OK; }, steps);
    if (!rc) set_region_windows(*steps, wins);
    return rc;
}

int check_region(const char *fn, w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int width, int height,
                 const int *window, const void *src, size_t src_stride_bytes, const void *out, size_t out_stride_bytes,
                 std::vector<Step> *steps) {
    return check_regions(fn, ctx, n_steps, models, kinds, 1, &width, &height, window, &src, &src_stride_bytes, &out, &out_stride_bytes, false,
                         steps);
}
}  // namespace

extern "C" {

int w2x_convert_chain_region(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int width, int height,
                             const int *window, const float *src, size_t src_stride_bytes, float *out, size_t out_stride_bytes,
                             w2x_step_fn on_step, void *user) {
    std::vector<Step> table;
    int rc = check_region("w2x_convert_chain_region", ctx, n_steps, models, kinds, width, height, window, src, src_stride_bytes, out,
                          out_stride_bytes, &table);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain region");
    std::vector<Part> parts{one_part(ctx, table)};
    Part &P = parts[0];
    const Rect s = P.steps.front().in[0];
    const int ow = P.steps.back().w[0], oh = P.steps.back().h[0];
    const size_t srow = (size_t)s.w * sizeof(float), orow = (size_t)ow * sizeof(float);
    rc = reserve_io(ctx, srow * s.h, orow * oh);
    P.ends = {PlaneIO{ctx->io_buf[0].get(), srow, ctx->io_buf[1].get(), orow}};
    if (!rc) rc = prepare_parts(parts, false, 0);
    if (rc) return rc;
    std::vector<HostGroup> one(1);
    one[0].up = {{ctx->io_buf[0].get(), srow, src, src_stride_bytes, srow, (size_t)s.h}};
    one[0].compute = [&] { return run_steps(ctx, P.steps, P.fd, 0, P.steps.size(), 0, on_step, user, false); };
    one[0].down = {{out, out_stride_bytes, ctx->io_buf[1].get(), orow, orow, (size_t)oh}};
    return run_host_groups(ctx, one);
}

int w2x_convert_chain_region_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int width, int height,
                                    const int *window, const float *d_src, size_t src_stride_bytes, float *d_out, size_t out_stride_bytes,
                                    w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_region("w2x_convert_chain_region_device", ctx, n_steps, models, kinds, width, height, window, d_src, src_stride_bytes,
                          d_out, out_stride_bytes, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain region");
    return planes_device(ctx, steps, &d_src, &src_stride_bytes, &d_out, &out_stride_bytes, false, 0, on_step, user);
}

int w2x_convert_chain_regions(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows, const int *widths,
                              const int *heights, const int *windows, const float *const *src, const size_t *src_strides, float *const *out,
                              const size_t *out_strides, w2x_step_fn on_step, void *user) {
    std::vector<Step> steps;
    int rc = check_regions("w2x_convert_chain_regions", ctx, n_steps, models, kinds, n_windows, widths, heights, windows,
                           reinterpret_cast<const void *const *>(src), src_strides, reinterpret_cast<const void *const *>(out), out_strides,
                           true, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain regions");
    std::vector<int> sw((size_t)n_windows), sh((size_t)n_windows);   // the source rectangles, staged densely
    for (size_t i = 0; i < sw.size(); i++) sw[i] = steps[0].in[i].w, sh[i] = steps[0].in[i].h;
    return planes_host(ctx, steps, src, sw.data(), sh.data(), src_strides, out, out_strides, on_step, user, false);
}

int w2x_convert_chain_regions_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows,
                                     const int *widths, const int *heights, const int *windows, const float *const *d_src,
                                     const size_t *src_strides, float *const *d_out, const size_t *out_strides, w2x_step_fn on_step,
                                     void *user) {
    std::vector<Step> steps;
    int rc = check_regions("w2x_convert_chain_regions_device", ctx, n_steps, models, kinds, n_windows, widths, heights, windows,
                           reinterpret_cast<const void *const *>(d_src), src_strides, reinterpret_cast<const void *const *>(d_out),
                           out_strides, true, &steps);
    if (rc) return rc;
    DeviceGuard g(ctx->device);
    NvtxRange nvtx("w2x convert chain regions");
    return planes_device(ctx, steps, d_src, src_strides, d_out, out_strides, true, 0, on_step, user);
}

// Test hook (not part of the stable ABI): the placement of w2x_multi_convert_chain_regions on n_devices GPUs, without a device.
// owner gets every window's GPU, load (n_devices entries) the planned work per GPU used.  Returns the number of GPUs used, or
// -W2X_ERR_ARG.
W2X_API int w2x_debug_plan_multi_regions(int n_devices, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows,
                                         const int *widths, const int *heights, const int *windows, int *owner, long long *load) {
    const char *fn = "w2x_debug_plan_multi_regions";
    if (n_devices < 1 || n_windows < 1 || !widths || !heights || !windows || !owner || !load) return -fail(W2X_ERR_ARG, "%s: bad argument", fn);
    std::vector<std::vector<Rect>> wins((size_t)n_windows);
    std::vector<int> sw((size_t)n_windows), sh((size_t)n_windows);
    for (int i = 0; i < n_windows; i++) {
        const std::string name = std::string(fn) + ": window " + std::to_string(i);
        if (int rc = region_windows(name.c_str(), n_steps, models, kinds, widths[i], heights[i], windows + 4 * i, &wins[(size_t)i])) return -rc;
        sw[(size_t)i] = wins[(size_t)i][0].w;
        sh[(size_t)i] = wins[(size_t)i][0].h;
    }
    std::vector<Step> steps = step_table(n_steps, models, kinds, n_windows, sw.data(), sh.data());
    set_region_windows(steps, wins);
    std::vector<int> own;
    std::vector<long long> ld;
    const int nd = plan_multi(n_devices, steps, &own, &ld);
    std::copy(own.begin(), own.end(), owner);
    std::copy(ld.begin(), ld.end(), load);
    return nd;
}

}  // extern "C"

namespace w2x {
namespace eng {
// w2x_convert_chain_regions with every window on one owner GPU (plan_multi on the windows' step table): the owner stages its
// source rectangle, holds its intermediate windows and writes its output, so nothing crosses devices.
int multi_regions(const char *fn, const std::vector<w2x_ctx *> &ctxs, int n_steps, const w2x_model *const *models, const int *kinds,
                  int n_windows, const int *widths, const int *heights, const int *windows, const float *const *src,
                  const size_t *src_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user) {
    w2x_ctx *ctx0 = ctxs[0];
    std::vector<Step> all;
    int rc = check_regions(fn, ctx0, n_steps, models, kinds, n_windows, widths, heights, windows,
                           reinterpret_cast<const void *const *>(src), src_strides, reinterpret_cast<const void *const *>(out), out_strides,
                           true, &all);
    if (rc) return rc;
    std::vector<int> owner;
    std::vector<long long> load;
    const int nd = plan_multi((int)ctxs.size(), all, &owner, &load);
    if (nd == 1)
        return w2x_convert_chain_regions(ctx0, n_steps, models, kinds, n_windows, widths, heights, windows, src, src_strides, out,
                                         out_strides, on_step, user);
    std::vector<Part> parts((size_t)nd);
    for (int i = 0; i < n_windows; i++) parts[(size_t)owner[(size_t)i]].own.push_back(i);
    for (int d = 0; d < nd; d++) {
        Part &P = parts[(size_t)d];
        P.ctx = ctxs[(size_t)d];
        P.ctx->precision = ctx0->precision;
        P.ctx->engine = ctx0->engine;
        P.steps = part_steps(all, P.own, std::vector<std::vector<int>>(all.size()));
    }
    NvtxRange nvtx("w2x multi convert chain regions");
    const Step &L = all.back();
    std::vector<int> sw((size_t)n_windows), sh((size_t)n_windows);   // the source rectangles, staged densely
    std::vector<HostRange> ranges;
    for (size_t i = 0; i < sw.size(); i++) {
        sw[i] = all[0].in[i].w, sh[i] = all[0].in[i].h;
        ranges.push_back({src[i], src_strides[i] * (size_t)(sh[i] - 1) + (size_t)sw[i] * 4});
        ranges.push_back({out[i], out_strides[i] * (size_t)(L.h[i] - 1) + (size_t)L.w[i] * 4});
    }
    HostPins pins(ranges);
    return planes_host(ctx0, all, parts, src, sw.data(), sh.data(), src_strides, out, out_strides, on_step, user, false);
}
}  // namespace eng
}  // namespace w2x
