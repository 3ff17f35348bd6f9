// engine_band.cu -- multi-GPU: row-band sessions with a halo exchange between layers, the peer-memory exchange itself, and
// the one-process N-GPU driver (w2x_multi_*).
//
// BASELINE.json north_star: "the full-resolution plane is tiled with halo overlap across the GPUs of one box, halos
// exchanged ... over NVLink between layers".  A plane is cut into contiguous row bands, one per GPU.  Every intermediate
// activation of a band lives in a frame of band_rows + one halo row per neighbour side (+ the replicated n-pixel ring at
// the image border, reference src/convertRoutine.cpp:35,96); after every layer each GPU stores its boundary row of the
// fresh activation straight into the neighbour's halo row.  Two ways to move those rows:
//   * w2x_band_exchange  -- inside the library: the neighbours' frames are peer-mapped (cudaDeviceEnablePeerAccess in one
//                           process, CUDA IPC between the ranks of a torchrun job) and ONE small kernel per layer stores
//                           the rows over NVLink, publishes a flag in the receiver's memory and waits for the neighbours'
//                           flags.  No host round trip, no collective library, nothing between two layer launches but that
//                           kernel.  w2x_band_run queues a whole pass; w2x_multi_* drives N GPUs from one host thread.
//   * w2x_band_halo      -- the segments are handed to the caller (ncclSend/ncclRecv, torch.distributed P2P): the
//                           cross-check path, bit-identical.
// The layer kernels never store a band's halo rows (their output tensor maps exclude them), so a neighbour may deliver
// its row as early as it likes.  Results are bit-identical to the single-GPU pass: every output pixel sees the same
// operands in the same order.
#include <functional>

#include "engine_internal.h"

using namespace w2x;
using namespace w2x::eng;

namespace {

int band_check(w2x_band *b) {
    if (!b || !b->ctx || !b->model) return fail(W2X_ERR_ARG, "NULL band session");
    return W2X_OK;
}

// The bytes of one row of the frame traded after `step` (-1 = the padded input frame).  A row is one contiguous range, and row r of
// a frame, the owner's or the neighbour's, is at base + r * row_bytes.
size_t row_bytes(const w2x_band *b, int step) {
    if (step == -1) return (size_t)b->pw * sizeof(float);
    if (step == b->n - 2) return (size_t)b->pw * 12 * sizeof(float);             // per-pixel tap partials [hf][pw][12] fp32
    return 4 * (size_t)b->pw * (size_t)b->model->layers[(size_t)step].n_out;    // RECORD frame: 4 bytes per element
}

// w2x_band_load_rows, also through the nearest 2x resize: with up2x the band's rows are 2x rows of a half-resolution plane, the band
// starts on an even one, and d_in points at the source row holding it; an overlap edge then reads the ceil(n / 2) source rows beyond.
int band_load_rows_from(w2x_band *band, const float *d_in, size_t in_stride_bytes, bool up2x) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (!d_in || in_stride_bytes % 4 || in_stride_bytes < (size_t)(up2x ? (band->width + 1) / 2 : band->width) * 4)
        return fail(W2X_ERR_ARG, "w2x_band_load_rows: bad input");
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    const FrameSource src{d_in, (long)(in_stride_bytes / 4), band->width, band->rows, band->n, band->pt, band->ov_up ? band->n : 0,
                          band->ov_down ? band->n : 0, up2x};
    CU_CHECK(launch_pad(src, band->pw, band->hf, band->pad.get(), ctx->stream, band->win_y0, band->win_rows));
    ctx->launches++;
    band->last_step = -1;
    band->cur = 0;
    return W2X_OK;
}

constexpr uint32_t BLOB_MAGIC = 0x77327862u;   // "w2xb"
struct BandBlob {                              // what w2x_band_export hands to the neighbour ranks
    uint32_t magic;
    int32_t pw, hf, n;
    int32_t precision;                         // the exchanged records' format (W2X_PRECISION_*)
    uint64_t act_bytes;
    cudaIpcMemHandle_t pad, act0, act1, flags;
};
static_assert(sizeof(BandBlob) <= W2X_BAND_BLOB_BYTES, "blob does not fit W2X_BAND_BLOB_BYTES");

int band_run_from(w2x_band *band, const float *d_in, size_t in_stride_bytes, bool up2x, float *d_out, size_t out_stride_bytes);

}  // namespace

extern "C" {

int w2x_band_create(w2x_ctx *ctx, const w2x_model *model, int width, int band_rows, int has_up, int has_down,
                    w2x_band **out_band) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || !out_band || width < 1 || band_rows < 1) return fail(W2X_ERR_ARG, "w2x_band_create: bad argument");
    *out_band = nullptr;
    if (!tc_eligible(model, ctx->precision) || ctx->engine == W2X_ENGINE_FP32)
        return fail(W2X_ERR_UNSUPPORTED, "w2x_band_create: the per-layer halo mode needs the tensor-core engine and a 1->{32,64,128}..->1 model");
    if (has_up < 0 || has_up > 2 || has_down < 0 || has_down > 2) return fail(W2X_ERR_ARG, "w2x_band_create: edge kind must be 0 (image border), 1 (neighbour GPU) or 2 (overlap rows)");
    // Refused here, before anything is allocated or queued: a band whose layers failed mid-pass would leave its neighbours'
    // exchange kernels waiting for rows that never come.
    const int n = (int)model->layers.size();
    const long frame_rows = (long)band_rows + (has_up == W2X_EDGE_NEIGHBOUR ? 1 : n) + (has_down == W2X_EDGE_NEIGHBOUR ? 1 : n);
    if (frame_rows > MAX_FRAME_ROWS)
        return fail(W2X_ERR_ARG, "w2x_band_create: the band's frame has %ld rows (%d owned + halo / border rows), more than the %ld a frame may have",
                    frame_rows, band_rows, MAX_FRAME_ROWS);
    DeviceGuard g(ctx->device);
    int rc = ensure_tc(ctx);
    if (rc) return rc;
    auto b = std::make_unique<w2x_band>();
    b->ctx = ctx;
    b->model = model;
    rc = get_dev_model(ctx, model, &b->dm);
    if (rc) return rc;
    if (ctx->precision == W2X_PRECISION_BF16X3) {   // now, not in the first pass: a pass must not stall neighbours that wait for its rows
        rc = upload_pack_bf16(ctx, model, b->dm);
        if (rc) return rc;
    }
    b->dm->band_sessions++;        // w2x_ctx_forget_model refuses until the session goes
    b->n = (int)model->layers.size();
    b->width = width;
    b->rows = band_rows;
    b->up = has_up == W2X_EDGE_NEIGHBOUR;
    b->down = has_down == W2X_EDGE_NEIGHBOUR;
    b->ov_up = has_up == W2X_EDGE_OVERLAP;
    b->ov_down = has_down == W2X_EDGE_OVERLAP;
    b->pt = b->up ? 1 : b->n;
    b->pb = b->down ? 1 : b->n;
    b->pw = width + 2 * b->n;
    b->hf = band_rows + b->pt + b->pb;
    b->win_y0 = b->up ? 1 : 0;
    b->win_rows = b->hf - b->win_y0 - (b->down ? 1 : 0);
    b->act_bytes = tc::act_bytes(max_channels(model), b->pw, b->hf);
    auto nomem = [](cudaError_t e) {
        cudaGetLastError();
        return fail(W2X_ERR_NOMEM, "w2x_band_create: cudaMalloc failed (%s)", cudaGetErrorString(e));
    };
    cudaError_t e;
    if ((e = b->pad.grow((size_t)b->pw * b->hf * sizeof(float))) != cudaSuccess) return nomem(e);
    for (int i = 0; i < 2; i++)
        if ((e = b->act[i].grow(b->act_bytes)) != cudaSuccess) return nomem(e);
    if ((e = b->flags.grow(64)) != cudaSuccess) return nomem(e);
    if ((e = cudaMemset(b->flags.get(), 0, 64)) != cudaSuccess) return nomem(e);
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return nomem(e);         // the flag words are zero before a neighbour can write them
    *out_band = b.release();
    return W2X_OK;
}

void w2x_band_destroy(w2x_band *band) {
    if (!band) return;
    DeviceGuard g(band->ctx->device);
    cudaStreamSynchronize(band->ctx->stream);
    delete band;
    cudaGetLastError();
}

// d_in: the band's rows PLUS one real row per neighbour side (the caller fetched them); every frame row is written.
int w2x_band_load(w2x_band *band, const float *d_in, size_t in_stride_bytes) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (!d_in || in_stride_bytes % 4 || in_stride_bytes < (size_t)band->width * 4) return fail(W2X_ERR_ARG, "w2x_band_load: bad input");
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    if (band->ov_up || band->ov_down) return fail(W2X_ERR_ARG, "w2x_band_load: overlap edges take their rows through w2x_band_load_rows");
    const long stride = (long)(in_stride_bytes / 4);
    const FrameSource src{d_in + (band->up ? stride : 0), stride, band->width, band->rows, band->n, band->pt, band->up ? 1 : 0,
                          band->down ? 1 : 0};
    CU_CHECK(launch_pad(src, band->pw, band->hf, band->pad.get(), ctx->stream));
    ctx->launches++;
    band->last_step = -1;
    band->cur = 0;
    return W2X_OK;
}

// d_in: the band's OWN rows; the halo rows of the input frame are left to the neighbours (w2x_band_exchange(band, -1)).  On an
// overlap edge (W2X_EDGE_OVERLAP) the n input rows beyond the band must be readable at d_in - n rows / d_in + rows.
int w2x_band_load_rows(w2x_band *band, const float *d_in, size_t in_stride_bytes) { return band_load_rows_from(band, d_in, in_stride_bytes, false); }

int w2x_band_step(w2x_band *band, int step) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (step != band->last_step + 1 || step < 0 || step > band->n - 2)
        return fail(W2X_ERR_ARG, "w2x_band_step: steps must run in order 0..%d (got %d after %d)", band->n - 2, step, band->last_step);
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    const w2x_model *m = band->model;
    DevModel *dm = band->dm;
    const Layer &L = m->layers[(size_t)step];
    if (step == 0) {
        LayerTimer t(ctx, 0);
        CU_CHECK(tc::launch_first(FrameSource::padded(band->pad.get(), band->pw, band->pw, band->hf), band->pw, band->hf, L.w.data(),
                                  dm->b_host[0].data(), L.n_out, band->act[0].get(), ctx->stream, tc::rec_format(ctx->precision), band->win_y0, band->win_rows));
        band->cur = 0;
        note_kernel(ctx, 0, "first_1xN");
        ctx->launches++;
    } else {
        int rc = launch_layer_tc(ctx, m, dm, step, band->act[band->cur].get(), band->act[band->cur ^ 1].get(), band->pw, band->hf, step == band->n - 2, false,
                                 band->win_y0, band->win_rows);
        if (rc) return rc;
        band->cur ^= 1;
    }
    band->last_step = step;
    return W2X_OK;
}

int w2x_band_halo(w2x_band *band, int step, int *n_segments, void **send_up, void **recv_up, void **send_down,
                  void **recv_down, size_t *seg_bytes) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (step != band->last_step || step < 0 || !n_segments || !send_up || !recv_up || !send_down || !recv_down || !seg_bytes)
        return fail(W2X_ERR_ARG, "w2x_band_halo: call it for the step that was queued last");
    char *base = reinterpret_cast<char *>(band->act[band->cur].get());
    const size_t bytes = row_bytes(band, step);
    *n_segments = 1;
    *seg_bytes = bytes;
    send_up[0] = band->up ? base + bytes : nullptr;                                   // first owned row
    recv_up[0] = band->up ? base : nullptr;                                           // halo row above
    send_down[0] = band->down ? base + bytes * (size_t)(band->hf - 2) : nullptr;      // last owned row
    recv_down[0] = band->down ? base + bytes * (size_t)(band->hf - 1) : nullptr;      // halo row below
    for (int s = 1; s < 4; s++) send_up[s] = recv_up[s] = send_down[s] = recv_down[s] = nullptr;
    return W2X_OK;
}

int w2x_band_finish(w2x_band *band, float *d_out, size_t out_stride_bytes) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (band->last_step != band->n - 2) return fail(W2X_ERR_ARG, "w2x_band_finish: steps 0..%d must have run", band->n - 2);
    if (!d_out || out_stride_bytes % 4 || out_stride_bytes < (size_t)band->width * 4) return fail(W2X_ERR_ARG, "w2x_band_finish: bad output");
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    const Layer &L = band->model->layers.back();
    {
        LayerTimer t(ctx, band->n - 1);
        CU_CHECK(tc::launch_last_gather(reinterpret_cast<const float *>(band->act[band->cur].get()), band->pw, band->hf,
                                        static_cast<float>(L.b[0]), band->n, band->pt, band->pb, d_out, (long)(out_stride_bytes / 4),
                                        ctx->stream));
    }
    note_kernel(ctx, band->n - 1, "last_gather");
    ctx->launches++;
    band->last_step = band->n - 1;
    return W2X_OK;
}

// ---- peer wiring ---------------------------------------------------------------------------------------------------------
int w2x_band_export(w2x_band *band, void *blob) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (!blob) return fail(W2X_ERR_ARG, "w2x_band_export: NULL blob");
    DeviceGuard g(band->ctx->device);
    BandBlob bl{};
    bl.magic = BLOB_MAGIC;
    bl.pw = band->pw;
    bl.hf = band->hf;
    bl.n = band->n;
    bl.precision = band->ctx->precision;
    bl.act_bytes = band->act_bytes;
    CU_CHECK(cudaIpcGetMemHandle(&bl.pad, band->pad.get()));
    CU_CHECK(cudaIpcGetMemHandle(&bl.act0, band->act[0].get()));
    CU_CHECK(cudaIpcGetMemHandle(&bl.act1, band->act[1].get()));
    CU_CHECK(cudaIpcGetMemHandle(&bl.flags, band->flags.get()));
    std::memset(blob, 0, W2X_BAND_BLOB_BYTES);
    std::memcpy(blob, &bl, sizeof bl);
    return W2X_OK;
}

int w2x_band_connect(w2x_band *band, const void *up_blob, const void *down_blob) {
    if (band_check(band)) return W2X_ERR_ARG;
    if ((band->up && !up_blob) || (band->down && !down_blob)) return fail(W2X_ERR_ARG, "w2x_band_connect: a neighbour's blob is missing");
    DeviceGuard g(band->ctx->device);
    const void *blobs[2] = {band->up ? up_blob : nullptr, band->down ? down_blob : nullptr};
    for (int side = 0; side < 2; side++) {
        if (!blobs[side]) continue;
        BandBlob bl;
        std::memcpy(&bl, blobs[side], sizeof bl);
        if (bl.magic != BLOB_MAGIC || bl.pw != band->pw || bl.n != band->n || bl.precision != band->ctx->precision || bl.hf < 3)
            return fail(W2X_ERR_ARG, "w2x_band_connect: the %s neighbour's session does not match (width / model / precision)", side ? "down" : "up");
        w2x_band::Peer &p = band->peer[side];
        void *q = nullptr;
        CU_CHECK(cudaIpcOpenMemHandle(&q, bl.pad, cudaIpcMemLazyEnablePeerAccess));
        p.pad = static_cast<float *>(q);
        CU_CHECK(cudaIpcOpenMemHandle(&q, bl.act0, cudaIpcMemLazyEnablePeerAccess));
        p.act[0] = static_cast<char *>(q);
        CU_CHECK(cudaIpcOpenMemHandle(&q, bl.act1, cudaIpcMemLazyEnablePeerAccess));
        p.act[1] = static_cast<char *>(q);
        CU_CHECK(cudaIpcOpenMemHandle(&q, bl.flags, cudaIpcMemLazyEnablePeerAccess));
        p.flags = static_cast<unsigned *>(q);
        p.hf = bl.hf;
        p.ipc = true;
    }
    return W2X_OK;
}

int w2x_band_connect_local(w2x_band *band, w2x_band *up, w2x_band *down) {
    if (band_check(band)) return W2X_ERR_ARG;
    if ((band->up && band_check(up)) || (band->down && band_check(down))) return fail(W2X_ERR_ARG, "w2x_band_connect_local: a neighbour session is missing");
    DeviceGuard g(band->ctx->device);
    w2x_band *nb[2] = {band->up ? up : nullptr, band->down ? down : nullptr};
    for (int side = 0; side < 2; side++) {
        w2x_band *o = nb[side];
        if (!o) continue;
        if (o->pw != band->pw || o->n != band->n || o->ctx->precision != band->ctx->precision)
            return fail(W2X_ERR_ARG, "w2x_band_connect_local: the %s neighbour's session does not match (width / model / precision)", side ? "down" : "up");
        if (o->ctx->device != band->ctx->device) {
            int can = 0;
            CU_CHECK(cudaDeviceCanAccessPeer(&can, band->ctx->device, o->ctx->device));
            if (!can) return fail(W2X_ERR_UNSUPPORTED, "device %d cannot map the memory of device %d (no peer access)", band->ctx->device, o->ctx->device);
            cudaError_t e = cudaDeviceEnablePeerAccess(o->ctx->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU_CHECK(e);
            cudaGetLastError();
        }
        w2x_band::Peer &p = band->peer[side];
        p.pad = o->pad.get();
        p.act[0] = reinterpret_cast<char *>(o->act[0].get());
        p.act[1] = reinterpret_cast<char *>(o->act[1].get());
        p.flags = o->flags.get();
        p.hf = o->hf;
        p.ipc = false;
    }
    return W2X_OK;
}

// After w2x_band_load_rows (step = -1) or w2x_band_step(step): this band's boundary rows -> the neighbours' halo rows, flag
// handshake; the context's stream continues once the neighbours' rows are here.  One kernel.
int w2x_band_exchange(w2x_band *band, int step) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (step != band->last_step || step < -1 || step > band->n - 2) return fail(W2X_ERR_ARG, "w2x_band_exchange: call it for the step that was queued last");
    if ((band->up && !band->peer[0].flags) || (band->down && !band->peer[1].flags))
        return fail(W2X_ERR_ARG, "w2x_band_exchange: the neighbours are not connected (w2x_band_connect / w2x_band_connect_local)");
    if (!band->up && !band->down) return W2X_OK;
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    const size_t bytes = row_bytes(band, step);
    char *mine = step < 0 ? reinterpret_cast<char *>(band->pad.get()) : reinterpret_cast<char *>(band->act[band->cur].get());
    HaloXArgs a{};
    if (band->up) {      // my first owned row -> the up neighbour's halo row below (its last frame row)
        const w2x_band::Peer &p = band->peer[0];
        char *theirs = step < 0 ? reinterpret_cast<char *>(p.pad) : p.act[band->cur];
        a.src[a.n] = mine + bytes;
        a.dst[a.n] = theirs + bytes * (size_t)(p.hf - 1);
        a.n++;
    }
    if (band->down) {    // my last owned row -> the down neighbour's halo row above (its frame row 0)
        const w2x_band::Peer &p = band->peer[1];
        char *theirs = step < 0 ? reinterpret_cast<char *>(p.pad) : p.act[band->cur];
        a.src[a.n] = mine + bytes * (size_t)(band->hf - 2);
        a.dst[a.n] = theirs;
        a.n++;
    }
    a.bytes = bytes;
    unsigned *const flags = band->flags.get();
    a.counter = flags + 4;
    a.value = ++band->seq;
    // I am the DOWN neighbour of my up peer (its flag 1) and the UP neighbour of my down peer (its flag 0)
    a.peer_flag[0] = band->up ? band->peer[0].flags + 1 : nullptr;
    a.peer_flag[1] = band->down ? band->peer[1].flags + 0 : nullptr;
    a.my_flag[0] = band->up ? flags + 0 : nullptr;
    a.my_flag[1] = band->down ? flags + 1 : nullptr;
    NvtxRange nvtx("w2x halo exchange");
    CU_CHECK(launch_halo_exchange(a, ctx->stream));
    ctx->launches++;
    return W2X_OK;
}

// One whole pass of a connected band: own rows in, own rows out; everything is queued on the context's stream.
int w2x_band_run(w2x_band *band, const float *d_in, size_t in_stride_bytes, float *d_out, size_t out_stride_bytes) {
    return band_run_from(band, d_in, in_stride_bytes, false, d_out, out_stride_bytes);
}

}  // extern "C"

namespace {
// w2x_band_run from a row source that may be a half-resolution plane (band_load_rows_from)
int band_run_from(w2x_band *band, const float *d_in, size_t in_stride_bytes, bool up2x, float *d_out, size_t out_stride_bytes) {
    int rc = band_load_rows_from(band, d_in, in_stride_bytes, up2x);
    if (rc) return rc;
    if ((rc = w2x_band_exchange(band, -1))) return rc;
    for (int k = 0; k <= band->n - 2; k++) {
        if ((rc = w2x_band_step(band, k))) return rc;
        if ((rc = w2x_band_exchange(band, k))) return rc;
    }
    return w2x_band_finish(band, d_out, out_stride_bytes);
}
}  // namespace

// =========================================================================================================================
// One GPU's slab of a multi-GPU plane with HOST buffers: upload, layers and download pipelined over sub-bands
// =========================================================================================================================
// A slab is what one rank (or one GPU of w2x_multi_*) owns of the plane.  It is cut into K sub-bands that run one after the
// other: the upload of sub-band t+1 and the download of t-1 overlap the layers of t (copy engines + SMs).  Seams INSIDE the
// slab are overlap edges (n real input rows, recomputed -- the data is local anyway); the slab's outer edges keep the
// per-layer halo exchange with the neighbour GPU.  Two neighbouring slabs must work on their common boundary at the same
// time, so even slabs walk top -> bottom and odd ones bottom -> top (`order`).
struct w2x_slab {
    w2x_ctx *ctx = nullptr;
    const w2x_model *model = nullptr;
    int width = 0, rows = 0, order = 0;
    bool up = false, down = false;
    bool half_in = false;                        // d_in holds the rows at half resolution: [rows / 2][width / 2], read through the 2x resize
    std::vector<w2x_band *> sub;
    std::vector<int> r0;                         // sub-band s owns slab rows [r0[s], r0[s+1])
    DevBuf<float> d_in, d_out;                   // [rows][width]
    std::vector<cudaEvent_t> ev_in, ev_done;
    cudaEvent_t ev_drained = nullptr;            // the previous pass's downloads have left d_out

    // The sub-bands and the events; d_in and d_out go after this body.  The caller has made the context's device current.
    ~w2x_slab() {
        for (auto b : sub) w2x_band_destroy(b);
        for (auto e : ev_in) cudaEventDestroy(e);
        for (auto e : ev_done) cudaEventDestroy(e);
        if (ev_drained) cudaEventDestroy(ev_drained);
    }
};

namespace {
// w2x_slab_create for a step of w2x_multi_convert_chain: without d_in when the slab's rows come from another slab's d_out; up2x: the
// slab's rows are read through the nearest 2x resize, so every sub-band starts on an even row (the first copy of a source row) and
// d_in, if any, holds the half-resolution rows.
int slab_create(w2x_ctx *ctx, const w2x_model *model, int width, int rows, int has_up, int has_down, int order, int n_sub, bool with_d_in,
                bool up2x, w2x_slab **out) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || !out || width < 1 || rows < 1) return fail(W2X_ERR_ARG, "w2x_slab_create: bad argument");
    *out = nullptr;
    const int n = (int)model->layers.size();
    if (n_sub <= 0) n_sub = std::min(4, rows / 512);            // like w2x_convert_plane's copy pipeline
    n_sub = std::max(1, std::min(n_sub, std::min(8, rows / (4 * n))));
    // ... and as many as it takes for every sub-band's frame (its rows + at most n above and below) to stay within MAX_FRAME_ROWS
    const long sub_max = MAX_FRAME_ROWS - 2 * n;
    n_sub = std::max(n_sub, (int)((rows + sub_max - 1) / sub_max));
    DeviceGuard g(ctx->device);   // before the slab: it is still current when an early return destroys what has been created
    auto s = std::make_unique<w2x_slab>();
    s->ctx = ctx;
    s->model = model;
    s->width = width;
    s->rows = rows;
    s->order = order ? 1 : 0;
    s->up = has_up != 0;
    s->down = has_down != 0;
    for (int i = 0; i <= n_sub; i++) s->r0.push_back(i == n_sub ? rows : (int)((long)rows * i / n_sub) & (up2x ? ~1 : ~0));
    for (int i = 0; i < n_sub; i++) {
        w2x_band *b = nullptr;
        const int ue = i == 0 ? (s->up ? W2X_EDGE_NEIGHBOUR : W2X_EDGE_BORDER) : W2X_EDGE_OVERLAP;
        const int de = i == n_sub - 1 ? (s->down ? W2X_EDGE_NEIGHBOUR : W2X_EDGE_BORDER) : W2X_EDGE_OVERLAP;
        int rc = w2x_band_create(ctx, model, width, s->r0[(size_t)i + 1] - s->r0[(size_t)i], ue, de, &b);
        if (rc) return rc;
        s->sub.push_back(b);
    }
    s->half_in = with_d_in && up2x;
    int rc = with_d_in ? s->d_in.reserve(s->half_in ? (size_t)(rows / 2) * (width / 2) * 4 : (size_t)rows * width * 4) : W2X_OK;
    if (!rc) rc = s->d_out.reserve((size_t)rows * width * 4);
    if (rc) return rc;
    for (int i = 0; i < n_sub; i++) {
        cudaEvent_t e;
        CU_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        s->ev_in.push_back(e);
        CU_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        s->ev_done.push_back(e);
    }
    CU_CHECK(cudaEventCreateWithFlags(&s->ev_drained, cudaEventDisableTiming));
    *out = s.release();
    return W2X_OK;
}
}  // namespace

extern "C" {

void w2x_slab_destroy(w2x_slab *s) {
    if (!s) return;
    DeviceGuard g(s->ctx->device);
    delete s;
    cudaGetLastError();
}

int w2x_slab_create(w2x_ctx *ctx, const w2x_model *model, int width, int rows, int has_up, int has_down, int order, int n_sub, w2x_slab **out) {
    return slab_create(ctx, model, width, rows, has_up, has_down, order, n_sub, true, false, out);
}

// blob = [top sub-band's session | bottom sub-band's session]
int w2x_slab_export(w2x_slab *s, void *blob) {
    if (!s || !blob) return fail(W2X_ERR_ARG, "w2x_slab_export: NULL argument");
    int rc = w2x_band_export(s->sub.front(), blob);
    if (rc) return rc;
    return w2x_band_export(s->sub.back(), static_cast<char *>(blob) + W2X_BAND_BLOB_BYTES);
}

int w2x_slab_connect(w2x_slab *s, const void *up_blob, const void *down_blob) {
    if (!s) return fail(W2X_ERR_ARG, "w2x_slab_connect: NULL slab");
    if ((s->up && !up_blob) || (s->down && !down_blob)) return fail(W2X_ERR_ARG, "w2x_slab_connect: a neighbour's blob is missing");
    const void *ub = s->up ? static_cast<const char *>(up_blob) + W2X_BAND_BLOB_BYTES : nullptr;   // the up slab's BOTTOM session
    const void *db = s->down ? down_blob : nullptr;                                                  // the down slab's TOP session
    if (s->sub.size() == 1) return w2x_band_connect(s->sub[0], ub, db);
    int rc = w2x_band_connect(s->sub.front(), ub, nullptr);
    if (rc) return rc;
    return w2x_band_connect(s->sub.back(), nullptr, db);
}

int w2x_slab_connect_local(w2x_slab *s, w2x_slab *up, w2x_slab *down) {
    if (!s) return fail(W2X_ERR_ARG, "w2x_slab_connect_local: NULL slab");
    if ((s->up && !up) || (s->down && !down)) return fail(W2X_ERR_ARG, "w2x_slab_connect_local: a neighbour slab is missing");
    w2x_band *ub = s->up ? up->sub.back() : nullptr, *db = s->down ? down->sub.front() : nullptr;
    if (s->sub.size() == 1) return w2x_band_connect_local(s->sub[0], ub, db);
    int rc = w2x_band_connect_local(s->sub.front(), ub, nullptr);
    if (rc) return rc;
    return w2x_band_connect_local(s->sub.back(), nullptr, db);
}

}  // extern "C"

namespace {
// Phase 1 of a pass, first half: the slab's rows from the host into d_in, one upload per sub-band.
int slab_enqueue_upload(w2x_slab *s, const float *in, size_t in_stride_bytes) {
    w2x_ctx *ctx = s->ctx;
    DeviceGuard g(ctx->device);
    const int K = (int)s->sub.size();
    const size_t rowb = (size_t)s->width * 4;
    auto at = [&](int t) { return s->order ? K - 1 - t : t; };      // t-th sub-band in processing order
    CU_CHECK(cudaStreamWaitEvent(ctx->copy_in, s->ev_done[(size_t)at(K - 1)], 0));   // the previous pass has finished reading d_in
    if (s->half_in) {   // a quarter of the slab's pixels: one upload, which every sub-band waits for
        const size_t half_rowb = (size_t)(s->width / 2) * 4;
        CU_CHECK(cudaMemcpy2DAsync(s->d_in.get(), half_rowb, in, in_stride_bytes, half_rowb, (size_t)(s->rows / 2), cudaMemcpyHostToDevice, ctx->copy_in));
        for (auto e : s->ev_in) CU_CHECK(cudaEventRecord(e, ctx->copy_in));
        return W2X_OK;
    }
    // Upload t carries the t-th sub-band's rows shifted by n towards the sub-band processed next: its own rows minus the n the previous
    // upload already brought, plus the n rows of overlap context it reads from the next one -- so a sub-band waits for ITS upload only.
    const int n = (int)s->model->layers.size();
    for (int t = 0; t < K; t++) {
        const int i = at(t);
        int ya, yb;
        if (!s->order) { ya = s->r0[(size_t)i] + (t == 0 ? 0 : n); yb = s->r0[(size_t)i + 1] + (t == K - 1 ? 0 : n); }
        else { ya = s->r0[(size_t)i] - (t == K - 1 ? 0 : n); yb = s->r0[(size_t)i + 1] - (t == 0 ? 0 : n); }
        CU_CHECK(cudaMemcpy2DAsync(s->d_in.get() + (size_t)ya * s->width, rowb, reinterpret_cast<const char *>(in) + (size_t)ya * in_stride_bytes, in_stride_bytes, rowb,
                                   (size_t)(yb - ya), cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(s->ev_in[(size_t)i], ctx->copy_in));
    }
    return W2X_OK;
}

// Second half: the layer loops of every sub-band from a device row source (nothing here can block the host on another GPU's
// progress).  `src` holds the slab's rows: d_in after slab_enqueue_upload (uploaded: each sub-band waits for its upload), or, in a
// chain, the d_out of the previous step's slab on this GPU, as it is or (up2x) at half resolution.  An overlap edge of an upscaling
// sub-band reads ceil(n / 2) source rows of the NEIGHBOURING sub-band's output of the previous step; all of that step's sub-bands
// were queued on this stream before any of this step's, so stream order alone has them written.
int slab_enqueue_run(w2x_slab *s, const float *src, size_t src_stride_bytes, bool up2x, bool uploaded) {
    w2x_ctx *ctx = s->ctx;
    DeviceGuard g(ctx->device);
    const int K = (int)s->sub.size();
    const size_t rowb = (size_t)s->width * 4;
    CU_CHECK(cudaStreamWaitEvent(ctx->stream, s->ev_drained, 0));                    // the previous pass's downloads have left d_out
    for (int t = 0; t < K; t++) {
        const int i = s->order ? K - 1 - t : t, y = s->r0[(size_t)i];
        if (uploaded) CU_CHECK(cudaStreamWaitEvent(ctx->stream, s->ev_in[(size_t)i], 0));   // own rows + the overlap rows (earlier uploads are ordered before it)
        const float *rows = reinterpret_cast<const float *>(reinterpret_cast<const char *>(src) + (size_t)(up2x ? y / 2 : y) * src_stride_bytes);
        int rc = band_run_from(s->sub[(size_t)i], rows, src_stride_bytes, up2x, s->d_out.get() + (size_t)y * s->width, rowb);
        if (rc) {
            cudaStreamSynchronize(ctx->copy_in);
            cudaStreamSynchronize(ctx->stream);
            return rc;
        }
        CU_CHECK(cudaEventRecord(s->ev_done[(size_t)i], ctx->stream));
    }
    return W2X_OK;
}

int slab_enqueue_compute(w2x_slab *s, const float *in, size_t in_stride_bytes) {
    int rc = slab_enqueue_upload(s, in, in_stride_bytes);
    if (rc) return rc;
    return slab_enqueue_run(s, s->d_in.get(), (size_t)(s->half_in ? s->width / 2 : s->width) * 4, s->half_in, true);
}

// Phase 2: every sub-band's rows go home as soon as its layers are done.  (A download into PAGEABLE memory blocks the host
// until the data is there -- which is why a multi-GPU driver must have queued phase 1 on every GPU first: this GPU's layers
// wait for its neighbours' halo rows.)
int slab_enqueue_download(w2x_slab *s, float *out, size_t out_stride_bytes) {
    w2x_ctx *ctx = s->ctx;
    DeviceGuard g(ctx->device);
    const int K = (int)s->sub.size();
    const size_t rowb = (size_t)s->width * 4;
    for (int t = 0; t < K; t++) {
        const int i = s->order ? K - 1 - t : t, y = s->r0[(size_t)i], rows = s->r0[(size_t)i + 1] - y;
        CU_CHECK(cudaStreamWaitEvent(ctx->copy_out, s->ev_done[(size_t)i], 0));
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(out) + (size_t)y * out_stride_bytes, out_stride_bytes, s->d_out.get() + (size_t)y * s->width, rowb, rowb,
                                   (size_t)rows, cudaMemcpyDeviceToHost, ctx->copy_out));
    }
    CU_CHECK(cudaEventRecord(s->ev_drained, ctx->copy_out));
    return W2X_OK;
}
}  // namespace

extern "C" {

// Queues one whole pass: host rows in -> host rows out (pinned host memory keeps every copy asynchronous).
int w2x_slab_convert_async(w2x_slab *s, const float *in, size_t in_stride_bytes, float *out, size_t out_stride_bytes) {
    if (!s || !in || !out) return fail(W2X_ERR_ARG, "w2x_slab_convert: NULL argument");
    if (in_stride_bytes < (size_t)s->width * 4 || out_stride_bytes < (size_t)s->width * 4) return fail(W2X_ERR_ARG, "w2x_slab_convert: row stride smaller than a row");
    int rc = slab_enqueue_compute(s, in, in_stride_bytes);
    if (rc) return rc;
    return slab_enqueue_download(s, out, out_stride_bytes);
}

int w2x_slab_synchronize(w2x_slab *s) {
    if (!s) return fail(W2X_ERR_ARG, "NULL slab");
    DeviceGuard g(s->ctx->device);
    CU_CHECK(cudaStreamSynchronize(s->ctx->copy_out));
    CU_CHECK(cudaStreamSynchronize(s->ctx->stream));
    return W2X_OK;
}

int w2x_slab_convert(w2x_slab *s, const float *in, size_t in_stride_bytes, float *out, size_t out_stride_bytes) {
    int rc = w2x_slab_convert_async(s, in, in_stride_bytes, out, out_stride_bytes);
    int rc2 = s ? w2x_slab_synchronize(s) : W2X_OK;
    return rc ? rc : rc2;
}

}  // extern "C"

// =========================================================================================================================
// One process, N GPUs
// =========================================================================================================================
struct w2x_multi {
    std::vector<w2x_ctx *> ctx;
    // The slabs of the last (models, kinds, width, height), one per step and GPU: jobs usually repeat a shape.
    struct Chain {
        std::vector<uint64_t> uids;
        std::vector<int> kinds;
        int w = 0, h = 0, precision = -1;
        std::vector<std::vector<w2x_slab *>> slabs;   // [step][GPU]; GPU i owns rows [r0[i] << u, r0[i + 1] << u) of a step after u upscales
        std::vector<int> r0;                          // in input rows
    };
    // [0]: w2x_multi_convert_plane's (a one-step W2X_STEP_SAME chain); [1]: every other chain's.  Kept side by side, so a job that
    // alternates planes and chains does not rebuild either.
    Chain plan[2];
};

namespace {

void drop(w2x_multi::Chain &c) {
    for (auto &step : c.slabs)
        for (auto b : step) w2x_slab_destroy(b);
    c = w2x_multi::Chain();
}

// w2x_convert_chain over the row bands of nd >= 2 GPUs, HOST rows in and out, through the plan in `c` (built here unless the steps,
// size, precision and nd are the plan's).  A nearest 2x step maps the rows [a, b) a GPU owns onto [2a, 2b), so the cut of step 0
// stays a valid cut at every later step and no row ever changes GPU: the rows a GPU's slab of step k leaves in its d_out are, on
// that GPU, the (half-resolution) source of its slab of step k + 1.  Only step 0 uploads and only the last step downloads; the one
// cross-GPU traffic a step adds is the halo row of its input frame, which w2x_band_exchange(band, -1) already moves.  Every step
// has sessions (frames, flags) of its own: a neighbour may deliver a halo row of step k + 1 while this GPU still reads step k.
// begin(k) runs before step k is queued on any GPU.
int multi_convert(w2x_multi *m, w2x_multi::Chain &c, int nd, int n_steps, const w2x_model *const *models, const int *kinds, const float *in,
                  int width, int height, size_t in_stride_bytes, float *out, size_t out_stride_bytes, const std::function<void(int)> &begin) {
    w2x_ctx *ctx0 = m->ctx[0];
    int rc = W2X_OK;
    // ---- plan: per step one slab per GPU, neighbours of a step wired through peer memory; all device memory is reserved here ----
    std::vector<uint64_t> uids;
    for (int k = 0; k < n_steps; k++) uids.push_back(models[k]->uid);
    const std::vector<int> kv(kinds, kinds + n_steps);
    if (c.uids != uids || c.kinds != kv || c.w != width || c.h != height || c.precision != ctx0->precision || c.slabs.empty() ||
        (int)c.slabs[0].size() != nd) {
        drop(c);
        for (int i = 0; i <= nd; i++) c.r0.push_back((int)((long)height * i / nd));
        c.slabs.resize((size_t)n_steps);
        int u = 0;
        for (int k = 0; k < n_steps && !rc; k++) {
            const bool up = (kinds[k] & W2X_STEP_UPSCALE2X) != 0;
            u += up;
            for (int i = 0; i < nd && !rc; i++) {
                m->ctx[(size_t)i]->precision = ctx0->precision;
                w2x_slab *sl = nullptr;
                rc = slab_create(m->ctx[(size_t)i], models[k], width << u, (c.r0[(size_t)i + 1] - c.r0[(size_t)i]) << u, i > 0, i + 1 < nd, i & 1, 0,
                                 k == 0, up, &sl);
                if (!rc) c.slabs[(size_t)k].push_back(sl);
            }
            for (int i = 0; i < nd && !rc; i++)
                rc = w2x_slab_connect_local(c.slabs[(size_t)k][(size_t)i], i > 0 ? c.slabs[(size_t)k][(size_t)i - 1] : nullptr,
                                            i + 1 < nd ? c.slabs[(size_t)k][(size_t)i + 1] : nullptr);
        }
        if (rc) { drop(c); return rc; }
        c.uids = uids;
        c.kinds = kv;
        c.w = width;
        c.h = height;
        c.precision = ctx0->precision;
    }
    const size_t last = (size_t)n_steps - 1;
    int u_last = 0;
    for (int k = 0; k < n_steps; k++) u_last += (kinds[k] & W2X_STEP_UPSCALE2X) != 0;
    const int ow = width << u_last;
    HostPin pin_in(in, in_stride_bytes * (size_t)(height - 1) + (size_t)width * 4),
        pin_out(out, out_stride_bytes * (size_t)(((size_t)height << u_last) - 1) + (size_t)ow * 4);
    // ---- queue step-major, every GPU from this one thread: begin(k) comes before step k is queued anywhere, and a GPU's step k + 1
    // follows its own step k in stream order.  Nothing queued here can block this thread on a GPU's progress. ----
    for (size_t k = 0; k <= last && rc == W2X_OK; k++) {
        begin((int)k);
        for (int i = 0; i < nd && rc == W2X_OK; i++) {
            w2x_slab *sl = c.slabs[k][(size_t)i];
            if (k == 0) {
                rc = slab_enqueue_compute(sl, reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + (size_t)c.r0[(size_t)i] * in_stride_bytes), in_stride_bytes);
            } else {
                const w2x_slab *prev = c.slabs[k - 1][(size_t)i];
                rc = slab_enqueue_run(sl, prev->d_out.get(), (size_t)prev->width * 4, (kinds[k] & W2X_STEP_UPSCALE2X) != 0, false);
            }
        }
    }
    for (int i = 0; i < nd && rc == W2X_OK; i++)      // every GPU's layers are queued: a download (into pageable memory) may block this thread now
        rc = slab_enqueue_download(c.slabs[last][(size_t)i], reinterpret_cast<float *>(reinterpret_cast<char *>(out) + ((size_t)c.r0[(size_t)i] << u_last) * out_stride_bytes),
                                   out_stride_bytes);
    for (int i = 0; i < nd; i++) {
        int r2 = w2x_slab_synchronize(c.slabs[last][(size_t)i]);
        if (rc == W2X_OK) rc = r2;
    }
    return rc;
}

}  // namespace

extern "C" {

int w2x_multi_create(const int *devices, int n_devices, w2x_multi **out) {
    if (!out || n_devices < 1 || n_devices > 64) return fail(W2X_ERR_ARG, "w2x_multi_create: bad argument");
    *out = nullptr;
    auto m = std::make_unique<w2x_multi>();
    for (int i = 0; i < n_devices; i++) {
        w2x_ctx *c = nullptr;
        int rc = w2x_ctx_create(devices ? devices[i] : i, &c);
        if (rc) {
            for (auto p : m->ctx) w2x_ctx_destroy(p);
            return rc;
        }
        m->ctx.push_back(c);
    }
    *out = m.release();
    return W2X_OK;
}

void w2x_multi_destroy(w2x_multi *m) {
    if (!m) return;
    for (auto &c : m->plan) drop(c);
    for (auto c : m->ctx) w2x_ctx_destroy(c);
    delete m;
}

int w2x_multi_device_count(const w2x_multi *m) { return m ? (int)m->ctx.size() : 0; }
w2x_ctx *w2x_multi_ctx(w2x_multi *m, int i) { return m && i >= 0 && i < (int)m->ctx.size() ? m->ctx[(size_t)i] : nullptr; }

int w2x_multi_convert_plane(w2x_multi *m, const w2x_model *model, const float *in, int width, int height, size_t in_stride_bytes,
                            float *out, size_t out_stride_bytes, int block_splitting) {
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "w2x_multi_convert_plane: NULL handle");
    if (!model || !in || !out || width < 1 || height < 1) return fail(W2X_ERR_ARG, "w2x_multi_convert_plane: bad argument");
    if (in_stride_bytes < (size_t)width * 4 || out_stride_bytes < (size_t)width * 4) return fail(W2X_ERR_ARG, "w2x_multi_convert_plane: row stride smaller than a row");
    const int n_layers = (int)model->layers.size();
    int nd = (int)m->ctx.size();
    // every band needs a few rows of its own; small planes (and models without a tensor-core form) stay on one GPU
    nd = std::min(nd, height / (4 * n_layers));
    if (nd < 2 || !tc_eligible(model, m->ctx[0]->precision) || m->ctx[0]->engine == W2X_ENGINE_FP32)
        return w2x_convert_plane(m->ctx[0], model, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting);
    const int same = W2X_STEP_SAME;
    return multi_convert(m, m->plan[0], nd, 1, &model, &same, in, width, height, in_stride_bytes, out, out_stride_bytes, [&](int) {
        emit_reference_progress(m->ctx[0], width, height, n_layers, block_splitting && w2x_requires_splitting(width, height));
    });
}

int w2x_multi_convert_chain(w2x_multi *m, int n_steps, const w2x_model *const *models, const int *kinds, const float *in, int width,
                            int height, size_t in_stride_bytes, float *out, size_t out_stride_bytes, int block_splitting,
                            w2x_step_fn on_step, void *user) {
    const char *fn = "w2x_multi_convert_chain";
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "%s: NULL handle", fn);
    w2x_ctx *ctx0 = m->ctx[0];
    int rc = check_chain_host(fn, ctx0, n_steps, models, kinds, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting);
    if (rc) return rc;
    for (int k = 0; k < n_steps; k++)
        if (kinds[k] & W2X_STEP_TTA)
            return fail(W2X_ERR_ARG, "%s: step %d: W2X_STEP_TTA has no multi-GPU form (its transposed variants would turn row bands into column bands)", fn, k);
    if (n_steps == 1 && kinds[0] == W2X_STEP_SAME) {
        if (on_step) on_step(0, user);
        return w2x_multi_convert_plane(m, models[0], in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting);
    }
    int n_max = 0;
    bool tc = ctx0->engine != W2X_ENGINE_FP32;
    for (int k = 0; k < n_steps; k++) {
        n_max = std::max(n_max, (int)models[k]->layers.size());
        tc = tc && tc_eligible(models[k], ctx0->precision);
    }
    // decided on the input height with the deepest model: later steps only get taller
    const int nd = std::min((int)m->ctx.size(), height / (4 * n_max));
    if (nd < 2 || !tc)
        return w2x_convert_chain(ctx0, n_steps, models, kinds, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting, on_step, user);
    int w = width, h = height;      // step k's output size: begin(k) runs once per step, in order
    return multi_convert(m, m->plan[1], nd, n_steps, models, kinds, in, width, height, in_stride_bytes, out, out_stride_bytes, [&](int k) {
        if (kinds[k] & W2X_STEP_UPSCALE2X) w *= 2, h *= 2;
        if (on_step) on_step(k, user);
        emit_plane_progress(ctx0, models[k], w, h, block_splitting, true);
    });
}

int w2x_multi_convert_planes_chain(w2x_multi *m, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                                   const float *const *in, const int *widths, const int *heights, const size_t *in_strides, float *const *out,
                                   const size_t *out_strides, w2x_step_fn on_step, void *user) {
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "w2x_multi_convert_planes_chain: NULL handle");
    return multi_planes_chain("w2x_multi_convert_planes_chain", m->ctx, n_steps, models, kinds, n_planes, in, widths, heights, in_strides,
                              out, out_strides, on_step, user);
}

int w2x_multi_convert_chain_regions(w2x_multi *m, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows,
                                    const int *widths, const int *heights, const int *windows, const float *const *src,
                                    const size_t *src_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step,
                                    void *user) {
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "w2x_multi_convert_chain_regions: NULL handle");
    return multi_regions("w2x_multi_convert_chain_regions", m->ctx, n_steps, models, kinds, n_windows, widths, heights, windows, src,
                         src_strides, out, out_strides, on_step, user);
}

int w2x_multi_convert_planes(w2x_multi *m, const w2x_model *model, int n_planes, const float *const *in, const int *widths,
                             const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides) {
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "w2x_multi_convert_planes: NULL handle");
    const int same = W2X_STEP_SAME;
    return multi_planes_chain("w2x_multi_convert_planes", m->ctx, 1, &model, &same, n_planes, in, widths, heights, in_strides, out,
                              out_strides, nullptr, nullptr);
}

// Independent planes of one shape (the reference's block loop, src/convertRoutine.cpp:114-165, and BASELINE config 5):
// tile t goes to GPU t mod N, every GPU runs its tiles as ONE batched pass; no exchange.
int w2x_multi_convert_tiles(w2x_multi *m, const w2x_model *model, const float *const *in_tiles, float *const *out_tiles, int n_tiles,
                            int width, int height, size_t in_stride_bytes, size_t out_stride_bytes) {
    if (!m || m->ctx.empty()) return fail(W2X_ERR_ARG, "w2x_multi_convert_tiles: NULL handle");
    if (!model || !in_tiles || !out_tiles || n_tiles < 1) return fail(W2X_ERR_ARG, "w2x_multi_convert_tiles: bad argument");
    const int nd = std::min((int)m->ctx.size(), n_tiles);
    std::vector<std::vector<const float *>> tin((size_t)nd);
    std::vector<std::vector<float *>> tout((size_t)nd);
    for (int t = 0; t < n_tiles; t++) {
        tin[(size_t)(t % nd)].push_back(in_tiles[t]);
        tout[(size_t)(t % nd)].push_back(out_tiles[t]);
    }
    // queue every GPU's batch without waiting, then wait for all of them
    int rc = W2X_OK;
    for (int i = 0; i < nd && rc == W2X_OK; i++)
        rc = tiles_enqueue_compute(m->ctx[(size_t)i], model, tin[(size_t)i].data(), tout[(size_t)i].data(), (int)tin[(size_t)i].size(), width, height, in_stride_bytes, out_stride_bytes);
    for (int i = 0; i < nd && rc == W2X_OK; i++)
        rc = tiles_enqueue_download(m->ctx[(size_t)i], tout[(size_t)i].data(), (int)tout[(size_t)i].size(), width, height, out_stride_bytes);
    for (int i = 0; i < nd; i++) {
        int r2 = w2x_ctx_synchronize(m->ctx[(size_t)i]);
        if (rc == W2X_OK) rc = r2;
    }
    return rc;
}

int w2x_multi_set_precision(w2x_multi *m, int precision) {
    if (!m) return fail(W2X_ERR_ARG, "NULL handle");
    for (auto c : m->ctx) {
        int rc = w2x_ctx_set_precision(c, precision);
        if (rc) return rc;
    }
    return W2X_OK;
}

int w2x_multi_set_log(w2x_multi *m, w2x_log_fn fn, void *user) {
    if (!m) return fail(W2X_ERR_ARG, "NULL handle");
    return w2x_ctx_set_log(m->ctx[0], fn, user);
}

// Test hook: launch_pad alone on HOST arrays.  `in` is in_rows x in_stride_floats and the source's pixel (0, 0) is its pixel
// (in_row0, in_col0); every row and column the source's clamps allow must lie inside it.  `out` is the dense pw x ph frame and comes
// back with the rows outside the store window [out_y0, out_y0 + out_rows) as the caller left them.
W2X_API int w2x_debug_pad(w2x_ctx *ctx, const float *in, int in_rows, long in_stride_floats, int in_row0, int in_col0, int w, int h, int pad_x,
                          int pad_top, int rows_above, int rows_below, int up2x, int cols_left, int cols_right, int pw, int ph, int out_y0,
                          int out_rows, float *out) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    const int sh = up2x ? 1 : 0;   // the source rows and columns the clamps can reach: [lo >> sh, hi >> sh] of each
    if (!in || !out || w < 1 || h < 1 || in_rows < 1 || pw < 1 || ph < 1 || -rows_above > h - 1 + rows_below || -cols_left > w - 1 + cols_right ||
        in_row0 + (-rows_above >> sh) < 0 || in_row0 + ((h - 1 + rows_below) >> sh) >= in_rows || in_col0 + (-cols_left >> sh) < 0 ||
        in_col0 + ((w - 1 + cols_right) >> sh) >= in_stride_floats)
        return fail(W2X_ERR_ARG, "w2x_debug_pad: bad argument");
    DeviceGuard g(ctx->device);
    const size_t in_bytes = (size_t)in_rows * in_stride_floats * 4, out_bytes = (size_t)pw * ph * 4;
    DevBuf<float> d_in, d_out;
    int rc = d_in.reserve(in_bytes);
    if (!rc) rc = d_out.reserve(out_bytes);
    if (rc) return rc;
    CU_CHECK(cudaMemcpyAsync(d_in.get(), in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    CU_CHECK(cudaMemcpyAsync(d_out.get(), out, out_bytes, cudaMemcpyHostToDevice, ctx->stream));
    const FrameSource src{d_in.get() + (size_t)in_row0 * in_stride_floats + in_col0, in_stride_floats, w, h, pad_x, pad_top, rows_above,
                          rows_below, up2x != 0, cols_left, cols_right};
    CU_CHECK(launch_pad(src, pw, ph, d_out.get(), ctx->stream, out_y0, out_rows));
    ctx->launches++;
    CU_CHECK(cudaMemcpyAsync(out, d_out.get(), out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CU_CHECK(cudaStreamSynchronize(ctx->stream));
    return W2X_OK;
}

}  // extern "C"
