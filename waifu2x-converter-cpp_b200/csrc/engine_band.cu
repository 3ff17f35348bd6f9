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
#include "engine_internal.h"

using namespace w2x;
using namespace w2x::eng;

namespace {

int band_check(w2x_band *b) {
    if (!b || !b->ctx || !b->model) return fail(W2X_ERR_ARG, "NULL band session");
    return W2X_OK;
}

// The rows traded after `step` (-1 = the padded input frame): up to 4 contiguous ranges per row, each `bytes` long, at
//   base + plane_mul * (pw * C * frame_rows) + row * pitch + in_row        (evaluated in the owner's OR the neighbour's frame)
struct RowSeg { size_t plane_mul, pitch, in_row; };
int row_segments(const w2x_band *b, int step, RowSeg seg[4], size_t *bytes, size_t *px_out) {
    const int n = b->n;
    if (step == -1) {
        *bytes = (size_t)b->pw * sizeof(float);
        seg[0] = {0, *bytes, 0};
        *px_out = 0;
        return 1;
    }
    if (step == n - 2) {              // per-pixel tap partials [hf][pw][12] fp32
        *bytes = (size_t)b->pw * 12 * sizeof(float);
        seg[0] = {0, *bytes, 0};
        *px_out = 0;
        return 1;
    }
    const size_t px = (size_t)b->pw * (size_t)b->model->layers[(size_t)step].n_out;
    *px_out = px;
    *bytes = 4 * px;                  // RECORD frame: a row is one contiguous range of 4 bytes per element
    seg[0] = {0, 4 * px, 0};
    return 1;
}

inline char *seg_at(char *base, int frame_rows, size_t px, const RowSeg &s, int row) {
    return base + s.plane_mul * px * (size_t)frame_rows + s.pitch * (size_t)row + s.in_row;
}

constexpr uint32_t BLOB_MAGIC = 0x77327862u;   // "w2xb"
struct BandBlob {                              // what w2x_band_export hands to the neighbour ranks
    uint32_t magic;
    int32_t pw, hf, n;
    uint64_t act_bytes;
    cudaIpcMemHandle_t pad, act0, act1, flags;
};
static_assert(sizeof(BandBlob) <= W2X_BAND_BLOB_BYTES, "blob does not fit W2X_BAND_BLOB_BYTES");

}  // namespace

extern "C" {

int w2x_band_create(w2x_ctx *ctx, const w2x_model *model, int width, int band_rows, int has_up, int has_down,
                    w2x_band **out_band) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || !out_band || width < 1 || band_rows < 1) return fail(W2X_ERR_ARG, "w2x_band_create: bad argument");
    *out_band = nullptr;
    if (!model->tc_eligible || ctx->engine == W2X_ENGINE_FP32)
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
    int maxc = 1;
    for (auto &L : model->layers) maxc = std::max(maxc, std::max(L.n_in, L.n_out));
    b->act_bytes = tc::act_bytes(maxc, b->pw, b->hf);
    auto cleanup = [&](cudaError_t e) {
        cudaFree(b->pad);
        cudaFree(b->act[0]);
        cudaFree(b->act[1]);
        cudaFree(b->flags);
        cudaGetLastError();
        return fail(W2X_ERR_NOMEM, "w2x_band_create: cudaMalloc failed (%s)", cudaGetErrorString(e));
    };
    cudaError_t e;
    if ((e = cudaMalloc(&b->pad, (size_t)b->pw * b->hf * sizeof(float))) != cudaSuccess) return cleanup(e);
    for (int i = 0; i < 2; i++)
        if ((e = cudaMalloc(&b->act[i], b->act_bytes)) != cudaSuccess) return cleanup(e);
    if ((e = cudaMalloc(&b->flags, 64)) != cudaSuccess) return cleanup(e);
    if ((e = cudaMemset(b->flags, 0, 64)) != cudaSuccess) return cleanup(e);
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return cleanup(e);       // the flag words are zero before a neighbour can write them
    *out_band = b.release();
    return W2X_OK;
}

void w2x_band_destroy(w2x_band *band) {
    if (!band) return;
    if (band->ctx) {
        DeviceGuard g(band->ctx->device);
        cudaStreamSynchronize(band->ctx->stream);
        for (auto &p : band->peer) {
            if (!p.ipc) continue;
            if (p.pad) cudaIpcCloseMemHandle(p.pad);
            if (p.act[0]) cudaIpcCloseMemHandle(p.act[0]);
            if (p.act[1]) cudaIpcCloseMemHandle(p.act[1]);
            if (p.flags) cudaIpcCloseMemHandle(p.flags);
        }
        cudaFree(band->pad);
        cudaFree(band->act[0]);
        cudaFree(band->act[1]);
        cudaFree(band->flags);
        cudaGetLastError();
    }
    delete band;
}

// d_in: the band's rows PLUS one real row per neighbour side (the caller fetched them); every frame row is written.
int w2x_band_load(w2x_band *band, const float *d_in, size_t in_stride_bytes) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (!d_in || in_stride_bytes % 4 || in_stride_bytes < (size_t)band->width * 4) return fail(W2X_ERR_ARG, "w2x_band_load: bad input");
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    if (band->ov_up || band->ov_down) return fail(W2X_ERR_ARG, "w2x_band_load: overlap edges take their rows through w2x_band_load_rows");
    const long stride = (long)(in_stride_bytes / 4);
    const float *band0 = d_in + (band->up ? stride : 0);
    CU_CHECK(launch_pad_replicate_xy(band0, band->width, band->rows, stride, band->n, band->pt, band->pb, band->up ? 1 : 0,
                                     band->down ? 1 : 0, band->pad, ctx->stream));
    ctx->launches++;
    band->last_step = -1;
    band->cur = 0;
    return W2X_OK;
}

// d_in: the band's OWN rows; the halo rows of the input frame are left to the neighbours (w2x_band_exchange(band, -1)).  On an
// overlap edge (W2X_EDGE_OVERLAP) the n input rows beyond the band must be readable at d_in - n rows / d_in + rows.
int w2x_band_load_rows(w2x_band *band, const float *d_in, size_t in_stride_bytes) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (!d_in || in_stride_bytes % 4 || in_stride_bytes < (size_t)band->width * 4) return fail(W2X_ERR_ARG, "w2x_band_load_rows: bad input");
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    CU_CHECK(launch_pad_replicate_xy(d_in, band->width, band->rows, (long)(in_stride_bytes / 4), band->n, band->pt, band->pb,
                                     band->ov_up ? band->n : 0, band->ov_down ? band->n : 0, band->pad, ctx->stream, band->up ? 1 : 0,
                                     band->down ? 1 : 0));
    ctx->launches++;
    band->last_step = -1;
    band->cur = 0;
    return W2X_OK;
}

int w2x_band_step(w2x_band *band, int step) {
    if (band_check(band)) return W2X_ERR_ARG;
    if (step != band->last_step + 1 || step < 0 || step > band->n - 2)
        return fail(W2X_ERR_ARG, "w2x_band_step: steps must run in order 0..%d (got %d after %d)", band->n - 2, step, band->last_step);
    w2x_ctx *ctx = band->ctx;
    DeviceGuard g(ctx->device);
    const w2x_model *m = band->model;
    DevModel *dm = band->dm;
    const Layer &L = m->layers[(size_t)step];
    const int f8 = ctx->precision == W2X_PRECISION_F16_F8X2 ? 1 : 0;
    // the halo rows belong to the neighbours: they are not part of this layer's store window
    const int y0 = band->up ? 1 : 0, rows = band->hf - y0 - (band->down ? 1 : 0);
    if (step == 0) {
        LayerTimer t(ctx, 0);
        const tc::FirstSource fsrc{band->pad, band->pw, band->pw, band->hf, 0, 0, 0, 0};       // the session's padded input frame (halo rows come from the neighbours)
        CU_CHECK(tc::launch_first(fsrc, band->pw, band->hf, L.w.data(), dm->b_host[0].data(), L.n_out, band->act[0], ctx->stream, f8, y0, rows));
        band->cur = 0;
        note_kernel(ctx, 0, "first_1xN");
        ctx->launches++;
    } else {
        int rc = launch_layer_tc(ctx, m, dm, step, band->act[band->cur], band->act[band->cur ^ 1], band->pw, band->hf, step == band->n - 2, false, y0, rows);
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
    char *base = reinterpret_cast<char *>(band->act[band->cur]);
    RowSeg seg[4];
    size_t bytes, px;
    const int nseg = row_segments(band, step, seg, &bytes, &px);
    *n_segments = nseg;
    *seg_bytes = bytes;
    for (int s = 0; s < 4; s++) {
        const bool on = s < nseg;
        send_up[s] = on && band->up ? seg_at(base, band->hf, px, seg[s], 1) : nullptr;                       // first owned row
        recv_up[s] = on && band->up ? seg_at(base, band->hf, px, seg[s], 0) : nullptr;                       // halo row above
        send_down[s] = on && band->down ? seg_at(base, band->hf, px, seg[s], band->hf - 2) : nullptr;        // last owned row
        recv_down[s] = on && band->down ? seg_at(base, band->hf, px, seg[s], band->hf - 1) : nullptr;        // halo row below
    }
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
        CU_CHECK(tc::launch_last_gather_xy(reinterpret_cast<const float *>(band->act[band->cur]), band->pw, band->hf,
                                           static_cast<float>(L.b[0]), band->n, band->pt, band->pb, d_out,
                                           (long)(out_stride_bytes / 4), ctx->stream));
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
    bl.act_bytes = band->act_bytes;
    CU_CHECK(cudaIpcGetMemHandle(&bl.pad, band->pad));
    CU_CHECK(cudaIpcGetMemHandle(&bl.act0, band->act[0]));
    CU_CHECK(cudaIpcGetMemHandle(&bl.act1, band->act[1]));
    CU_CHECK(cudaIpcGetMemHandle(&bl.flags, band->flags));
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
        if (bl.magic != BLOB_MAGIC || bl.pw != band->pw || bl.n != band->n || bl.hf < 3)
            return fail(W2X_ERR_ARG, "w2x_band_connect: the %s neighbour's session does not match (width / model)", side ? "down" : "up");
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
        p.pad = o->pad;
        p.act[0] = reinterpret_cast<char *>(o->act[0]);
        p.act[1] = reinterpret_cast<char *>(o->act[1]);
        p.flags = o->flags;
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
    RowSeg seg[4];
    size_t bytes, px;
    const int nseg = row_segments(band, step, seg, &bytes, &px);
    char *mine = step < 0 ? reinterpret_cast<char *>(band->pad) : reinterpret_cast<char *>(band->act[band->cur]);
    HaloXArgs a{};
    for (int s = 0; s < nseg; s++) {
        if (band->up) {      // my first owned row -> the up neighbour's halo row below (its last frame row)
            const w2x_band::Peer &p = band->peer[0];
            char *theirs = step < 0 ? reinterpret_cast<char *>(p.pad) : p.act[band->cur];
            a.src[a.n] = seg_at(mine, band->hf, px, seg[s], 1);
            a.dst[a.n] = seg_at(theirs, p.hf, px, seg[s], p.hf - 1);
            a.n++;
        }
        if (band->down) {    // my last owned row -> the down neighbour's halo row above (its frame row 0)
            const w2x_band::Peer &p = band->peer[1];
            char *theirs = step < 0 ? reinterpret_cast<char *>(p.pad) : p.act[band->cur];
            a.src[a.n] = seg_at(mine, band->hf, px, seg[s], band->hf - 2);
            a.dst[a.n] = seg_at(theirs, p.hf, px, seg[s], 0);
            a.n++;
        }
    }
    a.bytes = bytes;
    a.counter = band->flags + 4;
    a.value = ++band->seq;
    // I am the DOWN neighbour of my up peer (its flag 1) and the UP neighbour of my down peer (its flag 0)
    a.peer_flag[0] = band->up ? band->peer[0].flags + 1 : nullptr;
    a.peer_flag[1] = band->down ? band->peer[1].flags + 0 : nullptr;
    a.my_flag[0] = band->up ? band->flags + 0 : nullptr;
    a.my_flag[1] = band->down ? band->flags + 1 : nullptr;
    NvtxRange nvtx("w2x halo exchange");
    CU_CHECK(launch_halo_exchange(a, ctx->stream));
    ctx->launches++;
    return W2X_OK;
}

// One whole pass of a connected band: own rows in, own rows out; everything is queued on the context's stream.
int w2x_band_run(w2x_band *band, const float *d_in, size_t in_stride_bytes, float *d_out, size_t out_stride_bytes) {
    int rc = w2x_band_load_rows(band, d_in, in_stride_bytes);
    if (rc) return rc;
    if ((rc = w2x_band_exchange(band, -1))) return rc;
    for (int k = 0; k <= band->n - 2; k++) {
        if ((rc = w2x_band_step(band, k))) return rc;
        if ((rc = w2x_band_exchange(band, k))) return rc;
    }
    return w2x_band_finish(band, d_out, out_stride_bytes);
}

}  // extern "C"

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
    std::vector<w2x_band *> sub;
    std::vector<int> r0;                         // sub-band s owns slab rows [r0[s], r0[s+1])
    float *d_in = nullptr, *d_out = nullptr;     // [rows][width]
    std::vector<cudaEvent_t> ev_in, ev_done;
    cudaEvent_t ev_drained = nullptr;            // the previous pass's downloads have left d_out
};

extern "C" {

void w2x_slab_destroy(w2x_slab *s) {
    if (!s) return;
    for (auto b : s->sub) w2x_band_destroy(b);
    if (s->ctx) {
        DeviceGuard g(s->ctx->device);
        cudaFree(s->d_in);
        cudaFree(s->d_out);
        for (auto e : s->ev_in) cudaEventDestroy(e);
        for (auto e : s->ev_done) cudaEventDestroy(e);
        if (s->ev_drained) cudaEventDestroy(s->ev_drained);
        cudaGetLastError();
    }
    delete s;
}

int w2x_slab_create(w2x_ctx *ctx, const w2x_model *model, int width, int rows, int has_up, int has_down, int order, int n_sub, w2x_slab **out) {
    if (check_ctx(ctx)) return W2X_ERR_ARG;
    if (!model || !out || width < 1 || rows < 1) return fail(W2X_ERR_ARG, "w2x_slab_create: bad argument");
    *out = nullptr;
    const int n = (int)model->layers.size();
    if (n_sub <= 0) n_sub = std::min(4, rows / 512);            // like w2x_convert_plane's copy pipeline
    n_sub = std::max(1, std::min(n_sub, std::min(8, rows / (4 * n))));
    // ... and as many as it takes for every sub-band's frame (its rows + at most n above and below) to stay within MAX_FRAME_ROWS
    const long sub_max = MAX_FRAME_ROWS - 2 * n;
    n_sub = std::max(n_sub, (int)((rows + sub_max - 1) / sub_max));
    auto s = std::unique_ptr<w2x_slab, void (*)(w2x_slab *)>(new w2x_slab(), w2x_slab_destroy);
    s->ctx = ctx;
    s->model = model;
    s->width = width;
    s->rows = rows;
    s->order = order ? 1 : 0;
    s->up = has_up != 0;
    s->down = has_down != 0;
    for (int i = 0; i <= n_sub; i++) s->r0.push_back((int)((long)rows * i / n_sub));
    DeviceGuard g(ctx->device);
    for (int i = 0; i < n_sub; i++) {
        w2x_band *b = nullptr;
        const int ue = i == 0 ? (s->up ? W2X_EDGE_NEIGHBOUR : W2X_EDGE_BORDER) : W2X_EDGE_OVERLAP;
        const int de = i == n_sub - 1 ? (s->down ? W2X_EDGE_NEIGHBOUR : W2X_EDGE_BORDER) : W2X_EDGE_OVERLAP;
        int rc = w2x_band_create(ctx, model, width, s->r0[(size_t)i + 1] - s->r0[(size_t)i], ue, de, &b);
        if (rc) return rc;
        s->sub.push_back(b);
    }
    CU_CHECK(cudaMalloc(&s->d_in, (size_t)rows * width * 4));
    CU_CHECK(cudaMalloc(&s->d_out, (size_t)rows * width * 4));
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
// Phase 1 of a pass: uploads and the layer loops of every sub-band (nothing here can block the host on another GPU's progress).
int slab_enqueue_compute(w2x_slab *s, const float *in, size_t in_stride_bytes) {
    w2x_ctx *ctx = s->ctx;
    DeviceGuard g(ctx->device);
    const int K = (int)s->sub.size();
    const size_t rowb = (size_t)s->width * 4;
    auto at = [&](int t) { return s->order ? K - 1 - t : t; };      // t-th sub-band in processing order
    CU_CHECK(cudaStreamWaitEvent(ctx->copy_in, s->ev_done[(size_t)at(K - 1)], 0));   // the previous pass has finished reading d_in
    CU_CHECK(cudaStreamWaitEvent(ctx->stream, s->ev_drained, 0));                    // ... and its downloads have left d_out
    // Upload t carries the t-th sub-band's rows shifted by n towards the sub-band processed next: its own rows minus the n the previous
    // upload already brought, plus the n rows of overlap context it reads from the next one -- so a sub-band waits for ITS upload only.
    const int n = (int)s->model->layers.size();
    for (int t = 0; t < K; t++) {
        const int i = at(t);
        int ya, yb;
        if (!s->order) { ya = s->r0[(size_t)i] + (t == 0 ? 0 : n); yb = s->r0[(size_t)i + 1] + (t == K - 1 ? 0 : n); }
        else { ya = s->r0[(size_t)i] - (t == K - 1 ? 0 : n); yb = s->r0[(size_t)i + 1] - (t == 0 ? 0 : n); }
        CU_CHECK(cudaMemcpy2DAsync(s->d_in + (size_t)ya * s->width, rowb, reinterpret_cast<const char *>(in) + (size_t)ya * in_stride_bytes, in_stride_bytes, rowb,
                                   (size_t)(yb - ya), cudaMemcpyHostToDevice, ctx->copy_in));
        CU_CHECK(cudaEventRecord(s->ev_in[(size_t)i], ctx->copy_in));
    }
    for (int t = 0; t < K; t++) {
        const int i = at(t), y = s->r0[(size_t)i];
        CU_CHECK(cudaStreamWaitEvent(ctx->stream, s->ev_in[(size_t)i], 0));   // own rows + the overlap rows (earlier uploads are ordered before it)
        int rc = w2x_band_run(s->sub[(size_t)i], s->d_in + (size_t)y * s->width, rowb, s->d_out + (size_t)y * s->width, rowb);
        if (rc) {
            cudaStreamSynchronize(ctx->copy_in);
            cudaStreamSynchronize(ctx->stream);
            return rc;
        }
        CU_CHECK(cudaEventRecord(s->ev_done[(size_t)i], ctx->stream));
    }
    return W2X_OK;
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
        CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char *>(out) + (size_t)y * out_stride_bytes, out_stride_bytes, s->d_out + (size_t)y * s->width, rowb, rowb,
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
    // the slabs of the last (model, width, height): planes of one job usually share a shape
    uint64_t plan_uid = 0;
    int plan_w = 0, plan_h = 0, plan_precision = -1;
    std::vector<w2x_slab *> slabs;
    std::vector<int> r0;                       // first row of every slab (+ the plane height at the end)
};

namespace {

void multi_drop_plan(w2x_multi *m) {
    for (auto b : m->slabs) w2x_slab_destroy(b);
    m->slabs.clear();
    m->plan_uid = 0;
}

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
    ~HostPin() {
        if (p) cudaHostUnregister(p);
    }
};

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
    multi_drop_plan(m);
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
    if (nd < 2 || !model->tc_eligible || m->ctx[0]->engine == W2X_ENGINE_FP32)
        return w2x_convert_plane(m->ctx[0], model, in, width, height, in_stride_bytes, out, out_stride_bytes, block_splitting);
    // ---- plan: one slab per GPU (sub-bands for the copy pipeline), neighbours wired through peer memory ----
    if (m->plan_uid != model->uid || m->plan_w != width || m->plan_h != height || (int)m->slabs.size() != nd ||
        m->plan_precision != m->ctx[0]->precision) {
        multi_drop_plan(m);
        m->r0.assign((size_t)nd + 1, 0);
        for (int i = 0; i <= nd; i++) m->r0[(size_t)i] = (int)((long)height * i / nd);
        for (int i = 0; i < nd; i++) {
            m->ctx[(size_t)i]->precision = m->ctx[0]->precision;
            w2x_slab *sl = nullptr;
            int rc = w2x_slab_create(m->ctx[(size_t)i], model, width, m->r0[(size_t)i + 1] - m->r0[(size_t)i], i > 0, i + 1 < nd, i & 1, 0, &sl);
            if (rc) { multi_drop_plan(m); return rc; }
            m->slabs.push_back(sl);
        }
        for (int i = 0; i < nd; i++) {
            int rc = w2x_slab_connect_local(m->slabs[(size_t)i], i > 0 ? m->slabs[(size_t)i - 1] : nullptr, i + 1 < nd ? m->slabs[(size_t)i + 1] : nullptr);
            if (rc) { multi_drop_plan(m); return rc; }
        }
        m->plan_uid = model->uid;
        m->plan_w = width;
        m->plan_h = height;
        m->plan_precision = m->ctx[0]->precision;
    }
    emit_reference_progress(m->ctx[0], width, height, n_layers, block_splitting && w2x_requires_splitting(width, height));
    HostPin pin_in(in, in_stride_bytes * (size_t)(height - 1) + (size_t)width * 4), pin_out(out, out_stride_bytes * (size_t)(height - 1) + (size_t)width * 4);
    // ---- queue everything (uploads, the layer loops with their exchanges, downloads) for every GPU from this one thread ----
    int rc = W2X_OK;
    for (int i = 0; i < nd && rc == W2X_OK; i++)      // phase 1 on EVERY GPU before any download can block this thread
        rc = slab_enqueue_compute(m->slabs[(size_t)i], reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + (size_t)m->r0[(size_t)i] * in_stride_bytes), in_stride_bytes);
    for (int i = 0; i < nd && rc == W2X_OK; i++)
        rc = slab_enqueue_download(m->slabs[(size_t)i], reinterpret_cast<float *>(reinterpret_cast<char *>(out) + (size_t)m->r0[(size_t)i] * out_stride_bytes), out_stride_bytes);
    for (int i = 0; i < nd; i++) {
        int r2 = w2x_slab_synchronize(m->slabs[(size_t)i]);
        if (rc == W2X_OK) rc = r2;
    }
    return rc;
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
        rc = tiles_enqueue_compute(m->ctx[(size_t)i], model, tin[(size_t)i].data(), (int)tin[(size_t)i].size(), width, height, in_stride_bytes);
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

}  // extern "C"
