// geometry.cpp -- process-wide configuration and the block-split index arithmetic (host only).
//
// Config mirrors the w2xc::modelUtility singleton (reference src/modelHandler.hpp:92-113,
// src/modelHandler.cpp:161-224): nJob = 4, blockSplittingSize = 512 x 512 by default.
// block_table reproduces the loop bounds of convertWithModelsBlockSplit
// (src/convertRoutine.cpp:100-131 for the input ROI, :143-155 for the output ROI), including the
// float ceil of :100-105 and the use of blockSize.height for the output column offset at :153-154.
#include <algorithm>
#include <climits>
#include <cmath>

#include "w2x_internal.h"

namespace w2x {

Config &config() {
    static Config c;
    return c;
}

int block_table(int w, int h, int bw, int bh, int n_model, int *table, int capacity, int *sc_out, int *sr_out) {
    if (w < 1 || h < 1 || n_model < 0 || bw - 2 * n_model < 1 || bh - 2 * n_model < 1) return -W2X_ERR_ARG;
    const unsigned n = (unsigned)n_model;
    const unsigned sc = static_cast<unsigned>(std::ceil(static_cast<float>(w) / static_cast<float>(bw - 2 * (int)n)));
    const unsigned sr = static_cast<unsigned>(std::ceil(static_cast<float>(h) / static_cast<float>(bh - 2 * (int)n)));
    if (sc_out) *sc_out = (int)sc;
    if (sr_out) *sr_out = (int)sr;
    const int pw = w + 2 * n_model, ph = h + 2 * n_model;
    int idx = 0;
    for (unsigned r = 0; r < sr; r++) {
        const int y0 = (int)(r * (unsigned)(bh - 2 * (int)n));
        const int y1 = (r == sr - 1) ? ph : y0 + bh;
        for (unsigned c = 0; c < sc; c++) {
            const int x0 = (int)(c * (unsigned)(bw - 2 * (int)n));
            const int x1 = (c == sc - 1) ? pw : x0 + bw;
            if (table && idx < capacity) {
                int *t = table + 8 * idx;
                t[0] = (int)r; t[1] = (int)c;
                t[2] = y0; t[3] = y1; t[4] = x0; t[5] = x1;
                t[6] = (int)(r * (unsigned)(bh - 2 * (int)n));
                t[7] = (int)(c * (unsigned)(bh - 2 * (int)n));   // blockSize.height, as the reference
            }
            idx++;
        }
    }
    return idx;
}

// Shelf packing: rectangles sorted by height (tallest first) fill a shelf left to right; the next one that does not fit opens a
// shelf below, as tall as that rectangle; a shelf that would pass the frame's last row opens a new frame.
int plan_planes(int n, const int *widths, const int *heights, int n_layers, int max_channels, size_t scratch_limit, int *frame,
                int *x0, int *y0, std::vector<int> *fw, std::vector<int> *fh) {
    const long px_limit = (long)std::min<size_t>(scratch_limit / ((size_t)max_channels * 4), (size_t)1 << 40);
    fw->clear();
    fh->clear();
    std::vector<int> order;
    long area = 0, wmax = 0;
    for (int i = 0; i < n; i++) {
        frame[i] = -1;
        x0[i] = y0[i] = 0;
        const long pw = (long)widths[i] + 2 * n_layers, ph = (long)heights[i] + 2 * n_layers;
        if (pw * ph > px_limit || ph > MAX_FRAME_ROWS) continue;
        order.push_back(i);
        area += pw * ph;
        wmax = std::max(wmax, pw);
    }
    if (order.empty()) return 0;
    // Frame width: the side of a square that holds every rectangle (or one full frame), rounded up to the layer kernels' 16-pixel
    // tile-set, and never narrower than the widest rectangle.  Shelf packing wastes the end of each shelf (less than one
    // rectangle per shelf, small when the frame is wide) and the rest of the last shelf (less than one shelf per frame, small
    // when the frame is tall); a square keeps both small at once.
    const long side = (long)std::ceil(std::sqrt((double)std::min(area, px_limit)));
    const long W = std::max(wmax, (side + 15) / 16 * 16);
    const long rows = std::min(MAX_FRAME_ROWS, px_limit / W);
    auto pw_of = [&](int i) { return (long)widths[i] + 2 * n_layers; };
    auto ph_of = [&](int i) { return (long)heights[i] + 2 * n_layers; };
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ph_of(a) != ph_of(b) ? ph_of(a) > ph_of(b) : pw_of(a) > pw_of(b); });
    long x = 0, y = 0, shelf_h = 0;
    for (int i : order) {
        const long pw = pw_of(i), ph = ph_of(i);
        if (ph > rows) continue;                          // taller than a frame of this width may be: converted alone
        if (fw->empty() || x + pw > W) {                  // a new shelf ...
            y += shelf_h;
            x = 0;
            shelf_h = ph;
            if (fw->empty() || y + ph > rows) {           // ... in a new frame
                fw->push_back((int)W);
                fh->push_back(0);
                y = 0;
            }
        }
        frame[i] = (int)fw->size() - 1;
        x0[i] = (int)x;
        y0[i] = (int)y;
        x += pw;
        fh->back() = (int)(y + shelf_h);
    }
    return (int)fw->size();
}

int region_windows(const char *fn, int n_steps, const w2x_model *const *models, const int *kinds, int width, int height,
                   const int *window, std::vector<Rect> *wins) {
    if (n_steps < 1) return fail(W2X_ERR_ARG, "%s: n_steps is %d: at least one step (step 0) is needed", fn, n_steps);
    if (!models) return fail(W2X_ERR_ARG, "%s: step 0: NULL models array", fn);
    if (!kinds) return fail(W2X_ERR_ARG, "%s: step 0: NULL kinds array", fn);
    long W = width, H = height;
    for (int k = 0; k < n_steps; k++) {
        const w2x_model *m = models[k];
        if (!m) return fail(W2X_ERR_ARG, "%s: step %d: NULL model", fn, k);
        if (kinds[k] & W2X_STEP_TTA) return fail(W2X_ERR_ARG, "%s: step %d: a W2X_STEP_TTA step has no window form", fn, k);
        if (kinds[k] & ~W2X_STEP_UPSCALE2X)
            return fail(W2X_ERR_ARG, "%s: step %d: kind %d is neither W2X_STEP_SAME (0) nor W2X_STEP_UPSCALE2X (1)", fn, k, kinds[k]);
        if (m->layers.front().n_in != 1 || m->layers.back().n_out != 1)
            return fail(W2X_ERR_ARG, "%s: step %d: model must map 1 plane to 1 plane", fn, k);
    }
    if (width < 1 || height < 1) return fail(W2X_ERR_ARG, "%s: step 0: input size %d x %d", fn, width, height);
    for (int k = 0; k < n_steps; k++)
        if (kinds[k] & W2X_STEP_UPSCALE2X) {
            W *= 2;
            H *= 2;
            if (W > INT_MAX || H > INT_MAX) return fail(W2X_ERR_ARG, "%s: step %d: the output size %ld x %ld overflows int", fn, k, W, H);
        }
    if (!window) return fail(W2X_ERR_ARG, "%s: NULL window", fn);
    const Rect o{window[0], window[1], window[2], window[3]};
    if (o.w < 1 || o.h < 1) return fail(W2X_ERR_ARG, "%s: empty window %d x %d", fn, o.w, o.h);
    if (o.x0 < 0 || o.y0 < 0 || o.x0 > W - o.w || o.y0 > H - o.h)
        return fail(W2X_ERR_ARG, "%s: window {%d, %d, %d, %d} is not inside the %ld x %ld output", fn, o.x0, o.y0, o.w, o.h, W, H);
    wins->assign((size_t)n_steps + 1, o);
    for (int k = n_steps - 1; k >= 0; k--) {   // (W, H): step k's output plane
        const Rect &r = (*wins)[(size_t)k + 1];
        const int n = (int)models[k]->layers.size();
        int x0 = std::max(0, r.x0 - n), y0 = std::max(0, r.y0 - n);
        int x1 = (int)std::min<long>(W, (long)r.x1() + n), y1 = (int)std::min<long>(H, (long)r.y1() + n);
        if (kinds[k] & W2X_STEP_UPSCALE2X) {
            x0 >>= 1, y0 >>= 1, x1 = (x1 + 1) >> 1, y1 = (y1 + 1) >> 1;
            W /= 2, H /= 2;
        }
        (*wins)[(size_t)k] = Rect{x0, y0, x1 - x0, y1 - y0};
    }
    return W2X_OK;
}

}  // namespace w2x

extern "C" {

int w2x_chain_region_source(int n_steps, const w2x_model *const *models, const int *kinds, int width, int height, const int *window,
                            int *source) {
    std::vector<w2x::Rect> wins;
    int rc = w2x::region_windows("w2x_chain_region_source", n_steps, models, kinds, width, height, window, &wins);
    if (rc) return rc;
    if (!source) return w2x::fail(W2X_ERR_ARG, "w2x_chain_region_source: NULL source");
    source[0] = wins[0].x0;
    source[1] = wins[0].y0;
    source[2] = wins[0].w;
    source[3] = wins[0].h;
    return W2X_OK;
}

int w2x_set_jobs(int n_job) {
    if (n_job < 1) return w2x::fail(W2X_ERR_ARG, "w2x_set_jobs: number of jobs must be >= 1");
    w2x::config().n_job = n_job;
    return W2X_OK;
}
int w2x_get_jobs(void) { return w2x::config().n_job; }

int w2x_set_block_size(int width, int height) {
    if (width < 0 || height < 0) return w2x::fail(W2X_ERR_ARG, "w2x_set_block_size: negative size");
    w2x::config().block_w = width;
    w2x::config().block_h = height;
    return W2X_OK;
}
int w2x_set_block_size_exp2_square(int exp) {
    if (exp < 0 || exp > 30) return w2x::fail(W2X_ERR_ARG, "w2x_set_block_size_exp2_square: bad exponent");
    int len = 1 << exp;
    w2x::config().block_w = len;
    w2x::config().block_h = len;
    return W2X_OK;
}
void w2x_get_block_size(int *width, int *height) {
    if (width) *width = w2x::config().block_w;
    if (height) *height = w2x::config().block_h;
}

int w2x_requires_splitting(int width, int height) {
    const w2x::Config &c = w2x::config();
    return (width * height) > c.block_w * c.block_h * 3 / 2 ? 1 : 0;  // int math, src/convertRoutine.cpp:25-26
}

int w2x_block_table(int width, int height, int n_model, int *table, int capacity, int *split_cols, int *split_rows) {
    const w2x::Config &c = w2x::config();
    int n = w2x::block_table(width, height, c.block_w, c.block_h, n_model, table, capacity, split_cols, split_rows);
    if (n < 0) {
        w2x::fail(W2X_ERR_ARG, "w2x_block_table: bad plane size, pad width or block size");
        return -W2X_ERR_ARG;
    }
    return n;
}

// Probe hook (not part of the stable ABI, needs no device): the frame plan w2x_convert_planes makes for these plane sizes with a
// model of n_layers layers at most max_channels wide and the given scratch limit.  Per plane: frame index (-1 = converted alone)
// and the padded rectangle's top-left corner; frame_dims gets (width, height) of the first `capacity` frames.  Returns the
// frame count, or -W2X_ERR_ARG.
W2X_API int w2x_debug_plan_planes(int n_planes, const int *widths, const int *heights, int n_layers, int max_channels,
                                  size_t scratch_limit, int *frame, int *x0, int *y0, int *frame_dims, int capacity) {
    if (n_planes < 1 || !widths || !heights || !frame || !x0 || !y0 || n_layers < 1 || max_channels < 1 || !scratch_limit)
        return -w2x::fail(W2X_ERR_ARG, "w2x_debug_plan_planes: bad argument");
    for (int i = 0; i < n_planes; i++)
        if (widths[i] < 1 || heights[i] < 1) return -w2x::fail(W2X_ERR_ARG, "w2x_debug_plan_planes: plane %d has no pixels", i);
    std::vector<int> fw, fh;
    const int nf = w2x::plan_planes(n_planes, widths, heights, n_layers, max_channels, scratch_limit, frame, x0, y0, &fw, &fh);
    for (int f = 0; f < nf && f < capacity && frame_dims; f++) {
        frame_dims[2 * f] = fw[(size_t)f];
        frame_dims[2 * f + 1] = fh[(size_t)f];
    }
    return nf;
}

}  // extern "C"
