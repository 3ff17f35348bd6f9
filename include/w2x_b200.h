/*
 * w2x_b200.h -- C ABI of the H100-native (sm_90a) convolution hot path of waifu2x-converter-cpp.
 *
 * This is the drop-in boundary.  The reference (WL-Amigo/waifu2x-converter-cpp, C++11) has no
 * plugin/FFI layer; the functions its CLI calls for this path are the ones replaced here.  Every
 * entry point cites the reference interface it stands in for (paths relative to the reference
 * repository root).  Plain C types only: no OpenCV, no torch, no C++ in the signatures.
 *
 * Conventions
 *   - every function that can fail returns an int status (W2X_OK == 0); the reference's `bool`
 *     results and its std::exit(-1) paths (src/modelHandler.hpp:57,69, src/convertRoutine.cpp:69)
 *     both become non-zero statuses -- the library never calls exit();
 *   - w2x_last_error() returns the message the reference would have written to std::cerr
 *     (thread-local, valid until the next failing call on the same thread);
 *   - planes are fp32 (CV_32FC1), row-major, described by (pointer, width, height,
 *     row stride in BYTES) so a strided ROI (src/convertRoutine.cpp:116-131) can be passed as is;
 *   - there is NO CPU fallback: the compute entry points fail with W2X_ERR_NO_DEVICE when no
 *     sm_90 (H100) device is present.
 */
#ifndef W2X_B200_H_
#define W2X_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define W2X_API __attribute__((visibility("default")))
#else
#define W2X_API
#endif

/* ---- status codes ------------------------------------------------------------------------- */
#define W2X_OK 0
#define W2X_ERR_ARG 1          /* bad argument (NULL, non-positive size, plane-count mismatch) */
#define W2X_ERR_IO 2           /* "Error : couldn't open <file>"  (src/modelHandler.cpp:176-179) */
#define W2X_ERR_PARSE 3        /* "Error : PicoJSON Error : ..."  (src/modelHandler.cpp:183-187) */
#define W2X_ERR_MODEL 4        /* malformed model: non-square kernel (src/modelHandler.hpp:52-58),
                                  wrong types/shapes, layer chain mismatch, unsupported kernel size */
#define W2X_ERR_CUDA 5         /* a CUDA runtime/driver call failed */
#define W2X_ERR_NO_DEVICE 6    /* no CUDA device / not an sm_90 part: no CPU fallback exists */
#define W2X_ERR_UNSUPPORTED 7  /* layer shape not supported by the requested engine */
#define W2X_ERR_NOMEM 8

typedef struct w2x_model w2x_model; /* a loaded model = std::vector<std::unique_ptr<w2xc::Model>> */
typedef struct w2x_ctx w2x_ctx;     /* one GPU + stream + scratch buffers */

W2X_API const char *w2x_last_error(void);
W2X_API const char *w2x_version(void); /* "1.0.0-b200.<n>" ; the reference CLI is 1.0.0 (src/main.cpp:26) */

/* ---- model container ---------------------------------------------------------------------- */
/* Replaces w2xc::modelUtility::generateModelFromJSON(fileName, models)
 * (src/modelHandler.hpp:104-105, src/modelHandler.cpp:170-197) together with the Model
 * constructor and loadModelFromJSONObject (src/modelHandler.hpp:48-71, src/modelHandler.cpp:74-115):
 * same file format (array of {nInputPlane,nOutputPlane,kW,kH,weight[o][i][ky][kx],bias[o]}),
 * numbers parsed strtod-exactly, weights rounded double->float, biases kept double. */
W2X_API int w2x_model_load_json(const char *path, w2x_model **out_model);
/* Same container built from memory (what a binding that already holds the parsed arrays calls).
 * weights[l] is [n_out][n_in][3][3] fp32, biases[l] is [n_out] fp64. */
W2X_API int w2x_model_create(int n_layers, const int *n_in, const int *n_out,
                             const float *const *weights, const double *const *biases,
                             w2x_model **out_model);
W2X_API void w2x_model_free(w2x_model *model);
/* models.size() as used at src/convertRoutine.cpp:33,93 (nModel = pad width = 7). */
W2X_API int w2x_model_layer_count(const w2x_model *model);
/* Model::getNInputPlanes / getNOutputPlanes (src/modelHandler.hpp:81-82) + kernelSize. */
W2X_API int w2x_model_layer_dims(const w2x_model *model, int layer, int *n_in, int *n_out, int *k);
/* Read-only views of the stored parameters (the reference's printWeightMatrix/printBiases
 * debugging hooks, src/modelHandler.hpp:77-78). */
W2X_API int w2x_model_layer_params(const w2x_model *model, int layer, const float **weights,
                                   const double **biases);

/* ---- process-wide configuration: w2xc::modelUtility (src/modelHandler.hpp:92-113) ----------- */
W2X_API int w2x_set_jobs(int n_job);               /* setNumberOfJobs: <1 -> W2X_ERR_ARG. Parsed and
                                                      stored for drop-in compatibility; the GPU path
                                                      has no use for it. */
W2X_API int w2x_get_jobs(void);                     /* default 4 */
W2X_API int w2x_set_block_size(int width, int height);   /* setBlockSize */
W2X_API int w2x_set_block_size_exp2_square(int exp);     /* setBlockSizeExp2Square */
W2X_API void w2x_get_block_size(int *width, int *height); /* default 512 x 512 */

/* ---- block geometry of convertWithModelsBlockSplit (src/convertRoutine.cpp:84-169) ----------- */
/* The split decision of src/convertRoutine.cpp:25-26 (int arithmetic, current block size). */
W2X_API int w2x_requires_splitting(int width, int height);
/* Fills 8 ints per block in the reference's processing order (r outer, c inner):
 *   { r, c, in_y0, in_y1, in_x0, in_x1, out_y0, out_x0 }
 * in_* index the pad-n_model plane, out_* the output plane.  Returns the number of blocks, or a
 * negative status.  table may be NULL (count only); capacity counts blocks. */
W2X_API int w2x_block_table(int width, int height, int n_model, int *table, int capacity,
                            int *split_cols, int *split_rows);

/* ---- context ------------------------------------------------------------------------------ */
#define W2X_ENGINE_AUTO 0  /* tensor-core path when the model shape allows, else fp32 */
#define W2X_ENGINE_FP32 1  /* hand-written fp32 CUDA-core direct convolution (reference op order) */
#define W2X_ENGINE_TC 2    /* hand-written wgmma/TMA implicit-GEMM, 2-term fp16 split, fp32 accum */

W2X_API int w2x_ctx_create(int device, w2x_ctx **out_ctx);
W2X_API void w2x_ctx_destroy(w2x_ctx *ctx);
/* A context caches device copies of every model it has converted with; this drops one model's copies
 * (call before w2x_model_free when a long-lived context cycles through many models).  Returns W2X_ERR_ARG, and keeps
 * the copies, while band sessions on this context use the model: w2x_band_* sessions, the sub-bands of w2x_slab_*
 * and the plans w2x_multi_convert_plane and w2x_multi_convert_chain keep for their last (models, width, height).  Destroy those
 * first. */
W2X_API int w2x_ctx_forget_model(w2x_ctx *ctx, const w2x_model *model);
W2X_API int w2x_ctx_set_engine(w2x_ctx *ctx, int engine);
W2X_API int w2x_ctx_get_engine(const w2x_ctx *ctx);
/* Arithmetic of the tensor-core engine (both keep fp32 accumulators and meet the 1e-4 gate of BASELINE.json):
 *   W2X_PRECISION_F16X3     x*w = xh*wh + xl*wh + xh*wl, three fp16 tensor-core products
 *                           (measured on H100: <= 7.4e-6 max-abs against the reference CPU path on white noise;
 *                           283 Mpix/s on a 4096x4096 scale2.0x pass, H100 80GB HBM3 at a 400 W power limit)
 *   W2X_PRECISION_F16_F8X2  (default) the two correction products run on e4m3 copies of the operands at twice
 *                           the tensor rate: 2.0 instead of 3.0 pass-equivalents; measured on H100: <= 2.2e-5
 *                           max-abs on white noise, <= 5.9e-6 on a smooth image; 357 Mpix/s on the same pass and card
 *   W2X_PRECISION_F16       one fp16 product per MAC (xh*wh) with fp32 accumulation: a different accuracy contract,
 *                           NOT held to the 1e-4 gate; 8-bit outputs (rint(255 y)) stay within 1 LSB of the
 *                           reference's.  Measured on H100 (tools/precision_bench.py): 9.0e-4 max-abs against the
 *                           fp32 engine on sampled rows of a 4096x4096 white-noise scale2.0x pass (2.1 % of the 8-bit
 *                           values change, by 1); 566 Mpix/s on that pass against the default's 309 in the same run,
 *                           H100 80GB HBM3 at a 400 W power limit
 * Activation range (a = the largest |activation| entering any tensor-core layer; relative error = max-abs error /
 * max(1, max |reference|); the shipped models reach a = 1 on planes in [0, 1] and grow about linearly with the input's
 * scale, so a plane in 0..255 reaches a = 100 to 300).  Asserted by tests/test_activation_range.py:
 *   W2X_PRECISION_F16X3     <= 1e-6 relative to float64 arithmetic (2e-5 to the reference's own fp32 path) for
 *                           a < 4094 (16 a < 65520, the fp16 limit of the activation records)
 *   W2X_PRECISION_F16_F8X2  <= 6e-5 relative for a < 56 (16 a < 896).  From a = 56 the e4m3 copies saturate
 *                           (xh8 = e4m3(16 a / 2) at 448, from a = 64 also xl8) and the corrections are capped:
 *                           <= 1e-3 relative for a < 4094 (about 1e-4 at a = 150 to 300)
 *   W2X_PRECISION_F16       <= 4e-3 relative for a < 4094
 * Beyond a = 4094 every precision saturates its records at +-65504 (fp16 hi and lo): outputs stay finite, with no
 * accuracy bound (they no longer follow the reference).  The fp32 engine has no such limit.
 * Model scale: the records hold 16 a at a fixed scale, so a layer whose activations are small loses their low bits
 * (fp16 subnormals; e4m3 underflow of the default precision's copies) and later layers amplify the loss.  With
 * g = the largest ratio, over the inputs of the tensor-core layers (layers 1 .. L-2), of max(1, max |output|) to that
 * input's largest |activation| (about 7 for the shipped models on planes in [0, 1]), the ranges above hold for g <= 64
 * (the default precision also needs max |w| >= 1/16 in every tensor-core layer: below, the weight scale of the packed
 * operands, at most 2^14, no longer lifts them to the e4m3 copies' range).  Beyond, for a < 4094:
 *   W2X_PRECISION_F16X3     <= 4e-8 g relative to float64 (about 1.3e-4 at g = 3e4)
 *   W2X_PRECISION_F16_F8X2  <= 1e-3 relative (about 4e-4 at g = 3e4)
 * Asserted by tests/test_model_scale.py on power-of-two rescalings of the shipped models (one layer's output x 2^-12 to
 * 2^12), which the reference and the fp32 engine compute bit for bit as the originals.  A model whose tensor-core layers
 * hold a non-finite weight or one of |w| >= 65520 (past the fp16 limit) runs on the fp32 engine: W2X_ENGINE_AUTO picks
 * it; W2X_ENGINE_TC returns W2X_ERR_UNSUPPORTED for it, and for w2x_filter_layer of such a layer.
 *   W2X_PRECISION_BF16X3    x*w = xh*wh + xl*wh + xh*wl with h = the bf16 rounding: three bf16 tensor-core products
 *                           on records hi = bf16(16 a), lo = bf16(16 a - hi) and weights packed at scale 1.  bf16 has
 *                           fp32's exponent range, so nothing saturates or underflows where fp16 and e4m3 do:
 *                           <= 3e-5 relative to float64 for any activation and model scale whose activations stay
 *                           within fp32's normal range (measured on H100: 7e-6 to 1.5e-5 at input scales x1 to x1e6;
 *                           f16x3 stays the more accurate choice at a < 4094 and g <= 64).  A power-of-two rescaling of
 *                           a model's layers (as above) gives bit-identical outputs.  Eligibility: the same layer shapes
 *                           with finite inner weights, no 65520 limit; W2X_ENGINE_AUTO runs such a model on the tensor
 *                           cores in this precision only (every other precision still sends a weight of |w| >= 65520 to
 *                           the fp32 engine), and W2X_ENGINE_TC refuses only non-finite inner weights.  Measured with
 *                           tools/precision_bench.py on a 4096x4096 scale2.0x pass: 380 Mpix/s against f16x3's 366 in
 *                           the same run, H100 80GB HBM3 at a 700 W power limit and a 1980 MHz max SM clock.
 *                           Asserted by tests/test_precision_bf16.py. */
/* The environment variable W2X_PRECISION=f16x3|f8|f16|bf16x3 sets the initial value of new contexts. */
#define W2X_PRECISION_F16X3 0
#define W2X_PRECISION_F16_F8X2 1
#define W2X_PRECISION_F16 2
/* 3 is not a precision and stays one: w2x_ctx_set_precision(ctx, 3) returns W2X_ERR_ARG.  bf16x3 is 4. */
#define W2X_PRECISION_BF16X3 4
W2X_API int w2x_ctx_set_precision(w2x_ctx *ctx, int precision);
W2X_API int w2x_ctx_get_precision(const w2x_ctx *ctx);
/* Run on a caller-owned CUDA stream (cudaStream_t passed as void*); NULL = the ctx's own stream.
 * A host-buffer entry point starts its copies only after the work already queued on the context's stream.
 * Work queued after a switch starts after everything the context queued before it, on any stream: the new
 * stream waits for the previous one (one event, no host wait; setting the current stream again does nothing).
 * The previous stream must still be valid when it is replaced. */
W2X_API int w2x_ctx_set_stream(w2x_ctx *ctx, void *cuda_stream);
/* Block until everything queued by this context has finished. */
W2X_API int w2x_ctx_synchronize(w2x_ctx *ctx);
/* Progress lines exactly as the reference prints them to std::cout
 * ("Iteration #k..." src/convertRoutine.cpp:67, "start process block (c,r) ..." :133-134).
 * A call prints its lines before it queues the work they describe, and a call rejected by its argument checks prints none.
 * NULL disables (default). */
typedef void (*w2x_log_fn)(const char *line, void *user);
W2X_API int w2x_ctx_set_log(w2x_ctx *ctx, w2x_log_fn fn, void *user);
/* W2X_WALK_FUSED (default): a plane that the reference would block-split is processed in one pass
 * of whole-plane kernels (results are bit-identical to the block walk because every output pixel
 * sees the same operands in the same order).  W2X_WALK_BLOCKS: walk the reference's blocks one by
 * one in its order -- kept for fidelity tests and for the per-block progress lines. */
#define W2X_WALK_FUSED 0
#define W2X_WALK_BLOCKS 1
W2X_API int w2x_ctx_set_block_walk(w2x_ctx *ctx, int mode);
/* Upper bound in bytes for ONE activation scratch buffer (two are kept); larger planes are
 * processed in horizontal bands with a 7-row recompute halo.  0 = default (16 GiB). */
W2X_API int w2x_ctx_set_scratch_limit(w2x_ctx *ctx, size_t bytes);

/* Page-locked host memory for planes handed to the host-buffer entry points (optional: any host pointer works, pinned
 * ones make the copies asynchronous and link-rate).  NULL when no device / out of memory: fall back to malloc. */
W2X_API void *w2x_host_alloc(size_t bytes);
W2X_API void w2x_host_free(void *p);

/* ---- the hot path ------------------------------------------------------------------------- */
/* Device memory of w2x_convert_plane*, w2x_convert_planes*, w2x_convert_chain*, w2x_convert_planes_chain*,
 * w2x_convert_chain_region* and w2x_convert_chain_regions*: every buffer a call uses (the host entries' staging, the planes between steps, TTA variants, packed
 * frames, activation and padding scratch) is reserved before its first progress line, on_step call, copy or launch, so
 * W2X_ERR_NOMEM leaves nothing logged, called back or queued.  The context keeps its buffers for later calls. */
/* Replaces bool w2xc::convertWithModels(cv::Mat& in, cv::Mat& out, models, bool blockSplitting)
 * (src/convertRoutine.hpp:25-28, src/convertRoutine.cpp:21-51): out = crop_n(L_{n-1}(...L_0(
 * replicate_pad_n(in)))) with every layer = 3x3 correlation + bias + leaky-ReLU(0.1).
 * HOST buffers; host->device and device->host copies happen inside the call; synchronous.
 * in and out must not overlap (the reference's callers deep-copy first, src/main.cpp:94,140). */
W2X_API int w2x_convert_plane(w2x_ctx *ctx, const w2x_model *model, const float *in, int width,
                              int height, size_t in_stride_bytes, float *out,
                              size_t out_stride_bytes, int block_splitting);
/* Same, DEVICE buffers, asynchronous on the context's stream. */
W2X_API int w2x_convert_plane_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in,
                                     int width, int height, size_t in_stride_bytes, float *d_out,
                                     size_t out_stride_bytes, int block_splitting);
/* Replaces bool Model::filter(std::vector<cv::Mat>& in, std::vector<cv::Mat>& out)
 * (src/modelHandler.hpp:87-88, src/modelHandler.cpp:26-72,117-159): one layer, same-size output,
 * BORDER_REPLICATE.  n_in_planes must equal the layer's nInputPlane (mismatch -> W2X_ERR_ARG with
 * the reference's "number of input planes mismatch." message).  HOST plane pointers. */
W2X_API int w2x_filter_layer(w2x_ctx *ctx, const w2x_model *model, int layer,
                             const float *const *in_planes, int n_in_planes,
                             float *const *out_planes, int n_out_planes, int width, int height,
                             size_t in_stride_bytes, size_t out_stride_bytes);
/* Same on dense planar DEVICE tensors: d_in [n_in][h][w], d_out [n_out][h][w]; asynchronous. */
W2X_API int w2x_filter_layer_device(w2x_ctx *ctx, const w2x_model *model, int layer,
                                    const float *d_in, float *d_out, int width, int height);

/* ---- multi-GPU row-band mode (one process per GPU; the caller moves the halo rows) ----------- */
/* A plane of `height` rows is cut into contiguous bands, one per rank.  Each rank calls
 * w2x_band_begin with ITS band of the input plus up to n_layers rows of real neighbour data
 * above and below (rows_above/rows_below; 0 at the image border, where the library replicates
 * like src/convertRoutine.cpp:35,96).  This is the zero-exchange ("input halo, recompute")
 * variant: one call per rank, no collective on the data path.  d_in points at the first halo row
 * (i.e. band row -rows_above); d_out receives band_height rows. */
W2X_API int w2x_convert_band_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in,
                                    int width, int band_height, int rows_above, int rows_below,
                                    size_t in_stride_bytes, float *d_out, size_t out_stride_bytes);

/* ---- multi-GPU row-band mode with a halo exchange BETWEEN LAYERS ------------------------------ */
/* The variant BASELINE.json's north_star names: each GPU keeps only its own rows (+1 halo row per
 * neighbour side) of every intermediate activation and trades ONE boundary row with each neighbour
 * after every layer.  A session is one GPU's band; all calls are asynchronous on the context's stream.
 *
 * Exchange inside the library (the product path): the neighbours' frames are peer-mapped and
 * w2x_band_exchange stores the boundary rows straight into them over NVLink -- one small kernel per
 * layer (rows, a flag in the receiver's memory, wait for the neighbours' flags); no host round trip.
 *     w2x_band_connect_local(band, up, down)        neighbours in the same process (cudaDeviceEnablePeerAccess), or
 *     w2x_band_export(band, blob) + w2x_band_connect(band, up_blob, down_blob)   between processes (CUDA IPC):
 *                                                   every rank exports, the blobs travel over any host channel
 *     w2x_band_run(band, d_in, stride, d_out, stride)   one pass: own rows in -> own rows out
 *         = w2x_band_load_rows; w2x_band_exchange(-1); { w2x_band_step(k); w2x_band_exchange(k) } k = 0..n-2; w2x_band_finish
 * Every rank of a group must run the same sequence of exchanges (they are numbered).
 *
 * Exchange by the caller (cross-check path; ncclSend/ncclRecv, torch.distributed P2P):
 *     w2x_band_load(band, d_in, stride)            input: band rows + 1 real row per neighbour side
 *     for k in 0 .. n-2:  w2x_band_step(band, k);  w2x_band_halo(band, k, ...) -> move the segments
 *     w2x_band_finish(band, d_out, stride)
 * Step n-2 is the tensor-core layer with the last layer folded into its epilogue; its rows are per-pixel tap
 * partials instead of activations.  Requires the tensor-core engine.  The layer kernels never store a band's
 * halo rows, so a neighbour's row may arrive at any time after the previous exchange. */
typedef struct w2x_band w2x_band;
/* What lies beyond a band's first / last row: */
#define W2X_EDGE_BORDER 0      /* the image border: replicate (src/convertRoutine.cpp:35,96) */
#define W2X_EDGE_NEIGHBOUR 1   /* another GPU's band: one halo row, exchanged after every layer */
#define W2X_EDGE_OVERLAP 2     /* n_layers real input rows supplied with the band and recomputed (no exchange): the seam
                                  between two sub-bands of ONE GPU (w2x_slab_*), input read through w2x_band_load_rows */
/* A band's frame is band_rows plus 1 row per W2X_EDGE_NEIGHBOUR side and n_layers rows per other side; a frame of more than
 * 8 * 65535 = 524280 rows is refused with W2X_ERR_ARG before anything is allocated. */
W2X_API int w2x_band_create(w2x_ctx *ctx, const w2x_model *model, int width, int band_rows,
                            int up_edge, int down_edge, w2x_band **out_band);
W2X_API void w2x_band_destroy(w2x_band *band);
W2X_API int w2x_band_load(w2x_band *band, const float *d_in, size_t in_stride_bytes);
W2X_API int w2x_band_load_rows(w2x_band *band, const float *d_in_own_rows, size_t in_stride_bytes);
W2X_API int w2x_band_step(w2x_band *band, int step);
/* Segments to move after `step` was queued: n_segments (<= 4) contiguous device ranges of
 * seg_bytes each per direction; send_* hold this rank's boundary row, recv_* its halo row.
 * Pointers for a missing neighbour are NULL.  Arrays must have room for 4 entries. */
W2X_API int w2x_band_halo(w2x_band *band, int step, int *n_segments, void **send_up, void **recv_up,
                          void **send_down, void **recv_down, size_t *seg_bytes);
W2X_API int w2x_band_finish(w2x_band *band, float *d_out, size_t out_stride_bytes);
#define W2X_BAND_BLOB_BYTES 320
W2X_API int w2x_band_export(w2x_band *band, void *blob /* W2X_BAND_BLOB_BYTES */);
W2X_API int w2x_band_connect(w2x_band *band, const void *up_blob, const void *down_blob);
W2X_API int w2x_band_connect_local(w2x_band *band, w2x_band *up, w2x_band *down);
W2X_API int w2x_band_exchange(w2x_band *band, int step /* -1 after w2x_band_load_rows */);
W2X_API int w2x_band_run(w2x_band *band, const float *d_in_own_rows, size_t in_stride_bytes, float *d_out,
                         size_t out_stride_bytes);

/* ---- one GPU's slab of a multi-GPU plane, HOST buffers ------------------------------------------------ */
/* What a rank of a multi-process job (or one GPU of w2x_multi_*) owns of the plane: rows in pinned host memory go in,
 * rows come out.  The slab is cut into sub-bands so that uploads, layers and downloads overlap; seams inside the slab are
 * W2X_EDGE_OVERLAP (recomputed, local data), its outer edges exchange a halo row per layer with the neighbour slab.
 * order: 0 = walk the sub-bands top -> bottom, 1 = bottom -> top; neighbouring slabs must alternate (rank parity) so that
 * both sides of a boundary are in flight at the same time.  n_sub = 0: automatic.  Blobs are 2 * W2X_BAND_BLOB_BYTES.
 * n_sub is raised, past any number asked for, until every sub-band's frame has at most 524280 rows. */
typedef struct w2x_slab w2x_slab;
W2X_API int w2x_slab_create(w2x_ctx *ctx, const w2x_model *model, int width, int rows, int has_up_neighbour,
                            int has_down_neighbour, int order, int n_sub, w2x_slab **out_slab);
W2X_API void w2x_slab_destroy(w2x_slab *slab);
W2X_API int w2x_slab_export(w2x_slab *slab, void *blob /* 2 * W2X_BAND_BLOB_BYTES */);
W2X_API int w2x_slab_connect(w2x_slab *slab, const void *up_blob, const void *down_blob);
W2X_API int w2x_slab_connect_local(w2x_slab *slab, w2x_slab *up, w2x_slab *down);
W2X_API int w2x_slab_convert(w2x_slab *slab, const float *in_rows, size_t in_stride_bytes, float *out_rows,
                             size_t out_stride_bytes);
W2X_API int w2x_slab_convert_async(w2x_slab *slab, const float *in_rows, size_t in_stride_bytes, float *out_rows,
                                   size_t out_stride_bytes);
W2X_API int w2x_slab_synchronize(w2x_slab *slab);

/* ---- independent planes of one shape in one pass ---------------------------------------------- */
/* The reference's block loop (src/convertRoutine.cpp:114-165) and BASELINE config 5 (64 x 512x512 tiles):
 * n_tiles planes, each converted exactly like w2x_convert_plane(block_splitting = 0) would -- bit-identical --
 * but stacked into ONE frame so that every layer is one launch for the whole batch.  HOST pointers; batches of
 * eight tiles and more are cut into up to four such frames so that uploads, layers and downloads overlap. */
W2X_API int w2x_convert_tiles(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles,
                              float *const *out_tiles, int n_tiles, int width, int height,
                              size_t in_stride_bytes, size_t out_stride_bytes);
/* Same, returns once everything is queued (pinned host memory makes it truly asynchronous);
 * w2x_ctx_synchronize completes it. */
W2X_API int w2x_convert_tiles_async(w2x_ctx *ctx, const w2x_model *model, const float *const *in_tiles,
                                    float *const *out_tiles, int n_tiles, int width, int height,
                                    size_t in_stride_bytes, size_t out_stride_bytes);
/* Same on dense DEVICE batches d_in [n_tiles][height][width] -> d_out; asynchronous. */
W2X_API int w2x_convert_tiles_device(w2x_ctx *ctx, const w2x_model *model, const float *d_in, float *d_out,
                                     int n_tiles, int width, int height);

/* ---- independent planes of any sizes in one pass ------------------------------------------------ */
/* For collections of small images of different sizes (sprite and icon sets, dataset crops, thumbnails), which one
 * w2x_convert_plane call each would run on a fraction of the GPU.  The reference converts such a collection a plane at a time
 * (convertWithModels per image, src/main.cpp:96,148), and its own block loop converts blocks of up to four shapes one after
 * another (src/convertRoutine.cpp:114-165).
 * n_planes independent planes of any sizes, each converted exactly like w2x_convert_plane(block_splitting = 0) would convert it
 * -- bit-identical -- but packed side by side into as few frames as the scratch limit allows, so that every layer is one launch
 * per frame.  A plane whose padded rectangle fits no frame is converted alone.  Only the tensor-core engine with the fused last
 * layer packs; every other case converts plane by plane.  Every plane is checked before anything is queued: NULL pointers,
 * sizes < 1 and row strides that are not multiples of 4 or shorter than a row give W2X_ERR_ARG naming the plane index.
 * The progress lines are the ones the single-plane calls would log, plane by plane in order.
 * HOST buffers, synchronous; uploads, layers and downloads of successive frames overlap. */
W2X_API int w2x_convert_planes(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *in, const int *widths,
                               const int *heights, const size_t *in_strides, float *const *out, const size_t *out_strides);
/* Same on DEVICE planes (the pointer, size and stride arrays themselves are host arrays), asynchronous on the context's stream. */
W2X_API int w2x_convert_planes_device(w2x_ctx *ctx, const w2x_model *model, int n_planes, const float *const *d_in,
                                      const int *widths, const int *heights, const size_t *in_strides, float *const *d_out,
                                      const size_t *out_strides);

/* ---- a chain of conversions on one plane: noise reduction, then 2x scaling steps ------------------ */
/* The reference's main loop (src/main.cpp:82-156) runs the Y plane through the noise model (:96) and then through k scale
 * iterations, each a nearest-neighbour 2x resize followed by the scale model (:132-148).  Y after a step depends only on Y before
 * it (split, merge and an exact 2x INTER_NEAREST resize copy values; the bicubic Y channel is overwritten at :148-154), so the
 * whole sequence can run in one call that keeps the plane on the device between steps and never builds the 2x plane.
 * Step k computes P_{k+1} = convertWithModels(models[k], U_k(P_k)), P_0 = in, U_k = identity (W2X_STEP_SAME) or the nearest 2x
 * resize (W2X_STEP_UPSCALE2X); every P_{k+1} is bit-identical to w2x_convert_plane(ctx, models[k], U_k(P_k), ..., block_splitting)
 * on the same context settings.  The output is (width << u) x (height << u), u = the number of upscaling steps.  With n_steps == 1
 * and W2X_STEP_SAME this is w2x_convert_plane (w2x_convert_plane_device): same bits, same progress lines, same launches.
 * Before step k is queued, on_step(k, user) is called (if not NULL); then the step logs the progress lines w2x_convert_plane
 * (host entry) or w2x_convert_plane_device (device entry) logs for its plane, block lines included.
 * Every argument is checked before anything is queued; W2X_ERR_ARG names the step: n_steps < 1, a NULL models / kinds array or
 * model, an unknown kind, a model that does not map 1 plane to 1 plane, an output size that overflows int, bad row strides
 * (multiples of 4 bytes, >= the row) or NULL planes.  in and out must not overlap.
 * HOST buffers, synchronous. */
#define W2X_STEP_SAME 0        /* the model's output replaces the plane (noise pass, src/main.cpp:96) */
#define W2X_STEP_UPSCALE2X 1   /* cv::resize INTER_NEAREST to 2w x 2h (src/main.cpp:132-140), then the model (:148) */
/* Test-time augmentation, OR-ed into a step's kind (valid kinds: 0, 1, 4, 5): average the step over the 8 flips / transposes of its
 * plane(s), the "-tta" switch of later waifu2x front ends.  It damps the orientation bias of the SRCNN output (ringing along edges)
 * at 8x the layer work.  Variant j = 0..7 of a w x h plane X, with t = bit 2, fy = bit 1 and fx = bit 0 of j, is W' x H' =
 * (t ? h : w) x (t ? w : h) and V_j[y][x] = X[r][c], x' = fx ? W'-1-x : x, y' = fy ? H'-1-y : y, (r, c) = t ? (x', y') : (y', x');
 * V_0 = X.  The step maps P to (((O_0 + O_1) + O_2) + ... + O_7) * 0.125f in fp32, left to right, where O_j is
 * convertWithModels(models[k], V_j(U_k(P))) carried back through the same index map (out[r][c] = O_j[y][x]).  Every O_j is
 * bit-identical to w2x_convert_plane(block_splitting = 0) on V_j(U_k(P)) on the same context settings, so the step is bit-identical
 * to 8 such calls and an fp32 sum in that order.  The nearest 2x resize commutes with every V_j, so an upscaling TTA step
 * transforms the half-resolution plane and never builds the 2x one.  w2x_convert_planes_chain* packs the 8n variants of its n
 * planes into frames; w2x_convert_chain* converts each variant alone with the caller's block_splitting.  A TTA step logs the lines
 * of the same step without the flag, and launches what the plain step launches on the 8n variant planes, plus 2 (building the
 * variants, and the mean). */
#define W2X_STEP_TTA 4
typedef void (*w2x_step_fn)(int step, void *user);
W2X_API int w2x_convert_chain(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds,
                              const float *in, int width, int height, size_t in_stride_bytes,
                              float *out, size_t out_stride_bytes, int block_splitting, w2x_step_fn on_step, void *user);
/* Same on DEVICE planes, asynchronous on the context's stream (w2x_ctx_set_stream). */
W2X_API int w2x_convert_chain_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds,
                                     const float *d_in, int width, int height, size_t in_stride_bytes,
                                     float *d_out, size_t out_stride_bytes, int block_splitting, w2x_step_fn on_step,
                                     void *user);

/* ---- a window of a chain's output ------------------------------------------------------------------- */
/* Part of a chain's output without converting the rest: the visible part of a large page, the area around an edit patched into a
 * previous output, or the tiles of a plane too large to hold.  An output pixel of a step depends only on the (2 n + 1)^2
 * neighbourhood of its input pixel (n = the model's layer count), replicated only at the plane's own border, so a window computed
 * from real neighbours is the same window of the whole conversion, seams included.  window = {x0, y0, w, h} of the
 * (width << u) x (height << u) output (u = the number of upscaling steps).  Working back from the last step, a step's input window
 * is its output window grown by its model's layer count on every side and clamped to the step's input plane, then for an
 * upscaling step halved (floor at the top-left, ceil at the bottom-right); the first step's input window is the source rectangle.
 * w2x_chain_region_source writes it to source[4] = {x0, y0, w, h} of the width x height input plane; it needs no device.
 * W2X_STEP_TTA steps have no window form. */
W2X_API int w2x_chain_region_source(int n_steps, const w2x_model *const *models, const int *kinds, int width, int height,
                                    const int *window, int *source);
/* That window of w2x_convert_chain(..., block_splitting = 0) on the whole width x height plane, bit-identical on the same context
 * settings (engine, precision).  src points at the source rectangle's top-left pixel, and nothing outside the rectangle is read; out
 * receives the window (w x h).  Each step converts only its output window, reading real neighbours where the previous window has
 * them and replicating at the plane's border; intermediate windows stay on the device in the context's chain buffers.  Before
 * step k is queued, on_step(k, user) is called (if not NULL); then the step logs the lines w2x_convert_plane_device(...,
 * block_splitting = 0) logs for a plane the size of its output window, and launches the kernels that call launches for it.
 * Every argument is checked before anything is printed, allocated or queued: W2X_ERR_ARG names the step or the problem (the
 * checks of w2x_convert_chain, a W2X_STEP_TTA step, a NULL or empty window or one outside the output, NULL planes, row strides
 * that are not multiples of 4 bytes or shorter than the rectangle's / window's row); W2X_ERR_UNSUPPORTED a model the context's
 * engine refuses.
 * HOST buffers, synchronous. */
W2X_API int w2x_convert_chain_region(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int width,
                                     int height, const int *window, const float *src, size_t src_stride_bytes, float *out,
                                     size_t out_stride_bytes, w2x_step_fn on_step, void *user);
/* Same on DEVICE buffers, asynchronous on the context's stream. */
W2X_API int w2x_convert_chain_region_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int width,
                                            int height, const int *window, const float *d_src, size_t src_stride_bytes, float *d_out,
                                            size_t out_stride_bytes, w2x_step_fn on_step, void *user);
/* Many windows in one call, packed side by side into shared frames: the tiles of a scan too large to hold, the visible tiles of a
 * viewer, patches of many images for a dataset.  Window i is windows[4 i .. 4 i + 3] = {x0, y0, w, h} of the chain's output on a
 * widths[i] x heights[i] input plane; the steps are shared by every window.  src[i] points at the top-left pixel of window i's
 * source rectangle (w2x_chain_region_source), row stride src_strides[i] bytes, and nothing outside that rectangle is read; out[i]
 * receives the w x h window, row stride out_strides[i] bytes.  Several windows may come from one plane, and their source rectangles
 * may overlap or share memory; the outputs must not overlap one another or any source (as in w2x_convert_planes_chain).
 * Bits: every window is bit-identical to w2x_convert_chain_region on that window alone, and so to the same window of
 * w2x_convert_chain(..., block_splitting = 0), on the same context settings (both engines, every precision).
 * Packing: each step packs the windows' step outputs into frames as w2x_convert_planes* does, planned by their output-window sizes;
 * a frame's rectangle holds the window's real neighbours as its padding, so that only the plane's own border is replicated.  A
 * window too large for a frame is converted alone, in scratch bands if needed.  The fp32 engine, or a model without the fused last
 * layer, converts window by window.  Step k launches what w2x_convert_planes_device launches for planes of the step's output-window
 * sizes.
 * Before step k is queued, on_step(k, user) is called (if not NULL); then the step logs, window by window in order, the lines
 * w2x_convert_chain_region logs for that window at step k (both entries log them so).
 * Every argument is checked before anything is printed, allocated or queued.  W2X_ERR_ARG names the step or the window: n_windows
 * < 1 or a NULL array; a W2X_STEP_TTA step, an unknown kind or a model that does not map 1 plane to 1 plane (naming the step);
 * per window, every check of w2x_convert_chain_region, its message prefixed by "window i: ".  A model the context's engine refuses
 * gives W2X_ERR_UNSUPPORTED naming the step.  Every buffer is reserved first, so W2X_ERR_NOMEM leaves nothing queued.
 * HOST buffers, synchronous: each source rectangle is staged densely on the device, uploads overlap step 0 and downloads the last
 * step. */
W2X_API int w2x_convert_chain_regions(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_windows,
                                      const int *widths, const int *heights, const int *windows, const float *const *src,
                                      const size_t *src_strides, float *const *out, const size_t *out_strides, w2x_step_fn on_step,
                                      void *user);
/* Same on DEVICE buffers (the pointer, size, window and stride arrays themselves are host arrays), asynchronous on the context's
 * stream. */
W2X_API int w2x_convert_chain_regions_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds,
                                             int n_windows, const int *widths, const int *heights, const int *windows,
                                             const float *const *d_src, const size_t *src_strides, float *const *d_out,
                                             const size_t *out_strides, w2x_step_fn on_step, void *user);

/* ---- a chain of conversions on a collection of planes of any sizes ------------------------------------ */
/* w2x_convert_chain for every plane of a w2x_convert_planes collection, in one call: the default noise_scale mode of a sprite set,
 * say.  Step k maps every plane P to convertWithModels(models[k], U_k(P)), U_k as in w2x_convert_chain, with block splitting off;
 * plane i comes out (widths[i] << u) x (heights[i] << u), u = the number of W2X_STEP_UPSCALE2X steps.  Every output is
 * bit-identical to w2x_convert_chain(..., block_splitting = 0) on that plane alone, and to the per-step loop of w2x_convert_planes
 * on the resized planes, on the same context settings.  Each step packs its planes into frames as w2x_convert_planes does, planned
 * on the step's output sizes (a plane may pack at one step and be converted alone after a 2x step); an upscaling step packs
 * straight from the half-resolution planes and never builds the 2x ones.  With n_steps == 1 and W2X_STEP_SAME this is
 * w2x_convert_planes: same bits, same progress lines, same launches.
 * Before step k is queued, on_step(k, user) is called (if not NULL); then the step logs the lines w2x_convert_planes (host entry) or
 * w2x_convert_planes_device (device entry) logs for its planes, in plane order.
 * Every argument is checked before anything is printed, allocated or queued; W2X_ERR_ARG names the step or the plane: n_steps or
 * n_planes < 1, a NULL array, model or plane, an unknown kind, a model that does not map 1 plane to 1 plane, an output size that
 * overflows int, row strides that are not multiples of 4 bytes or shorter than the plane's input (in_strides) or output
 * (out_strides) row.  A model the engine refuses gives W2X_ERR_UNSUPPORTED naming the step.  Planes must not overlap one another's
 * outputs (as in w2x_convert_planes).
 * Device memory: two buffers of the context, each holding one step's outputs for the whole collection (only with 2 steps and
 * more), plus the frame scratch of w2x_convert_planes; the host entry also stages every input and every output plane on the device.
 * HOST buffers, synchronous; uploads overlap the first step and downloads the last. */
W2X_API int w2x_convert_planes_chain(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds, int n_planes,
                                     const float *const *in, const int *widths, const int *heights, const size_t *in_strides,
                                     float *const *out, const size_t *out_strides, w2x_step_fn on_step, void *user);
/* Same on DEVICE planes (the pointer, size and stride arrays themselves are host arrays), asynchronous on the context's stream. */
W2X_API int w2x_convert_planes_chain_device(w2x_ctx *ctx, int n_steps, const w2x_model *const *models, const int *kinds,
                                            int n_planes, const float *const *d_in, const int *widths, const int *heights,
                                            const size_t *in_strides, float *const *d_out, const size_t *out_strides,
                                            w2x_step_fn on_step, void *user);

/* ---- one process, N GPUs ---------------------------------------------------------------------- */
/* The sibling of the reference's -j (src/main.cpp:58-60, modelUtility::setNumberOfJobs): N contexts driven by
 * one host thread.  w2x_multi_convert_plane = w2x_convert_plane with the plane cut into N row bands and the
 * per-layer halo exchange above between them (bit-identical to one GPU); planes too small to cut run on the
 * first GPU.  w2x_multi_convert_tiles = w2x_convert_tiles with tile t on GPU t mod N (no exchange).
 * devices == NULL means 0 .. n_devices-1. */
typedef struct w2x_multi w2x_multi;
W2X_API int w2x_multi_create(const int *devices, int n_devices, w2x_multi **out);
W2X_API void w2x_multi_destroy(w2x_multi *multi);
W2X_API int w2x_multi_device_count(const w2x_multi *multi);
W2X_API w2x_ctx *w2x_multi_ctx(w2x_multi *multi, int index);   /* the i-th GPU's context (settings, timing) */
W2X_API int w2x_multi_set_precision(w2x_multi *multi, int precision);
W2X_API int w2x_multi_set_log(w2x_multi *multi, w2x_log_fn fn, void *user);
W2X_API int w2x_multi_convert_plane(w2x_multi *multi, const w2x_model *model, const float *in, int width,
                                    int height, size_t in_stride_bytes, float *out, size_t out_stride_bytes,
                                    int block_splitting);
W2X_API int w2x_multi_convert_tiles(w2x_multi *multi, const w2x_model *model, const float *const *in_tiles,
                                    float *const *out_tiles, int n_tiles, int width, int height,
                                    size_t in_stride_bytes, size_t out_stride_bytes);
/* w2x_convert_chain on N GPUs: the noise pass and the 2x steps of one plane in one call, the plane's row bands staying on their GPUs
 * between the steps.  A nearest 2x resize maps the rows [a, b) a GPU owns onto [2a, 2b), so the cut of step 0 holds at every step
 * and no row changes GPU: step 0 uploads, every later step reads the previous step's rows where its GPU left them (an upscaling
 * step through the resize, into the band's padded input frame; the 2x plane is never built), only the last step downloads, and
 * the host sees no intermediate plane.  Between GPUs a step trades the halo row of its input frame and one row per layer.
 * Every step's plane, and so the output, is bit-identical to w2x_convert_chain on one context with the same precision and the
 * same arguments.
 * Arguments are checked as by w2x_convert_chain, before anything is printed, allocated or queued, W2X_ERR_ARG (or, for a model
 * the engine refuses, W2X_ERR_UNSUPPORTED) naming the step.  A step with W2X_STEP_TTA is refused with W2X_ERR_ARG naming the step:
 * it has no row-band form (the transposed variants would turn row bands into column bands).  w2x_multi_convert_planes_chain runs TTA
 * steps across GPUs, a plane's variants on different GPUs; call it with the one plane.
 * Before step k is queued on any GPU, on_step(k, user) is called (if not NULL); then the step logs, through the first context's log
 * function (w2x_multi_set_log), the lines w2x_convert_chain logs for it.
 * GPUs used: min(n_devices, height / (4 * the largest n_layers of the steps)), decided on the INPUT height (later steps only get
 * taller).  Fewer than 2, a model without a tensor-core form, or W2X_ENGINE_FP32 on the first context: the whole call is
 * w2x_convert_chain on the first context.  With n_steps == 1 and W2X_STEP_SAME the call is w2x_multi_convert_plane: same bits,
 * same lines, same launches.
 * Device memory: every step keeps sessions of its own (a neighbour may deliver a halo row of step k + 1 while this GPU still reads
 * step k), about 1 KiB per frame pixel a GPU owns per step (two activation frames of up to 128 channels at 4 bytes per element):
 * 1920 x 1080 noise + 2x on 2 GPUs is about 1 + 4.3 GB per GPU.  It is kept, like w2x_multi_convert_plane's plan and beside it,
 * for the next call with the same models, kinds, size and precision, and freed by any other chain call or w2x_multi_destroy.  All of
 * it is reserved before the first copy or launch: W2X_ERR_NOMEM leaves nothing queued and no plan behind.
 * HOST buffers, synchronous. */
W2X_API int w2x_multi_convert_chain(w2x_multi *multi, int n_steps, const w2x_model *const *models, const int *kinds,
                                    const float *in, int width, int height, size_t in_stride_bytes,
                                    float *out, size_t out_stride_bytes, int block_splitting,
                                    w2x_step_fn on_step, void *user);

/* w2x_convert_planes_chain on N GPUs: a collection of planes of any sizes, each plane on one GPU, and each W2X_STEP_TTA step's 8
 * variants of a plane spread over the GPUs.  A TTA step is 8 independent conversions and an ordered mean, so its variants split across
 * GPUs with no per-layer exchange: one large image's TTA step spreads as evenly as a collection's.  w2x_multi_convert_planes is the
 * one-step W2X_STEP_SAME case (w2x_convert_planes on N GPUs).
 * Every output is bit-identical to w2x_convert_planes_chain on the first context with the same kinds, precision and engine, W2X_STEP_TTA
 * steps included: every context the call uses takes the first context's precision and engine.
 * Arguments are checked exactly as w2x_convert_planes_chain checks them, with the same messages naming the step or the plane, before
 * anything is printed, allocated or queued on any context.
 * Before step k is queued on any GPU, on_step(k, user) is called (if not NULL); then, through the first context's log function
 * (w2x_multi_set_log), the lines w2x_convert_planes_chain logs for step k, in plane order.
 * Placement (a pure function of the sizes, kinds, models and N): the work of a plane at a step is its output pixels times the step
 * model's multiply-adds per pixel (9 Cin Cout summed over its layers), a TTA step counting 8 times.  Every plane has one owner GPU for
 * the whole call, which holds its input, its intermediate planes and its output and runs its plain steps.  In a TTA step, variant j of
 * plane i is converted on GPU (owner(i) + j) mod nd; the owner builds the variants and writes the mean.  When nd divides 8, every GPU
 * converts 8 / nd variants of every plane.  Owners are chosen greedily: planes in decreasing order of total work (ties: the lower
 * index), each taking the owner that minimises the largest per-GPU load once its work is added (ties: the owner with the smaller load
 * before the plane, then the lower GPU index).
 * GPUs used: nd = min(n_devices, 8 n_planes) when a step has W2X_STEP_TTA, else min(n_devices, n_planes).  With nd == 1 the call is
 * w2x_convert_planes_chain on the first context: same bits, same lines, same launches.
 * A TTA step needs peer access between every two distinct devices it uses (contexts of one device always qualify); without it the call
 * returns W2X_ERR_UNSUPPORTED naming the pair, before anything is queued.
 * Device memory: each GPU holds the staging of the planes it owns, the two chain buffers of its planes, the TTA buffers of the variants
 * it converts and its frame scratch.  All of it is reserved on every GPU before the first copy or launch anywhere: W2X_ERR_NOMEM leaves
 * nothing queued on any context.
 * Every dependency between GPUs is a CUDA event (a converting GPU waits for the owner's variants kernel, the owner's mean for every
 * converting GPU); no kernel waits on a flag, so contexts of one device cannot hold each other up.
 * HOST buffers, synchronous; pageable buffers are pinned for the call.  Every GPU's work is queued before any is waited for. */
W2X_API int w2x_multi_convert_planes(w2x_multi *multi, const w2x_model *model, int n_planes, const float *const *in,
                                     const int *widths, const int *heights, const size_t *in_strides,
                                     float *const *out, const size_t *out_strides);
W2X_API int w2x_multi_convert_planes_chain(w2x_multi *multi, int n_steps, const w2x_model *const *models, const int *kinds,
                                           int n_planes, const float *const *in, const int *widths, const int *heights,
                                           const size_t *in_strides, float *const *out, const size_t *out_strides,
                                           w2x_step_fn on_step, void *user);

/* w2x_convert_chain_regions on N GPUs: the tiles of a scan too large to hold, the visible tiles of a viewer or patches of many images,
 * each window on one GPU.  The arguments mean what they mean for w2x_convert_chain_regions.
 * Every window is bit-identical to w2x_convert_chain_regions on the first context with the same precision and engine, and so to the
 * same window of w2x_convert_chain(..., block_splitting = 0): every context the call uses takes the first context's precision and
 * engine.
 * Arguments are checked exactly as w2x_convert_chain_regions checks them, with the same messages naming the step or "window i: ",
 * before anything is printed, allocated or queued on any context.  A W2X_STEP_TTA step is refused: windows have no TTA form.
 * Before step k is queued on any GPU, on_step(k, user) is called (if not NULL); then, through the first context's log function
 * (w2x_multi_set_log), the lines w2x_convert_chain_regions logs for step k, window by window in order.
 * Placement (a pure function of the windows, the steps and N): the work of a window is, summed over the steps, its output-window
 * pixels at the step times the step model's multiply-adds per pixel.  Every window has one owner GPU, which stages its source
 * rectangle, holds its intermediate windows and writes its output; owners are chosen as in w2x_multi_convert_planes_chain: windows
 * in decreasing order of work (ties: the lower index), each on the owner that minimises the largest per-GPU load once its work is
 * added (ties: the owner with the smaller load before it, then the lower GPU index).  Each context launches what
 * w2x_convert_chain_regions launches on the windows it owns, in order, under its own scratch limit.
 * GPUs used: nd = min(n_devices, n_windows).  With nd == 1 the call is w2x_convert_chain_regions on the first context: same bits,
 * same lines, same launches.  No window leaves its GPU, so the call needs no peer access.
 * Device memory: each GPU holds what w2x_convert_chain_regions holds for its windows.  All of it is reserved on every GPU before the
 * first copy or launch anywhere: W2X_ERR_NOMEM leaves nothing queued on any context.
 * HOST buffers, synchronous; pageable buffers are pinned for the call: the page-rounded union of every source rectangle's and every
 * output's rows, registered as merged intervals of 4 MiB and more, so that windows sharing pages are pinned too.  Every GPU's work
 * is queued before any is waited for. */
W2X_API int w2x_multi_convert_chain_regions(w2x_multi *multi, int n_steps, const w2x_model *const *models, const int *kinds,
                                            int n_windows, const int *widths, const int *heights, const int *windows,
                                            const float *const *src, const size_t *src_strides, float *const *out,
                                            const size_t *out_strides, w2x_step_fn on_step, void *user);

/* ---- instrumentation ---------------------------------------------------------------------- */
/* Number of kernels of THIS library launched by the context so far. */
W2X_API int w2x_ctx_launch_count(const w2x_ctx *ctx, uint64_t *n_launches);
/* When enabled, every layer kernel launched by convert_* is bracketed by CUDA events on the
 * launching stream; w2x_ctx_layer_times returns, per layer, the summed milliseconds and launch
 * count since the last reset (synchronises the stream; W2X_ERR_CUDA when a timed span cannot be read). */
W2X_API int w2x_ctx_set_timing(w2x_ctx *ctx, int enabled);
W2X_API int w2x_ctx_layer_times(w2x_ctx *ctx, int max_layers, float *ms, int *launches,
                                int *n_layers_out, int reset);
/* Name of the kernel family the last convert call used for `layer` ("fp32_direct",
 * "wgmma_f16x3", "wgmma_f16+f8x2", "wgmma_f16", each with "+last" when the last layer is folded in, "first_1xN",
 * "first_1xN+up2x" (the first layer reading a half-resolution plane through the nearest 2x resize, w2x_convert_chain),
 * "last_Nx1", "last_gather"). */
W2X_API const char *w2x_ctx_layer_kernel_name(const w2x_ctx *ctx, int layer);

#ifdef __cplusplus
}
#endif
#endif /* W2X_B200_H_ */
