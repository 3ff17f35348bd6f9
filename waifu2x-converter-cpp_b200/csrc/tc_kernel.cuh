// tc_kernel.cuh -- tc_conv3x3_kernel, conv3x3_bf16x3_kernel: the layer kernel (warp roles, pipelines, epilogue)
// Part of the tensor-core engine's single translation unit: included by kernels_tc.cu inside namespace w2x::tc, in this order:
//   tc_ptx.cuh, tc_wgmma.cuh, tc_config.cuh, tc_kernel.cuh, tc_edge_kernels.cuh
// (pure code organisation: the generated SASS is the same as with one file).

// Bias, scale and leaky-ReLU of one accumulator value: = ACT_SCALE * leaky(conv + bias)
__device__ __forceinline__ float activate(float acc, float scale, float bias) {
    const float v = fmaf(acc, scale, bias);
    return fmaxf(v, 0.1f * v);                                           // leaky 0.1: min(v,0)*0.1 + max(v,0)
}

// The record of activated channels cc, cc + 1 (cc even, within the 32-channel block) of one pixel, written into the staging
// row at rowaddr (swizzle phase sw = row & 7) in the TMA SWIZZLE_128B pattern: fp16 at byte 2 cc, then xh8 at 64 + cc and
// xl8 at 96 + cc (Rec::F8) or lo fp16 at 64 + 2 cc (Rec::F16); Rec::BF16: hi = bf16(v) at 2 cc, lo = bf16(v - hi) at 64 + 2 cc.
template <Rec R>
__device__ __forceinline__ void store_record_pair(uint32_t rowaddr, uint32_t sw, uint32_t cc, float v0, float v1) {
    constexpr bool F8 = R == Rec::F8;
    if constexpr (R == Rec::BF16) {
        const uint32_t hh = f32x2_to_bf16x2_sat(v0, v1);
        const float2 hf = bf16x2_to_f32x2(hh);
        const uint32_t lo = f32x2_to_bf16x2_sat(v0 - hf.x, v1 - hf.y);                  // v - hi: exact in fp32
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(rowaddr + (((cc >> 3) ^ sw) << 4) + 2u * (cc & 7u)), "r"(hh) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(rowaddr + (((4u + (cc >> 3)) ^ sw) << 4) + 2u * (cc & 7u)), "r"(lo) : "memory");
        return;
    }
    const __half2 hh = f32x2_to_f16x2_sat(v0, v1);
    const float2 hf = __half22float2(hh);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(rowaddr + (((cc >> 3) ^ sw) << 4) + 2u * (cc & 7u)), "r"(*reinterpret_cast<const uint32_t *>(&hh)) : "memory");
    if constexpr (F8) {
        constexpr float kDown = 1.0f / (float)(1 << F8_C), kUp = (float)(1 << F8_A);
        const __half2 hd = __hmul2(hh, __float2half2_rn(kDown));
        const uint16_t h8 = __nv_cvt_halfraw2_to_fp8x2(static_cast<__half2_raw>(hd), __NV_SATFINITE, __NV_E4M3);
        const uint16_t l8 = __nv_cvt_float2_to_fp8x2(make_float2((v0 - hf.x) * kUp, (v1 - hf.y) * kUp), __NV_SATFINITE, __NV_E4M3);
        asm volatile("st.shared.b16 [%0], %1;" ::"r"(rowaddr + (((4u + (cc >> 4)) ^ sw) << 4) + (cc & 15u)), "h"(h8) : "memory");
        asm volatile("st.shared.b16 [%0], %1;" ::"r"(rowaddr + (((6u + (cc >> 4)) ^ sw) << 4) + (cc & 15u)), "h"(l8) : "memory");
    } else {
        const __half2 lo = f32x2_to_f16x2_sat(v0 - hf.x, v1 - hf.y);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(rowaddr + (((4u + (cc >> 3)) ^ sw) << 4) + 2u * (cc & 7u)), "r"(*reinterpret_cast<const uint32_t *>(&lo)) : "memory");
    }
}

// One consumer warpgroup's M-tile (8 wide x 16 tall pixels = two m64 halves) of a tile-set: accumulators -> scale, bias,
// leaky-ReLU -> records of each 32-channel block written into the warpgroup's staging tile in the TMA SWIZZLE_128B pattern
// (staging row = pixel = y * 8 + x, conflict-free: the eight rows a warp writes at once fall into eight different 16-byte
// units) and sent as ONE 8x16-pixel TMA store box; the frame edge is clipped by the TMA unit.
template <int COUT, Rec R>
__device__ __forceinline__ void epilogue_store(const TcParams &p, const float *bias, const CUtensorMap *tmap_out, const float (&acc)[2][COUT / 2],
                                               uint32_t stg, int wg, int wq, int lane, int gx0, int gy0) {
    const int q = lane & 3, r_lo = wq * 16 + (lane >> 2);
#pragma unroll
    for (int cb = 0; cb < COUT / 32; cb++) {
        if (wq == 0) {                    // the lanes of warp 0 wait for their own store of the previous block to have left
            bulk_wait_read();
            __syncwarp();
        }
        named_sync(1 + wg, 128);
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const uint32_t row = (uint32_t)(64 * h + r_lo + 8 * e), sw = row & 7u, rowaddr = stg + row * 128u;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int jj = cb * 4 + j, ch = 8 * jj + 2 * q;
                    const float v0 = activate(acc[h][4 * jj + 2 * e], p.out_scale, bias[ch]);
                    const float v1 = activate(acc[h][4 * jj + 2 * e + 1], p.out_scale, bias[ch + 1]);
                    store_record_pair<R>(rowaddr, sw, (uint32_t)(8 * j + 2 * q), v0, v1);
                }
            }
        }
        fence_proxy_async();
        named_sync(1 + wg, 128);
        if (wq == 0) {
            tma_store_4d(tmap_out, stg, 0, cb, gx0, gy0);
            bulk_commit();
        }
    }
}

// epilogue_store for channel-major accumulators (Cfg::SWAP, Cout = 64): the thread holds channels ch = 16 wq + r + 8e
// (r = lane / 4) of the pixels n = 8j + 2q + {0, 1} (y = j, x = 2q + {0, 1}) at acc[4j + 2e + {0, 1}].  Lanes r and r ^ 1
// swap one value each, so the even lane holds channels ch, ch + 1 of pixel x = 2q and the odd lane those of x = 2q + 1:
// the same channel pairs, expressions and stores as epilogue_store.  Warps 0, 1 hold block 0 and warps 2, 3 block 1, each
// written into its own staging tile; warp 0 sends both boxes.
template <Rec R>
__device__ __forceinline__ void epilogue_store_swapped(const TcParams &p, const float *bias, const CUtensorMap *tmap_out, const float (&acc)[64],
                                                       uint32_t stg, int wg, int wq, int lane, int gx0, int gy0) {
    const int q = lane & 3, r = lane >> 2, odd = r & 1;
    const uint32_t blk = stg + (uint32_t)(wq >> 1) * (128u * 128u), x = (uint32_t)(2 * q + odd);
    if (wq == 0) {                        // the lanes of warp 0 wait for their own stores of the previous tile-set to have left
        bulk_wait_read();
        __syncwarp();
    }
    named_sync(1 + wg, 128);
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int ch = 16 * wq + (r & ~1) + 8 * e;
        const float b0 = bias[ch], b1 = bias[ch + 1];
        const uint32_t cc = (uint32_t)(ch & 31);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const float a0 = acc[4 * j + 2 * e], a1 = acc[4 * j + 2 * e + 1];
            const float other = __shfl_xor_sync(0xffffffffu, odd ? a0 : a1, 4);
            const float v0 = activate(odd ? other : a0, p.out_scale, b0);
            const float v1 = activate(odd ? a1 : other, p.out_scale, b1);
            const uint32_t row = 8u * (uint32_t)j + x;
            store_record_pair<R>(blk + row * 128u, x, cc, v0, v1);
        }
    }
    fence_proxy_async();
    named_sync(1 + wg, 128);
    if (wq == 0) {
        tma_store_4d(tmap_out, stg, 0, 0, gx0, gy0);
        tma_store_4d(tmap_out, stg + 128u * 128u, 0, 1, gx0, gy0);
        bulk_commit();
    }
}

// The last layer folded in: per pixel the nine tap dot products over this layer's activated channels.  The four lanes of
// a quad hold the pixel's channels (8j + 2q, +1); their partial sums meet through two shuffles.  The thread's four pixels
// (h, e) are summed side by side, so each channel pair's nine weight pairs are loaded once (a weight set per pixel would
// not fit in registers next to the accumulators); per pixel the sums still run over the channels in ascending order.
template <int COUT>
__device__ __forceinline__ void epilogue_fuse(const TcParams &p, const float *bias, const float *last_w, const float (&acc)[2][COUT / 2], int wq, int lane,
                                              int fx0, int fy0) {
    const int q = lane & 3, r_lo = wq * 16 + (lane >> 2);
    float pt[2][2][9];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int e = 0; e < 2; e++)
#pragma unroll
            for (int t = 0; t < 9; t++) pt[h][e][t] = 0.f;
#pragma unroll
    for (int jj = 0; jj < COUT / 8; jj++) {
        const int ch = 8 * jj + 2 * q;
        const float2 b2 = *reinterpret_cast<const float2 *>(bias + ch);
        float2 w[9];
#pragma unroll
        for (int t = 0; t < 9; t++) w[t] = *reinterpret_cast<const float2 *>(last_w + t * COUT + ch);
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const float a0 = activate(acc[h][4 * jj + 2 * e], p.out_scale, b2.x);
                const float a1 = activate(acc[h][4 * jj + 2 * e + 1], p.out_scale, b2.y);
#pragma unroll
                for (int t = 0; t < 9; t++) pt[h][e][t] = fmaf(a1, w[t].y, fmaf(a0, w[t].x, pt[h][e][t]));
            }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
            float (&pe)[9] = pt[h][e];
#pragma unroll
            for (int t = 0; t < 9; t++) {
                pe[t] += __shfl_xor_sync(0xffffffffu, pe[t], 1);
                pe[t] += __shfl_xor_sync(0xffffffffu, pe[t], 2);
            }
            const int row = 64 * h + r_lo + 8 * e;
            const int fx = fx0 + (row & 7), fy = fy0 + (row >> 3);
            if (q == 0 && fy < p.Hp && fx < p.Wp && fy >= p.out_y0 && fy < p.out_y0 + p.out_rows) {
                float4 *dst = reinterpret_cast<float4 *>(p.partial + ((size_t)fy * p.Wp + fx) * 12);
                dst[0] = make_float4(pe[0], pe[1], pe[2], pe[3]);
                dst[1] = make_float4(pe[4], pe[5], pe[6], pe[7]);
                dst[2] = make_float4(pe[8], 0.f, 0.f, 0.f);
            }
        }
    }
}

// ================================================================================================
// The layer kernel
// ================================================================================================
// Persistent, one CTA per SM, tile-sets of 16x16 output pixels round-robin over the CTAs.  Each consumer warpgroup owns an
// 8-wide x 16-tall M-tile (two m64 wgmma halves: halo rows 0..7 and 8..15), N = Cout; the 3x3 taps are descriptor start
// offsets into the staged 18x18 box.  Every commit is followed by a wait for the group before it, so one group is always in
// flight while the warpgroup works on the previous one's results.  f16x3 (and xh_only, with the xh * wh K steps alone): one
// group per tap.  F8: one group per (half h,
// 64-column slice s) of a tap, [h's f16 product if s == 0 | the slice's two e4m3 corrections into a fresh buffer]; the
// buffers alternate between two register sets, and a group's buffer is added to acc[h] once the NEXT group has been issued
// (that group never writes acc[h]: it is a correction-only group or the other half's).  Per accumulator element the order
// stays f16 product of tap t, correction of tap t, f16 product of tap t + 1.  A weight stage is handed back once every group
// reading it has completed: after the first wait of the next tap (F8: tap 8's stage and the activation slot after the wait
// for all groups that ends each 32-channel chunk).
//
// Register budget: 384 threads at one CTA per SM get 168 registers each.  The producer warpgroup (warps 0-3) drops to
// PRODUCER_REGS, and the consumer warpgroups take the rest: the accumulators alone are COUT fp32 registers per thread.
constexpr uint32_t PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS == NUM_THREADS * 168, "register hand-off must balance");

// The 16-bit product of a hi/lo record format: bf16 wgmmas on Rec::BF16 records and weights, f16 ones otherwise.  The two
// formats share the record layout, the weight image layout and the descriptors; only the element type differs.
template <int N, Rec R>
__device__ __forceinline__ void mma16(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (R == Rec::BF16) Wgmma<N>::bf16(d, a, b, scale_d);
    else Wgmma<N>::f16(d, a, b, scale_d);
}

// The consumer warpgroup of a Cout = 64 layer (Cfg::SWAP): D[channel][pixel], A = the stage's 64 weight rows (the packed
// image as it is: fp16 rows of 64 B, SWIZZLE_64B; e4m3 rows of 32 B, SWIZZLE_32B), B = the M-tile's 128 pixels (N = 128;
// the record box with the same descriptor the m64 halves use, eight pixels per halo row).  Per (tap, chunk) one m64n128
// per K step reads 24 KB of shared memory where two m64n64 halves read 32 KB: a tile-set of these layers is bound by the
// shared-memory operand traffic, not by the tensor cores.  Each element sees the same products in the same order, and
// the tensor cores' sums do not depend on which operand is A.
//   f16x3 / xh_only: one group per tap, as in the kernel below.
//   F8: F_t = the f16 product of tap t into acc, X_t = its e4m3 corrections into the fresh buffer corr[t & 1].  Issue order
//   F_0 X_0 | X_1 [wait: F_0, X_0 done; acc += corr[0]] F_1 | X_2 [wait; acc += corr[1]] F_2 | ... F_8 [wait all]: the
//   next tap's corrections run while the adds do, and per element the order stays f16 product of tap t, correction of
//   tap t, f16 product of tap t + 1.  Taps unrolled, the chunk ends with an empty pipe (see below).
template <int CIN, Rec R>
__device__ __forceinline__ void consume_swapped(const TcParams &p, const CUtensorMap *tmap_out, uint32_t a_base, uint32_t b_base, uint32_t stg,
                                                uint32_t bar_base, const float *prm, int wg, int wq, int lane, unsigned long long *prof) {
    constexpr bool F8 = R == Rec::F8;
    using C = Cfg<CIN, 64, false, F8>;
    auto a_full = [&](uint32_t i) { return bar_base + 8u * i; };
    auto a_empty = [&](uint32_t i) { return bar_base + 8u * (2u + i); };
    auto b_full = [&](uint32_t i) { return bar_base + 8u * (4u + i); };
    auto b_empty = [&](uint32_t i) { return bar_base + 8u * (4u + C::NB + i); };
    constexpr uint32_t ROWB = C::ROWB;
    constexpr uint32_t X_HI = desc_hi(HALO * ROWB, SW128);      // B: next 8-pixel group = next halo row
    constexpr uint32_t W_HI = desc_hi(8 * 64, SW64);             // A: fp16 weight rows of 64 B
    constexpr uint32_t W8_HI = desc_hi(8 * 32, SW32);            // A: e4m3 weight rows of 32 B
    const bool prof_on = prof != nullptr;
    float acc[64];
    float corr[F8 ? 2 : 1][64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.f;
    uint32_t a_it = 0, stage = 0, phase = 0, n = 0;
    unsigned long long w_af = 0, w_bf = 0;
    // the next weight stage, once it has arrived
    auto next_stage = [&]() -> uint32_t {
        if (!C::RESIDENT) mbar_wait_prof(b_full(stage), phase, prof_on, w_bf);
        else if (n == 0) mbar_wait_prof(b_full(stage), 0u, prof_on, w_bf);   // the stages arrive once, during the first tile-set
        const uint32_t s = stage;
        if (++stage == (uint32_t)C::NB) { stage = 0; phase ^= 1u; }
        return s;
    };
    const long long t_begin = clock64();
    for (int ts = blockIdx.x; ts < p.n_tilesets; ts += gridDim.x, n++) {
        const int ty = ts / p.tiles_x, tx = ts - ty * p.tiles_x;
        if constexpr (F8) {
            for (int c = 0; c < C::NCHUNK; c++, a_it++) {
                const uint32_t slot = a_it & 1u;
                mbar_wait_prof(a_full(slot), (a_it >> 1) & 1u, prof_on, w_af);
                const uint32_t x0 = a_base + slot * C::A_SLOT + (uint32_t)wg * 8u * ROWB;
                auto px = [&](int t) { return x0 + (uint32_t)((t / 3) * HALO + t % 3) * ROWB; };
                auto issue_f16 = [&](int t, uint32_t s, uint32_t scale_d) {
                    const uint32_t w = b_base + s * C::B_STAGE, x = px(t);
                    acc_fence(acc);
                    wgmma_fence();
                    Wgmma<128>::f16(acc, make_desc(W_HI, w), make_desc(X_HI, x), scale_d);               // wh * xh
                    Wgmma<128>::f16(acc, make_desc(W_HI, w + 32u), make_desc(X_HI, x + 32u), 1u);
                    wgmma_commit();
                };
                auto issue_corr = [&](int t, uint32_t s) {
                    const uint32_t w = b_base + s * C::B_STAGE, x = px(t);
                    acc_fence(corr[t & 1]);
                    wgmma_fence();
                    Wgmma<128>::e4m3(corr[t & 1], make_desc(W8_HI, w + 64u * 64u), make_desc(X_HI, x + 96u), 0u);   // wh8 * xl8
                    Wgmma<128>::e4m3(corr[t & 1], make_desc(W8_HI, w + 64u * 96u), make_desc(X_HI, x + 64u), 1u);   // wl8 * xh8
                    wgmma_commit();
                };
                uint32_t st_cur = next_stage();
                issue_f16(0, st_cur, c != 0 ? 1u : 0u);
                issue_corr(0, st_cur);
#pragma unroll 9
                for (int t = 0; t < 9; t++) {
                    uint32_t st_next = 0;
                    if (t < 8) {
                        st_next = next_stage();
                        issue_corr(t + 1, st_next);
                        wgmma_wait<1>();                     // all but X_{t+1}: F_t and X_t have completed
                    } else {
                        wgmma_wait<0>();
                    }
                    acc_fence(acc);
                    acc_fence(corr[t & 1]);
#pragma unroll
                    for (int i = 0; i < 64; i++) acc[i] += corr[t & 1][i];
                    acc_fence(acc);
                    if (lane == 0) {                         // tap t's stage (and after tap 8 the slot) is read by no group any more
                        if (!C::RESIDENT) mbar_arrive(b_empty(st_cur));
                        if (t == 8) mbar_arrive(a_empty(slot));
                    }
                    if (t < 8) {
                        issue_f16(t + 1, st_next, 1u);
                        st_cur = st_next;
                    }
                }
            }
        } else {
            // f16x3, or with p.xh_only the xh * wh K steps alone, chosen once per tile-set (no group in flight)
            auto chunks = [&](auto xh_only_tag) {
                constexpr bool XH_ONLY = decltype(xh_only_tag)::value;
                int pend_b = -1, pend_a = -1;                // stage / slot read by the previous tap's group
                for (int c = 0; c < C::NCHUNK; c++, a_it++) {
                    const uint32_t slot = a_it & 1u;
                    mbar_wait_prof(a_full(slot), (a_it >> 1) & 1u, prof_on, w_af);
                    const uint32_t x0 = a_base + slot * C::A_SLOT + (uint32_t)wg * 8u * ROWB;
#pragma unroll 1
                    for (int t = 0; t < 9; t++) {
                        const uint32_t x = x0 + (uint32_t)((t / 3) * HALO + t % 3) * ROWB;
                        const uint32_t s = next_stage(), w = b_base + s * C::B_STAGE, wl = w + 64u * 64u;
                        const uint32_t first = (c | t) != 0 ? 1u : 0u;
                        acc_fence(acc);
                        wgmma_fence();
                        mma16<128, R>(acc, make_desc(W_HI, w), make_desc(X_HI, x), first);              // wh * xh
                        mma16<128, R>(acc, make_desc(W_HI, w + 32u), make_desc(X_HI, x + 32u), 1u);
                        if constexpr (!XH_ONLY) {
                            mma16<128, R>(acc, make_desc(W_HI, w), make_desc(X_HI, x + 64u), 1u);       // wh * xl
                            mma16<128, R>(acc, make_desc(W_HI, w + 32u), make_desc(X_HI, x + 96u), 1u);
                            mma16<128, R>(acc, make_desc(W_HI, wl), make_desc(X_HI, x), 1u);             // wl * xh
                            mma16<128, R>(acc, make_desc(W_HI, wl + 32u), make_desc(X_HI, x + 32u), 1u);
                        }
                        wgmma_commit();
                        wgmma_wait<1>();                             // the previous group is done: its stage / slot may be refilled
                        acc_fence(acc);
                        if (lane == 0) {
                            if (!C::RESIDENT && pend_b >= 0) mbar_arrive(b_empty((uint32_t)pend_b));
                            if (pend_a >= 0) mbar_arrive(a_empty((uint32_t)pend_a));
                        }
                        pend_b = (int)s;
                        pend_a = t == 8 ? (int)slot : -1;
                    }
                }
                wgmma_wait<0>();
                acc_fence(acc);
                if (lane == 0) {
                    if (!C::RESIDENT && pend_b >= 0) mbar_arrive(b_empty((uint32_t)pend_b));
                    if (pend_a >= 0) mbar_arrive(a_empty((uint32_t)pend_a));
                }
            };
            if (R == Rec::F16 && p.xh_only) chunks(std::true_type{});
            else chunks(std::false_type{});
        }
        epilogue_store_swapped<R>(p, prm, tmap_out, acc, stg, wg, wq, lane, tx * REGION + 8 * wg, ty * REGION);
    }
    if (wq == 0) bulk_wait_all();    // this warpgroup's TMA stores are complete before the CTA may exit
    if (prof_on && wg == 0 && wq == 0 && lane == 0) {
        prof[PROF_TOTAL] += (unsigned long long)(clock64() - t_begin);
        prof[PROF_MMA_WAIT_A] += w_af;
        prof[PROF_MMA_WAIT_B] += w_bf;
        prof[PROF_TILESETS] += n;
    }
}

// The kernel body, for every record format; tc_conv3x3_kernel and conv3x3_bf16x3_kernel below are its entry points.
template <int CIN, int COUT, bool FUSE, Rec R>
__device__ __forceinline__ void conv3x3_body(const CUtensorMap &tmap_in, const CUtensorMap &tmap_out, const TcParams &p) {
    constexpr bool F8 = R == Rec::F8;
    using C = Cfg<CIN, COUT, FUSE, F8>;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment: the SWIZZLE_128B pattern repeats every 1024 B
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t a_base = smem_base;
    const uint32_t b_base = a_base + C::A_SLOTS * C::A_SLOT;
    const uint32_t stg_base = b_base + C::NB * C::B_STAGE;
    const uint32_t bar_base = stg_base + C::STG_BYTES;
    float *prm = reinterpret_cast<float *>(smem_raw + (bar_base + C::BAR_BYTES - smem_u32(smem_raw)));   // [bias (COUT)][last_w (9 x COUT)]
    // barrier map (8 bytes each)
    auto a_full = [&](uint32_t i) { return bar_base + 8u * i; };
    auto a_empty = [&](uint32_t i) { return bar_base + 8u * (2u + i); };
    auto b_full = [&](uint32_t i) { return bar_base + 8u * (4u + i); };
    auto b_empty = [&](uint32_t i) { return bar_base + 8u * (4u + C::NB + i); };
    constexpr uint32_t CONSUMER_WARPS = 8;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const bool prof_on = p.prof != nullptr;
    unsigned long long *prof = prof_on ? p.prof + (size_t)blockIdx.x * PROF_N : nullptr;

    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < 2; i++) {
            mbar_init(a_full(i), 1);
            mbar_init(a_empty(i), CONSUMER_WARPS);   // lane 0 of every consumer warp, after its wgmma wait
        }
        for (uint32_t i = 0; i < (uint32_t)C::NB; i++) {
            mbar_init(b_full(i), 1);
            mbar_init(b_empty(i), CONSUMER_WARPS);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&tmap_in);
        if constexpr (!FUSE) prefetch_tmap(&tmap_out);
    }
    for (int i = threadIdx.x; i < COUT; i += NUM_THREADS) prm[i] = p.bias[i];
    if constexpr (FUSE)
        for (int i = threadIdx.x; i < 9 * COUT; i += NUM_THREADS) prm[COUT + i] = p.last_w[i];
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<PRODUCER_REGS>();   // all four warps, idle warps 2 and 3 included: the instruction is warpgroup-wide
        if (warp == 0) {
            // ===================== A producer: one halo'd box of records per (tile-set, 32-channel block) ==============
            // (whole warp walks the loop; the arrive and the TMA instructions elect one lane)
            uint32_t it = 0;
            unsigned long long w_a = 0;
            for (int ts = blockIdx.x; ts < p.n_tilesets; ts += gridDim.x) {
                const int ty = ts / p.tiles_x, tx = ts - ty * p.tiles_x;
                const int x0 = tx * REGION - 1, y0 = p.out_y0 + ty * REGION - 1;   // box origin incl. ring (may be -1); tile-sets tile the store window
                for (int c = 0; c < C::NCHUNK; c++, it++) {
                    const uint32_t slot = it & 1u, round = it >> 1;
                    mbar_wait_prof(a_empty(slot), (round & 1u) ^ 1u, prof_on, w_a);
                    mbar_arrive_expect_tx(a_full(slot), (uint32_t)C::A_TX);
                    tma_load_4d(a_base + slot * C::A_SLOT, &tmap_in, a_full(slot), 0, c, x0, y0);
                }
            }
            if (prof_on && lane == 0) prof[PROF_APROD_WAIT] += w_a;
        } else if (warp == 1) {
            // ===================== B producer: stream the packed weights in consumption order ============
            uint32_t stage = 0, phase = 0;
            unsigned long long w_b = 0;
            const uint8_t *src = reinterpret_cast<const uint8_t *>(p.wpack);
            const uint32_t b_bytes = R == Rec::F16 && p.xh_only ? (uint32_t)C::B_BLOCK : (uint32_t)C::B_STAGE;   // xh_only: the wh half of each stage
            for (int ts = blockIdx.x; ts < p.n_tilesets; ts += gridDim.x) {
                if (C::RESIDENT && ts != (int)blockIdx.x) break;           // resident weights: one pass fills every stage for good
                for (int blk = 0; blk < C::STAGES_PER_TILESET; blk++) {
                    if constexpr (!C::RESIDENT) mbar_wait_prof(b_empty(stage), phase ^ 1u, prof_on, w_b);
                    mbar_arrive_expect_tx(b_full(stage), b_bytes);
                    bulk_load(b_base + stage * C::B_STAGE, src + (size_t)blk * C::B_STAGE, b_bytes, b_full(stage));
                    if (++stage == (uint32_t)C::NB) { stage = 0; phase ^= 1u; }
                }
            }
            if (prof_on && lane == 0) prof[PROF_BPROD_WAIT] += w_b;
        }
    } else if constexpr (C::SWAP) {
        setmaxnreg_inc<CONSUMER_REGS>();
        consume_swapped<CIN, R>(p, &tmap_out, a_base, b_base, stg_base + (uint32_t)((warp - 4) >> 2) * C::STG_WG, bar_base, prm, (warp - 4) >> 2,
                                 warp & 3, lane, prof);
    } else {
        setmaxnreg_inc<CONSUMER_REGS>();
        // ===================== consumers: warpgroup wg = M-tile wg (pixels x in [8 wg, 8 wg + 8) of the tile-set) ===========
        const int wg = (warp - 4) >> 2, wq = warp & 3;
        constexpr uint32_t ROWB = C::ROWB;
        constexpr uint32_t A_HI = desc_hi(HALO * ROWB, SW128);      // next 8-pixel group = next halo row
        constexpr uint32_t B_HI = desc_hi(8 * 64, SW64);             // fp16 weight rows of 64 B
        constexpr uint32_t HALF = 8 * HALO * ROWB;                   // second m64 half: eight halo rows down
        // F8: e4m3 corrections of NS columns per wgmma, S slices per half, 2 S groups per tap; group g = h S + s uses buffer g & 1
        constexpr int NS = COUT < 64 ? COUT : 64, S = COUT / NS, LAST = 2 * S - 1;
        constexpr uint32_t B8_HI = desc_hi(8 * 32, SW32);            // e4m3 weight rows of 32 B
        float acc[2][COUT / 2];
        float corr[F8 ? 2 : 1][NS / 2];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int i = 0; i < COUT / 2; i++) acc[h][i] = 0.f;
        // Adds the correction of the tap's group gq (completed) to the columns of its slice.
        auto add_corr = [&](int gq) {
            const int h = gq / S, s = gq % S;
            acc_fence(corr[gq & 1]);
            acc_fence(acc[h]);
#pragma unroll
            for (int i = 0; i < NS / 2; i++) acc[h][s * (NS / 2) + i] += corr[gq & 1][i];
            acc_fence(acc[h]);
        };
        uint32_t a_it = 0, stage = 0, phase = 0, n = 0;
        unsigned long long w_af = 0, w_bf = 0;
        const long long t_begin = clock64();
        for (int ts = blockIdx.x; ts < p.n_tilesets; ts += gridDim.x, n++) {
            const int ty = ts / p.tiles_x, tx = ts - ty * p.tiles_x;
            int pend_b = -1, pend_a = -1;                            // stage / slot read by the groups of the previous tap
            auto release = [&] {                                     // ... which have all completed
                if (lane == 0) {
                    if (!C::RESIDENT && pend_b >= 0) mbar_arrive(b_empty((uint32_t)pend_b));
                    if (pend_a >= 0) mbar_arrive(a_empty((uint32_t)pend_a));
                }
            };
            if constexpr (F8) {
                for (int c = 0; c < C::NCHUNK; c++, a_it++) {
                    const uint32_t slot = a_it & 1u;
                    mbar_wait_prof(a_full(slot), (a_it >> 1) & 1u, prof_on, w_af);
                    const uint32_t a0 = a_base + slot * C::A_SLOT + (uint32_t)wg * 8u * ROWB;
                    // The taps are unrolled and the chunk ends with an empty pipe.  A group still in flight across a loop's back
                    // edge while its registers are read after the next wait makes ptxas serialise every wgmma of the loop.
#pragma unroll 9
                    for (int t = 0; t < 9; t++) {
                        const uint32_t tap = (uint32_t)((t / 3) * HALO + t % 3) * ROWB;
                        if (!C::RESIDENT) mbar_wait_prof(b_full(stage), phase, prof_on, w_bf);
                        else if (n == 0) mbar_wait_prof(b_full(stage), 0u, prof_on, w_bf);   // the stages arrive once, during the first tile-set
                        const uint32_t b = b_base + stage * C::B_STAGE;
                        const uint32_t first = (c | t) != 0 ? 1u : 0u;
                        // a record's quarters: +0 / +32 the fp16 K steps, +64 xh8, +96 xl8.  Hopper's e4m3 wgmma accumulates in
                        // reduced precision, which would also round the fp32 sums it adds to: each slice's two corrections go into a
                        // fresh buffer (scale_d = 0) and reach the fp32 sums through ordinary adds.
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const uint32_t ah = a0 + (uint32_t)h * HALF + tap;
#pragma unroll
                            for (int s = 0; s < S; s++) {
                                const int g = h * S + s;
                                if (s == 0) acc_fence(acc[h]);
                                acc_fence(corr[g & 1]);
                                wgmma_fence();
                                if (s == 0) {
                                    Wgmma<COUT>::f16(acc[h], make_desc(A_HI, ah), make_desc(B_HI, b), first);           // xh * wh
                                    Wgmma<COUT>::f16(acc[h], make_desc(A_HI, ah + 32u), make_desc(B_HI, b + 32u), 1u);
                                }
                                Wgmma<NS>::e4m3(corr[g & 1], make_desc(A_HI, ah + 96u), make_desc(B8_HI, b + COUT * 64u + s * NS * 32u), 0u);   // xl8 * wh8
                                Wgmma<NS>::e4m3(corr[g & 1], make_desc(A_HI, ah + 64u), make_desc(B8_HI, b + COUT * 96u + s * NS * 32u), 1u);   // xh8 * wl8
                                wgmma_commit();
                                wgmma_wait<1>();                             // every group but this one has completed
                                if (g > 0) {
                                    add_corr(g - 1);
                                } else if (t > 0) {                          // the previous tap's last group
                                    add_corr(LAST);
                                    release();
                                }
                            }
                        }
                        pend_b = (int)stage;
                        pend_a = t == 8 ? (int)slot : -1;
                        if (++stage == (uint32_t)C::NB) { stage = 0; phase ^= 1u; }
                    }
                    wgmma_wait<0>();
                    acc_fence(acc[0]);
                    acc_fence(acc[1]);
                    add_corr(LAST);
                    release();
                }
            } else {
                // f16x3, or with p.xh_only the xh * wh K steps alone: the loop is chosen once per tile-set, where no wgmma group
                // is in flight, so each of the two is straight-line wgmma code.
                auto chunks = [&](auto xh_only_tag) {
                    constexpr bool XH_ONLY = decltype(xh_only_tag)::value;
                    for (int c = 0; c < C::NCHUNK; c++, a_it++) {
                        const uint32_t slot = a_it & 1u;
                        mbar_wait_prof(a_full(slot), (a_it >> 1) & 1u, prof_on, w_af);
                        const uint32_t a0 = a_base + slot * C::A_SLOT + (uint32_t)wg * 8u * ROWB;
#pragma unroll 1
                        for (int t = 0; t < 9; t++) {
                            const uint32_t tap = (uint32_t)((t / 3) * HALO + t % 3) * ROWB;
                            if (!C::RESIDENT) mbar_wait_prof(b_full(stage), phase, prof_on, w_bf);
                            else if (n == 0) mbar_wait_prof(b_full(stage), 0u, prof_on, w_bf);   // the stages arrive once, during the first tile-set
                            const uint32_t b = b_base + stage * C::B_STAGE;
                            const uint32_t first = (c | t) != 0 ? 1u : 0u;
                            // a record's quarters: +0 / +32 the fp16 K steps of hi, +64 / +96 those of lo
                            acc_fence(acc[0]);
                            acc_fence(acc[1]);
                            wgmma_fence();
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const uint32_t ah = a0 + (uint32_t)h * HALF + tap;
                                mma16<COUT, R>(acc[h], make_desc(A_HI, ah), make_desc(B_HI, b), first);                   // xh * wh
                                mma16<COUT, R>(acc[h], make_desc(A_HI, ah + 32u), make_desc(B_HI, b + 32u), 1u);
                                if constexpr (!XH_ONLY) {
                                    mma16<COUT, R>(acc[h], make_desc(A_HI, ah + 64u), make_desc(B_HI, b), 1u);            // xl * wh
                                    mma16<COUT, R>(acc[h], make_desc(A_HI, ah + 96u), make_desc(B_HI, b + 32u), 1u);
                                    mma16<COUT, R>(acc[h], make_desc(A_HI, ah), make_desc(B_HI, b + COUT * 64u), 1u);     // xh * wl
                                    mma16<COUT, R>(acc[h], make_desc(A_HI, ah + 32u), make_desc(B_HI, b + COUT * 64u + 32u), 1u);
                                }
                            }
                            wgmma_commit();
                            wgmma_wait<1>();                             // the previous group is done: its stage / slot may be refilled
                            acc_fence(acc[0]);
                            acc_fence(acc[1]);
                            release();
                            pend_b = (int)stage;
                            pend_a = t == 8 ? (int)slot : -1;
                            if (++stage == (uint32_t)C::NB) { stage = 0; phase ^= 1u; }
                        }
                    }
                };
                if (R == Rec::F16 && p.xh_only) chunks(std::true_type{});
                else chunks(std::false_type{});
                wgmma_wait<0>();
                acc_fence(acc[0]);
                acc_fence(acc[1]);
                release();
            }
            if constexpr (FUSE)
                epilogue_fuse<COUT>(p, prm, prm + COUT, acc, wq, lane, tx * REGION + 8 * wg, p.out_y0 + ty * REGION);
            else
                epilogue_store<COUT, R>(p, prm, &tmap_out, acc, stg_base + (uint32_t)wg * C::STG_WG, wg, wq, lane, tx * REGION + 8 * wg, ty * REGION);
        }
        if constexpr (!FUSE) {
            if (wq == 0) bulk_wait_all();    // this warpgroup's TMA stores are complete before the CTA may exit
        }
        if (prof_on && wg == 0 && wq == 0 && lane == 0) {
            prof[PROF_TOTAL] += (unsigned long long)(clock64() - t_begin);
            prof[PROF_MMA_WAIT_A] += w_af;
            prof[PROF_MMA_WAIT_B] += w_bf;
            prof[PROF_TILESETS] += n;
        }
    }
}

// The fp16 record formats: F8 = false Rec::F16 (f16x3, and f16 through TcParams::xh_only), F8 = true Rec::F8.
template <int CIN, int COUT, bool FUSE, bool F8>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_conv3x3_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ TcParams p) {
    conv3x3_body<CIN, COUT, FUSE, F8 ? Rec::F8 : Rec::F16>(tmap_in, tmap_out, p);
}

// bf16x3 (Rec::BF16): the f16x3 kernel with bf16 records, weights and wgmmas (TcParams::xh_only is ignored).
template <int CIN, int COUT, bool FUSE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3x3_bf16x3_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ TcParams p) {
    conv3x3_body<CIN, COUT, FUSE, Rec::BF16>(tmap_in, tmap_out, p);
}
