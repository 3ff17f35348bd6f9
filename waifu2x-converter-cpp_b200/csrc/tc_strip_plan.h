// tc_strip_plan.h -- the row-strip design's schedule (narrow layers, ky taps stacked along N, a ring of accumulator blocks)
// as plain integer arithmetic, checked by a CPU test that replays it against the reference model
// (tests/test_strip_kernel_model.py, tests/cpp/strip_plan_dump.cpp).  No kernel of this build includes it.  No CUDA types: compiles with g++ as is.
//
// A unit is `rows` output rows [y0, y0 + rows) of one 128-pixel column.  Its strips are the input rows r = y0 - 1 + j,
// j = j_first .. j_last (j_first = 1 at the frame's top edge, j_last = rows at its bottom edge, else 0 .. rows + 1).
// Input row r feeds output row r + 1 - ky with tap row ky; output rows own TMEM blocks in DESCENDING order,
// block(n) = NB-1 - (n mod NB) for the CTA's n-th output row, so the taps of one strip are adjacent ascending blocks:
// run 0 = cnt0 blocks from b0, and where the ring wraps run 1 = cnt1 blocks from block 0.
#ifndef W2X_TC_STRIP_PLAN_H_
#define W2X_TC_STRIP_PLAN_H_

#include <stdint.h>

#if defined(__CUDACC__)
#define W2X_PLAN_FN __host__ __device__ __forceinline__
#else
#define W2X_PLAN_FN inline
#endif

struct StripPlan {
    uint32_t ky_lo;            // first tap row of the strip (B rows start at ky_lo * Cout)
    uint32_t b0, cnt0, cnt1;   // run 0: cnt0 taps into blocks b0.., run 1: cnt1 taps into blocks 0..
    uint32_t acq_n, acq_cnt;   // output rows (CTA-global index) that receive their FIRST tap: their blocks must have been drained
    uint32_t com_n, com_cnt;   // output rows complete after this strip
};

// j_first_strip / j_last_strip: whether j is the unit's first / last strip; nbase: CTA-global index of the unit's row 0;
// NB a power of two.
W2X_PLAN_FN StripPlan strip_plan(int j, bool j_first_strip, bool j_last_strip, int rows, uint32_t nbase, uint32_t NB) {
    StripPlan P;
    const int ky_hi = j < 2 ? j : 2;
    const int ky_lo = j + 1 - rows > 0 ? j + 1 - rows : 0;
    const int i_top = j - ky_lo;                                           // = min(j, rows - 1): highest output row reached
    const int next_new = j_first_strip ? 0 : (j < rows ? j : rows);        // rows acquired by the strips before
    const int i_done = j_last_strip ? rows - 1 : j - 2;                    // rows whose ky = 2 tap is in
    const int next_done = j_first_strip ? 0 : (j - 2 > 0 ? j - 2 : 0);
    const uint32_t nky = (uint32_t)(ky_hi - ky_lo + 1);
    P.ky_lo = (uint32_t)ky_lo;
    P.b0 = NB - 1u - ((nbase + (uint32_t)i_top) & (NB - 1u));
    P.cnt0 = nky < NB - P.b0 ? nky : NB - P.b0;
    P.cnt1 = nky - P.cnt0;
    P.acq_n = nbase + (uint32_t)next_new;
    P.acq_cnt = (uint32_t)(i_top + 1 - next_new);
    P.com_n = nbase + (uint32_t)next_done;
    P.com_cnt = i_done + 1 > next_done ? (uint32_t)(i_done + 1 - next_done) : 0u;
    return P;
}

// strips of a unit: first / last j
W2X_PLAN_FN int strip_j_first(int y0) { return y0 == 0 ? 1 : 0; }
W2X_PLAN_FN int strip_j_last(int y1, int rows, int Hp) { return y1 == Hp ? rows : rows + 1; }

#endif
