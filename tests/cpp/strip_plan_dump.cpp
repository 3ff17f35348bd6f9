// strip_plan_dump.cpp -- walks the row-strip kernel's units exactly as the design's MMA issuer walks them
// using the shared schedule arithmetic of csrc/tc_strip_plan.h, and prints one line per strip:
//   cta u col y0 j ky_lo b0 cnt0 cnt1 acq_n acq_cnt com_n com_cnt
// tests/test_strip_kernel_model.py compares the lines with its own literal replay of the schedule.
#include <cstdio>
#include <cstdlib>

#include "tc_strip_plan.h"

int main(int argc, char **argv) {
    if (argc != 6) return 2;
    const int Hp = std::atoi(argv[1]), seg_rows = std::atoi(argv[2]), NB = std::atoi(argv[3]), n_ctas = std::atoi(argv[4]),
              ncols = std::atoi(argv[5]);
    const int n_units = ncols * ((Hp + seg_rows - 1) / seg_rows);
    for (int cta = 0; cta < n_ctas; cta++) {
        uint32_t nbase = 0;
        for (int u = cta; u < n_units; u += n_ctas) {
            const int seg = u / ncols, col = u - seg * ncols, y0 = seg * seg_rows, y1 = y0 + seg_rows < Hp ? y0 + seg_rows : Hp;
            const int rows = y1 - y0, j_first = strip_j_first(y0), j_last = strip_j_last(y1, rows, Hp);
            for (int j = j_first; j <= j_last; j++) {
                const StripPlan P = strip_plan(j, j == j_first, j == j_last, rows, nbase, (uint32_t)NB);
                std::printf("%d %d %d %d %d %u %u %u %u %u %u %u %u\n", cta, u, col, y0, j, P.ky_lo, P.b0, P.cnt0, P.cnt1, P.acq_n, P.acq_cnt,
                            P.com_n, P.com_cnt);
            }
            nbase += (uint32_t)rows;
        }
    }
    return 0;
}
