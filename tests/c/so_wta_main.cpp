// Prints whether the last scanline pass takes the WTA as its epilogue (so_wta_fused, adcensus_b200/csrc/so_plan.h), and
// the record counts the choice rests on.
// Usage: so_wta_main W H D dmin opt_export confidence discontinuity debug_run force
//   ->   "fused band row_records plane_floats vol_floats"
//        so_wta_main domain
//   ->   one line "D K LPS FULL n_fit w_first" per disparity range D = 1 .. 256: the k_scanline_wta instantiation D
//        selects, and how many widths W = 1 .. 10000 - D (adc_create's limits) the forced rule fuses, the first of them
//        (0 when none).  Whether the records fit does not depend on H or dmin.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../adcensus_b200/csrc/so_plan.h"

int main(int argc, char** argv) {
    if (argc == 2 && !strcmp(argv[1], "domain")) {
        for (int D = 1; D <= 256; D++) {
            const int Dp = (D + 3) / 4 * 4, lps = so_lanes_per_line(Dp), K = (Dp + lps - 1) / lps;
            int n = 0, first = 0;
            for (int W = 1; W <= 10000 - D; W++)
                if (so_wta_fused(SoVolumeUse{}, SO_WTA_ALWAYS, W, 1, D, Dp, 0, (long long)W * Dp)) {
                    if (!n) first = W;
                    n++;
                }
            printf("%d %d %d %d %d %d\n", D, K, lps, D == K * lps ? 1 : 0, n, first);
        }
        return 0;
    }
    if (argc != 10) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), D = atoi(argv[3]), dmin = atoi(argv[4]);
    const int Dp = (D + 3) / 4 * 4;
    SoVolumeUse use{};
    use.opt_export = atoi(argv[5]) != 0;
    use.confidence = atoi(argv[6]) != 0;
    use.discontinuity = atoi(argv[7]) != 0;
    use.debug_run = atoi(argv[8]) != 0;
    const long long vol = (long long)W * H * Dp;
    printf("%d %d %lld %lld %lld\n", so_wta_fused(use, atoi(argv[9]), W, H, D, Dp, dmin, vol) ? 1 : 0, so_wta_band(Dp),
           so_wta_row_records(W, D, Dp, dmin), so_wta_plane(W, H, D, Dp), vol);
    return 0;
}
