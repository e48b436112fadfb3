// Prints whether the last scanline pass takes the WTA as its epilogue (so_wta_fused, adcensus_b200/csrc/so_plan.h), and
// the record counts the choice rests on.
// Usage: so_wta_main W H D dmin opt_export confidence discontinuity debug_run force
//   ->   "fused band row_records plane_floats vol_floats"
#include <stdio.h>
#include <stdlib.h>

#include "../../adcensus_b200/csrc/so_plan.h"

int main(int argc, char** argv) {
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
