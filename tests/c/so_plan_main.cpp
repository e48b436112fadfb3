// Prints the scanline launch plan (adcensus_b200/csrc/so_plan.h) of one pass on an H100 SXM (132 SMs, 228 KB of shared
// memory per SM, 1 KB reserved per CTA).  Usage: so_plan_main W H Dp S axis   ->   "T NS smem ctas ctas_per_sm waves"
#include <stdio.h>
#include <stdlib.h>

#include "../../adcensus_b200/csrc/so_plan.h"

int main(int argc, char** argv) {
    if (argc != 6) return 2;
    const SoPlan p = so_plan(atoi(argv[1]), atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), 132, 228 * 1024, 1024);
    printf("%d %d %zu %d %d %d\n", p.T, p.NS, p.smem, p.ctas, p.ctas_per_sm, p.waves);
    return p.T ? 0 : 1;
}
