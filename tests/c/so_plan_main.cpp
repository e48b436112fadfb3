// Prints the scanline launch plan (adcensus_b200/csrc/so_plan.h) of one pass, by default on an H100 SXM (132 SMs, 228 KB
// of shared memory per SM, 1 KB reserved per CTA).
// Usage: so_plan_main W H Dp S axis [sm_count smem_per_sm smem_reserved_per_cta]   ->   "T NS smem ctas ctas_per_sm waves"
#include <stdio.h>
#include <stdlib.h>

#include "../../adcensus_b200/csrc/so_plan.h"

int main(int argc, char** argv) {
    if (argc != 6 && argc != 9) return 2;
    const int sms = argc == 9 ? atoi(argv[6]) : 132;
    const size_t smem_sm = argc == 9 ? (size_t)atol(argv[7]) : 228 * 1024, smem_res = argc == 9 ? (size_t)atol(argv[8]) : 1024;
    const SoPlan p = so_plan(atoi(argv[1]), atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), sms, smem_sm, smem_res);
    printf("%d %d %zu %d %d %d\n", p.T, p.NS, p.smem, p.ctas, p.ctas_per_sm, p.waves);
    return p.T ? 0 : 1;
}
