// Prints the launch plan of the fused cost + first horizontal arm sum (adcensus_b200/csrc/ca_plan.h) for one shape, then
// the output and cost ranges of every segment of a row.
// Usage: ca_plan_main W Dp L1   ->   "qc Ls nseg nchunks gm lpc threads smem ok budget" then one "s0 s1 m0 m1" line per segment
#include <stdio.h>
#include <stdlib.h>

#include "../../adcensus_b200/csrc/ca_plan.h"

int main(int argc, char** argv) {
    if (argc != 4) return 2;
    const int W = atoi(argv[1]), Dp = atoi(argv[2]), L1 = atoi(argv[3]);
    const CaPlan p = ca_plan(W, Dp, L1);
    printf("%d %d %d %d %d %d %d %zu %d %d\n", p.qc, p.Ls, p.nseg, p.nchunks, p.gm, p.lpc, p.threads, p.smem, (int)p.ok,
           CA_SMEM_BUDGET);
    for (int k = 0; p.ok && k < p.nseg; k++) {
        const int s0 = k * p.Ls, s1 = s0 + p.Ls < W ? s0 + p.Ls : W;
        int m0, m1;
        ca_cost_range(W, arm_L1c(L1), s0, s1, &m0, &m1);
        printf("%d %d %d %d\n", s0, s1, m0, m1);
    }
    return 0;
}
