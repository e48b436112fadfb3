// Prints the launch plans of adcensus_b200/csrc/ca_plan.h for one shape.
// Usage: ca_plan_main W Dp L1   ->   the fused cost + first horizontal arm sum:
//                                    "qc Ls nseg nchunks gm lpc threads smem ok budget" then one "s0 s1 m0 m1" line per segment
//        ca_plan_main arm W H Dp L1   ->   the double passes, one line per axis (dir 0 = rows, then dir 1 = columns):
//                                    "dir t_ok t_qc t_Ls t_nseg t_nchunks t_lpc t_threads t_smem  ldg_qc_log2 ldg_Ls ldg_nseg ldg_smem
//                                     form smem_attr"
//                                    (t_*: k_arm_sum2t's plan, ldg_*: k_arm_sum2's, form: the kernel arm_sum2_form picks,
//                                     A2_TMA or A2_LDG, smem_attr: the dynamic shared memory both are launched under)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../adcensus_b200/csrc/ca_plan.h"

int main(int argc, char** argv) {
    if (argc == 6 && strcmp(argv[1], "arm") == 0) {
        const int W = atoi(argv[2]), H = atoi(argv[3]), Dp = atoi(argv[4]), L1 = atoi(argv[5]);
        for (int dir = 0; dir < 2; dir++) {
            const ArmSum2tPlan t = plan_arm_sum2t(W, H, Dp, L1, dir);
            const ArmSum2Plan g = plan_arm_sum2(W, H, Dp, L1, dir);
            printf("%d %d %d %d %d %d %d %d %zu %d %d %d %zu %d %d\n", dir, (int)t.ok, t.qc, t.Ls, t.nseg, t.nchunks, t.lpc,
                   t.threads, t.smem, g.qc_log2, g.Ls, g.nseg, g.smem, arm_sum2_form(W, H, Dp, L1, dir), A2_SMEM_ATTR);
        }
        return 0;
    }
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
