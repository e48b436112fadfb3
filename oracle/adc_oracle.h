/* oracle/adc_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * C-ABI of the CPU restatement of the reference's AD-Census hot path (oracle/adc_oracle.c).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this; the product library (adcensus_b200/csrc) never does.
 *
 * Parity status: PINNED.  tests/test_oracle_vs_ref.py compares every stage of this restatement
 * bit-for-bit with the real reference (oracle/_ref, built from a checkout of the reference by oracle/Makefile)
 * on Cone and on synthetic pairs, and tests/test_oracle_golden.py compares it with the committed
 * golden vectors in tests/golden/ that were produced by the real reference (tools/make_golden.py).
 */
#ifndef ADC_ORACLE_H_
#define ADC_ORACLE_H_

#include <stddef.h>
#include <stdint.h>
#include "adc_taps.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Same 60-byte layout as the reference's ADCensusOption (adcensus_types.h:45-75). */
typedef struct orc_option {
    int32_t min_disparity, max_disparity;
    int32_t lambda_ad, lambda_census;
    int32_t cross_L1, cross_L2, cross_t1, cross_t2;
    float so_p1, so_p2;
    int32_t so_tso;
    int32_t irv_ts;
    float irv_th;
    float lrcheck_thres;
    uint8_t do_lr_check, do_filling, do_discontinuity_adjustment, pad_;
} orc_option;

typedef struct orc_ctx orc_ctx;

/* Tie counters: each is one increment at a comparison that an exact equality decided, where the neighbouring
 * comparison (>= for >, another reduction order) would have decided otherwise.  They never change a result.
 *   WTA_L / WTA_R   a later d with cost == the best so far (the strict > keeps the first minimum)
 *   SUBPIX_FLAT     the parabola's neighbours are equal or its denominator is 0
 *   LR_EQ           |disp - disp_r| == lrcheck_thres (kept)
 *   OCCL_EQ         disp_l[col_rl] == disp (a mismatch, not an occlusion)
 *   VOTE_PEAK       a filled pixel whose histogram has a later bin equal to the peak (the lowest disparity keeps it)
 *   VOTE_TS         total == irv_ts (not filled);  VOTE_TH  peak / total == irv_th (not filled)
 *   INTERP_DIST     a mismatch whose later ray meets the best colour distance with another disparity (the earliest
 *                   ray keeps it; occlusions take the smallest disparity, which no tie decides)
 *   INTERP_NONE     no ray found a candidate (the pixel becomes 0.0)
 *   EDGE_EQ         |gx| + |gy| == 5 (not an edge);  DISC_EQ  cc == c0 (not adjusted)
 *   ARM_T1 / ARM_T2 a colour distance equal to cross_t1 / cross_t2 where it is compared (the arm stops)
 *   ARM_L2          a step at exactly n + 1 == cross_L2 whose anchor distance is >= cross_t2 (the arm goes on)
 *   VOTE_PAIR       a filled pixel whose peak is an even bin 2k with bin 2k + 1 equal to it (the two bins of one word of
 *                   the GPU's narrow histogram, where the lane's own scan, not the cross-lane minimum, breaks the tie) */
enum { ORC_TIE_WTA_L, ORC_TIE_WTA_R, ORC_TIE_SUBPIX_FLAT, ORC_TIE_LR_EQ, ORC_TIE_OCCL_EQ, ORC_TIE_VOTE_PEAK,
       ORC_TIE_VOTE_TS, ORC_TIE_VOTE_TH, ORC_TIE_INTERP_DIST, ORC_TIE_INTERP_NONE, ORC_TIE_EDGE_EQ, ORC_TIE_DISC_EQ,
       ORC_TIE_ARM_T1, ORC_TIE_ARM_T2, ORC_TIE_ARM_L2, ORC_TIE_VOTE_PAIR, ORC_TIE_N };

void orc_default_option(orc_option* o);
orc_ctx* orc_create(int width, int height, const orc_option* opt);
void orc_destroy(orc_ctx* c);
/* whole pipeline, like ADCensusStereo::Match; returns 1 on success */
int orc_match(orc_ctx* c, const uint8_t* left, const uint8_t* right, float* disp_left);
/* staged runner, mirrors oracle/ref_harness.cpp */
int orc_begin(orc_ctx* c, const uint8_t* left, const uint8_t* right);
int orc_step(orc_ctx* c);
/* the staged runner from OUTLIER on, from given WTA maps (float [H][W] each); the arms come from the left image and the
 * cost volumes are never touched.  Returns 0 with do_discontinuity_adjustment set (that stage reads the volume). */
int orc_begin_refine(orc_ctx* c, const uint8_t* left, const uint8_t* right, const float* disp_left, const float* disp_right);
size_t orc_tap(orc_ctx* c, int tap, void* dst, size_t cap);
/* the tie counters accumulated since orc_begin / orc_begin_refine (ORC_TIE_N values) */
void orc_tie_counts(const orc_ctx* c, uint64_t* out);
double orc_time_match(orc_ctx* c, const uint8_t* left, const uint8_t* right, float* disp, int iters);

/* leaf functions exposed for exhaustive micro-tests */
uint8_t orc_gray(uint8_t b, uint8_t g, uint8_t r);
int orc_hamming64(uint64_t a, uint64_t b);
float orc_cost_value(int sum_abs_diff, int hamming, int lambda_ad, int lambda_census);

#ifdef __cplusplus
}
#endif
#endif
