/* oracle/adc_oracle.c -- TEST INFRASTRUCTURE ONLY (see adc_oracle.h for who may load it).
 *
 * A plain-C, single-threaded restatement of the reference's AD-Census pipeline, written from the
 * algorithm's description stage by stage.  Every function names the reference lines it follows
 * (paths relative to the reference's AD-Census/ directory).  It keeps the reference's *sequential in-place*
 * semantics everywhere (LR check, region voting, median) because those define the answer.
 *
 * Arithmetic conventions that matter for bit-exactness (SURVEY.md section 8c):
 *   - the author's build resolves exp(float) to expf and abs(float) to a float abs, so this file
 *     uses expf / fabsf;  lround(float) and lround(double of the same value) agree, lroundf is used;
 *   - no FMA contraction anywhere (compile with -ffp-contract=off);
 *   - int operands are converted to float exactly where C++'s usual conversions would.
 */
#include "adc_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#define ORC_INVALID INFINITY /* adcensus_types.h:33 */
#define ORC_LARGE 99999.0f   /* adcensus_types.h:35 */

typedef struct { uint8_t left, right, top, bottom; } orc_arm; /* cross_aggregator.h:17-20 */

struct orc_ctx {
    int w, h, dmin, dmax, D;
    orc_option opt;
    const uint8_t *left, *right;
    uint8_t *gray_l, *gray_r;
    uint64_t *census_l, *census_r;
    float *vol_init, *vol_aggr; /* [H][W][D] */
    orc_arm* arms;
    uint16_t *sup_h, *sup_v, *sup_tmp;
    float *slice0, *slice1;
    float *disp_l, *disp_r;
    int32_t *mism, *occl; /* (x,y) pairs */
    size_t n_mism, n_occl;
    uint8_t* edge;
    int next_stage;
    int horizontal_first;
    uint64_t tie[ORC_TIE_N]; /* orc_tie_counts: since orc_begin / orc_begin_refine */
};

/* ------------------------------------------------------------------------------------------ */
void orc_default_option(orc_option* o) { /* adcensus_types.h:67-74 */
    memset(o, 0, sizeof(*o));
    o->min_disparity = 0;  o->max_disparity = 64;
    o->lambda_ad = 10;     o->lambda_census = 30;
    o->cross_L1 = 34;      o->cross_L2 = 17;
    o->cross_t1 = 20;      o->cross_t2 = 6;
    o->so_p1 = 1.0f;       o->so_p2 = 3.0f;
    o->so_tso = 15;        o->irv_ts = 20;
    o->irv_th = 0.4f;      o->lrcheck_thres = 1.0f;
    o->do_lr_check = 1;    o->do_filling = 1;
    o->do_discontinuity_adjustment = 0;
}

orc_ctx* orc_create(int width, int height, const orc_option* opt) { /* ADCensusStereo.cpp:21-67 */
    if (width <= 0 || height <= 0 || !opt) return NULL;
    if (opt->max_disparity - opt->min_disparity <= 0) return NULL;
    orc_ctx* c = (orc_ctx*)calloc(1, sizeof(orc_ctx));
    if (!c) return NULL;
    c->w = width; c->h = height; c->opt = *opt;
    c->dmin = opt->min_disparity; c->dmax = opt->max_disparity; c->D = c->dmax - c->dmin;
    const size_t n = (size_t)width * height, nd = n * (size_t)c->D;
    c->gray_l = (uint8_t*)calloc(n, 1);   c->gray_r = (uint8_t*)calloc(n, 1);
    c->census_l = (uint64_t*)calloc(n, 8); c->census_r = (uint64_t*)calloc(n, 8);
    c->vol_init = (float*)calloc(nd, 4);  c->vol_aggr = (float*)calloc(nd, 4);
    c->arms = (orc_arm*)calloc(n, sizeof(orc_arm));
    c->sup_h = (uint16_t*)calloc(n, 2); c->sup_v = (uint16_t*)calloc(n, 2); c->sup_tmp = (uint16_t*)calloc(n, 2);
    c->slice0 = (float*)calloc(n, 4);   c->slice1 = (float*)calloc(n, 4);
    c->disp_l = (float*)calloc(n, 4);   c->disp_r = (float*)calloc(n, 4);
    c->mism = (int32_t*)calloc(n, 8);   c->occl = (int32_t*)calloc(n, 8);
    c->edge = (uint8_t*)calloc(n, 1);
    c->next_stage = ADC_STAGE_COUNT;
    return c;
}

void orc_destroy(orc_ctx* c) {
    if (!c) return;
    free(c->gray_l); free(c->gray_r); free(c->census_l); free(c->census_r);
    free(c->vol_init); free(c->vol_aggr); free(c->arms);
    free(c->sup_h); free(c->sup_v); free(c->sup_tmp); free(c->slice0); free(c->slice1);
    free(c->disp_l); free(c->disp_r); free(c->mism); free(c->occl); free(c->edge);
    free(c);
}

/* ---- stage 1: gray, census, AD-census cost ------------------------------------------------- */
uint8_t orc_gray(uint8_t b, uint8_t g, uint8_t r) { /* cost_computor.cpp:69, double, truncation */
    return (uint8_t)(r * 0.299 + g * 0.587 + b * 0.114);
}

static void gray_image(const uint8_t* bgr, uint8_t* gray, size_t n) { /* cost_computor.cpp:58-73 */
    for (size_t i = 0; i < n; i++) gray[i] = orc_gray(bgr[3 * i], bgr[3 * i + 1], bgr[3 * i + 2]);
}

/* adcensus_util.cpp:10-39: 9 rows x 7 columns, MSB = first neighbour, border pixels stay 0 */
static void census_9x7(const uint8_t* g, uint64_t* out, int w, int h) {
    if (w <= 9 || h <= 7) return;
    for (int y = 4; y < h - 4; y++)
        for (int x = 3; x < w - 3; x++) {
            const uint8_t centre = g[y * w + x];
            uint64_t bits = 0;
            for (int dy = -4; dy <= 4; dy++)
                for (int dx = -3; dx <= 3; dx++)
                    bits = (bits << 1) | (uint64_t)(g[(y + dy) * w + x + dx] < centre);
            out[y * w + x] = bits;
        }
}

int orc_hamming64(uint64_t a, uint64_t b) { /* adcensus_util.cpp:42-53 */
    uint64_t v = a ^ b;
    int n = 0;
    while (v) { v &= v - 1; n++; }
    return n;
}

/* cost_computor.cpp:110-117, float32 throughout, left-to-right */
float orc_cost_value(int sum_abs_diff, int hamming, int lambda_ad, int lambda_census) {
    const float cost_ad = (float)sum_abs_diff / 3.0f;
    const float cost_census = (float)hamming;
    const float e_ad = expf(-cost_ad / (float)lambda_ad);
    const float e_cen = expf(-cost_census / (float)lambda_census);
    float c = 1.0f - e_ad;
    c = c + 1.0f;
    c = c - e_cen;
    return c;
}

static void stage_cost(orc_ctx* c) { /* cost_computor.cpp:123-137 */
    const int w = c->w, h = c->h;
    const size_t n = (size_t)w * h;
    gray_image(c->left, c->gray_l, n);
    gray_image(c->right, c->gray_r, n);
    /* the reference zero-fills the census vectors once at Initialize (cost_computor.cpp:37-38) and
     * never rewrites the border, so it stays 0 across calls */
    census_9x7(c->gray_l, c->census_l, w, h);
    census_9x7(c->gray_r, c->census_r, w, h);
    float* row_cost = c->vol_init;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint8_t* pl = c->left + ((size_t)y * w + x) * 3;
            const uint64_t cl = c->census_l[(size_t)y * w + x];
            for (int d = c->dmin; d < c->dmax; d++, row_cost++) {
                const int xr = x - d;
                if (xr < 0 || xr >= w) { *row_cost = 1.0f; continue; } /* :101-104 */
                const uint8_t* pr = c->right + ((size_t)y * w + xr) * 3;
                const int sad = abs(pl[0] - pr[0]) + abs(pl[1] - pr[1]) + abs(pl[2] - pr[2]);
                const int ham = orc_hamming64(cl, c->census_r[(size_t)y * w + xr]);
                *row_cost = orc_cost_value(sad, ham, c->opt.lambda_ad, c->opt.lambda_census);
            }
        }
}

/* ---- stage 2: cross arms, support counts, aggregation ------------------------------------- */
static int colour_dist(const uint8_t* a, const uint8_t* b) { /* cross_aggregator.h:78-80 (max channel) */
    int d0 = abs(a[0] - b[0]), d1 = abs(a[1] - b[1]), d2 = abs(a[2] - b[2]);
    int m = d0 > d1 ? d0 : d1;
    return m > d2 ? m : d2;
}

/* One arm: walk from (x,y) in direction (sx,sy).  cross_aggregator.cpp:135-201 / 203-269. */
static uint8_t grow_arm(orc_ctx* c, int x, int y, int sx, int sy) {
    const int w = c->w, h = c->h;
    const int limit = c->opt.cross_L1 < 255 ? c->opt.cross_L1 : 255; /* min(L1, MAX_ARM_LENGTH) :151 */
    const uint8_t* p0 = c->left + ((size_t)y * w + x) * 3;
    const uint8_t* prev = p0;
    int len = 0;
    int px = x + sx, py = y + sy;
    for (int n = 0; n < limit; n++) {
        if (px < 0 || px >= w || py < 0 || py >= h) break;          /* :154-163 */
        const uint8_t* p = c->left + ((size_t)py * w + px) * 3;
        const int dist_anchor = colour_dist(p, p0);
        c->tie[ORC_TIE_ARM_T1] += dist_anchor == c->opt.cross_t1;
        if (dist_anchor >= c->opt.cross_t1) break;                    /* :169-172 */
        const int dist_prev = n > 0 ? colour_dist(p, prev) : 0;
        c->tie[ORC_TIE_ARM_T1] += n > 0 && dist_prev == c->opt.cross_t1;
        if (n > 0 && dist_prev >= c->opt.cross_t1) break;             /* :175-180 (t1 again) */
        c->tie[ORC_TIE_ARM_L2] += n + 1 == c->opt.cross_L2 && dist_anchor >= c->opt.cross_t2;
        c->tie[ORC_TIE_ARM_T2] += n + 1 > c->opt.cross_L2 && dist_anchor == c->opt.cross_t2;
        if (n + 1 > c->opt.cross_L2 && dist_anchor >= c->opt.cross_t2) break; /* :183-187 */
        len++;
        prev = p;
        px += sx; py += sy;
    }
    return (uint8_t)len;
}

static void build_arms(orc_ctx* c) { /* cross_aggregator.cpp:76-86 */
    for (int y = 0; y < c->h; y++)
        for (int x = 0; x < c->w; x++) {
            orc_arm* a = &c->arms[(size_t)y * c->w + x];
            a->left = grow_arm(c, x, y, -1, 0);
            a->right = grow_arm(c, x, y, +1, 0);
            a->top = grow_arm(c, x, y, 0, -1);
            a->bottom = grow_arm(c, x, y, 0, +1);
        }
}

static void support_counts(orc_ctx* c) { /* cross_aggregator.cpp:271-325; u16 storage wraps like the reference */
    const int w = c->w, h = c->h;
    /* horizontal first: row extent, then summed along the vertical arm */
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const orc_arm a = c->arms[(size_t)y * w + x];
            c->sup_tmp[(size_t)y * w + x] = (uint16_t)(a.left + a.right + 1);
        }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const orc_arm a = c->arms[(size_t)y * w + x];
            int32_t cnt = 0;
            for (int t = -a.top; t <= a.bottom; t++) cnt += c->sup_tmp[(size_t)(y + t) * w + x];
            c->sup_h[(size_t)y * w + x] = (uint16_t)cnt;
        }
    /* vertical first */
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const orc_arm a = c->arms[(size_t)y * w + x];
            c->sup_tmp[(size_t)y * w + x] = (uint16_t)(a.top + a.bottom + 1);
        }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const orc_arm a = c->arms[(size_t)y * w + x];
            int32_t cnt = 0;
            for (int t = -a.left; t <= a.right; t++) cnt += c->sup_tmp[(size_t)y * w + x + t];
            c->sup_v[(size_t)y * w + x] = (uint16_t)cnt;
        }
}

/* One iteration over every disparity slice.  cross_aggregator.cpp:327-394.
 * The sums are sequential float32 additions in ascending tap order starting from 0.0f. */
static void aggregate_iteration(orc_ctx* c, int horizontal_first) {
    const int w = c->w, h = c->h, D = c->D;
    const uint16_t* sup = horizontal_first ? c->sup_h : c->sup_v;
    for (int d = 0; d < D; d++) {
        for (size_t i = 0; i < (size_t)w * h; i++) c->slice0[i] = c->vol_aggr[i * D + d];
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const orc_arm a = c->arms[(size_t)y * w + x];
                float s = 0.0f;
                if (horizontal_first) for (int t = -a.left; t <= a.right; t++) s += c->slice0[(size_t)y * w + x + t];
                else                  for (int t = -a.top; t <= a.bottom; t++) s += c->slice0[(size_t)(y + t) * w + x];
                c->slice1[(size_t)y * w + x] = s;
            }
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const orc_arm a = c->arms[(size_t)y * w + x];
                float s = 0.0f;
                if (horizontal_first) for (int t = -a.top; t <= a.bottom; t++) s += c->slice1[(size_t)(y + t) * w + x];
                else                  for (int t = -a.left; t <= a.right; t++) s += c->slice1[(size_t)y * w + x + t];
                /* float / (u16 -> int -> float), :389 */
                c->vol_aggr[((size_t)y * w + x) * D + d] = s / (float)(int)sup[(size_t)y * w + x];
            }
    }
}

/* ---- stage 3: scanline optimisation -------------------------------------------------------- */
static float fminf2(float a, float b) { return b < a ? b : a; } /* std::min */

/* One directional pass.  scanline_optimizer.cpp:63-171 (horizontal) and :173-279 (vertical).
 * (sx,sy) is the path direction; lines are indexed by the other coordinate. */
static void so_pass(const orc_ctx* c, const float* src, float* dst, int sx, int sy) {
    const int w = c->w, h = c->h, D = c->D, dmin = c->dmin;
    const float p1 = c->opt.so_p1, p2 = c->opt.so_p2;
    const int tso = c->opt.so_tso;
    const int n_lines = sx ? h : w, n_steps = sx ? w : h;
    float* last = (float*)malloc(sizeof(float) * (size_t)(D + 2));
    for (int line = 0; line < n_lines; line++) {
        int x = sx ? (sx > 0 ? 0 : w - 1) : line;
        int y = sy ? (sy > 0 ? 0 : h - 1) : line;
        /* path head copies its costs (:99-100) */
        const float* s = src + ((size_t)y * w + x) * D;
        float* o = dst + ((size_t)y * w + x) * D;
        last[0] = last[D + 1] = ORC_LARGE;
        for (int d = 0; d < D; d++) { o[d] = s[d]; last[d + 1] = s[d]; }
        float min_last = ORC_LARGE;
        for (int d = 0; d < D + 2; d++) min_last = fminf2(min_last, last[d]); /* pads included, :107-110 */
        const uint8_t* prev_px = c->left + ((size_t)y * w + x) * 3;
        for (int step = 1; step < n_steps; step++) {
            x += sx; y += sy;
            const uint8_t* px = c->left + ((size_t)y * w + x) * 3;
            const uint8_t d1 = (uint8_t)colour_dist(px, prev_px);
            uint8_t d2 = d1; /* declared once per pixel: "sticky" across the d loop, :116 */
            s = src + ((size_t)y * w + x) * D;
            o = dst + ((size_t)y * w + x) * D;
            float min_cur = ORC_LARGE;
            for (int d = 0; d < D; d++) {
                const int xr = x - d - dmin;
                if (xr > 0 && xr < w - 1) { /* :120 */
                    const uint8_t* r = c->right + ((size_t)y * w + xr) * 3;
                    const uint8_t* rp = c->right + ((size_t)(y - sy) * w + (xr - sx)) * 3;
                    d2 = (uint8_t)colour_dist(r, rp);
                }
                float P1 = 0.0f, P2 = 0.0f; /* :129-141 */
                if (d1 < tso && d2 < tso) { P1 = p1; P2 = p2; }
                else if (d1 < tso && d2 >= tso) { P1 = p1 / 4; P2 = p2 / 4; }
                else if (d1 >= tso && d2 < tso) { P1 = p1 / 4; P2 = p2 / 4; }
                else if (d1 >= tso && d2 >= tso) { P1 = p1 / 10; P2 = p2 / 10; }
                const float l1 = last[d + 1];
                const float l2 = last[d] + P1;
                const float l3 = last[d + 2] + P1;
                const float l4 = min_last + P2;
                float v = s[d] + fminf2(fminf2(l1, l2), fminf2(l3, l4)); /* :144-151, no "- min" term */
                v /= 2;
                o[d] = v;
                min_cur = fminf2(min_cur, v);
            }
            min_last = min_cur;
            memcpy(last + 1, o, sizeof(float) * (size_t)D);
            prev_px = px;
        }
    }
    free(last);
}

/* ---- stage 4: winner-takes-all with parabola ---------------------------------------------- */
static float subpixel(orc_ctx* c, float c1, float c2, float cmin, int best) { /* ADCensusStereo.cpp:234-240 */
    const float denom = c1 + c2 - 2 * cmin;
    c->tie[ORC_TIE_SUBPIX_FLAT] += c1 == c2 || denom == 0.0f;
    if (denom != 0.0f) return (float)best + (c1 - c2) / (denom * 2.0f);
    return (float)best;
}

static void wta_left(orc_ctx* c) { /* ADCensusStereo.cpp:188-243 */
    const int w = c->w, h = c->h, D = c->D, dmin = c->dmin, dmax = c->dmax;
    for (size_t p = 0; p < (size_t)w * h; p++) {
        const float* v = c->vol_aggr + p * D;
        float best_cost = ORC_LARGE;
        int best = 0;
        for (int d = dmin; d < dmax; d++) {
            c->tie[ORC_TIE_WTA_L] += v[d - dmin] == best_cost;
            if (best_cost > v[d - dmin]) { best_cost = v[d - dmin]; best = d; } /* strict: first minimum */
        }
        if (best == dmin || best == dmax - 1) { c->disp_l[p] = ORC_INVALID; continue; }
        c->disp_l[p] = subpixel(c, v[best - 1 - dmin], v[best + 1 - dmin], best_cost, best);
    }
}

static void wta_right(orc_ctx* c) { /* ADCensusStereo.cpp:245-310: cost_R(x,d) = cost_L(x+d,d) */
    const int w = c->w, h = c->h, D = c->D, dmin = c->dmin, dmax = c->dmax;
    float* local = (float*)malloc(sizeof(float) * (size_t)D);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float best_cost = ORC_LARGE;
            int best = 0;
            for (int d = dmin; d < dmax; d++) {
                const int xl = x + d;
                if (xl >= 0 && xl < w) {
                    const float v = c->vol_aggr[((size_t)y * w + xl) * D + (d - dmin)];
                    local[d - dmin] = v;
                    c->tie[ORC_TIE_WTA_R] += v == best_cost;
                    if (best_cost > v) { best_cost = v; best = d; }
                } else {
                    local[d - dmin] = ORC_LARGE; /* :286 */
                }
            }
            float* out = &c->disp_r[(size_t)y * w + x];
            if (best == dmin || best == dmax - 1) { *out = (float)best; continue; } /* :290-293, NOT invalid */
            /* note: for dmin > 0 the reference can index local[] out of range here (best stays 0);
             * guarded, the reference's behaviour is undefined in that corner (SURVEY 8a/A10) */
            const int i1 = best - 1 - dmin, i2 = best + 1 - dmin;
            if (i1 < 0 || i2 >= D) { *out = (float)best; continue; }
            *out = subpixel(c, local[i1], local[i2], best_cost, best);
        }
    free(local);
}

/* ---- stage 5: multi-step refinement ---------------------------------------------------------- */
static void outlier_detection(orc_ctx* c) { /* multistep_refiner.cpp:90-151, raster order, in place */
    const int w = c->w, h = c->h;
    const float thres = c->opt.lrcheck_thres;
    c->n_mism = c->n_occl = 0;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float* dp = &c->disp_l[(size_t)y * w + x];
            const float disp = *dp;
            if (disp == ORC_INVALID) { c->mism[2 * c->n_mism] = x; c->mism[2 * c->n_mism + 1] = y; c->n_mism++; continue; }
            const long col_r = lroundf((float)x - disp);
            if (col_r >= 0 && col_r < w) {
                const float disp_r = c->disp_r[(size_t)y * w + col_r];
                c->tie[ORC_TIE_LR_EQ] += fabsf(disp - disp_r) == thres;
                if (fabsf(disp - disp_r) > thres) {
                    const int col_rl = (int)lroundf((float)col_r + disp_r);
                    int is_occl = 0;
                    if (col_rl > 0 && col_rl < w) {
                        const float dl = c->disp_l[(size_t)y * w + col_rl]; /* may already be +inf */
                        c->tie[ORC_TIE_OCCL_EQ] += dl == disp;
                        is_occl = dl > disp;
                    }
                    if (is_occl) { c->occl[2 * c->n_occl] = x; c->occl[2 * c->n_occl + 1] = y; c->n_occl++; }
                    else         { c->mism[2 * c->n_mism] = x; c->mism[2 * c->n_mism + 1] = y; c->n_mism++; }
                    *dp = ORC_INVALID;
                }
            } else {
                *dp = ORC_INVALID;
                c->mism[2 * c->n_mism] = x; c->mism[2 * c->n_mism + 1] = y; c->n_mism++;
            }
        }
}

static void region_voting(orc_ctx* c) { /* multistep_refiner.cpp:153-227 */
    const int w = c->w, D = c->D, dmin = c->dmin;
    int* hist = (int*)malloc(sizeof(int) * (size_t)D);
    for (int it = 0; it < 5; it++)
        for (int k = 0; k < 2; k++) {
            int32_t* list = k == 0 ? c->mism : c->occl;
            size_t* cnt = k == 0 ? &c->n_mism : &c->n_occl;
            for (size_t i = 0; i < *cnt; i++) {
                const int x = list[2 * i], y = list[2 * i + 1];
                float* dp = &c->disp_l[(size_t)y * w + x];
                if (*dp != ORC_INVALID) continue;
                memset(hist, 0, sizeof(int) * (size_t)D);
                const orc_arm a = c->arms[(size_t)y * w + x];
                for (int t = -a.top; t <= a.bottom; t++) {
                    const int yt = y + t;
                    const orc_arm a2 = c->arms[(size_t)yt * w + x];
                    for (int s = -a2.left; s <= a2.right; s++) {
                        const float d = c->disp_l[(size_t)yt * w + x + s];
                        if (d != ORC_INVALID) {
                            const long di = lroundf(d) - dmin;
                            if (di >= 0 && di < D) hist[di]++; /* reference would write out of range otherwise */
                        }
                    }
                }
                int best = 0, total = 0, peak = 0;
                for (int d = 0; d < D; d++) {
                    if (peak < hist[d]) { peak = hist[d]; best = d; }
                    total += hist[d];
                }
                c->tie[ORC_TIE_VOTE_TS] += peak > 0 && total == c->opt.irv_ts;
                c->tie[ORC_TIE_VOTE_TH] += peak > 0 && total > c->opt.irv_ts && (float)peak * 1.0f / (float)total == c->opt.irv_th;
                if (peak > 0 && total > c->opt.irv_ts && (float)peak * 1.0f / (float)total > c->opt.irv_th) {
                    int later = 0;
                    for (int d = best + 1; d < D; d++) later |= hist[d] == peak;
                    c->tie[ORC_TIE_VOTE_PEAK] += later;
                    c->tie[ORC_TIE_VOTE_PAIR] += best % 2 == 0 && best + 1 < D && hist[best + 1] == peak;
                    *dp = (float)(best + dmin); /* visible to later pixels of this sweep */
                }
            }
            size_t keep = 0; /* erase filled, order preserved (:217-224) */
            for (size_t i = 0; i < *cnt; i++) {
                const int x = list[2 * i], y = list[2 * i + 1];
                if (c->disp_l[(size_t)y * w + x] == ORC_INVALID) { list[2 * keep] = x; list[2 * keep + 1] = y; keep++; }
            }
            *cnt = keep;
        }
    free(hist);
}

static void proper_interpolation(orc_ctx* c) { /* multistep_refiner.cpp:229-305 */
    const int w = c->w, h = c->h;
    const float pi = 3.1415926f;
    const int a1 = abs(c->dmax), a2 = abs(c->dmin);
    const int max_len = a1 > a2 ? a1 : a2;
    float* fill = (float*)malloc(sizeof(float) * ((size_t)w * h + 1));
    for (int k = 0; k < 2; k++) {
        const int32_t* list = k == 0 ? c->mism : c->occl;
        const size_t cnt = k == 0 ? c->n_mism : c->n_occl;
        if (cnt == 0) continue;
        for (size_t i = 0; i < cnt; i++) {
            const int x = list[2 * i], y = list[2 * i + 1];
            fill[i] = 0.0f; /* value-initialised vector: "no candidate" leaves 0.0 (:244,270) */
            int n_cand = 0;
            int best_dist = 9999;
            float best_d = 0.0f, min_d = ORC_LARGE;
            const uint8_t* pc = c->left + ((size_t)y * w + x) * 3;
            double ang = 0.0;
            for (int s = 0; s < 16; s++) {
                const double sina = sin(ang), cosa = cos(ang);
                for (int m = 1; m < max_len; m++) {
                    const long yy = lround(y + m * sina);
                    const long xx = lround(x + m * cosa);
                    if (yy < 0 || yy >= h || xx < 0 || xx >= w) break;
                    const float d = c->disp_l[(size_t)yy * w + xx];
                    if (d != ORC_INVALID) {
                        const uint8_t* q = c->left + ((size_t)yy * w + xx) * 3;
                        const int dist = abs(pc[0] - q[0]) + abs(pc[1] - q[1]) + abs(pc[2] - q[2]);
                        c->tie[ORC_TIE_INTERP_DIST] += k == 0 && dist == best_dist && d != best_d;
                        if (best_dist > dist) { best_dist = dist; best_d = d; } /* first closest wins */
                        min_d = fminf2(min_d, d);
                        n_cand++;
                        break;
                    }
                }
                ang += pi / 16; /* float quotient accumulated in double (:234,268) */
            }
            c->tie[ORC_TIE_INTERP_NONE] += n_cand == 0;
            if (n_cand == 0) continue;
            fill[i] = k == 0 ? best_d : min_d;
        }
        for (size_t i = 0; i < cnt; i++) /* written after the whole list (:298-303) */
            c->disp_l[(size_t)list[2 * i + 1] * w + list[2 * i]] = fill[i];
    }
    free(fill);
}

static void discontinuity_adjustment(orc_ctx* c) { /* multistep_refiner.cpp:307-371 */
    const int w = c->w, h = c->h, D = c->D;
    const float* p = c->disp_l;
    memset(c->edge, 0, (size_t)w * h);
    for (int y = 1; y < h - 1; y++)
        for (int x = 1; x < w - 1; x++) {
            const float* r0 = p + (size_t)(y - 1) * w + x;
            const float* r1 = p + (size_t)y * w + x;
            const float* r2 = p + (size_t)(y + 1) * w + x;
            const float gx = (-r0[-1] + r0[1]) + (-2 * r1[-1] + 2 * r1[1]) + (-r2[-1] + r2[1]);
            const float gy = (-r0[-1] - 2 * r0[0] - r0[1]) + (r2[-1] + 2 * r2[0] + r2[1]);
            c->tie[ORC_TIE_EDGE_EQ] += fabsf(gx) + fabsf(gy) == 5.0f;
            if (fabsf(gx) + fabsf(gy) > 5.0f) c->edge[(size_t)y * w + x] = 1;
        }
    for (int y = 0; y < h; y++)
        for (int x = 1; x < w - 1; x++) {
            if (c->edge[(size_t)y * w + x] != 1) continue;
            float* row = c->disp_l + (size_t)y * w;
            if (row[x] == ORC_INVALID) continue;
            const float* cost = c->vol_aggr + ((size_t)y * w + x) * D;
            const long di = lroundf(row[x]); /* the reference does not subtract dmin here (:331) */
            if (di < 0 || di >= D) continue;  /* out of range is undefined in the reference */
            float c0 = cost[di];
            for (int k = 0; k < 2; k++) {
                const int x2 = k == 0 ? x - 1 : x + 1;
                const float d2 = row[x2];
                if (d2 == ORC_INVALID) continue;
                const long d2i = lroundf(d2);
                if (d2i < 0 || d2i >= D) continue;
                const float cc = k == 0 ? cost[-D + d2i] : cost[D + d2i];
                c->tie[ORC_TIE_DISC_EQ] += cc == c0;
                if (cc < c0) { row[x] = d2; c0 = cc; }
            }
        }
}

static int cmp_float(const void* a, const void* b) {
    const float fa = *(const float*)a, fb = *(const float*)b;
    return (fa > fb) - (fa < fb);
}

static void median3_inplace(float* img, int w, int h) { /* adcensus_util.cpp:55-81 with in == out */
    float win[9];
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int n = 0;
            for (int dy = -1; dy <= 1; dy++)
                for (int dx = -1; dx <= 1; dx++) {
                    const int yy = y + dy, xx = x + dx;
                    if (yy >= 0 && yy < h && xx >= 0 && xx < w) win[n++] = img[(size_t)yy * w + xx];
                }
            qsort(win, (size_t)n, sizeof(float), cmp_float);
            img[(size_t)y * w + x] = win[n / 2];
        }
}

/* ---- staged runner --------------------------------------------------------------------------- */
int orc_begin(orc_ctx* c, const uint8_t* left, const uint8_t* right) {
    if (!c || !left || !right) return 0;
    c->left = left; c->right = right;
    memset(c->tie, 0, sizeof(c->tie));
    c->next_stage = ADC_STAGE_COST;
    c->horizontal_first = 1;
    return 1;
}

/* Refinement only: the staged runner from OUTLIER on, with the given WTA maps and the arms of the left image.  It never
 * touches the cost volumes (calloc leaves them unmapped), so it runs at sizes whose volumes would not fit in host
 * memory.  The discontinuity adjustment reads the aggregated volume, so a context with it enabled is refused. */
int orc_begin_refine(orc_ctx* c, const uint8_t* left, const uint8_t* right, const float* disp_left, const float* disp_right) {
    if (!c || !left || !right || !disp_left || !disp_right || c->opt.do_discontinuity_adjustment) return 0;
    const size_t n = (size_t)c->w * c->h;
    c->left = left; c->right = right;
    memcpy(c->disp_l, disp_left, n * sizeof(float));
    memcpy(c->disp_r, disp_right, n * sizeof(float));
    memset(c->tie, 0, sizeof(c->tie));
    build_arms(c);
    support_counts(c);
    c->n_mism = c->n_occl = 0;
    c->next_stage = ADC_STAGE_OUTLIER;
    return 1;
}

int orc_step(orc_ctx* c) {
    const int st = c->next_stage;
    const size_t nd = (size_t)c->w * c->h * c->D;
    switch (st) {
    case ADC_STAGE_COST: stage_cost(c); break;
    case ADC_STAGE_ARMS:
        build_arms(c);
        support_counts(c);
        memcpy(c->vol_aggr, c->vol_init, nd * sizeof(float)); /* cross_aggregator.cpp:108 */
        c->horizontal_first = 1;
        break;
    case ADC_STAGE_AGG1: case ADC_STAGE_AGG2: case ADC_STAGE_AGG3: case ADC_STAGE_AGG4:
        aggregate_iteration(c, c->horizontal_first);
        c->horizontal_first = !c->horizontal_first;
        break;
    case ADC_STAGE_SO1: so_pass(c, c->vol_aggr, c->vol_init, +1, 0); break; /* scanline_optimizer.cpp:54-60 */
    case ADC_STAGE_SO2: so_pass(c, c->vol_init, c->vol_aggr, -1, 0); break;
    case ADC_STAGE_SO3: so_pass(c, c->vol_aggr, c->vol_init, 0, +1); break;
    case ADC_STAGE_SO4: so_pass(c, c->vol_init, c->vol_aggr, 0, -1); break;
    case ADC_STAGE_WTA: wta_left(c); wta_right(c); break;
    case ADC_STAGE_OUTLIER: if (c->opt.do_lr_check) outlier_detection(c); break;
    case ADC_STAGE_VOTE:    if (c->opt.do_filling) region_voting(c); break;      /* ADCensusStereo.cpp:183 */
    case ADC_STAGE_INTERP:  if (c->opt.do_filling) proper_interpolation(c); break;
    case ADC_STAGE_DISC:    if (c->opt.do_discontinuity_adjustment) discontinuity_adjustment(c); break;
    case ADC_STAGE_MEDIAN:  median3_inplace(c->disp_l, c->w, c->h); break;
    default: return -1;
    }
    c->next_stage = st + 1;
    return st;
}

int orc_match(orc_ctx* c, const uint8_t* left, const uint8_t* right, float* disp_left) {
    if (!c || !left || !right || !disp_left) return 0; /* ADCensusStereo.cpp:71-76 */
    orc_begin(c, left, right);
    /* the reference only clears its outlier lists inside OutlierDetection; a fresh context starts empty */
    while (orc_step(c) >= 0) {}
    memcpy(disp_left, c->disp_l, sizeof(float) * (size_t)c->w * c->h);
    return 1;
}

static size_t put(void* dst, size_t cap, const void* src, size_t bytes) {
    if (dst && cap >= bytes) memcpy(dst, src, bytes);
    return bytes;
}

size_t orc_tap(orc_ctx* c, int tap, void* dst, size_t cap) {
    const size_t n = (size_t)c->w * c->h, nd = n * (size_t)c->D;
    switch (tap) {
    case ADC_TAP_GRAY_L:   return put(dst, cap, c->gray_l, n);
    case ADC_TAP_GRAY_R:   return put(dst, cap, c->gray_r, n);
    case ADC_TAP_CENSUS_L: return put(dst, cap, c->census_l, n * 8);
    case ADC_TAP_CENSUS_R: return put(dst, cap, c->census_r, n * 8);
    case ADC_TAP_VOL_INIT: return put(dst, cap, c->vol_init, nd * 4);
    case ADC_TAP_VOL_AGGR: return put(dst, cap, c->vol_aggr, nd * 4);
    case ADC_TAP_ARMS:     return put(dst, cap, c->arms, n * 4);
    case ADC_TAP_SUPCNT_H: return put(dst, cap, c->sup_h, n * 2);
    case ADC_TAP_SUPCNT_V: return put(dst, cap, c->sup_v, n * 2);
    case ADC_TAP_DISP_L:   return put(dst, cap, c->disp_l, n * 4);
    case ADC_TAP_DISP_R:   return put(dst, cap, c->disp_r, n * 4);
    case ADC_TAP_MISMATCHES: return put(dst, cap, c->mism, c->n_mism * 8);
    case ADC_TAP_OCCLUSIONS: return put(dst, cap, c->occl, c->n_occl * 8);
    default: return 0;
    }
}

void orc_tie_counts(const orc_ctx* c, uint64_t* out) { memcpy(out, c->tie, sizeof(c->tie)); }

double orc_time_match(orc_ctx* c, const uint8_t* left, const uint8_t* right, float* disp, int iters) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int i = 0; i < iters; i++) orc_match(c, left, right, disp);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    const double s = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
    return s / (iters > 0 ? iters : 1);
}
