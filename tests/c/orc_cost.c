/* tests/c/orc_cost.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The C restatement of the reference (oracle/adc_oracle.c, compiled in unchanged) with a caller-supplied cost volume:
 * orc_begin_cost's COST step installs the given [H][W][D] f32 volume as cost_init instead of computing the AD-census
 * cost; every later step is the restatement's own.  The gray / census buffers are not computed in that mode.
 * Exported under the prefix occ_ with the staged API of the other checkers (tests/cost_testlib.py), built by
 * tests/cost_testlib.py into oracle/_build/libadc_oracle_cost.so.
 */
#include "adc_oracle.c"

typedef struct occ_ctx {
    orc_ctx* c;
    float* cost;   /* [H][W][D], the volume the next COST step installs */
    int injected;
} occ_ctx;

occ_ctx* occ_create(int width, int height, const orc_option* opt) {
    orc_ctx* c = orc_create(width, height, opt);
    if (!c) return NULL;
    occ_ctx* x = (occ_ctx*)calloc(1, sizeof(occ_ctx));
    x->c = c;
    x->cost = (float*)calloc((size_t)width * height * c->D, sizeof(float));
    return x;
}

void occ_destroy(occ_ctx* x) {
    if (!x) return;
    orc_destroy(x->c);
    free(x->cost);
    free(x);
}

int occ_begin(occ_ctx* x, const uint8_t* left, const uint8_t* right) {
    x->injected = 0;
    return orc_begin(x->c, left, right);
}

int orc_begin_cost(occ_ctx* x, const uint8_t* left, const uint8_t* right, const float* cost_hwd_f32) {
    if (!x || !cost_hwd_f32 || !orc_begin(x->c, left, right)) return 0;
    memcpy(x->cost, cost_hwd_f32, (size_t)x->c->w * x->c->h * x->c->D * sizeof(float));
    x->injected = 1;
    return 1;
}
int occ_begin_cost(occ_ctx* x, const uint8_t* left, const uint8_t* right, const float* cost_hwd_f32) {
    return orc_begin_cost(x, left, right, cost_hwd_f32);
}

int occ_step(occ_ctx* x) {
    orc_ctx* c = x->c;
    if (x->injected && c->next_stage == ADC_STAGE_COST) {
        memcpy(c->vol_init, x->cost, (size_t)c->w * c->h * c->D * sizeof(float));
        c->next_stage = ADC_STAGE_ARMS;
        return ADC_STAGE_COST;
    }
    return orc_step(c);
}

size_t occ_tap(occ_ctx* x, int tap, void* dst, size_t cap) { return orc_tap(x->c, tap, dst, cap); }

/* the whole pipeline on the given volume, like orc_match; returns 1 on success */
int orc_match_cost(occ_ctx* x, const uint8_t* left, const uint8_t* right, const float* cost_hwd_f32, float* disp_left) {
    if (!disp_left || !orc_begin_cost(x, left, right, cost_hwd_f32)) return 0;
    while (occ_step(x) >= 0) {}
    memcpy(disp_left, x->c->disp_l, sizeof(float) * (size_t)x->c->w * x->c->h);
    return 1;
}

double occ_time_match(occ_ctx* x, const uint8_t* left, const uint8_t* right, float* disp, int iters) {
    x->injected = 0;
    return orc_time_match(x->c, left, right, disp, iters);
}

void occ_tie_counts(const occ_ctx* x, uint64_t* out) { orc_tie_counts(x->c, out); }
