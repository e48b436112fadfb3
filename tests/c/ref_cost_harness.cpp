// tests/c/ref_cost_harness.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product library).
//
// The staged harness around the UNMODIFIED reference (oracle/ref_harness.cpp, compiled in unchanged) with a
// caller-supplied cost volume: ref_begin_cost's COST step writes the given [H][W][D] f32 volume into the reference's
// cost_computer_.cost_init_ instead of calling ComputeCost; every later step runs the reference's own code.  Exported
// under the prefix refc_ with the staged API of the other checkers.  tools/make_golden_cost.py compiles it with the
// reference's sources (flags of oracle/Makefile) to produce tests/golden/golden_cost_cases.json.
#include "ref_harness.cpp"

namespace {
struct RefCostCtx {
    RefCtx* r = nullptr;
    std::vector<float> cost;
    bool injected = false;
};
}  // namespace

extern "C" {

void* refc_create(int width, int height, const void* opt_bytes) {
    RefCtx* r = static_cast<RefCtx*>(ref_create(width, height, opt_bytes));
    if (!r) return nullptr;
    RefCostCtx* x = new RefCostCtx();
    x->r = r;
    return x;
}

void refc_destroy(void* h) {
    RefCostCtx* x = static_cast<RefCostCtx*>(h);
    ref_destroy(x->r);
    delete x;
}

int refc_begin(void* h, const uint8_t* left, const uint8_t* right) {
    RefCostCtx* x = static_cast<RefCostCtx*>(h);
    x->injected = false;
    return ref_begin(x->r, left, right);
}

int ref_begin_cost(void* h, const uint8_t* left, const uint8_t* right, const float* cost_hwd_f32) {
    RefCostCtx* x = static_cast<RefCostCtx*>(h);
    if (!cost_hwd_f32 || !ref_begin(x->r, left, right)) return 0;
    const size_t nd = (size_t)x->r->w * x->r->h * (x->r->opt.max_disparity - x->r->opt.min_disparity);
    x->cost.assign(cost_hwd_f32, cost_hwd_f32 + nd);
    x->injected = true;
    return 1;
}
int refc_begin_cost(void* h, const uint8_t* left, const uint8_t* right, const float* cost_hwd_f32) {
    return ref_begin_cost(h, left, right, cost_hwd_f32);
}

int refc_step(void* h) {
    RefCostCtx* x = static_cast<RefCostCtx*>(h);
    if (x->injected && x->r->next_stage == ADC_STAGE_COST) {
        std::vector<float>& dst = x->r->stereo.cost_computer_.cost_init_;
        std::copy(x->cost.begin(), x->cost.end(), dst.begin());
        x->r->next_stage = ADC_STAGE_ARMS;
        return ADC_STAGE_COST;
    }
    return ref_step(x->r);
}

size_t refc_tap(void* h, int tap, void* dst, size_t cap) { return ref_tap(static_cast<RefCostCtx*>(h)->r, tap, dst, cap); }

double refc_time_match(void* h, const uint8_t* left, const uint8_t* right, float* disp, int iters) {
    return ref_time_match(static_cast<RefCostCtx*>(h)->r, left, right, disp, iters);
}

}  // extern "C"
