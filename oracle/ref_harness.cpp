// oracle/ref_harness.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product library).
//
// Thin C-ABI harness around the UNMODIFIED reference sources (AD-Census/ of a checkout of the reference).
// It is compiled together with the reference's six algorithm .cpp files (where they lie, nothing
// is copied into this repo) into oracle/_ref/libadcensus_ref.so by oracle/Makefile.  It exists to
//   (1) pin oracle/adc_oracle.c (our own restatement) against the real reference, stage by stage,
//   (2) generate the golden fixtures under tests/golden/ (tools/make_golden.py),
//   (3) serve as the CPU baseline ("kind": "reference") in bench.py.
//
// The reference keeps every intermediate private, so the class is opened up with the usual
// `#define private public` trick; the staged runner below then calls the reference's own stage
// methods in exactly the order ADCensusStereo::Match (ADCensusStereo.cpp:69-132) and
// CrossAggregator::Aggregate (cross_aggregator.cpp:89-118) / ScanlineOptimizer::Optimize
// (scanline_optimizer.cpp:40-61) / MultiStepRefiner::Refine (multistep_refiner.cpp:60-87) do,
// stopping between stages so that a test can read the live buffers.
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <utility>
#include <vector>
#include <unistd.h>
#include <fcntl.h>

#define private public
#include "ADCensusStereo.h"
#include "adcensus_util.h"
#undef private

#include "adc_taps.h"

namespace {

struct RefCtx {
    ADCensusStereo stereo;
    ADCensusOption opt;
    int w = 0, h = 0;
    int next_stage = ADC_STAGE_COST;
    bool horizontal_first = true;
    const uint8_t* left = nullptr;
    const uint8_t* right = nullptr;
};

struct StdoutMute {
    int saved = -1;
    StdoutMute() {
        fflush(stdout);
        saved = dup(1);
        int nul = open("/dev/null", O_WRONLY);
        if (nul >= 0) { dup2(nul, 1); close(nul); }
    }
    ~StdoutMute() {
        fflush(stdout);
        if (saved >= 0) { dup2(saved, 1); close(saved); }
    }
};

size_t put(void* dst, size_t cap, const void* src, size_t bytes) {
    if (dst && cap >= bytes) memcpy(dst, src, bytes);
    return bytes;
}

}  // namespace

extern "C" {

int ref_option_size() { return (int)sizeof(ADCensusOption); }

// Writes the reference's default-constructed option block (adcensus_types.h:67-74).
void ref_default_option(void* opt_out) {
    ADCensusOption o;
    memset(opt_out, 0, sizeof(ADCensusOption));
    memcpy(opt_out, &o, sizeof(ADCensusOption));
}

void* ref_create(int width, int height, const void* opt_bytes) {
    RefCtx* c = new RefCtx();
    memcpy(&c->opt, opt_bytes, sizeof(ADCensusOption));
    c->w = width;
    c->h = height;
    if (!c->stereo.Initialize(width, height, c->opt)) {
        delete c;
        return nullptr;
    }
    return c;
}

void ref_destroy(void* h) { delete static_cast<RefCtx*>(h); }

// The stock entry point, untouched: ADCensusStereo::Match (ADCensusStereo.cpp:69).  The six
// timing printf lines it emits are muted so that a caller's stdout stays clean.
int ref_match(void* h, const uint8_t* left, const uint8_t* right, float* disp, int mute) {
    RefCtx* c = static_cast<RefCtx*>(h);
    if (mute) {
        StdoutMute m;
        return c->stereo.Match(left, right, disp) ? 1 : 0;
    }
    return c->stereo.Match(left, right, disp) ? 1 : 0;
}

// ---- staged runner -------------------------------------------------------------------------
int ref_begin(void* h, const uint8_t* left, const uint8_t* right) {
    RefCtx* c = static_cast<RefCtx*>(h);
    if (!left || !right) return 0;
    c->left = left;
    c->right = right;
    c->stereo.img_left_ = left;
    c->stereo.img_right_ = right;
    c->next_stage = ADC_STAGE_COST;
    c->horizontal_first = true;
    return 1;
}

// Executes the next stage; returns the id of the stage just executed, or -1 when finished.
int ref_step(void* h) {
    RefCtx* c = static_cast<RefCtx*>(h);
    ADCensusStereo& s = c->stereo;
    const ADCensusOption& o = s.option_;
    const int st = c->next_stage;
    switch (st) {
    case ADC_STAGE_COST:
        s.ComputeCost();
        break;
    case ADC_STAGE_ARMS: {
        CrossAggregator& a = s.aggregator_;
        a.SetData(s.img_left_, s.img_right_, s.cost_computer_.get_cost_ptr());
        a.SetParams(o.cross_L1, o.cross_L2, o.cross_t1, o.cross_t2);
        a.BuildArms();
        a.ComputeSupPixelCount();
        memcpy(&a.cost_aggr_[0], a.cost_init_,
               sizeof(float) * (size_t)a.width_ * a.height_ * (a.max_disparity_ - a.min_disparity_));
        c->horizontal_first = true;
        break;
    }
    case ADC_STAGE_AGG1: case ADC_STAGE_AGG2: case ADC_STAGE_AGG3: case ADC_STAGE_AGG4: {
        CrossAggregator& a = s.aggregator_;
        for (int d = a.min_disparity_; d < a.max_disparity_; d++) a.AggregateInArms(d, c->horizontal_first);
        c->horizontal_first = !c->horizontal_first;
        break;
    }
    case ADC_STAGE_SO1: {
        ScanlineOptimizer& so = s.scan_line_;
        so.SetData(s.img_left_, s.img_right_, s.cost_computer_.get_cost_ptr(), s.aggregator_.get_cost_ptr());
        so.SetParam(s.width_, s.height_, o.min_disparity, o.max_disparity, o.so_p1, o.so_p2, o.so_tso);
        so.ScanlineOptimizeLeftRight(so.cost_aggr_, so.cost_init_, true);
        break;
    }
    case ADC_STAGE_SO2: s.scan_line_.ScanlineOptimizeLeftRight(s.scan_line_.cost_init_, s.scan_line_.cost_aggr_, false); break;
    case ADC_STAGE_SO3: s.scan_line_.ScanlineOptimizeUpDown(s.scan_line_.cost_aggr_, s.scan_line_.cost_init_, true); break;
    case ADC_STAGE_SO4: s.scan_line_.ScanlineOptimizeUpDown(s.scan_line_.cost_init_, s.scan_line_.cost_aggr_, false); break;
    case ADC_STAGE_WTA:
        s.ComputeDisparity();
        s.ComputeDisparityRight();
        break;
    case ADC_STAGE_OUTLIER: {
        MultiStepRefiner& r = s.refiner_;
        r.SetData(s.img_left_, s.aggregator_.get_cost_ptr(), s.aggregator_.get_arms_ptr(), s.disp_left_, s.disp_right_);
        r.SetParam(o.min_disparity, o.max_disparity, o.irv_ts, o.irv_th, o.lrcheck_thres,
                   o.do_lr_check, o.do_filling, o.do_filling, o.do_discontinuity_adjustment);
        if (r.do_lr_check_) r.OutlierDetection();
        break;
    }
    case ADC_STAGE_VOTE:   if (s.refiner_.do_region_voting_) s.refiner_.IterativeRegionVoting(); break;
    case ADC_STAGE_INTERP: if (s.refiner_.do_interpolating_) s.refiner_.ProperInterpolation(); break;
    case ADC_STAGE_DISC:   if (s.refiner_.do_discontinuity_adjustment_) s.refiner_.DepthDiscontinuityAdjustment(); break;
    case ADC_STAGE_MEDIAN:
        adcensus_util::MedianFilter(s.disp_left_, s.disp_left_, s.width_, s.height_, 3);
        break;
    default:
        return -1;
    }
    c->next_stage = st + 1;
    return st;
}

// Copies a live buffer; returns its size in bytes (call with dst==NULL to query).
size_t ref_tap(void* h, int tap, void* dst, size_t cap) {
    RefCtx* c = static_cast<RefCtx*>(h);
    ADCensusStereo& s = c->stereo;
    const size_t n = (size_t)c->w * c->h;
    const size_t nd = n * (size_t)(c->opt.max_disparity - c->opt.min_disparity);
    switch (tap) {
    case ADC_TAP_GRAY_L:    return put(dst, cap, s.cost_computer_.gray_left_.data(), n);
    case ADC_TAP_GRAY_R:    return put(dst, cap, s.cost_computer_.gray_right_.data(), n);
    case ADC_TAP_CENSUS_L:  return put(dst, cap, s.cost_computer_.census_left_.data(), n * 8);
    case ADC_TAP_CENSUS_R:  return put(dst, cap, s.cost_computer_.census_right_.data(), n * 8);
    case ADC_TAP_VOL_INIT:  return put(dst, cap, s.cost_computer_.cost_init_.data(), nd * 4);
    case ADC_TAP_VOL_AGGR:  return put(dst, cap, s.aggregator_.cost_aggr_.data(), nd * 4);
    case ADC_TAP_ARMS:      return put(dst, cap, s.aggregator_.vec_cross_arms_.data(), n * 4);
    case ADC_TAP_SUPCNT_H:  return put(dst, cap, s.aggregator_.vec_sup_count_[0].data(), n * 2);
    case ADC_TAP_SUPCNT_V:  return put(dst, cap, s.aggregator_.vec_sup_count_[1].data(), n * 2);
    case ADC_TAP_DISP_L:    return put(dst, cap, s.disp_left_, n * 4);
    case ADC_TAP_DISP_R:    return put(dst, cap, s.disp_right_, n * 4);
    case ADC_TAP_MISMATCHES:
    case ADC_TAP_OCCLUSIONS: {
        const auto& v = (tap == ADC_TAP_MISMATCHES) ? s.refiner_.mismatches_ : s.refiner_.occlusions_;
        const size_t bytes = v.size() * 8;
        if (dst && cap >= bytes) {
            int32_t* o = static_cast<int32_t*>(dst);
            for (size_t i = 0; i < v.size(); i++) { o[2 * i] = v[i].first; o[2 * i + 1] = v[i].second; }
        }
        return bytes;
    }
    default: return 0;
    }
}

// Loops the stock Match `iters` times on one pair and returns the mean seconds per call
// (steady_clock, like the reference's own timers).  Used for the cpu_baseline leg of bench.py.
double ref_time_match(void* h, const uint8_t* left, const uint8_t* right, float* disp, int iters) {
    RefCtx* c = static_cast<RefCtx*>(h);
    StdoutMute m;
    auto t0 = std::chrono::steady_clock::now();
    for (int i = 0; i < iters; i++) c->stereo.Match(left, right, disp);
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count() / (iters > 0 ? iters : 1);
}

}  // extern "C"
