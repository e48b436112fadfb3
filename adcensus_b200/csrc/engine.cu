// engine.cu -- host side of the H100 AD-Census engine and its C ABI (include/adcensus_b200.h).
//
// An engine owns `lanes` independent pipelines.  A lane = one CUDA stream + a device arena for a
// wave of up to `wave_pairs` stereo pairs (two cost volumes per pair dominate: 2*4*N*Dp bytes) +
// pinned staging for callers that hand in pageable memory.  A batch is cut into waves that are
// dealt round-robin to the lanes; every kernel of a wave is one batched launch over all its pairs
// (pair index = outermost grid dimension), and the lanes overlap each other's copies, bandwidth
// kernels and the latency-bound refinement kernels.  Nothing here ever falls back to a CPU path:
// if the CUDA library cannot run, the call fails.
#include <cuda_runtime.h>

#include <float.h>
#include <math.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/adcensus_b200.h"
#include "../../include/adcensus_b200_preview.h"
#include "adc_common.cuh"
#include "ca_plan.h"
#include "so_plan.h"

static_assert(sizeof(adc_option) == 60, "adc_option must match the reference's ADCensusOption (60 bytes)");
static_assert(offsetof(adc_option, so_p1) == 32 && offsetof(adc_option, irv_th) == 48 &&
              offsetof(adc_option, do_lr_check) == 56 && offsetof(adc_option, do_discontinuity_adjustment) == 58,
              "adc_option field offsets must match adcensus_types.h:45-75");
static_assert(sizeof(adc_image_desc) == 32 && offsetof(adc_image_desc, reserved) == 4 &&
              offsetof(adc_image_desc, row_pitch) == 8 && offsetof(adc_image_desc, plane_pitch) == 16 &&
              offsetof(adc_image_desc, image_stride) == 24, "adc_image_desc layout (include/adcensus_b200.h)");
static_assert(sizeof(adc_remap) == 32 && offsetof(adc_remap, map2) == 8 && offsetof(adc_remap, map1_pitch) == 16 &&
              offsetof(adc_remap, map2_pitch) == 24, "adc_remap layout (include/adcensus_b200.h)");
static_assert(sizeof(adc_rectification) == 80 && offsetof(adc_rectification, src_height) == 4 &&
              offsetof(adc_rectification, map_type) == 8 && offsetof(adc_rectification, reserved) == 12 &&
              offsetof(adc_rectification, view) == 16, "adc_rectification layout (include/adcensus_b200.h)");
static_assert(sizeof(adc_speckle_params) == 32 && offsetof(adc_speckle_params, max_size) == 4 &&
              offsetof(adc_speckle_params, new_val) == 8 && offsetof(adc_speckle_params, max_diff) == 16 &&
              offsetof(adc_speckle_params, reserved) == 24, "adc_speckle_params layout (include/adcensus_b200.h)");
static_assert(sizeof(adc_reproject_out) == 16 && offsetof(adc_reproject_out, kind) == 8 &&
              offsetof(adc_reproject_out, reserved) == 12, "adc_reproject_out layout (include/adcensus_b200.h)");
static_assert(sizeof(adc_preview_params) == 48 && offsetof(adc_preview_params, alpha) == 8 &&
              offsetof(adc_preview_params, dst_width) == 24 && offsetof(adc_preview_params, invalid_bgr) == 32 &&
              offsetof(adc_preview_params, reserved) == 40, "adc_preview_params layout (include/adcensus_b200_preview.h)");
static_assert(sizeof(adc_cloud_out) == 48 && offsetof(adc_cloud_out, colors) == 8 && offsetof(adc_cloud_out, pixels) == 16 &&
              offsetof(adc_cloud_out, counts) == 24 && offsetof(adc_cloud_out, capacity) == 32 &&
              offsetof(adc_cloud_out, reserved) == 40, "adc_cloud_out layout (include/adcensus_b200.h)");

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                 \
    do {                                                                                         \
        cudaError_t err__ = (call);                                                              \
        if (err__ != cudaSuccess)                                                                \
            return fail(ADC_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)

struct Lane {
    cudaStream_t st = nullptr;
    cudaEvent_t ev_done = nullptr;     // all work of the lane's latest wave (incl. D2H) finished
    cudaEvent_t ev_in_free = nullptr;  // the H2D of the latest wave has consumed the staging-in buffer
    void* arena = nullptr;
    AdcWave w{};                       // device pointers, capacity S pairs
    AdcArmTmaps arm_tm{};              // TMA descriptors of this lane's volumes (aggregation double passes)
    AdcSoTmaps so_tm{};                // TMA descriptors of this lane's volumes and penalty records (scanline passes)
    uint8_t* pin_in = nullptr;         // [S][2][N*3] pinned staging (pageable callers only)
    float* pin_out = nullptr;          // [S][N]
    // pending copy-out of a staged wave (pageable callers)
    int drain_n = 0;
    float* const* drain_ptrs = nullptr;
    float* drain_base = nullptr;
    int drain_first = 0;
};

}  // namespace

struct adc_engine {
    int W = 0, H = 0;
    adc_option opt{};
    adc_config cfg{};
    AdcParams P{};
    int S = 0;
    std::vector<Lane> lanes;
    cudaStream_t main_st = nullptr;
    cudaEvent_t ev_fork = nullptr;
    float* d_lut_ad = nullptr;
    float* d_lut_cen = nullptr;
    double* d_rays = nullptr;  // [32]: sin[16], cos[16]
    short2* d_ray_off = nullptr;  // [16][max_search] integer ray offsets, when verified exact for this image size
    bool pipelined = false;            // adc_set_pipelined: batch calls do not join the caller's stream themselves
    bool agg_fused = false;            // same-axis aggregation passes of neighbouring iterations run as one kernel (k_arm_sum2t / k_arm_sum2)
    unsigned long long launches = 0;
    float stage_ms[6] = {0, 0, 0, 0, 0, 0};
    cudaEvent_t ev_stage[8] = {};
    // debug state (adc_debug_run): which buffer plays the reference's cost_init_ / cost_aggr_
    const float* dbg_init = nullptr;
    const float* dbg_aggr = nullptr;   // nullptr also after a run whose last scanline pass took the WTA (dbg_so_wta)
    bool dbg_so_wta = false;           // the last run's pass 4 stored partial WTA records, not the optimised volume
    int dbg_stage = -1;
    // layout / element type of the last cost-input call (adc_profile_kernel's ingestion timing)
    int cost_layout = ADC_COST_DHW, cost_dtype = ADC_COST_F32;
    // layout / element type of the last volume export (adc_profile_kernel's export timing)
    int export_layout = ADC_COST_DHW, export_dtype = ADC_COST_F32;
    // image format of the last adc_match_images* call (adc_profile_kernel's ingestion timing)
    int img_format = ADC_IMG_RGB_PLANAR;
    // rectification (adc_set_rectification): its r->map_type, -1 = none set; for maps (ADC_REMAP_*) both views' maps in
    // the internal form, [2][N], for a resize (ADC_RESIZE_*) nullptr
    int rect_type = -1;
    uint2* rect_map = nullptr;
    int rect_src_w = 0, rect_src_h = 0;
    // raw frame format of the last adc_match_rectified* call (adc_profile_kernel's rectified ingestion timing)
    int rect_format = ADC_IMG_BGR;
    // device staging of adc_match_volumes' exported volumes: allocated on first use, grown when needed
    void* vol_stage = nullptr;
    size_t vol_stage_bytes = 0;
    // [N] pinned: the right-view map of the latest one-pair host match with a final map (adc_get_right_disparity), kept
    // apart from lane 0's arena, which every batch call's first wave overwrites
    float* pin_disp_r = nullptr;
};

namespace {

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Carver {
    char* base;
    size_t off = 0;
    explicit Carver(void* b) : base(static_cast<char*>(b)) {}
    template <typename T> T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off = align_up(off + count * sizeof(T), 256);
        return p;
    }
};

// Carves (or, with base == nullptr, just sizes) one lane's arena.
size_t carve_lane(void* base, const AdcDims& dm, int L1, int S, AdcWave* w) {
    Carver c(base);
    const size_t N = (size_t)dm.N;
    AdcWave t{};
    t.volA = c.take<float>((size_t)S * dm.vol_stride);
    t.volB = c.take<float>((size_t)S * dm.vol_stride);
    c.take<float>(adc_arm_overread_floats(dm));           // the arm-sum walks may load (never use) a few taps past a volume's end
    t.bgr = c.take<uint8_t>((size_t)S * 2 * N * 3);
    t.gray = c.take<uint8_t>((size_t)S * 2 * N);
    t.bgrx = c.take<unsigned>((size_t)S * 2 * N);
    t.census = c.take<unsigned long long>((size_t)S * 2 * N);
    t.arms = c.take<uchar4>((size_t)S * N);
    t.arm_rec = c.take<unsigned>((size_t)S * adc_arm_rec_bytes(dm, L1) / 4);
    t.sup_h = c.take<uint16_t>((size_t)S * N);
    t.sup_v = c.take<uint16_t>((size_t)S * N);
    t.dmap = c.take<uint8_t>((size_t)S * 4 * N);
    t.disp_l = c.take<float>((size_t)S * N);
    t.disp_r = c.take<float>((size_t)S * N);
    t.disp_t = c.take<float>((size_t)S * N);
    t.label = c.take<uint8_t>((size_t)S * N);
    t.flag = c.take<uint8_t>((size_t)S * N);
    t.pend = c.take<int>((size_t)S * 2 * N);
    t.vlist = c.take<int>((size_t)S * 2 * N);
    t.counters = c.take<int>((size_t)S * ADC_CNT);
    t.vote_alr = c.take<uchar2>((size_t)S * N);
    t.vote_chg = c.take<int2>((size_t)S * N);
    t.vote_atbT = c.take<uchar2>((size_t)S * N);
    t.vote_pslotT = c.take<int>((size_t)S * N);
    t.vote_val = c.take<uint16_t>((size_t)S * N);
    t.vote_dirtyb = c.take<uint8_t>((size_t)S * N);
    t.vote_state = c.take<int>((size_t)S * N);
    t.vote_off = c.take<int>((size_t)S * (N + 1));
    t.rowcnt = c.take<int>((size_t)S * 2 * dm.H);
    t.so_bitrows = c.take<unsigned>((size_t)S * adc_so_bitrow_bytes(dm) / 4);
    t.so_rec = c.take<unsigned>((size_t)S * adc_so_rec_bytes(dm) / 4);
    t.vote_work = c.take<int>((size_t)S * N);
    t.vote_hist = reinterpret_cast<unsigned*>(t.volB);   // idle after the last scanline pass
    if (w) *w = t;
    return c.off;
}

void build_params(adc_engine* e) {
    const adc_option& o = e->opt;
    AdcParams& P = e->P;
    P.dm.W = e->W; P.dm.H = e->H;
    P.dm.dmin = o.min_disparity; P.dm.dmax = o.max_disparity;
    P.dm.D = o.max_disparity - o.min_disparity;
    P.dm.Dp = (P.dm.D + 3) / 4 * 4;
    P.dm.N = e->W * e->H;
    P.dm.vol_stride = (long long)P.dm.N * P.dm.Dp;
    P.L1 = std::min(o.cross_L1, 255);  // min(cross_L1_, MAX_ARM_LENGTH), cross_aggregator.cpp:151
    P.L2 = o.cross_L2; P.t1 = o.cross_t1; P.t2 = o.cross_t2;
    // scanline_optimizer.cpp:133-140: p/4 and p/10 are float / int -> IEEE float division
    P.p1 = o.so_p1; P.p2 = o.so_p2;
    P.p1_4 = o.so_p1 / 4; P.p2_4 = o.so_p2 / 4;
    P.p1_10 = o.so_p1 / 10; P.p2_10 = o.so_p2 / 10;
    P.tso = o.so_tso;
    P.irv_ts = o.irv_ts; P.irv_th = o.irv_th;
    P.lr_thres = o.lrcheck_thres;
    P.max_search = std::max(abs(o.max_disparity), abs(o.min_disparity));  // multistep_refiner.cpp:236
    P.dbg = e->cfg.debug_flags;
}

int upload_tables(adc_engine* e) {
    // exp() factors of the AD-census cost on their integer domains, with THIS host's libm expf and
    // the reference's operation order (cost_computor.cpp:110-117): the device never calls exp.
    std::vector<float> ad(766), cen(64);
    for (int s = 0; s < 766; s++) {
        const float cost_ad = (float)s / 3.0f;
        const float e_ad = expf(-cost_ad / (float)e->opt.lambda_ad);
        float t = 1.0f - e_ad;
        t = t + 1.0f;
        ad[s] = t;
    }
    for (int h = 0; h < 64; h++) cen[h] = expf(-(float)h / (float)e->opt.lambda_census);
    // ray directions of ProperInterpolation (multistep_refiner.cpp:234,252-254,268)
    double rays[32];
    const float pi = 3.1415926f;
    double ang = 0.0;
    for (int s = 0; s < 16; s++) {
        rays[s] = sin(ang);
        rays[16 + s] = cos(ang);
        ang += pi / 16;
    }
    CK(cudaMalloc(&e->d_lut_ad, sizeof(float) * 766));
    CK(cudaMalloc(&e->d_lut_cen, sizeof(float) * 64));
    CK(cudaMalloc(&e->d_rays, sizeof(double) * 32));
    CK(cudaMemcpy(e->d_lut_ad, ad.data(), sizeof(float) * 766, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(e->d_lut_cen, cen.data(), sizeof(float) * 64, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(e->d_rays, rays, sizeof(double) * 32, cudaMemcpyHostToDevice));
    // ProperInterpolation evaluates lround(y + m*sin) per step (multistep_refiner.cpp:252-254).  For integer y
    // that equals y + lround(m*sin) unless a rounding of the double sum (or a half-way case) intervenes;
    // check every (ray, m, coordinate) the image can produce and only then let the kernel use the table.
    const int L = e->P.max_search;
    if (L > 1 && L < 4096 && !(e->cfg.debug_flags & ADC_DBG_NO_RAY_TABLE)) {
        std::vector<short2> off((size_t)16 * L);
        bool exact = true;
        for (int s = 0; s < 16 && exact; s++)
            for (int m = 1; m < L && exact; m++) {
                const long dy = lround(m * rays[s]), dx = lround(m * rays[16 + s]);
                for (int y = 0; y < e->H && exact; y++) exact = lround(y + m * rays[s]) == y + dy;
                for (int x = 0; x < e->W && exact; x++) exact = lround(x + m * rays[16 + s]) == x + dx;
                off[(size_t)s * L + m] = make_short2((short)dx, (short)dy);
            }
        if (exact) {
            CK(cudaMalloc(&e->d_ray_off, sizeof(short2) * off.size()));
            CK(cudaMemcpy(e->d_ray_off, off.data(), sizeof(short2) * off.size(), cudaMemcpyHostToDevice));
        }
    }
    return ADC_OK;
}

bool poisoned(const adc_engine* e) { return (e->cfg.debug_flags & ADC_DBG_POISON) != 0; }
int poison_byte(const adc_engine* e) { return (e->cfg.debug_flags >> 8) & 0xff; }

// Fills lane ln's whole arena on its stream: every buffer carve_lane cuts, the unused slots of a partial wave and the
// arm-sum over-read tail behind the volumes.  With ADC_DBG_POISON the fill is the test pattern, so that a kernel that
// reads what its wave or call did not write shows in the outputs; otherwise zeros, which nothing relies on (the poison
// tests run every entry point without them) but which keep a fresh engine's buffers deterministic for adc_debug_get and
// adc_profile_kernel before its first run.  Then comes the state a kernel relies on from adc_create, restored after
// every poison fill; each entry names the kernel.  There is none: every buffer a kernel reads is written earlier in the
// same wave or call.
int fill_arena(adc_engine* e, Lane& ln) {
    const size_t bytes = carve_lane(nullptr, e->P.dm, e->P.L1, e->S, nullptr);
    CK(cudaMemsetAsync(ln.arena, poisoned(e) ? poison_byte(e) : 0, bytes, ln.st));
    return ADC_OK;
}

AdcWave wave_view(const adc_engine* e, const Lane& ln, int nS) {
    AdcWave w = ln.w;
    w.S = nS;
    w.lut_ad = e->d_lut_ad;
    w.lut_cen = e->d_lut_cen;
    w.ray_sin = e->d_rays;
    w.ray_cos = e->d_rays + 16;
    w.ray_off = e->d_ray_off;
    return w;
}

// Where stage 1's volume comes from: the AD-census cost of the images (p == nullptr), or the caller's volumes of the
// wave at device address p (pair stride N*D elements).
struct CostSrc {
    const void* p = nullptr;
    int layout = ADC_COST_HWD, dtype = ADC_COST_F32;
};

// Volumes a call exports (adc_volume_out, at most one per ADC_VOL_* stage), with the wave's destinations.
struct VolOuts {
    adc_volume_out o[3] = {};
    int n = 0;
};

// Side maps a call requests (adc_map_out), indexed by ADC_MAP_* kind, with the wave's destinations; nullptr = not requested.
struct MapOuts {
    void* dst[5] = {};
};

size_t map_elem_bytes(int kind) { return kind == ADC_MAP_OUTLIERS ? 1 : sizeof(float); }

// One match call, as its entry point describes it once the arguments are checked (DESIGN.md section 2, "Host
// drivers").  Host entries hold one pair's cost volume in cost.p, device entries the first pair's; the volume and map
// destinations are the caller's, of one pair (host) or of pair 0 (device).
struct MatchReq {
    CostSrc cost;
    const adc_volume_out* vols = nullptr;
    int n_vols = 0;
    const adc_map_out* maps = nullptr;
    int n_maps = 0;
    const AdcImageGeom* img = nullptr;   // the views' resolved geometry; nullptr = tight packed BGR
    const AdcRectGeom* rect = nullptr;   // with img: the views are raw frames, resampled through these maps
    bool final_map = true;               // the refined disparity map is wanted
    int debug_stage = -1;                // adc_debug_run*: the stage to stop after
};

// The stage a request's run stops after: the debug entries' own; with a final map everything; otherwise the latest
// requested volume's or map's (the outlier map is taken after the LR check, every other map right after the WTA).
int last_stage(const MatchReq& q) {
    if (q.debug_stage >= 0) return q.debug_stage;
    if (q.final_map) return ADC_STAGE_MEDIAN;
    static const int vol_stage[3] = {ADC_STAGE_COST, ADC_STAGE_AGG4, ADC_STAGE_SO4};
    int last = ADC_STAGE_COST;
    for (int i = 0; i < q.n_vols; i++) last = std::max(last, vol_stage[q.vols[i].stage]);
    for (int i = 0; i < q.n_maps; i++)
        last = std::max(last, q.maps[i].kind == ADC_MAP_OUTLIERS ? (int)ADC_STAGE_OUTLIER : (int)ADC_STAGE_WTA);
    return last;
}

// Records the formats of a request that runs, for adc_profile_kernel's ingestion and export timings.
void note_formats(adc_engine* e, const MatchReq& q) {
    if (q.cost.p) {
        e->cost_layout = q.cost.layout;
        e->cost_dtype = q.cost.dtype;
    }
    if (q.n_vols > 0) {
        e->export_layout = q.vols[q.n_vols - 1].layout;
        e->export_dtype = q.vols[q.n_vols - 1].dtype;
    }
    if (q.rect) e->rect_format = q.img->format;
    else if (q.img) e->img_format = q.img->format;
}

// Whether a request's views go through an ingestion kernel into the wave's bgr: raw frames and formats other than
// packed BGR do.  Packed BGR rows are copied, one pair's whatever their pitch; the pairs of a batch (one_pair false)
// only when they are tight and back to back.
bool needs_ingest(const adc_engine* e, const MatchReq& q, bool one_pair) {
    if (q.rect) return true;
    if (!q.img) return false;
    if (q.img->format != ADC_IMG_BGR) return true;
    return !one_pair && (q.img->row_pitch != 3ll * e->W || q.img->image_stride != 3ll * e->W * e->H);
}

// A run that has to stop between aggregation iterations (debug taps AGG1..AGG3) takes the single passes.
bool agg_fused_for(const adc_engine* e, int last_stage) {
    return e->agg_fused && !(last_stage >= ADC_STAGE_AGG1 && last_stage <= ADC_STAGE_AGG3);
}

// The lane volumes of a run that stops after `last_stage`: c0, the one stage 1 writes (the cost volume), and the other
// one.  Host images and raw frames are staged in c0, whose contents nothing reads before their ingestion; a host cost
// volume waits for its ingestion in the other one, which stage 1 only reads.
struct LaneVols {
    float* c0;
    float* other;
};
LaneVols lane_volumes(const adc_engine* e, const AdcWave& w, int last_stage) {
    return agg_fused_for(e, last_stage) ? LaneVols{w.volB, w.volA} : LaneVols{w.volA, w.volB};
}

// Enqueues the whole pipeline for the nS pairs whose images already sit in ln.w.bgr.  Stops after
// `last_stage` (ADC_STAGE_MEDIAN = everything).  ev[] (optional, 6 events) are recorded at the
// stage boundaries the reference times in Match (ADCensusStereo.cpp:81-129).  `outs` (possibly none) are exported at the one
// point where their volume is live (DESIGN.md section 11): COST in C0 right after stage 1, before the first aggregation
// launch (the fused passes overwrite volB) -- or, where the cost is computed inside the first aggregation pass, right after
// that kernel, which then also stores the cost volume to C0; AGGR in volA after the last aggregation pass, before scanline pass 2 writes volA;
// OPT in volA after scanline pass 4, which nothing later writes.  `maps` (possibly none) likewise (DESIGN.md section 12): the
// WTA maps and the confidence right after the WTA (disp_l is overwritten by the LR check), the outlier map right after
// the LR check (region voting changes label).
int enqueue_pipeline(adc_engine* e, Lane& ln, int nS, int last_stage, bool debug_run, cudaEvent_t* ev, const CostSrc& cost,
                     const VolOuts& outs, const MapOuts& maps) {
    const AdcParams& P = e->P;
    const AdcWave w = wave_view(e, ln, nS);
    cudaStream_t st = ln.st;
    unsigned long long* L = &e->launches;
    const size_t mapN = (size_t)nS * P.dm.N;
    // The two volumes play the reference's cost_init_ / cost_aggr_.  The aggregation leaves its result in volA either way:
    //   eight single passes:   cost -> A | H: A->B, V/: B->A | V: A->B, H/: B->A | ...                          (8 x 2 = 16 volume transfers)
    //   same-axis passes fused (second pass of iteration k + first pass of iteration k+1 in one kernel):
    //                          cost -> B | H: B->A | V/ V: A->B | H/ H: B->A | V/ V: A->B | H/: B->A           (5 x 2 = 10 volume transfers)
    const bool fused = agg_fused_for(e, last_stage);
    float* A = w.volA;
    float* B = w.volB;
    float* C0 = lane_volumes(e, w, last_stage).c0;   // where the cost volume is written
    // The fused path computes the AD-census cost inside iteration 0's horizontal pass (k_cost_arm_sum_h): the cost volume
    // is not materialised, C0 is written only for a COST export.  The host staging of images and raw frames in C0 (volB
    // here) stays valid: volB is first written by the first fused vertical double pass, after the ingestion kernels have
    // read it.
    const bool cost_in_agg = fused && last_stage > ADC_STAGE_ARMS && !cost.p && adc_cost_arm_sum_h_available(P);
    bool cost_exported = false;
    for (int i = 0; i < outs.n; i++) cost_exported |= outs.o[i].stage == ADC_VOL_COST;
    e->dbg_init = cost_in_agg && !cost_exported ? nullptr : C0;   // no tap of a cost volume that was never written
    e->dbg_aggr = C0;
    e->dbg_so_wta = false;
    auto stop = [&](int stage) { e->dbg_stage = stage; return stage >= last_stage; };
    // launch errors surface where they happen: a stage boundary reports the first failed launch since the previous one
    auto launched = [&](const char* what) -> int {
        const cudaError_t err = cudaGetLastError();
        if (err != cudaSuccess) return fail(ADC_ERR_CUDA, "%s: kernel launch failed: %s", what, cudaGetErrorString(err));
        return ADC_OK;
    };
    auto export_vol = [&](int stage, const float* vol) {
        for (int i = 0; i < outs.n; i++)
            if (outs.o[i].stage == stage)
                adc_launch_cost_export(P, w, vol, outs.o[i].dst, outs.o[i].layout, outs.o[i].dtype, st, L);
    };
    int rc;

    // ---- stage 1: cost (cost_computor.cpp:123-137), or the caller's volume.  Gray / census run either way: the
    // kernels after this stage read the packed pixels (bgrx) the census kernel writes.
    adc_launch_gray_census(P, w, st, L);
    if (cost.p) adc_launch_cost_ingest(P, w, cost.p, cost.layout, cost.dtype, C0, st, L);
    else if (!cost_in_agg) adc_launch_cost(P, w, C0, st, L);
    if (!cost_in_agg) export_vol(ADC_VOL_COST, C0);
    if ((rc = launched("cost volume"))) return rc;
    if (ev) CK(cudaEventRecord(ev[1], st));
    if (stop(ADC_STAGE_COST)) return ADC_OK;

    // ---- stage 2: arms, support counts, window records, 4 aggregation iterations (cross_aggregator.cpp:89-118)
    adc_launch_arms(P, w, st, L);
    if ((rc = launched("cross arms"))) return rc;
    if (stop(ADC_STAGE_ARMS)) return ADC_OK;
    if (fused) {
        if (cost_in_agg) {                                                       // cost + it 0: H
            if (!adc_launch_cost_arm_sum_h(P, w, A, cost_exported ? C0 : nullptr, st, L))
                return fail(ADC_ERR_UNSUPPORTED, "fused cost and aggregation pass not applicable");
            export_vol(ADC_VOL_COST, C0);
        } else {
            adc_launch_arm_sum(P, w, B, A, 0, nullptr, st, L);                   // it 0: H
        }
        adc_launch_arm_sum2(P, w, A, B, 1, w.sup_h, st, L);                      // it 0: V /   + it 1: V
        adc_launch_arm_sum2(P, w, B, A, 0, w.sup_v, st, L);                      // it 1: H /   + it 2: H
        adc_launch_arm_sum2(P, w, A, B, 1, w.sup_h, st, L);                      // it 2: V /   + it 3: V
        adc_launch_arm_sum(P, w, B, A, 0, w.sup_v, st, L);                       // it 3: H /
        export_vol(ADC_VOL_AGGR, A);
        e->dbg_aggr = A;
        e->dbg_stage = ADC_STAGE_AGG4;
    } else {
        for (int it = 0; it < 4; it++) {
            const bool hfirst = (it % 2) == 0;  // H,V | V,H | H,V | V,H  (:102,116)
            adc_launch_arm_sum(P, w, A, B, hfirst ? 0 : 1, nullptr, st, L);
            adc_launch_arm_sum(P, w, B, A, hfirst ? 1 : 0, hfirst ? w.sup_h : w.sup_v, st, L);
            if (it == 3) export_vol(ADC_VOL_AGGR, A);
            if (stop(ADC_STAGE_AGG1 + it)) return launched("aggregation");
        }
    }
    if ((rc = launched("aggregation"))) return rc;
    if (ev) CK(cudaEventRecord(ev[2], st));
    if (last_stage <= ADC_STAGE_AGG4) return ADC_OK;

    // ---- stage 3: scanline optimisation, 4 chained passes (scanline_optimizer.cpp:54-60)
    adc_launch_diffmaps(P, w, st, L);
    adc_launch_so_bitrows(P, w, st, L);
    // Pass 4 takes both WTA views as its epilogue where nothing else reads the optimised volume: it then writes disp_l and
    // the right view's partial records into A instead of the volume, and k_wta_merge finishes disp_r (so_plan.h).
    SoVolumeUse vol_use{};
    for (int i = 0; i < outs.n; i++) vol_use.opt_export |= outs.o[i].stage == ADC_VOL_OPT;
    vol_use.confidence = maps.dst[ADC_MAP_MIN_COST] || maps.dst[ADC_MAP_PEAK_RATIO];
    vol_use.discontinuity = e->opt.do_discontinuity_adjustment != 0;
    vol_use.debug_run = debug_run || last_stage < ADC_STAGE_WTA;
    const int wta_force = (e->cfg.debug_flags & ADC_DBG_UNFUSED_SO_WTA) ? SO_WTA_NEVER
                          : (e->cfg.debug_flags & ADC_DBG_FUSED_SO_WTA) ? SO_WTA_ALWAYS : SO_WTA_AUTO;
    const bool so_wta = so_wta_fused(vol_use, wta_force, P.dm.W, P.dm.H, P.dm.D, P.dm.Dp, P.dm.dmin, P.dm.vol_stride);
    static const int dirs[4][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}};
    for (int ps = 0; ps < 4; ps++) {
        const float* src = (ps % 2 == 0) ? A : B;
        float* dst = (ps % 2 == 0) ? B : A;
        if (ps == 3 && so_wta ? adc_launch_scanline_wta(P, w, src, dst, st, L)
                              : adc_launch_scanline(P, w, src, dst, dirs[ps][0], dirs[ps][1], st, L))
            return fail(ADC_ERR_UNSUPPORTED, "scanline pass not launched (disparity range %d, limit 256)", P.dm.D);
        if (ps % 2 == 0) e->dbg_init = B; else e->dbg_aggr = ps == 3 && so_wta ? nullptr : A;   // the fused pass leaves records in A
        if (ps == 3) e->dbg_so_wta = so_wta;
        if (ps == 3) export_vol(ADC_VOL_OPT, A);
        if (stop(ADC_STAGE_SO1 + ps)) return launched("scanline optimisation");
    }
    if ((rc = launched("scanline optimisation"))) return rc;
    if (ev) CK(cudaEventRecord(ev[3], st));

    // ---- stage 4: left + right disparity (ADCensusStereo.cpp:108-109)
    if (so_wta) adc_launch_wta_merge(P, w, A, st, L);
    else if (adc_launch_wta(P, w, A, st, L)) return fail(ADC_ERR_UNSUPPORTED, "WTA launch failed");
    if (maps.dst[ADC_MAP_WTA_LEFT])
        CK(cudaMemcpyAsync(maps.dst[ADC_MAP_WTA_LEFT], w.disp_l, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (maps.dst[ADC_MAP_WTA_RIGHT])
        CK(cudaMemcpyAsync(maps.dst[ADC_MAP_WTA_RIGHT], w.disp_r, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (maps.dst[ADC_MAP_MIN_COST] || maps.dst[ADC_MAP_PEAK_RATIO])
        adc_launch_confidence(P, w, A, static_cast<float*>(maps.dst[ADC_MAP_MIN_COST]),
                              static_cast<float*>(maps.dst[ADC_MAP_PEAK_RATIO]), st, L);
    if ((rc = launched("winner-takes-all"))) return rc;
    if (ev) CK(cudaEventRecord(ev[4], st));
    if (stop(ADC_STAGE_WTA)) return ADC_OK;

    // ---- stage 5: multi-step refinement (multistep_refiner.cpp:60-87)
    if (e->opt.do_lr_check) {
        adc_launch_outlier(P, w, st, L);  // disp_l (orig) -> disp_t, label
        CK(cudaMemcpyAsync(w.disp_l, w.disp_t, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else {
        CK(cudaMemsetAsync(w.label, 0, mapN, st));
        CK(cudaMemcpyAsync(w.disp_t, w.disp_l, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (maps.dst[ADC_MAP_OUTLIERS]) CK(cudaMemcpyAsync(maps.dst[ADC_MAP_OUTLIERS], w.label, mapN, cudaMemcpyDeviceToDevice, st));
    if (stop(ADC_STAGE_OUTLIER)) return launched("outlier detection");
    if (e->opt.do_filling) {  // gates voting AND interpolation (ADCensusStereo.cpp:183)
        CK(cudaMemsetAsync(w.counters, 0, (size_t)nS * ADC_CNT * sizeof(int), st));
        adc_launch_build_lists(P, w, st, L);
        adc_launch_voting(P, w, st, L);
        if ((rc = launched("region voting"))) return rc;
        if (stop(ADC_STAGE_VOTE)) return ADC_OK;
        for (int k = 0; k < 2; k++) {
            adc_launch_interp_list(P, w, k, st, L);
            CK(cudaMemcpyAsync(w.disp_l, w.disp_t, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
        if (stop(ADC_STAGE_INTERP)) return launched("interpolation");
    } else if (last_stage <= ADC_STAGE_INTERP) {
        e->dbg_stage = last_stage;
        return launched("refinement");
    }
    if (e->opt.do_discontinuity_adjustment) adc_launch_discontinuity(P, w, A, st, L);
    if (stop(ADC_STAGE_DISC)) return launched("discontinuity adjustment");
    // median: disp_l -> disp_t, then back so that disp_l always holds the current map
    if (adc_launch_median(P, w, w.disp_l, w.disp_t, st, L))
        return fail(ADC_ERR_UNSUPPORTED, "image height %d exceeds the median kernel's limit", P.dm.H);
    CK(cudaMemcpyAsync(w.disp_l, w.disp_t, mapN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (ev) CK(cudaEventRecord(ev[5], st));
    e->dbg_stage = ADC_STAGE_MEDIAN;
    return launched("refinement");
}

bool is_pinned(const void* p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged;
}

int drain_lane(adc_engine* e, Lane& ln) {
    if (ln.drain_n == 0) return ADC_OK;
    CK(cudaEventSynchronize(ln.ev_done));
    const size_t N = (size_t)e->P.dm.N;
    for (int i = 0; i < ln.drain_n; i++) {
        float* dst = ln.drain_ptrs ? ln.drain_ptrs[ln.drain_first + i] : ln.drain_base + (size_t)(ln.drain_first + i) * N;
        memcpy(dst, ln.pin_out + (size_t)i * N, N * sizeof(float));
    }
    ln.drain_n = 0;
    return ADC_OK;
}

// n pairs of views at left / right (pair i at byte i * g.image_stride; geometry g, resolved, over the raw frames of
// `rect` or the engine's size) -> `bgr` as packed BGR [n][2][N*3] on st: one ingestion launch per
// adc_view_ingest_max_pairs pairs.
void ingest_views(adc_engine* e, int n, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                  const AdcRectGeom* rect, uint8_t* bgr, cudaStream_t st) {
    const int chunk = adc_view_ingest_max_pairs(e->P.dm);
    for (int first = 0; first < n; first += chunk) {
        const long long off = (long long)first * g.image_stride;
        adc_launch_view_ingest(e->P.dm, std::min(n - first, chunk), left + off, right + off, g, rect,
                               bgr + (size_t)first * 6 * e->P.dm.N, st, &e->launches);
    }
}

enum SrcKind { SRC_HOST_PTRS, SRC_HOST_STRIDED, SRC_DEVICE_STRIDED };

// Where the pairs of a batch live: strided views and maps (ls / rs / ds, pair i at i times a tight pair's size, or at
// i * image_stride for described images) in pinned or pageable host memory or in device memory, or host pointer
// arrays (lp / rp / dp, one pointer per pair).  A device call without a final map has ds == nullptr.
struct BatchIO {
    SrcKind kind;
    bool pinned;
    const uint8_t* ls = nullptr;
    const uint8_t* rs = nullptr;
    float* ds = nullptr;
    const uint8_t* const* lp = nullptr;
    const uint8_t* const* rp = nullptr;
    float* const* dp = nullptr;
};

// The batch driver (arguments checked, device set): the n pairs of request q, where `io` says they live, cut into
// waves dealt round-robin to the lanes.  `user` = stream to fork from / join to.  `force_join`: the call is one of the
// synchronous entry points, whose results must be complete on return whatever the engine's pipelined setting
// (adc_set_pipelined only changes the asynchronous entry points).
int run_batch(adc_engine* e, int n, const BatchIO& io, const MatchReq& q, cudaStream_t user, bool force_join) {
    const size_t N = (size_t)e->P.dm.N, IMG = N * 3;
    const int S = e->S, nl = (int)e->lanes.size();
    const int last = last_stage(q);
    const bool ingest = needs_ingest(e, q, false);   // only device entries describe their images
    const bool on_device = io.kind == SRC_DEVICE_STRIDED;
    const bool strided_copy = on_device || (io.pinned && io.kind == SRC_HOST_STRIDED);   // one 2D copy per view and wave
    note_formats(e, q);
    CK(cudaEventRecord(e->ev_fork, user));
    const int n_waves = (n + S - 1) / S;
    for (int li = 0; li < std::min(nl, n_waves); li++) CK(cudaStreamWaitEvent(e->lanes[li].st, e->ev_fork, 0));
    for (int wv = 0; wv < n_waves; wv++) {
        Lane& ln = e->lanes[wv % nl];
        const int first = wv * S, nS = std::min(S, n - first);
        const AdcWave& w = ln.w;   // where the images go in and the map comes out
        if (poisoned(e)) {
            int rcp = fill_arena(e, ln);
            if (rcp) return rcp;
        }
        // ---- inputs -> w.bgr  ([S][2][IMG])
        if (ingest) {
            const long long off = (long long)first * q.img->image_stride;
            ingest_views(e, nS, io.ls + off, io.rs + off, *q.img, q.rect, w.bgr, ln.st);
        } else if (strided_copy) {
            const cudaMemcpyKind k = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
            CK(cudaMemcpy2DAsync(w.bgr, 2 * IMG, io.ls + (size_t)first * IMG, IMG, IMG, nS, k, ln.st));
            CK(cudaMemcpy2DAsync(w.bgr + IMG, 2 * IMG, io.rs + (size_t)first * IMG, IMG, IMG, nS, k, ln.st));
        } else if (io.pinned) {
            for (int i = 0; i < nS; i++) {
                CK(cudaMemcpyAsync(w.bgr + (size_t)i * 2 * IMG, io.lp[first + i], IMG, cudaMemcpyHostToDevice, ln.st));
                CK(cudaMemcpyAsync(w.bgr + (size_t)i * 2 * IMG + IMG, io.rp[first + i], IMG, cudaMemcpyHostToDevice, ln.st));
            }
        } else {
            // pageable caller memory: finish the lane's previous wave (copy-out), then stage through pinned memory
            int rcd = drain_lane(e, ln);
            if (rcd) return rcd;
            CK(cudaEventSynchronize(ln.ev_in_free));
            for (int i = 0; i < nS; i++) {
                const uint8_t* l = io.kind == SRC_HOST_PTRS ? io.lp[first + i] : io.ls + (size_t)(first + i) * IMG;
                const uint8_t* r = io.kind == SRC_HOST_PTRS ? io.rp[first + i] : io.rs + (size_t)(first + i) * IMG;
                memcpy(ln.pin_in + (size_t)i * 2 * IMG, l, IMG);
                memcpy(ln.pin_in + (size_t)i * 2 * IMG + IMG, r, IMG);
            }
            CK(cudaMemcpyAsync(w.bgr, ln.pin_in, (size_t)nS * 2 * IMG, cudaMemcpyHostToDevice, ln.st));
            CK(cudaEventRecord(ln.ev_in_free, ln.st));
        }
        // ---- compute
        cudaStream_t rst = ln.st;   // stream on which the map becomes available
        CostSrc wave_cost = q.cost;
        if (q.cost.p)
            wave_cost.p = static_cast<const char*>(q.cost.p) + (size_t)first * N * e->P.dm.D * adc_cost_elem_bytes(q.cost.dtype);
        VolOuts wave_outs;
        wave_outs.n = q.n_vols;
        for (int i = 0; i < q.n_vols; i++) {
            wave_outs.o[i] = q.vols[i];
            wave_outs.o[i].dst = static_cast<char*>(q.vols[i].dst) + (size_t)first * N * e->P.dm.D * adc_cost_elem_bytes(q.vols[i].dtype);
        }
        MapOuts wave_maps;
        for (int i = 0; i < q.n_maps; i++)
            wave_maps.dst[q.maps[i].kind] = static_cast<char*>(q.maps[i].dst) + (size_t)first * N * map_elem_bytes(q.maps[i].kind);
        int rc = enqueue_pipeline(e, ln, nS, last, q.debug_stage >= 0, nullptr, wave_cost, wave_outs, wave_maps);
        if (rc) return rc;
        // ---- outputs (a device call without a map output gives exported volumes / side maps only)
        if (strided_copy) {
            if (io.ds)
                CK(cudaMemcpyAsync(io.ds + (size_t)first * N, w.disp_l, (size_t)nS * N * sizeof(float),
                                   on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, rst));
        } else if (io.pinned) {
            for (int i = 0; i < nS; i++)
                CK(cudaMemcpyAsync(io.dp[first + i], w.disp_l + (size_t)i * N, N * sizeof(float), cudaMemcpyDeviceToHost, rst));
        } else {
            CK(cudaMemcpyAsync(ln.pin_out, w.disp_l, (size_t)nS * N * sizeof(float), cudaMemcpyDeviceToHost, rst));
            ln.drain_n = nS; ln.drain_first = first;
            ln.drain_ptrs = io.kind == SRC_HOST_PTRS ? io.dp : nullptr;
            ln.drain_base = io.ds;
        }
        CK(cudaEventRecord(ln.ev_done, rst));
    }
    // join: the caller's stream waits for every lane -- unless the engine is in pipelined mode, where consecutive
    // batch calls flow into each other (a lane starts the next call's wave while other lanes still finish the
    // previous call's) and the caller joins once with adc_join
    const bool pageable = !io.pinned && !on_device;
    if (!e->pipelined || force_join || pageable)
        for (int li = 0; li < std::min(nl, n_waves); li++) CK(cudaStreamWaitEvent(user, e->lanes[li].ev_done, 0));
    if (pageable)
        for (auto& ln : e->lanes) { int rc = drain_lane(e, ln); if (rc) return rc; }
    return ADC_OK;
}

bool layout_known(int layout) { return layout == ADC_COST_HWD || layout == ADC_COST_DHW; }
bool dtype_known(int dtype) { return dtype == ADC_COST_F32 || dtype == ADC_COST_F16 || dtype == ADC_COST_BF16; }

// The rules of a caller's cost volume format, when the call has a volume (`have`).
int check_cost(const char* fn, bool have, int layout, int dtype) {
    if (!have) return ADC_OK;
    if (!layout_known(layout)) return fail(ADC_ERR_ARG, "%s: unknown cost_layout %d", fn, layout);
    if (!dtype_known(dtype)) return fail(ADC_ERR_ARG, "%s: unknown cost_dtype %d (not an element type)", fn, dtype);
    return ADC_OK;
}

// The rules every request array shares (volumes, side maps, reprojection outputs): n in lo..hi, the array not NULL,
// each request's `key` field (named key_name) in 0..n_keys-1 and not repeated; `more` checks the rest of request i.
template <typename Req, typename More>
int check_requests(const char* fn, const char* what, const Req* reqs, int n, int lo, int hi, int32_t Req::*key,
                   const char* key_name, int n_keys, More more) {
    if (n < lo || n > hi) return fail(ADC_ERR_ARG, "%s: n_%s %d outside %d..%d", fn, what, n, lo, hi);
    if (n > 0 && !reqs) return fail(ADC_ERR_ARG, "%s: %s is NULL with n_%s %d", fn, what, what, n);
    for (int i = 0; i < n; i++) {
        const int k = reqs[i].*key;
        if (k < 0 || k >= n_keys) return fail(ADC_ERR_ARG, "%s: %s[%d].%s %d unknown", fn, what, i, key_name, k);
        for (int j = 0; j < i; j++)
            if (reqs[j].*key == k) return fail(ADC_ERR_ARG, "%s: %s[%d].%s %d requested twice", fn, what, i, key_name, k);
        const int rc = more(reqs[i], i);
        if (rc) return rc;
    }
    return ADC_OK;
}

// The rules of a volume request array.  `device`: the destinations are the caller's device buffers, written by the
// export kernel directly, and must be aligned to their element size.  `what`: the array's name in the entry point's
// signature ("outs" / "vols").
int check_volumes(const char* fn, const char* what, const adc_volume_out* vols, int n, bool device) {
    return check_requests(fn, what, vols, n, 0, 3, &adc_volume_out::stage, "stage", 3, [&](const adc_volume_out& o, int i) -> int {
        if (!layout_known(o.layout)) return fail(ADC_ERR_ARG, "%s: %s[%d].layout %d unknown", fn, what, i, o.layout);
        if (!dtype_known(o.dtype)) return fail(ADC_ERR_ARG, "%s: %s[%d].dtype %d unknown", fn, what, i, o.dtype);
        if (o.reserved != 0) return fail(ADC_ERR_ARG, "%s: %s[%d].reserved must be zero", fn, what, i);
        if (!o.dst) return fail(ADC_ERR_ARG, "%s: %s[%d].dst is NULL", fn, what, i);
        if (device && (uintptr_t)o.dst % adc_cost_elem_bytes(o.dtype))
            return fail(ADC_ERR_ARG, "%s: %s[%d].dst is not aligned to its element size", fn, what, i);
        return ADC_OK;
    });
}

// The argument rules of adc_match_volumes*, checked before any device work: the volume requests, then some output,
// then the cost format.
int check_volume_args(const char* fn, const adc_volume_out* outs, int n_outs, bool have_disp, bool have_cost,
                      int cost_layout, int cost_dtype, bool device) {
    int rc = check_volumes(fn, "outs", outs, n_outs, device);
    if (rc) return rc;
    if (n_outs == 0 && !have_disp) return fail(ADC_ERR_ARG, "%s: disp is NULL and no volume is requested (n_outs 0)", fn);
    return check_cost(fn, have_cost, cost_layout, cost_dtype);
}

// The argument rules of adc_match_outputs*, images* and rectified*: the volume requests, the cost format, the map
// requests, then some output.  `device`: f32 map destinations are written by kernels and device copies directly and
// must be 4-byte aligned.
int check_output_args(const char* fn, const adc_volume_out* vols, int n_vols, const adc_map_out* maps, int n_maps,
                      bool have_disp, bool have_cost, int cost_layout, int cost_dtype, bool device) {
    int rc = check_volumes(fn, "vols", vols, n_vols, device);
    if (rc || (rc = check_cost(fn, have_cost, cost_layout, cost_dtype))) return rc;
    rc = check_requests(fn, "maps", maps, n_maps, 0, 5, &adc_map_out::kind, "kind", 5, [&](const adc_map_out& m, int i) -> int {
        if (m.reserved != 0) return fail(ADC_ERR_ARG, "%s: maps[%d].reserved must be zero", fn, i);
        if (!m.dst) return fail(ADC_ERR_ARG, "%s: maps[%d].dst is NULL", fn, i);
        if (device && (uintptr_t)m.dst % map_elem_bytes(m.kind))
            return fail(ADC_ERR_ARG, "%s: maps[%d].dst is not 4-byte aligned", fn, i);
        return ADC_OK;
    });
    if (rc) return rc;
    if (!have_disp && n_vols == 0 && n_maps == 0)
        return fail(ADC_ERR_ARG, "%s: disp is NULL and no volume or map is requested (n_vols 0, n_maps 0)", fn);
    return ADC_OK;
}

// The request of the entries with outputs, from their arguments (checked).
MatchReq output_req(const void* cost, int cost_layout, int cost_dtype, const float* disp, const adc_volume_out* vols,
                    int n_vols, const adc_map_out* maps, int n_maps) {
    MatchReq q;
    q.cost = CostSrc{cost, cost_layout, cost_dtype};
    q.vols = vols;
    q.n_vols = n_vols;
    q.maps = maps;
    q.n_maps = n_maps;
    q.final_map = disp != nullptr;
    return q;
}

// The rules of an image descriptor that need no image size (adc_match_images*, checked before the engine).
int check_image_desc(const char* fn, const adc_image_desc* img) {
    if (!img) return ADC_OK;
    switch (img_code_error(img->format)) {
        case 1: return fail(ADC_ERR_ARG, "%s: img->format %d unknown", fn, img->format);
        case 2: return fail(ADC_ERR_ARG, "%s: img->format %d: ADC_IMG_YUV_BT709 and ADC_IMG_YUV_FULL_RANGE apply to the "
                            "YUV formats only", fn, img->format);
    }
    if (img->reserved != 0) return fail(ADC_ERR_ARG, "%s: img->reserved must be zero", fn);
    if (img->row_pitch < 0) return fail(ADC_ERR_ARG, "%s: img->row_pitch %lld is negative", fn, (long long)img->row_pitch);
    if (img->plane_pitch < 0) return fail(ADC_ERR_ARG, "%s: img->plane_pitch %lld is negative", fn, (long long)img->plane_pitch);
    if (img->image_stride < 0) return fail(ADC_ERR_ARG, "%s: img->image_stride %lld is negative", fn, (long long)img->image_stride);
    if (img_planes(img->format) == 1 && img->plane_pitch != 0)
        return fail(ADC_ERR_ARG, "%s: img->plane_pitch must be 0 for a format other than ADC_IMG_RGB_PLANAR and the 4:2:0 "
                    "YUV formats", fn);
    if (img_yuv_planar(img->format) && img->row_pitch % 2)
        return fail(ADC_ERR_ARG, "%s: img->row_pitch %lld must be even for I420 / YV12 (the chroma pitch is row_pitch / 2)",
                    fn, (long long)img->row_pitch);
    return ADC_OK;
}

// The rule the device entries add for the formats with one sample per 16-bit word (img_words), whose words the kernels
// load whole: both bases, the row pitch, the plane pitch (P016's chroma plane) and the image stride are even.  Needs no
// image size.
int check_image_align(const char* fn, const adc_image_desc* img, const void* left, const void* right) {
    if (!img || !img_words(img->format)) return ADC_OK;
    if ((uintptr_t)left % 2) return fail(ADC_ERR_ARG, "%s: d_left must be 2-byte aligned for a 16-bit format", fn);
    if ((uintptr_t)right % 2) return fail(ADC_ERR_ARG, "%s: d_right must be 2-byte aligned for a 16-bit format", fn);
    if (img->row_pitch % 2) return fail(ADC_ERR_ARG, "%s: img->row_pitch %lld must be even for a 16-bit format", fn, (long long)img->row_pitch);
    if (img->plane_pitch % 2) return fail(ADC_ERR_ARG, "%s: img->plane_pitch %lld must be even for a 16-bit format", fn, (long long)img->plane_pitch);
    if (img->image_stride % 2) return fail(ADC_ERR_ARG, "%s: img->image_stride %lld must be even for a 16-bit format", fn, (long long)img->image_stride);
    return ADC_OK;
}

// The size-dependent rules of an image descriptor (NULL = tight packed BGR) for n pairs of views of w x h pixels (the
// engine's size, or the raw frame size of the rectified entries); `g` receives the geometry with every zero default
// replaced.
int resolve_image(const char* fn, int w, int h, const adc_image_desc* img, int n, AdcImageGeom* g) {
    const adc_image_desc d = img ? *img : adc_image_desc{};
    const long long H = h, min_row = img_row_pitch(d.format, w);
    g->format = d.format;
    g->row_pitch = d.row_pitch ? (long long)d.row_pitch : min_row;
    if (g->row_pitch < min_row)
        return fail(ADC_ERR_ARG, "%s: img->row_pitch %lld is less than %s (%lld)", fn, g->row_pitch, img_row_rule(d.format),
                    min_row);
    long long foot = 0;
    if (__builtin_mul_overflow(H, g->row_pitch, &foot)) return fail(ADC_ERR_ARG, "%s: img->row_pitch %lld is too large", fn, g->row_pitch);
    g->plane_pitch = 0;
    if (img_planes(d.format) > 1) {
        g->plane_pitch = d.plane_pitch ? (long long)d.plane_pitch : foot;
        if (g->plane_pitch < foot)
            return fail(ADC_ERR_ARG, "%s: img->plane_pitch %lld is less than H * row_pitch (%lld)", fn, g->plane_pitch, foot);
        if (!img_footprint(d.format, H, g->row_pitch, g->plane_pitch, &foot))
            return fail(ADC_ERR_ARG, "%s: img->plane_pitch %lld is too large", fn, g->plane_pitch);
    }
    g->image_stride = d.image_stride ? (long long)d.image_stride : foot;
    if (g->image_stride < foot)
        return fail(ADC_ERR_ARG, "%s: img->image_stride %lld is less than the view's footprint (%lld)", fn, g->image_stride, foot);
    long long last_view = 0;
    if (n > 1 && __builtin_mul_overflow((long long)(n - 1), g->image_stride, &last_view))
        return fail(ADC_ERR_ARG, "%s: img->image_stride %lld * (n - 1) overflows", fn, g->image_stride);
    return ADC_OK;
}

// The engine's rectification (set) as the ingestion kernel takes it.
AdcRectGeom rect_geom(const adc_engine* e) {
    const uint2* m = e->rect_map;
    return AdcRectGeom{{m, m ? m + e->P.dm.N : nullptr}, e->rect_src_w, e->rect_src_h, e->rect_type};
}

// The rules the rectified entries add to the image entries' (after the engine check): a rectification is set, and
// the descriptor's size-dependent rules hold for the raw frame size.
int resolve_rectified(adc_engine* e, const char* fn, const adc_image_desc* img, int n, AdcImageGeom* g, AdcRectGeom* r) {
    if (e->rect_type < 0) return fail(ADC_ERR_ARG, "%s: no rectification is set (adc_set_rectification)", fn);
    int rc = resolve_image(fn, e->rect_src_w, e->rect_src_h, img, n, g);
    if (rc) return rc;
    *r = rect_geom(e);
    return ADC_OK;
}

// Lays out the device staging of a one-pair host call (e->vol_stage): `carve` takes the call's parts from a Carver, first
// to size them, then to point them into the staging, which is freed and re-allocated when it is smaller (ADC_ERR_NOMEM
// if that fails).  With ADC_DBG_POISON the whole staging is filled with the pattern on lane 0's stream, which every
// caller (a one-pair host call) works on.
template <typename Carve>
int grow_stage(adc_engine* e, const char* fn, const char* what, Carve carve) {
    Carver sizing(nullptr);
    carve(sizing);
    const size_t need = sizing.off;
    if (need > e->vol_stage_bytes) {
        if (e->vol_stage) CK(cudaFree(e->vol_stage));
        e->vol_stage = nullptr;
        e->vol_stage_bytes = 0;
        if (cudaMalloc(&e->vol_stage, need) != cudaSuccess) {
            cudaGetLastError();
            e->vol_stage = nullptr;
            return fail(ADC_ERR_NOMEM, "%s: device staging of %zu bytes for %s", fn, need, what);
        }
        e->vol_stage_bytes = need;
    }
    if (poisoned(e) && e->vol_stage) CK(cudaMemsetAsync(e->vol_stage, poison_byte(e), e->vol_stage_bytes, e->lanes[0].st));
    Carver parts(e->vol_stage);
    carve(parts);
    return ADC_OK;
}

// The prologue of the one-pair host calls, which all run on lane 0: sets the engine's device, finishes the lane's
// pending copy-out and waits for its stream.
int idle_lane0(adc_engine* e) {
    CK(cudaSetDevice(e->cfg.device));
    int rc = drain_lane(e, e->lanes[0]);
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->lanes[0].st));
    return ADC_OK;
}

// The tight geometry of a view of `format`: over the raw frames of `rect`, or the engine's size without one.
AdcImageGeom tight_view(const adc_engine* e, int format, const AdcRectGeom* rect) {
    return rect ? adc_image_tight(format, rect->src_w, rect->src_h) : adc_image_tight(format, e->W, e->H);
}

// One pair's host views (geometry g, resolved) -> `bgr` as packed BGR [2][N*3] on st: the views are uploaded tightly,
// view after view, to `raw` (2 * the tight footprint) and converted from there by ingest_views.
int ingest_host_pair(adc_engine* e, const AdcImageGeom& g, const AdcRectGeom* rect, const uint8_t* left,
                     const uint8_t* right, uint8_t* raw, uint8_t* bgr, cudaStream_t st) {
    const size_t sh = rect ? rect->src_h : e->H;
    const AdcImageGeom tight = tight_view(e, g.format, rect);
    const size_t foot = (size_t)tight.image_stride, tp = (size_t)tight.row_pitch;
    // one block of tight rows per plane
    for (int v = 0; v < 2; v++)
        for (int c = 0; c < img_planes(g.format); c++) {
            const size_t ctp = (size_t)img_plane_row_pitch(g.format, c, (long long)tp);
            CK(cudaMemcpy2DAsync(raw + v * foot + img_plane_offset(g.format, c, sh, tight.row_pitch, tight.plane_pitch), ctp,
                                 (v ? right : left) + img_plane_offset(g.format, c, sh, g.row_pitch, g.plane_pitch),
                                 (size_t)img_plane_row_pitch(g.format, c, g.row_pitch), ctp,
                                 (size_t)img_plane_rows(g.format, c, sh), cudaMemcpyHostToDevice, st));
        }
    ingest_views(e, 1, raw, raw + foot, tight, rect, bgr, st);
    return ADC_OK;
}

// One pair's host inputs of request q -> lane ln, for a run that stops after `last`.  Packed BGR rows (raw ==
// nullptr) are gathered into the pinned ring and copied into ln.w.bgr at once.  Other formats and raw frames are
// uploaded tightly, view after view, to `raw` and converted from there by the (rectified) ingestion kernel.  A host
// cost volume goes into the lane volume that stage 1 does not write, where `src` then points.  `start` (optional) is
// recorded before the first copy.
int upload_pair(adc_engine* e, Lane& ln, const MatchReq& q, const uint8_t* left, const uint8_t* right, uint8_t* raw,
                int last, cudaEvent_t start, CostSrc* src) {
    const size_t W = (size_t)e->W, H = (size_t)e->H, IMG = W * H * 3;
    if (!raw) {
        const size_t pitch = q.img ? (size_t)q.img->row_pitch : 3 * W;
        for (int v = 0; v < 2; v++) {
            const uint8_t* s = v ? right : left;
            if (pitch == 3 * W) memcpy(ln.pin_in + v * IMG, s, IMG);
            else for (size_t y = 0; y < H; y++) memcpy(ln.pin_in + v * IMG + y * 3 * W, s + y * pitch, 3 * W);
        }
    }
    if (start) CK(cudaEventRecord(start, ln.st));
    if (!raw) {
        CK(cudaMemcpyAsync(ln.w.bgr, ln.pin_in, 2 * IMG, cudaMemcpyHostToDevice, ln.st));
    } else {
        int rc = ingest_host_pair(e, *q.img, q.rect, left, right, raw, ln.w.bgr, ln.st);
        if (rc) return rc;
    }
    if (q.cost.p) {
        float* staging = lane_volumes(e, ln.w, last).other;
        CK(cudaMemcpyAsync(staging, q.cost.p, W * H * e->P.dm.D * adc_cost_elem_bytes(q.cost.dtype), cudaMemcpyHostToDevice,
                           ln.st));
        *src = q.cost;
        src->p = staging;
    }
    return ADC_OK;
}

// The one-pair host driver: runs request q for the views at left / right on lane 0 and hands every output to the
// caller.  Exported volumes and maps go to the device staging first, one after the other, and so do raw frames that do
// not fit in the lane volume that stage 1 writes.  With a final map (disp) the stage times are taken.
int match_host(adc_engine* e, const char* fn, const MatchReq& q, const uint8_t* left, const uint8_t* right, float* disp) {
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (!left || !right) return fail(ADC_ERR_ARG, "%s: NULL image", fn);
    int rc = idle_lane0(e);
    if (rc) return rc;
    Lane& ln = e->lanes[0];
    note_formats(e, q);
    const int last = last_stage(q);
    const size_t N = (size_t)e->P.dm.N, ND = N * e->P.dm.D;
    const bool ingest = needs_ingest(e, q, true);
    const size_t raw_bytes = ingest ? 2 * (size_t)tight_view(e, q.img->format, q.rect).image_stride : 0;
    const bool raw_in_volume = raw_bytes <= (size_t)e->S * e->P.dm.vol_stride * sizeof(float);
    VolOuts dev;
    dev.n = q.n_vols;
    MapOuts dev_maps;
    uint8_t* raw = ingest && raw_in_volume ? reinterpret_cast<uint8_t*>(lane_volumes(e, ln.w, last).c0) : nullptr;
    rc = grow_stage(e, fn, "the exported volumes and maps", [&](Carver& c) {
        for (int i = 0; i < q.n_vols; i++) {
            dev.o[i] = q.vols[i];
            dev.o[i].dst = c.take<char>(ND * adc_cost_elem_bytes(q.vols[i].dtype));
        }
        for (int i = 0; i < q.n_maps; i++) dev_maps.dst[q.maps[i].kind] = c.take<char>(N * map_elem_bytes(q.maps[i].kind));
        if (!raw_in_volume) raw = c.take<uint8_t>(raw_bytes);
    });
    if (rc) return rc;
    if (poisoned(e) && (rc = fill_arena(e, ln))) return rc;
    cudaEvent_t* ev = disp ? e->ev_stage : nullptr;
    CostSrc src;
    if ((rc = upload_pair(e, ln, q, left, right, raw, last, ev ? ev[0] : nullptr, &src))) return rc;
    if ((rc = enqueue_pipeline(e, ln, 1, last, q.debug_stage >= 0, ev, src, dev, dev_maps))) return rc;
    if (disp) {
        CK(cudaMemcpyAsync(ln.pin_out, ln.w.disp_l, N * sizeof(float), cudaMemcpyDeviceToHost, ln.st));
        CK(cudaEventRecord(ev[6], ln.st));
        CK(cudaMemcpyAsync(e->pin_disp_r, ln.w.disp_r, N * sizeof(float), cudaMemcpyDeviceToHost, ln.st));
    }
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    if (disp) {
        memcpy(disp, ln.pin_out, N * sizeof(float));
        for (int i = 0; i < 6; i++) CK(cudaEventElapsedTime(&e->stage_ms[i], ev[i], ev[i + 1]));
    }
    for (int i = 0; i < q.n_vols; i++)
        CK(cudaMemcpy(q.vols[i].dst, dev.o[i].dst, ND * adc_cost_elem_bytes(q.vols[i].dtype), cudaMemcpyDeviceToHost));
    for (int i = 0; i < q.n_maps; i++)
        CK(cudaMemcpy(q.maps[i].dst, dev_maps.dst[q.maps[i].kind], N * map_elem_bytes(q.maps[i].kind), cudaMemcpyDeviceToHost));
    return ADC_OK;
}

// The device batch driver: runs request q for n pairs of strided device views, enqueued on `stream`.
int match_device(adc_engine* e, const char* fn, int n, const uint8_t* d_left, const uint8_t* d_right, float* d_disp,
                 const MatchReq& q, void* stream) {
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (n < 0 || (n > 0 && (!d_left || !d_right || (q.final_map && !d_disp)))) return fail(ADC_ERR_ARG, "%s: bad arguments", fn);
    if (n == 0) return ADC_OK;
    CK(cudaSetDevice(e->cfg.device));
    return run_batch(e, n, BatchIO{SRC_DEVICE_STRIDED, true, d_left, d_right, d_disp}, q, (cudaStream_t)stream, false);
}

// Reprojection outputs by kind (ADC_REPROJ_*), nullptr = not requested.
struct ReprojOuts {
    void* dst[3] = {nullptr, nullptr, nullptr};
};
size_t reproj_elem_bytes(int kind) { return kind == ADC_REPROJ_POINTS ? 3 * sizeof(float) : kind == ADC_REPROJ_DEPTH ? sizeof(float) : sizeof(int16_t); }

// The rules of the reprojection entries, none of which needs the engine (device: the alignment rules too).
int check_reproject_args(const char* fn, int n, const float* disp, const double* Q, const adc_reproject_out* outs,
                         int n_outs, bool device, ReprojOuts* by_kind) {
    int rc = check_requests(fn, "outs", outs, n_outs, 1, 3, &adc_reproject_out::kind, "kind", 3,
                            [&](const adc_reproject_out& o, int i) -> int {
        if (!o.dst) return fail(ADC_ERR_ARG, "%s: outs[%d].dst is NULL", fn, i);
        if (o.reserved != 0) return fail(ADC_ERR_ARG, "%s: outs[%d].reserved must be zero", fn, i);
        const uintptr_t align = o.kind == ADC_REPROJ_DISP_S16 ? 2 : 4;
        if (device && (uintptr_t)o.dst % align)
            return fail(ADC_ERR_ARG, "%s: outs[%d].dst is not %d-byte aligned", fn, i, (int)align);
        by_kind->dst[o.kind] = o.dst;
        return ADC_OK;
    });
    if (rc) return rc;
    if (!disp) return fail(ADC_ERR_ARG, "%s: disp is NULL", fn);
    if (!Q) return fail(ADC_ERR_ARG, "%s: Q is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (device && (uintptr_t)disp % 4) return fail(ADC_ERR_ARG, "%s: disp is not 4-byte aligned", fn);
    return ADC_OK;
}

AdcReprojQ reproj_q(const double* Q) {
    AdcReprojQ q;
    memcpy(q.q, Q, sizeof(q.q));
    return q;
}

// Reprojects n maps at device address disp into the device outputs `o` on st.  A +inf pixel's DISP_S16 value is
// (min_disparity - 1) * 16 saturated to int16.
int reproject_enqueue(adc_engine* e, long long n, const float* disp, const double* Q, const ReprojOuts& o, cudaStream_t st) {
    const long long s16_invalid = std::min(32767ll, std::max(-32768ll, ((long long)e->opt.min_disparity - 1) * 16));
    adc_launch_reproject(e->P.dm, n, disp, reproj_q(Q), static_cast<float*>(o.dst[ADC_REPROJ_POINTS]),
                         static_cast<float*>(o.dst[ADC_REPROJ_DEPTH]), static_cast<int16_t*>(o.dst[ADC_REPROJ_DISP_S16]),
                         (int16_t)s16_invalid, st, &e->launches);
    CK(cudaGetLastError());
    return ADC_OK;
}

// cvRound on x86 (cvtsd2si): round half to even, INT_MIN for NaN and for anything outside int32.
int cv_round(double v) {
    const double r = nearbyint(v);
    return r >= -2147483648.0 && r <= 2147483647.0 ? (int)r : INT32_MIN;
}

// The largest float not above v (v not NaN): (double)f <= v  <=>  f <= this, for every float f.
float float_at_most(double v) {
    if (v >= (double)FLT_MAX) return v == INFINITY ? INFINITY : FLT_MAX;
    if (v < -(double)FLT_MAX) return -INFINITY;
    const float f = (float)v;
    return (double)f > v ? nextafterf(f, -INFINITY) : f;
}

size_t speckle_elem_bytes(int type) { return type == ADC_SPECKLE_S16 ? sizeof(int16_t) : sizeof(float); }

// The rules of the speckle entries that need no engine (device: the alignment rules too).
int check_speckle_args(const char* fn, int n, const void* maps, const adc_speckle_params* p, const void* work,
                       bool device) {
    if (!p) return fail(ADC_ERR_ARG, "%s: params is NULL", fn);
    if (p->type != ADC_SPECKLE_S16 && p->type != ADC_SPECKLE_F32)
        return fail(ADC_ERR_ARG, "%s: params.type %d unknown", fn, p->type);
    if (p->reserved != 0) return fail(ADC_ERR_ARG, "%s: params.reserved must be zero", fn);
    if (p->type == ADC_SPECKLE_F32 && std::isnan(p->max_diff))
        return fail(ADC_ERR_ARG, "%s: params.max_diff is NaN (F32 maps take a number)", fn);
    if (!maps) return fail(ADC_ERR_ARG, "%s: map is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (device) {
        const int a = (int)speckle_elem_bytes(p->type);
        if ((uintptr_t)maps % a) return fail(ADC_ERR_ARG, "%s: maps are not %d-byte aligned", fn, a);
        if ((uintptr_t)work % 4) return fail(ADC_ERR_ARG, "%s: work is not 4-byte aligned", fn);
    }
    return ADC_OK;
}

// Filters n maps at device address maps in place on st, with the workspace at device address work.
int speckles_enqueue(adc_engine* e, long long n, void* maps, void* work, const adc_speckle_params& p, cudaStream_t st) {
    AdcSpeckle s;
    s.nv_i = cv_round(p.new_val);
    s.md_i = cv_round(p.max_diff);
    s.nv_f = (float)p.new_val;
    s.md_f = p.type == ADC_SPECKLE_F32 ? float_at_most(p.max_diff) : 0.0f;
    s.max_size = p.max_size;
    adc_launch_speckles(e->P.dm, n, p.type == ADC_SPECKLE_F32, maps, work, s, st, &e->launches);
    CK(cudaGetLastError());
    return ADC_OK;
}

size_t speckle_work_bytes(const adc_engine* e, long long n) { return 8 * (size_t)n * (size_t)e->P.dm.N; }

// The rules of the view entries that need no engine: the image entries' rules on img, then rectified and views.
int check_views_args(const char* fn, const adc_image_desc* img, int rectified, const void* views, bool device,
                     const void* left, const void* right) {
    int rc = check_image_desc(fn, img);
    if (rc || (device && (rc = check_image_align(fn, img, left, right)))) return rc;
    if (rectified != 0 && rectified != 1) return fail(ADC_ERR_ARG, "%s: rectified %d is not 0 or 1", fn, rectified);
    if (!views) return fail(ADC_ERR_ARG, "%s: views is NULL", fn);
    return ADC_OK;
}

// The rules of the view entries after the engine check: the size-dependent rules of img against the engine's size
// (plain) or the raw frame size (rectified, which needs a rectification set).
int resolve_views(adc_engine* e, const char* fn, const adc_image_desc* img, int rectified, int n, AdcImageGeom* g,
                  AdcRectGeom* r) {
    return rectified ? resolve_rectified(e, fn, img, n, g, r) : resolve_image(fn, e->W, e->H, img, n, g);
}

// The rules of the point-cloud entries that need no engine (device: the alignment rules too).
int check_cloud_args(const char* fn, int n, const float* disp, const double* Q, const uint8_t* bgr, long long bgr_stride,
                     float z_min, float z_max, const adc_cloud_out* o, const void* work, bool device) {
    if (!o) return fail(ADC_ERR_ARG, "%s: out is NULL", fn);
    if (!o->points) return fail(ADC_ERR_ARG, "%s: out->points is NULL", fn);
    if (!o->counts) return fail(ADC_ERR_ARG, "%s: out->counts is NULL", fn);
    if (!disp) return fail(ADC_ERR_ARG, "%s: disp is NULL", fn);
    if (!Q) return fail(ADC_ERR_ARG, "%s: Q is NULL", fn);
    if (!o->colors != !bgr)
        return fail(ADC_ERR_ARG, "%s: out->colors is %s but bgr is %s (colours need an image, an image needs colours)", fn,
                    o->colors ? "given" : "NULL", bgr ? "given" : "NULL");
    if (o->capacity < 1) return fail(ADC_ERR_ARG, "%s: out->capacity %lld is below 1", fn, (long long)o->capacity);
    if (o->reserved != 0) return fail(ADC_ERR_ARG, "%s: out->reserved must be zero", fn);
    if (std::isnan(z_min)) return fail(ADC_ERR_ARG, "%s: z_min is NaN", fn);
    if (std::isnan(z_max)) return fail(ADC_ERR_ARG, "%s: z_max is NaN", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (bgr_stride < 0) return fail(ADC_ERR_ARG, "%s: bgr_stride %lld is negative", fn, bgr_stride);
    if (device) {
        if ((uintptr_t)disp % 4) return fail(ADC_ERR_ARG, "%s: disp is not 4-byte aligned", fn);
        if ((uintptr_t)o->points % 4) return fail(ADC_ERR_ARG, "%s: out->points is not 4-byte aligned", fn);
        if ((uintptr_t)o->pixels % 4) return fail(ADC_ERR_ARG, "%s: out->pixels is not 4-byte aligned", fn);
        if ((uintptr_t)o->counts % 4) return fail(ADC_ERR_ARG, "%s: out->counts is not 4-byte aligned", fn);
        if ((uintptr_t)work % 8) return fail(ADC_ERR_ARG, "%s: work is not 8-byte aligned", fn);
    }
    return ADC_OK;
}

int check_cloud_capacity(const adc_engine* e, const char* fn, const adc_cloud_out* o) {
    if (o->capacity > e->P.dm.N)
        return fail(ADC_ERR_ARG, "%s: out->capacity %lld is above H * W (%d)", fn, (long long)o->capacity, e->P.dm.N);
    return ADC_OK;
}

// The point clouds of n maps at device address disp into the device outputs `o` on st: zeroes the workspace `work`,
// then one launch.  bgr_stride 0 = tight images (3 * N bytes apart).
int cloud_enqueue(adc_engine* e, long long n, const float* disp, const double* Q, const uint8_t* bgr, long long bgr_stride,
                  float z_min, float z_max, const adc_cloud_out& o, void* work, cudaStream_t st) {
    CK(cudaMemsetAsync(work, 0, adc_point_cloud_work_bytes(e->P.dm, n), st));
    adc_launch_point_cloud(e->P.dm, n, disp, reproj_q(Q), bgr, bgr_stride ? bgr_stride : 3ll * e->P.dm.N, z_min, z_max,
                           AdcCloudOut{o.points, o.colors, o.pixels, o.counts, (long long)o.capacity}, work, st,
                           &e->launches);
    CK(cudaGetLastError());
    return ADC_OK;
}

// The output formats of the previews.
bool preview_format(int f) {
    switch (f) {
        case ADC_IMG_BGR: case ADC_IMG_BGRA: case ADC_IMG_RGBA: case ADC_IMG_GRAY:
        case ADC_IMG_NV12: case ADC_IMG_NV21: case ADC_IMG_I420: case ADC_IMG_YV12: return true;
        default: return false;
    }
}

// The rules of the preview entries that need no engine (device: the alignment rules too).
int check_preview_args(const char* fn, int n, const float* maps, const adc_preview_params* p, const void* dst,
                       const adc_image_desc* desc, const void* work, bool device) {
    if (!p) return fail(ADC_ERR_ARG, "%s: p is NULL", fn);
    if (p->colormap < ADC_COLORMAP_NONE || p->colormap >= ADC_COLORMAP_COUNT)
        return fail(ADC_ERR_ARG, "%s: p->colormap %d unknown (ADC_COLORMAP_NONE or 0..%d)", fn, p->colormap,
                    ADC_COLORMAP_COUNT - 1);
    if (p->range != ADC_PREVIEW_MINMAX && p->range != ADC_PREVIEW_FIXED)
        return fail(ADC_ERR_ARG, "%s: p->range %d unknown", fn, p->range);
    if (!std::isfinite(p->alpha)) return fail(ADC_ERR_ARG, "%s: p->alpha is not finite", fn);
    if (!std::isfinite(p->beta)) return fail(ADC_ERR_ARG, "%s: p->beta is not finite", fn);
    if (p->range == ADC_PREVIEW_MINMAX && (p->alpha != 0 || p->beta != 0))
        return fail(ADC_ERR_ARG, "%s: p->alpha and p->beta must be 0 with ADC_PREVIEW_MINMAX", fn);
    for (int i = 0; i < 5; i++)
        if (p->reserved_[i]) return fail(ADC_ERR_ARG, "%s: p->reserved_ must be zero", fn);
    if (p->reserved != 0) return fail(ADC_ERR_ARG, "%s: p->reserved must be zero", fn);
    const int format = desc ? desc->format : ADC_IMG_BGR;
    if (!preview_format(format))
        return fail(ADC_ERR_ARG, "%s: dst->format %d is not a preview format (BGR, BGRA, RGBA, GRAY, NV12, NV21, I420, "
                    "YV12, without flags)", fn, format);
    const bool yuv = img_yuv420(format);
    if (p->dst_width < 0 || p->dst_width > 32767)
        return fail(ADC_ERR_ARG, "%s: p->dst_width %d outside 0..32767", fn, p->dst_width);
    if (p->dst_height < 0 || p->dst_height > 32767)
        return fail(ADC_ERR_ARG, "%s: p->dst_height %d outside 0..32767", fn, p->dst_height);
    if (yuv && p->dst_width % 2) return fail(ADC_ERR_ARG, "%s: p->dst_width %d must be even for a 4:2:0 format", fn, p->dst_width);
    if (yuv && p->dst_height % 2) return fail(ADC_ERR_ARG, "%s: p->dst_height %d must be even for a 4:2:0 format", fn, p->dst_height);
    int rc = check_image_desc(fn, desc);
    if (rc) return rc;
    if (!maps) return fail(ADC_ERR_ARG, "%s: maps is NULL", fn);
    if (!dst) return fail(ADC_ERR_ARG, "%s: dst is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (device && (uintptr_t)maps % 4) return fail(ADC_ERR_ARG, "%s: maps are not 4-byte aligned", fn);
    if (device && (uintptr_t)work % 4) return fail(ADC_ERR_ARG, "%s: work is not 4-byte aligned", fn);
    return ADC_OK;
}

// The rules of the preview entries after the engine check: the frame size (0 = the engine's; even for 4:2:0) and the
// descriptor's size-dependent rules for n frames.  `a` receives everything but the pointers.
int resolve_preview(const adc_engine* e, const char* fn, int n, const adc_preview_params* p, const adc_image_desc* desc,
                    AdcPreviewArgs* a) {
    const int w = p->dst_width ? p->dst_width : e->W, h = p->dst_height ? p->dst_height : e->H;
    const int format = desc ? desc->format : ADC_IMG_BGR;
    if (img_yuv420(format) && (w % 2 || h % 2))
        return fail(ADC_ERR_ARG, "%s: the frame size %d x %d (0 = the engine's) must be even for a 4:2:0 format", fn, w, h);
    adc_image_desc d = desc ? *desc : adc_image_desc{};
    AdcImageGeom g;
    int rc = resolve_image(fn, w, h, &d, std::max(n, 1), &g);
    if (rc) return rc;
    *a = AdcPreviewArgs{};
    a->row_pitch = g.row_pitch;
    a->plane_pitch = g.plane_pitch;
    a->image_stride = g.image_stride;
    a->inv_x = 1.0 / ((double)w / e->W);
    a->inv_y = 1.0 / ((double)h / e->H);
    a->alpha = (float)p->alpha;
    a->beta = (float)p->beta;
    a->format = format;
    a->colormap = p->colormap;
    a->dst_w = w;
    a->dst_h = h;
    memcpy(a->invalid, p->invalid_bgr, 3);
    return ADC_OK;
}

size_t preview_work_bytes(long long n) { return 8 * (size_t)n; }

// Renders n maps at device address maps into the frames at dst on st; work (MINMAX) is zeroed first.
int preview_enqueue(adc_engine* e, long long n, const float* maps, AdcPreviewArgs a, bool minmax, void* dst, void* work,
                    cudaStream_t st) {
    a.dst = static_cast<uint8_t*>(dst);
    a.work = minmax ? static_cast<unsigned*>(work) : nullptr;
    if (minmax) CK(cudaMemsetAsync(work, 0, preview_work_bytes(n), st));
    adc_launch_preview(e->P.dm, n, maps, a, st, &e->launches);
    CK(cudaGetLastError());
    return ADC_OK;
}

}  // namespace

// =============================================================================================
extern "C" {

const char* adc_last_error(void) { return g_err.c_str(); }
const char* adc_version(void) { return "adcensus_b200 0.1 (sm_90a)"; }

void adc_default_option(adc_option* o) {
    if (!o) return;
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

void adc_destroy(adc_engine* e) {
    if (!e) return;
    cudaSetDevice(e->cfg.device);
    cudaDeviceSynchronize();
    for (auto& ln : e->lanes) {
        if (ln.arena) cudaFree(ln.arena);
        if (ln.pin_in) cudaFreeHost(ln.pin_in);
        if (ln.pin_out) cudaFreeHost(ln.pin_out);
        if (ln.ev_done) cudaEventDestroy(ln.ev_done);
        if (ln.ev_in_free) cudaEventDestroy(ln.ev_in_free);
        if (ln.st) cudaStreamDestroy(ln.st);
    }
    if (e->d_lut_ad) cudaFree(e->d_lut_ad);
    if (e->d_lut_cen) cudaFree(e->d_lut_cen);
    if (e->d_rays) cudaFree(e->d_rays);
    if (e->d_ray_off) cudaFree(e->d_ray_off);
    if (e->vol_stage) cudaFree(e->vol_stage);
    if (e->rect_map) cudaFree(e->rect_map);
    if (e->pin_disp_r) cudaFreeHost(e->pin_disp_r);
    if (e->ev_fork) cudaEventDestroy(e->ev_fork);
    for (auto& ev : e->ev_stage) if (ev) cudaEventDestroy(ev);
    if (e->main_st) cudaStreamDestroy(e->main_st);
    delete e;
}

int adc_create(int32_t width, int32_t height, const adc_option* opt, const adc_config* cfg, adc_engine** out) {
    if (!out) return fail(ADC_ERR_ARG, "adc_create: out is NULL");
    *out = nullptr;
    if (!opt) return fail(ADC_ERR_ARG, "adc_create: option is NULL");
    if (width <= 0 || height <= 0) return fail(ADC_ERR_ARG, "adc_create: non-positive image size %dx%d", width, height);
    const long long dmin = opt->min_disparity, dmax = opt->max_disparity;
    if (dmax - dmin <= 0)
        return fail(ADC_ERR_ARG, "adc_create: empty disparity range [%d,%d)", opt->min_disparity, opt->max_disparity);
    // The option domain (include/adcensus_b200.h, adc_option): values for which the reference's arithmetic is undefined
    // or leaves its cost volume non-finite.  All in 64 bits, before any device work.
    if (dmax - dmin > INT32_MAX || dmin == INT32_MIN || dmax == INT32_MIN)
        return fail(ADC_ERR_ARG, "adc_create: min_disparity %d / max_disparity %d: max - min or abs() overflows int32",
                    opt->min_disparity, opt->max_disparity);
    if ((width - 1) - dmin > INT32_MAX || (width - 1) + (dmax - 1) > INT32_MAX)
        return fail(ADC_ERR_ARG, "adc_create: min_disparity %d / max_disparity %d: a candidate column x - d or x + d "
                    "overflows int32 at width %d", opt->min_disparity, opt->max_disparity, width);
    if (opt->lambda_ad < 1) return fail(ADC_ERR_ARG, "adc_create: lambda_ad %d < 1", opt->lambda_ad);
    if (opt->lambda_census < 1) return fail(ADC_ERR_ARG, "adc_create: lambda_census %d < 1", opt->lambda_census);
    if (!std::isfinite(opt->so_p1) || opt->so_p1 < 0)
        return fail(ADC_ERR_ARG, "adc_create: so_p1 %g is negative or not finite", (double)opt->so_p1);
    if (!std::isfinite(opt->so_p2) || opt->so_p2 < 0)
        return fail(ADC_ERR_ARG, "adc_create: so_p2 %g is negative or not finite", (double)opt->so_p2);
    // Limits of the kernels (the reference has none; INTEGRATION.md lists them).  They are checked HERE, so that a caller
    // never sees Initialize() succeed and Match() fail for a size: whatever adc_create accepts, adc_match runs.
    const int drange = (int)(dmax - dmin);
    if ((long long)width * height > (1ll << 28)) return fail(ADC_ERR_UNSUPPORTED, "adc_create: image too large (more than 2^28 pixels)");
    if (drange > ADC_MAX_DISPARITY_RANGE)
        return fail(ADC_ERR_UNSUPPORTED, "adc_create: disparity range %d > %d is not supported (scanline kernel: 8 disparities per lane)", drange, ADC_MAX_DISPARITY_RANGE);
    if (height > ADC_MAX_HEIGHT)
        return fail(ADC_ERR_UNSUPPORTED, "adc_create: image height %d > %d is not supported (in-place median: one CTA per image)", height, ADC_MAX_HEIGHT);
    if (width > ADC_MAX_WIDTH || width + drange > ADC_MAX_WIDTH)
        return fail(ADC_ERR_UNSUPPORTED, "adc_create: image width %d (+ disparity range %d) > %d is not supported (widest size the kernels are validated for)", width, drange, ADC_MAX_WIDTH);

    adc_engine* e = new adc_engine();
    e->W = width; e->H = height; e->opt = *opt;
    if (cfg) e->cfg = *cfg;
    build_params(e);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        delete e;
        return fail(ADC_ERR_CUDA, "adc_create: no CUDA device available (this library has no CPU fallback)");
    }
    if (e->cfg.device < 0 || e->cfg.device >= ndev) { delete e; return fail(ADC_ERR_ARG, "adc_create: bad device ordinal"); }
    auto bail = [&](int rc) { adc_destroy(e); return rc; };
    if (cudaSetDevice(e->cfg.device) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "cudaSetDevice failed"));

    // wave size: enough scanlines in flight for the line-per-lane-group scanline kernels (32 pairs per wave
    // x 4 lanes for Cone: the scanline passes only have W or H lines per pair to spread over the SMs)
    int S = e->cfg.wave_pairs;
    if (S <= 0) S = std::min(32, std::max(2, (12288 + std::min(width, height) - 1) / std::min(width, height)));
    int nl = e->cfg.lanes > 0 ? e->cfg.lanes : 4;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "cudaMemGetInfo failed"));
    while (true) {
        const size_t need = carve_lane(nullptr, e->P.dm, e->P.L1, S, nullptr) * nl;
        if (need < free_b * 8 / 10) break;
        if (nl > 1) nl--; else if (S > 1) S--; else return bail(fail(ADC_ERR_NOMEM, "adc_create: one pair does not fit in device memory"));
    }
    e->S = S;
    e->cfg.wave_pairs = S; e->cfg.lanes = nl;
    e->agg_fused = !(e->cfg.debug_flags & ADC_DBG_UNFUSED_AGG);

    int rc = upload_tables(e);
    if (rc) return bail(rc);
    if (cudaStreamCreateWithFlags(&e->main_st, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "stream create failed"));
    if (cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "event create failed"));
    for (auto& ev : e->ev_stage) if (cudaEventCreate(&ev) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "event create failed"));
    e->lanes.resize(nl);
    const size_t N = (size_t)e->P.dm.N;
    for (auto& ln : e->lanes) {
        if (cudaStreamCreateWithFlags(&ln.st, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "stream create failed"));
        if (cudaEventCreateWithFlags(&ln.ev_done, cudaEventDisableTiming) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "event create failed"));
        if (cudaEventCreateWithFlags(&ln.ev_in_free, cudaEventDisableTiming) != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "event create failed"));
        const size_t bytes = carve_lane(nullptr, e->P.dm, e->P.L1, S, nullptr);
        if (cudaMalloc(&ln.arena, bytes) != cudaSuccess) { cudaGetLastError(); return bail(fail(ADC_ERR_NOMEM, "device arena of %zu bytes", bytes)); }
        carve_lane(ln.arena, e->P.dm, e->P.L1, S, &ln.w);
        if (!adc_arm_tmaps_encode(e->P, S, ln.w.volA, ln.w.volB, &ln.arm_tm))
            return bail(fail(ADC_ERR_CUDA, "adc_create: the aggregation passes' tensor maps could not be encoded (cuTensorMapEncodeTiled)"));
        ln.w.arm_tm = &ln.arm_tm;
        if (!adc_so_tmaps_encode(e->P, S, ln.w.volA, ln.w.volB, ln.w.so_rec, &ln.so_tm))
            return bail(fail(ADC_ERR_CUDA, "adc_create: the scanline passes' tensor maps could not be encoded (cuTensorMapEncodeTiled)"));
        ln.w.so_tm = &ln.so_tm;
        if ((rc = fill_arena(e, ln))) return bail(rc);
        if (cudaHostAlloc((void**)&ln.pin_in, (size_t)S * 2 * N * 3, cudaHostAllocDefault) != cudaSuccess ||
            cudaHostAlloc((void**)&ln.pin_out, (size_t)S * N * sizeof(float), cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return bail(fail(ADC_ERR_NOMEM, "pinned staging allocation failed"));
        }
    }
    if (cudaHostAlloc((void**)&e->pin_disp_r, N * sizeof(float), cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return bail(fail(ADC_ERR_NOMEM, "pinned staging allocation failed"));
    }
    memset(e->pin_disp_r, 0, N * sizeof(float));
    if (cudaDeviceSynchronize() != cudaSuccess) return bail(fail(ADC_ERR_CUDA, "device sync failed: %s", cudaGetErrorString(cudaGetLastError())));
    *out = e;
    return ADC_OK;
}

int adc_match(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, float* disp_left) {
    if (!e) return fail(ADC_ERR_ARG, "adc_match: engine is NULL (Match before Initialize)");
    if (!img_left || !img_right || !disp_left) return fail(ADC_ERR_ARG, "adc_match: NULL image or output pointer");
    return match_host(e, "adc_match", MatchReq(), img_left, img_right, disp_left);
}

int adc_match_cost(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, const void* cost, int32_t layout,
                   int32_t dtype, float* disp_left) {
    const char* fn = "adc_match_cost";
    int rc = check_cost(fn, true, layout, dtype);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (!img_left || !img_right || !cost || !disp_left) return fail(ADC_ERR_ARG, "%s: NULL image, cost or output pointer", fn);
    MatchReq q;
    q.cost = CostSrc{cost, layout, dtype};
    return match_host(e, fn, q, img_left, img_right, disp_left);
}

int adc_get_right_disparity(adc_engine* e, float* disp_right) {
    if (!e || !disp_right) return fail(ADC_ERR_ARG, "adc_get_right_disparity: bad arguments");
    memcpy(disp_right, e->pin_disp_r, (size_t)e->P.dm.N * sizeof(float));   // complete: match_host synchronised
    return ADC_OK;
}

int adc_match_batch(adc_engine* e, int32_t n, const uint8_t* const* img_left, const uint8_t* const* img_right,
                    float* const* disp_left) {
    if (!e) return fail(ADC_ERR_ARG, "adc_match_batch: engine is NULL");
    if (n < 0 || (n > 0 && (!img_left || !img_right || !disp_left))) return fail(ADC_ERR_ARG, "adc_match_batch: bad arguments");
    if (n == 0) return ADC_OK;
    bool pinned = true;
    for (int i = 0; i < n; i++) {
        if (!img_left[i] || !img_right[i] || !disp_left[i]) return fail(ADC_ERR_ARG, "adc_match_batch: NULL pointer for pair %d", i);
    }
    CK(cudaSetDevice(e->cfg.device));
    for (int i = 0; i < n && pinned; i++) pinned = is_pinned(img_left[i]) && is_pinned(img_right[i]) && is_pinned(disp_left[i]);
    const BatchIO io{SRC_HOST_PTRS, pinned, nullptr, nullptr, nullptr, img_left, img_right, disp_left};
    int rc = run_batch(e, n, io, MatchReq(), e->main_st, true);
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->main_st));
    return ADC_OK;
}

int adc_match_batch_strided(adc_engine* e, int32_t n, const uint8_t* left, const uint8_t* right, float* disp) {
    if (!e) return fail(ADC_ERR_ARG, "adc_match_batch_strided: engine is NULL");
    if (n < 0 || (n > 0 && (!left || !right || !disp))) return fail(ADC_ERR_ARG, "adc_match_batch_strided: bad arguments");
    if (n == 0) return ADC_OK;
    CK(cudaSetDevice(e->cfg.device));
    const bool pinned = is_pinned(left) && is_pinned(right) && is_pinned(disp);
    int rc = run_batch(e, n, BatchIO{SRC_HOST_STRIDED, pinned, left, right, disp}, MatchReq(), e->main_st, true);
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->main_st));
    return ADC_OK;
}

int adc_match_batch_pinned_async(adc_engine* e, int32_t n, const uint8_t* left, const uint8_t* right, float* disp, void* stream) {
    if (!e) return fail(ADC_ERR_ARG, "adc_match_batch_pinned_async: engine is NULL");
    if (n < 0 || (n > 0 && (!left || !right || !disp))) return fail(ADC_ERR_ARG, "adc_match_batch_pinned_async: bad arguments");
    if (n == 0) return ADC_OK;
    CK(cudaSetDevice(e->cfg.device));
    if (!(is_pinned(left) && is_pinned(right) && is_pinned(disp)))
        return fail(ADC_ERR_ARG, "adc_match_batch_pinned_async: buffers must be pinned host memory");
    return run_batch(e, n, BatchIO{SRC_HOST_STRIDED, true, left, right, disp}, MatchReq(), (cudaStream_t)stream, false);
}

int adc_match_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right, float* d_disp, void* stream) {
    return match_device(e, "adc_match_batch_device", n, d_left, d_right, d_disp, MatchReq(), stream);
}

int adc_match_cost_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right, const void* d_cost,
                                int32_t layout, int32_t dtype, float* d_disp, void* stream) {
    const char* fn = "adc_match_cost_batch_device";
    int rc = check_cost(fn, true, layout, dtype);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (n < 0 || (n > 0 && (!d_left || !d_right || !d_cost || !d_disp))) return fail(ADC_ERR_ARG, "%s: bad arguments", fn);
    MatchReq q;
    q.cost = CostSrc{d_cost, layout, dtype};
    return match_device(e, fn, n, d_left, d_right, d_disp, q, stream);
}

int adc_match_volumes_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right, const void* d_cost,
                                   int32_t cost_layout, int32_t cost_dtype, float* d_disp, const adc_volume_out* outs,
                                   int32_t n_outs, void* stream) {
    const char* fn = "adc_match_volumes_batch_device";
    int rc = check_volume_args(fn, outs, n_outs, d_disp != nullptr, d_cost != nullptr, cost_layout, cost_dtype, true);
    if (rc) return rc;
    return match_device(e, fn, n, d_left, d_right, d_disp,
                        output_req(d_cost, cost_layout, cost_dtype, d_disp, outs, n_outs, nullptr, 0), stream);
}

int adc_match_volumes(adc_engine* e, const uint8_t* left, const uint8_t* right, const void* cost, int32_t cost_layout,
                      int32_t cost_dtype, float* disp, const adc_volume_out* outs, int32_t n_outs) {
    const char* fn = "adc_match_volumes";
    int rc = check_volume_args(fn, outs, n_outs, disp != nullptr, cost != nullptr, cost_layout, cost_dtype, false);
    if (rc) return rc;
    return match_host(e, fn, output_req(cost, cost_layout, cost_dtype, disp, outs, n_outs, nullptr, 0), left, right, disp);
}

int adc_match_outputs_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right, const void* d_cost,
                                   int32_t cost_layout, int32_t cost_dtype, float* d_disp, const adc_volume_out* vols,
                                   int32_t n_vols, const adc_map_out* maps, int32_t n_maps, void* stream) {
    const char* fn = "adc_match_outputs_batch_device";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, d_disp != nullptr, d_cost != nullptr, cost_layout, cost_dtype, true);
    if (rc) return rc;
    return match_device(e, fn, n, d_left, d_right, d_disp,
                        output_req(d_cost, cost_layout, cost_dtype, d_disp, vols, n_vols, maps, n_maps), stream);
}

int adc_match_outputs(adc_engine* e, const uint8_t* left, const uint8_t* right, const void* cost, int32_t cost_layout,
                      int32_t cost_dtype, float* disp, const adc_volume_out* vols, int32_t n_vols, const adc_map_out* maps,
                      int32_t n_maps) {
    const char* fn = "adc_match_outputs";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, disp != nullptr, cost != nullptr, cost_layout, cost_dtype, false);
    if (rc) return rc;
    return match_host(e, fn, output_req(cost, cost_layout, cost_dtype, disp, vols, n_vols, maps, n_maps), left, right, disp);
}

int adc_match_images_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                  const adc_image_desc* img, const void* d_cost, int32_t cost_layout, int32_t cost_dtype,
                                  float* d_disp, const adc_volume_out* vols, int32_t n_vols, const adc_map_out* maps,
                                  int32_t n_maps, void* stream) {
    const char* fn = "adc_match_images_batch_device";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, d_disp != nullptr, d_cost != nullptr, cost_layout, cost_dtype, true);
    if (rc || (rc = check_image_desc(fn, img)) || (rc = check_image_align(fn, img, d_left, d_right))) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcImageGeom g;
    if ((rc = resolve_image(fn, e->W, e->H, img, n, &g))) return rc;
    MatchReq q = output_req(d_cost, cost_layout, cost_dtype, d_disp, vols, n_vols, maps, n_maps);
    q.img = &g;
    return match_device(e, fn, n, d_left, d_right, d_disp, q, stream);
}

int adc_match_images(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img, const void* cost,
                     int32_t cost_layout, int32_t cost_dtype, float* disp, const adc_volume_out* vols, int32_t n_vols,
                     const adc_map_out* maps, int32_t n_maps) {
    const char* fn = "adc_match_images";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, disp != nullptr, cost != nullptr, cost_layout, cost_dtype, false);
    if (rc || (rc = check_image_desc(fn, img))) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcImageGeom g;
    if ((rc = resolve_image(fn, e->W, e->H, img, 1, &g))) return rc;
    MatchReq q = output_req(cost, cost_layout, cost_dtype, disp, vols, n_vols, maps, n_maps);
    q.img = &g;
    return match_host(e, fn, q, left, right, disp);
}

int adc_set_rectification(adc_engine* e, const adc_rectification* r) {
    const char* fn = "adc_set_rectification";
    const bool f32 = r && r->map_type == ADC_REMAP_F32;
    const bool resize = r && adc_is_resize(r->map_type);   // no maps: nothing to copy or convert
    const long long e1 = 4, e2 = f32 ? 4 : 2;   // bytes per element of map1 (float, int16 pair) and map2 (float, uint16)
    if (r) {
        if (r->src_width < 1 || r->src_width > 32767) return fail(ADC_ERR_ARG, "%s: r->src_width %d outside 1..32767", fn, r->src_width);
        if (r->src_height < 1 || r->src_height > 32767) return fail(ADC_ERR_ARG, "%s: r->src_height %d outside 1..32767", fn, r->src_height);
        if (r->map_type != ADC_REMAP_F32 && r->map_type != ADC_REMAP_FIXED && !resize)
            return fail(ADC_ERR_ARG, "%s: r->map_type %d unknown", fn, r->map_type);
        if (r->reserved != 0) return fail(ADC_ERR_ARG, "%s: r->reserved must be zero", fn);
        for (int v = 0; v < 2 && resize; v++) {
            const adc_remap& m = r->view[v];
            if (m.map1) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1 must be NULL for a resize", fn, v);
            if (m.map2) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2 must be NULL for a resize", fn, v);
            if (m.map1_pitch) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1_pitch must be 0 for a resize", fn, v);
            if (m.map2_pitch) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2_pitch must be 0 for a resize", fn, v);
        }
        for (int v = 0; v < 2 && !resize; v++) {
            const adc_remap& m = r->view[v];
            if (!m.map1) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1 is NULL", fn, v);
            if (!m.map2) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2 is NULL", fn, v);
            if (m.map1_pitch < 0) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1_pitch %lld is negative", fn, v, (long long)m.map1_pitch);
            if (m.map2_pitch < 0) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2_pitch %lld is negative", fn, v, (long long)m.map2_pitch);
            if ((uintptr_t)m.map1 % (f32 ? 4 : 2) || m.map1_pitch % (f32 ? 4 : 2))
                return fail(ADC_ERR_ARG, "%s: r->view[%d].map1 or map1_pitch is not aligned to its element", fn, v);
            if ((uintptr_t)m.map2 % e2 || m.map2_pitch % e2)
                return fail(ADC_ERR_ARG, "%s: r->view[%d].map2 or map2_pitch is not aligned to its element", fn, v);
        }
    }
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    const long long W = e->W, H = e->H;
    if (r && r->map_type == ADC_RESIZE_AREA) {
        const long long kx = r->src_width / W, ky = r->src_height / H;
        if (r->src_width < W || r->src_width % W)
            return fail(ADC_ERR_ARG, "%s: r->src_width %d is not a multiple of W (%lld) for ADC_RESIZE_AREA", fn,
                        r->src_width, W);
        if (r->src_height < H || r->src_height % H)
            return fail(ADC_ERR_ARG, "%s: r->src_height %d is not a multiple of H (%lld) for ADC_RESIZE_AREA", fn,
                        r->src_height, H);
        // cv::resize takes the integer-block rule only where its scale 1 / (W / src_width), in double, is the factor
        // exactly; for 640 of the factors 1..4096 it is not, and OpenCV's general area path rounds differently
        if (1.0 / ((double)W / r->src_width) != (double)kx)
            return fail(ADC_ERR_ARG, "%s: r->src_width %d: the factor %lld is not exact in double (1 / (W / src_width)) "
                        "for ADC_RESIZE_AREA", fn, r->src_width, kx);
        if (1.0 / ((double)H / r->src_height) != (double)ky)
            return fail(ADC_ERR_ARG, "%s: r->src_height %d: the factor %lld is not exact in double "
                        "(1 / (H / src_height)) for ADC_RESIZE_AREA", fn, r->src_height, ky);
        if (kx * ky > 4096)
            return fail(ADC_ERR_ARG, "%s: r->src_width %d / W times r->src_height %d / H is more than 4096 for "
                        "ADC_RESIZE_AREA", fn, r->src_width, r->src_height);
    }
    long long p1[2] = {0, 0}, p2[2] = {0, 0};
    if (r && !resize) {
        for (int v = 0; v < 2; v++) {
            const adc_remap& m = r->view[v];
            p1[v] = m.map1_pitch ? (long long)m.map1_pitch : W * e1;
            p2[v] = m.map2_pitch ? (long long)m.map2_pitch : W * e2;
            long long foot = 0;
            if (p1[v] < W * e1) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1_pitch %lld is less than a row (%lld bytes)", fn, v, p1[v], W * e1);
            if (p2[v] < W * e2) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2_pitch %lld is less than a row (%lld bytes)", fn, v, p2[v], W * e2);
            if (__builtin_mul_overflow(H, p1[v], &foot)) return fail(ADC_ERR_ARG, "%s: r->view[%d].map1_pitch %lld is too large", fn, v, p1[v]);
            if (__builtin_mul_overflow(H, p2[v], &foot)) return fail(ADC_ERR_ARG, "%s: r->view[%d].map2_pitch %lld is too large", fn, v, p2[v]);
        }
    }
    CK(cudaSetDevice(e->cfg.device));
    const size_t N = (size_t)e->P.dm.N;
    uint2* maps = nullptr;
    void* tmp = nullptr;
    bool host[2][2] = {};
    if (r && !resize) {
        bool any_host = false;
        for (int v = 0; v < 2; v++)
            for (int k = 0; k < 2; k++) {
                cudaPointerAttributes at{};
                const void* p = k ? r->view[v].map2 : r->view[v].map1;
                if (cudaPointerGetAttributes(&at, p) != cudaSuccess) cudaGetLastError();
                host[v][k] = at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged;
                any_host |= host[v][k];
            }
        // the maps in the internal form, and (host maps) device staging of one view's tight maps
        if (cudaMalloc(&maps, 2 * N * sizeof(uint2)) != cudaSuccess ||
            (any_host && cudaMalloc(&tmp, N * (size_t)(e1 + e2)) != cudaSuccess)) {
            cudaGetLastError();
            if (maps) cudaFree(maps);
            return fail(ADC_ERR_NOMEM, "%s: device memory for the maps (%zu bytes)", fn, 2 * N * sizeof(uint2) + N * (size_t)(e1 + e2));
        }
    }
    // join the engine's outstanding work (and whatever work of the caller's wrote device maps)
    cudaError_t err = cudaDeviceSynchronize();
    for (int v = 0; r && !resize && v < 2 && err == cudaSuccess; v++) {
        const adc_remap& m = r->view[v];
        const void* s1 = m.map1;
        const void* s2 = m.map2;
        long long q1 = p1[v], q2 = p2[v];
        uint8_t* t = static_cast<uint8_t*>(tmp);
        if (host[v][0] && err == cudaSuccess) {
            err = cudaMemcpy2DAsync(t, W * e1, s1, q1, W * e1, H, cudaMemcpyDefault, e->main_st);
            s1 = t, q1 = W * e1;
        }
        if (host[v][1] && err == cudaSuccess) {
            err = cudaMemcpy2DAsync(t + N * e1, W * e2, s2, q2, W * e2, H, cudaMemcpyDefault, e->main_st);
            s2 = t + N * e1, q2 = W * e2;
        }
        if (err == cudaSuccess) {
            adc_launch_remap_convert(e->P.dm, r->map_type, s1, q1, s2, q2, maps + v * N, e->main_st);
            err = cudaGetLastError();
        }
        if (err == cudaSuccess) err = cudaStreamSynchronize(e->main_st);   // the staging is reused by the next view
    }
    if (tmp) cudaFree(tmp);
    if (err != cudaSuccess) {
        if (maps) cudaFree(maps);
        return fail(ADC_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(err));
    }
    if (e->rect_map) CK(cudaFree(e->rect_map));
    e->rect_map = maps;
    e->rect_type = r ? r->map_type : -1;
    e->rect_src_w = r ? r->src_width : 0;
    e->rect_src_h = r ? r->src_height : 0;
    return ADC_OK;
}

int adc_match_rectified_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                     const adc_image_desc* img, const void* d_cost, int32_t cost_layout,
                                     int32_t cost_dtype, float* d_disp, const adc_volume_out* vols, int32_t n_vols,
                                     const adc_map_out* maps, int32_t n_maps, void* stream) {
    const char* fn = "adc_match_rectified_batch_device";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, d_disp != nullptr, d_cost != nullptr, cost_layout, cost_dtype, true);
    if (rc || (rc = check_image_desc(fn, img)) || (rc = check_image_align(fn, img, d_left, d_right))) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcImageGeom g;
    AdcRectGeom r;
    if ((rc = resolve_rectified(e, fn, img, n, &g, &r))) return rc;
    MatchReq q = output_req(d_cost, cost_layout, cost_dtype, d_disp, vols, n_vols, maps, n_maps);
    q.img = &g;
    q.rect = &r;
    return match_device(e, fn, n, d_left, d_right, d_disp, q, stream);
}

int adc_match_rectified(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img, const void* cost,
                        int32_t cost_layout, int32_t cost_dtype, float* disp, const adc_volume_out* vols, int32_t n_vols,
                        const adc_map_out* maps, int32_t n_maps) {
    const char* fn = "adc_match_rectified";
    int rc = check_output_args(fn, vols, n_vols, maps, n_maps, disp != nullptr, cost != nullptr, cost_layout, cost_dtype, false);
    if (rc || (rc = check_image_desc(fn, img))) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcImageGeom g;
    AdcRectGeom r;
    if ((rc = resolve_rectified(e, fn, img, 1, &g, &r))) return rc;
    MatchReq q = output_req(cost, cost_layout, cost_dtype, disp, vols, n_vols, maps, n_maps);
    q.img = &g;
    q.rect = &r;
    return match_host(e, fn, q, left, right, disp);
}

int adc_reproject_batch_device(adc_engine* e, int32_t n, const float* d_disp, const double Q[16],
                               const adc_reproject_out* outs, int32_t n_outs, void* stream) {
    const char* fn = "adc_reproject_batch_device";
    ReprojOuts o;
    int rc = check_reproject_args(fn, n, d_disp, Q, outs, n_outs, true, &o);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (n == 0) return ADC_OK;
    CK(cudaSetDevice(e->cfg.device));
    return reproject_enqueue(e, n, d_disp, Q, o, (cudaStream_t)stream);
}

int adc_reproject(adc_engine* e, const float* disp, const double Q[16], const adc_reproject_out* outs, int32_t n_outs) {
    const char* fn = "adc_reproject";
    ReprojOuts o;
    int rc = check_reproject_args(fn, 1, disp, Q, outs, n_outs, false, &o);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if ((rc = idle_lane0(e))) return rc;
    Lane& ln = e->lanes[0];
    const size_t N = (size_t)e->P.dm.N;
    float* d_disp = nullptr;
    ReprojOuts d;
    rc = grow_stage(e, fn, "the disparity map and its reprojection", [&](Carver& c) {
        d_disp = c.take<float>(N);
        for (int k = 0; k < 3; k++) d.dst[k] = o.dst[k] ? c.take<char>(N * reproj_elem_bytes(k)) : nullptr;
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_disp, disp, N * sizeof(float), cudaMemcpyHostToDevice, ln.st));
    if ((rc = reproject_enqueue(e, 1, d_disp, Q, d, ln.st))) return rc;
    for (int k = 0; k < 3; k++)
        if (o.dst[k]) CK(cudaMemcpyAsync(o.dst[k], d.dst[k], N * reproj_elem_bytes(k), cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    return ADC_OK;
}

int adc_speckle_workspace_bytes(const adc_engine* e, int32_t n, size_t* out) {
    const char* fn = "adc_speckle_workspace_bytes";
    if (!out) return fail(ADC_ERR_ARG, "%s: out is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    *out = speckle_work_bytes(e, n);
    return ADC_OK;
}

int adc_filter_speckles_batch_device(adc_engine* e, int32_t n, void* d_maps, const adc_speckle_params* params,
                                     void* d_work, size_t work_bytes, void* stream) {
    const char* fn = "adc_filter_speckles_batch_device";
    int rc = check_speckle_args(fn, n, d_maps, params, d_work, true);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    const size_t need = speckle_work_bytes(e, n);
    if (work_bytes < need) return fail(ADC_ERR_ARG, "%s: work_bytes %zu below the %zu bytes of %d maps", fn, work_bytes, need, n);
    if (n == 0) return ADC_OK;
    if (!d_work) return fail(ADC_ERR_ARG, "%s: work is NULL", fn);
    CK(cudaSetDevice(e->cfg.device));
    return speckles_enqueue(e, n, d_maps, d_work, *params, (cudaStream_t)stream);
}

int adc_filter_speckles(adc_engine* e, void* map, const adc_speckle_params* params) {
    const char* fn = "adc_filter_speckles";
    int rc = check_speckle_args(fn, 1, map, params, nullptr, false);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if ((rc = idle_lane0(e))) return rc;
    Lane& ln = e->lanes[0];
    const size_t bytes = (size_t)e->P.dm.N * speckle_elem_bytes(params->type);
    char *work = nullptr, *d_map = nullptr;
    rc = grow_stage(e, fn, "the map and its speckle workspace", [&](Carver& c) {
        work = c.take<char>(speckle_work_bytes(e, 1));
        d_map = c.take<char>(bytes);
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_map, map, bytes, cudaMemcpyHostToDevice, ln.st));
    if ((rc = speckles_enqueue(e, 1, d_map, work, *params, ln.st))) return rc;
    CK(cudaMemcpyAsync(map, d_map, bytes, cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    return ADC_OK;
}

int adc_ingest_views_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                  const adc_image_desc* img, int32_t rectified, uint8_t* d_views, void* stream) {
    const char* fn = "adc_ingest_views_batch_device";
    int rc = check_views_args(fn, img, rectified, d_views, true, d_left, d_right);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (n > 0 && (!d_left || !d_right)) return fail(ADC_ERR_ARG, "%s: NULL image", fn);
    AdcImageGeom g;
    AdcRectGeom r;
    if ((rc = resolve_views(e, fn, img, rectified, n, &g, &r))) return rc;
    if (n == 0) return ADC_OK;
    CK(cudaSetDevice(e->cfg.device));
    ingest_views(e, n, d_left, d_right, g, rectified ? &r : nullptr, d_views, (cudaStream_t)stream);
    CK(cudaGetLastError());
    return ADC_OK;
}

int adc_ingest_views(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img,
                     int32_t rectified, uint8_t* views) {
    const char* fn = "adc_ingest_views";
    int rc = check_views_args(fn, img, rectified, views, false, left, right);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (!left || !right) return fail(ADC_ERR_ARG, "%s: NULL image", fn);
    AdcImageGeom g;
    AdcRectGeom r;
    if ((rc = resolve_views(e, fn, img, rectified, 1, &g, &r))) return rc;
    if ((rc = idle_lane0(e))) return rc;
    Lane& ln = e->lanes[0];
    const AdcRectGeom* rect = rectified ? &r : nullptr;
    const size_t out_bytes = 6 * (size_t)e->P.dm.N;
    uint8_t *d_views = nullptr, *raw = nullptr;
    rc = grow_stage(e, fn, "the raw views and the packed BGR views", [&](Carver& c) {
        d_views = c.take<uint8_t>(out_bytes);
        raw = c.take<uint8_t>(2 * (size_t)tight_view(e, g.format, rect).image_stride);
    });
    if (rc || (rc = ingest_host_pair(e, g, rect, left, right, raw, d_views, ln.st))) return rc;
    CK(cudaMemcpyAsync(views, d_views, out_bytes, cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    return ADC_OK;
}

int adc_point_cloud_workspace_bytes(const adc_engine* e, int32_t n, size_t* out) {
    const char* fn = "adc_point_cloud_workspace_bytes";
    if (!out) return fail(ADC_ERR_ARG, "%s: out is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    *out = adc_point_cloud_work_bytes(e->P.dm, n);
    return ADC_OK;
}

int adc_point_cloud_batch_device(adc_engine* e, int32_t n, const float* d_disp, const double Q[16], const uint8_t* d_bgr,
                                 int64_t bgr_stride, float z_min, float z_max, const adc_cloud_out* out, void* d_work,
                                 size_t work_bytes, void* stream) {
    const char* fn = "adc_point_cloud_batch_device";
    int rc = check_cloud_args(fn, n, d_disp, Q, d_bgr, bgr_stride, z_min, z_max, out, d_work, true);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if ((rc = check_cloud_capacity(e, fn, out))) return rc;
    const size_t need = adc_point_cloud_work_bytes(e->P.dm, n);
    if (work_bytes < need) return fail(ADC_ERR_ARG, "%s: work_bytes %zu below the %zu bytes of %d maps", fn, work_bytes, need, n);
    if (n == 0) return ADC_OK;
    if (!d_work) return fail(ADC_ERR_ARG, "%s: work is NULL", fn);
    CK(cudaSetDevice(e->cfg.device));
    return cloud_enqueue(e, n, d_disp, Q, d_bgr, bgr_stride, z_min, z_max, *out, d_work, (cudaStream_t)stream);
}

int adc_point_cloud(adc_engine* e, const float* disp, const double Q[16], const uint8_t* bgr, float z_min, float z_max,
                    const adc_cloud_out* out) {
    const char* fn = "adc_point_cloud";
    int rc = check_cloud_args(fn, 1, disp, Q, bgr, 0, z_min, z_max, out, nullptr, false);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if ((rc = check_cloud_capacity(e, fn, out))) return rc;
    if ((rc = idle_lane0(e))) return rc;
    Lane& ln = e->lanes[0];
    const size_t N = (size_t)e->P.dm.N, cap = (size_t)out->capacity;
    void* work = nullptr;
    float* d_disp = nullptr;
    uint8_t* d_bgr = nullptr;
    adc_cloud_out o = *out;
    rc = grow_stage(e, fn, "the map, its image and its point cloud", [&](Carver& c) {
        work = c.take<char>(adc_point_cloud_work_bytes(e->P.dm, 1));
        d_disp = c.take<float>(N);
        d_bgr = bgr ? c.take<uint8_t>(3 * N) : nullptr;
        o.points = c.take<float>(3 * cap);
        o.colors = out->colors ? c.take<uint8_t>(3 * cap) : nullptr;
        o.pixels = out->pixels ? c.take<int32_t>(cap) : nullptr;
        o.counts = c.take<int32_t>(1);
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_disp, disp, N * sizeof(float), cudaMemcpyHostToDevice, ln.st));
    if (bgr) CK(cudaMemcpyAsync(d_bgr, bgr, 3 * N, cudaMemcpyHostToDevice, ln.st));
    if ((rc = cloud_enqueue(e, 1, d_disp, Q, d_bgr, 0, z_min, z_max, o, work, ln.st))) return rc;
    CK(cudaMemcpyAsync(out->counts, o.counts, sizeof(int32_t), cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    const size_t kept = std::min((size_t)std::max(out->counts[0], 0), cap);
    CK(cudaMemcpy(out->points, o.points, 12 * kept, cudaMemcpyDeviceToHost));
    if (out->colors) CK(cudaMemcpy(out->colors, o.colors, 3 * kept, cudaMemcpyDeviceToHost));
    if (out->pixels) CK(cudaMemcpy(out->pixels, o.pixels, 4 * kept, cudaMemcpyDeviceToHost));
    return ADC_OK;
}

int adc_preview_workspace_bytes(const adc_engine* e, int32_t n, size_t* out) {
    const char* fn = "adc_preview_workspace_bytes";
    if (!out) return fail(ADC_ERR_ARG, "%s: out is NULL", fn);
    if (n < 0) return fail(ADC_ERR_ARG, "%s: n %d is negative", fn, n);
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    *out = preview_work_bytes(n);
    return ADC_OK;
}

int adc_preview_batch_device(adc_engine* e, int32_t n, const float* d_maps, const adc_preview_params* p, void* d_dst,
                             const adc_image_desc* dst, void* d_work, size_t work_bytes, void* stream) {
    const char* fn = "adc_preview_batch_device";
    int rc = check_preview_args(fn, n, d_maps, p, d_dst, dst, d_work, true);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcPreviewArgs a;
    if ((rc = resolve_preview(e, fn, n, p, dst, &a))) return rc;
    const bool minmax = p->range == ADC_PREVIEW_MINMAX;
    if (minmax && work_bytes < preview_work_bytes(n))
        return fail(ADC_ERR_ARG, "%s: work_bytes %zu below the %zu bytes of %d maps", fn, work_bytes, preview_work_bytes(n), n);
    if (n == 0) return ADC_OK;
    if (minmax && !d_work) return fail(ADC_ERR_ARG, "%s: work is NULL", fn);
    CK(cudaSetDevice(e->cfg.device));
    return preview_enqueue(e, n, d_maps, a, minmax, d_dst, d_work, (cudaStream_t)stream);
}

int adc_preview(adc_engine* e, const float* map, const adc_preview_params* p, void* dst, const adc_image_desc* desc) {
    const char* fn = "adc_preview";
    int rc = check_preview_args(fn, 1, map, p, dst, desc, nullptr, false);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    AdcPreviewArgs a;
    if ((rc = resolve_preview(e, fn, 1, p, desc, &a))) return rc;
    if ((rc = idle_lane0(e))) return rc;
    Lane& ln = e->lanes[0];
    const size_t N = (size_t)e->P.dm.N;
    // the frame is rendered tightly into the staging, then each plane's rows are copied to the caller's pitches
    const AdcImageGeom tight = adc_image_tight(a.format, a.dst_w, a.dst_h);
    AdcPreviewArgs t = a;
    t.row_pitch = tight.row_pitch;
    t.plane_pitch = tight.plane_pitch;
    t.image_stride = tight.image_stride;
    float* d_map = nullptr;
    uint8_t* d_frame = nullptr;
    void* work = nullptr;
    rc = grow_stage(e, fn, "the map and its preview", [&](Carver& c) {
        work = c.take<unsigned>(2);
        d_map = c.take<float>(N);
        d_frame = c.take<uint8_t>((size_t)tight.image_stride);
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_map, map, N * sizeof(float), cudaMemcpyHostToDevice, ln.st));
    if ((rc = preview_enqueue(e, 1, d_map, t, p->range == ADC_PREVIEW_MINMAX, d_frame, work, ln.st))) return rc;
    const int format = a.format;
    const long long row_bytes = img_row_pitch(format, a.dst_w);
    for (int c = 0; c < img_planes(format); c++) {
        uint8_t* to = static_cast<uint8_t*>(dst) + img_plane_offset(format, c, a.dst_h, a.row_pitch, a.plane_pitch);
        const uint8_t* from = d_frame + img_plane_offset(format, c, a.dst_h, t.row_pitch, t.plane_pitch);
        CK(cudaMemcpy2DAsync(to, (size_t)img_plane_row_pitch(format, c, a.row_pitch), from,
                             (size_t)img_plane_row_pitch(format, c, t.row_pitch),
                             (size_t)img_plane_row_pitch(format, c, row_bytes), (size_t)img_plane_rows(format, c, a.dst_h),
                             cudaMemcpyDeviceToHost, ln.st));
    }
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    return ADC_OK;
}

void* adc_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void adc_host_free(void* p) { if (p) cudaFreeHost(p); }

int adc_synchronize(adc_engine* e) {
    if (!e) return fail(ADC_ERR_ARG, "adc_synchronize: engine is NULL");
    CK(cudaSetDevice(e->cfg.device));
    for (auto& ln : e->lanes) {
        CK(cudaStreamSynchronize(ln.st));
    }
    CK(cudaStreamSynchronize(e->main_st));
    return ADC_OK;
}

int adc_set_pipelined(adc_engine* e, int32_t on) {
    if (!e) return fail(ADC_ERR_ARG, "adc_set_pipelined: engine is NULL");
    e->pipelined = on != 0;
    return ADC_OK;
}

int adc_join(adc_engine* e, void* stream) {
    if (!e) return fail(ADC_ERR_ARG, "adc_join: engine is NULL");
    CK(cudaSetDevice(e->cfg.device));
    for (auto& ln : e->lanes) CK(cudaStreamWaitEvent((cudaStream_t)stream, ln.ev_done, 0));
    return ADC_OK;
}

uint64_t adc_launch_count(const adc_engine* e) { return e ? e->launches : 0; }

int adc_last_stage_ms(const adc_engine* e, float out[6]) {
    if (!e || !out) return fail(ADC_ERR_ARG, "adc_last_stage_ms: bad arguments");
    // ev_stage[0..6]: start | cost | aggregation | scanline | wta | refine | output copy
    for (int i = 0; i < 6; i++) out[i] = e->stage_ms[i];
    return ADC_OK;
}

int adc_get_config(const adc_engine* e, adc_config* out) {
    if (!e || !out) return fail(ADC_ERR_ARG, "adc_get_config: bad arguments");
    *out = e->cfg;
    return ADC_OK;
}

// ---- output side of the reference's demo (main.cpp:147-230), SURVEY.md 8(f) rank 3 ----------------------------
int adc_render_disparity(adc_engine* e, const float* disp, uint8_t* gray8, uint8_t* jet_bgr, float* min_max) {
    if (!e) return fail(ADC_ERR_ARG, "adc_render_disparity: engine is NULL");
    if (!disp || (!gray8 && !jet_bgr && !min_max)) return fail(ADC_ERR_ARG, "adc_render_disparity: NULL map or no output requested");
    int rc = idle_lane0(e);
    if (rc) return rc;
    Lane& ln = e->lanes[0];
    const size_t N = (size_t)e->P.dm.N;
    // lane 0's buffers are idle between calls: disp_t holds the map, flag the 8-bit image, bgr the colour image,
    // the first words of rowcnt the min/max keys and (as floats) the values handed back
    float* d_disp = ln.w.disp_t;
    unsigned* d_mm = reinterpret_cast<unsigned*>(ln.w.rowcnt);
    float* d_mm_out = reinterpret_cast<float*>(ln.w.rowcnt) + 2;
    if (poisoned(e) && (rc = fill_arena(e, ln))) return rc;
    CK(cudaMemcpyAsync(d_disp, disp, N * sizeof(float), cudaMemcpyHostToDevice, ln.st));
    if (adc_launch_render(e->P.dm, d_disp, d_mm, ln.w.flag, ln.w.bgr, d_mm_out, ln.st, &e->launches))
        return fail(ADC_ERR_CUDA, "adc_render_disparity: colour table upload failed");
    if (gray8) CK(cudaMemcpyAsync(gray8, ln.w.flag, N, cudaMemcpyDeviceToHost, ln.st));
    if (jet_bgr) CK(cudaMemcpyAsync(jet_bgr, ln.w.bgr, 3 * N, cudaMemcpyDeviceToHost, ln.st));
    if (min_max) CK(cudaMemcpyAsync(min_max, d_mm_out, 2 * sizeof(float), cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    CK(cudaGetLastError());
    return ADC_OK;
}

int adc_disparity_cloud(adc_engine* e, const uint8_t* img_left, const float* disp, float* cloud, int32_t* n_points) {
    if (!e) return fail(ADC_ERR_ARG, "adc_disparity_cloud: engine is NULL");
    if (!img_left || !disp || !cloud || !n_points) return fail(ADC_ERR_ARG, "adc_disparity_cloud: NULL pointer");
    int rc = idle_lane0(e);
    if (rc) return rc;
    Lane& ln = e->lanes[0];
    const size_t N = (size_t)e->P.dm.N;
    const AdcWave w1 = wave_view(e, ln, 1);
    float* d_cloud = ln.w.volA;                       // 6 floats per pixel at most; a volume has Dp >= 4 ... use both volumes' span
    if ((size_t)e->P.dm.vol_stride * 2 < N * 6) return fail(ADC_ERR_UNSUPPORTED, "adc_disparity_cloud: disparity range too small for the scratch volume");
    if (poisoned(e) && (rc = fill_arena(e, ln))) return rc;
    CK(cudaMemcpyAsync(ln.w.disp_t, disp, N * sizeof(float), cudaMemcpyHostToDevice, ln.st));
    CK(cudaMemcpyAsync(ln.w.bgr, img_left, 3 * N, cudaMemcpyHostToDevice, ln.st));
    CK(cudaMemsetAsync(ln.w.counters, 0, ADC_CNT * sizeof(int), ln.st));
    adc_launch_cloud(e->P, w1, ln.w.disp_t, ln.w.bgr, d_cloud, ln.st, &e->launches);
    int n = 0;
    CK(cudaMemcpyAsync(&n, ln.w.counters, sizeof(int), cudaMemcpyDeviceToHost, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    if (n > 0) CK(cudaMemcpy(cloud, d_cloud, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost));
    *n_points = n;
    CK(cudaGetLastError());
    return ADC_OK;
}

// ---- per-kernel timing for the roofline figures of bench.py ------------------------------------
// Re-launches ONE kernel of the pipeline `reps` times on lane 0's wave buffers (which hold whatever
// the last batch left there; every kernel below is data-oblivious in its memory traffic except for
// the arm lengths, which are real) and reports the mean device time per launch, measured with CUDA
// events on the lane's own stream, plus the algorithmic bytes one launch moves (SURVEY.md 8d model).
int adc_profile_kernel(adc_engine* e, int32_t kernel_id, int32_t reps, float* avg_ms, double* algorithmic_bytes) {
    if (!e || !avg_ms || reps <= 0) return fail(ADC_ERR_ARG, "adc_profile_kernel: bad arguments");
    CK(cudaSetDevice(e->cfg.device));
    Lane& ln = e->lanes[0];
    const AdcParams& P = e->P;
    const AdcWave w = wave_view(e, ln, e->S);
    const double V = (double)P.dm.N * P.dm.D * 4.0, N = (double)P.dm.N;
    double bytes = 0;
    CK(cudaStreamSynchronize(ln.st));
    cudaEvent_t e0 = e->ev_stage[0], e1 = e->ev_stage[1];
    for (int r = -1; r < reps; r++) {   // r = -1: warm-up launch
        if (r == 0) CK(cudaEventRecord(e0, ln.st));
        switch (kernel_id) {
            case 0: adc_launch_cost(P, w, w.volB, ln.st, &e->launches); bytes = V + 6 * N + 16 * N; break;
            case 1: adc_launch_arm_sum(P, w, w.volA, w.volB, 0, nullptr, ln.st, &e->launches); bytes = 2 * V + 4 * N; break;
            case 2: adc_launch_arm_sum(P, w, w.volA, w.volB, 1, w.sup_h, ln.st, &e->launches); bytes = 2 * V + 6 * N; break;
            case 3: if (adc_launch_scanline(P, w, w.volA, w.volB, 1, 0, ln.st, &e->launches)) return fail(ADC_ERR_UNSUPPORTED, "scanline"); bytes = 2 * V + 6 * N; break;
            case 4: if (adc_launch_scanline(P, w, w.volA, w.volB, 0, 1, ln.st, &e->launches)) return fail(ADC_ERR_UNSUPPORTED, "scanline"); bytes = 2 * V + 6 * N; break;
            case 5: if (adc_launch_wta(P, w, w.volA, ln.st, &e->launches)) return fail(ADC_ERR_UNSUPPORTED, "wta"); bytes = V + 8 * N; break;
            case 6: adc_launch_arm_sum2(P, w, w.volA, w.volB, 1, w.sup_h, ln.st, &e->launches); bytes = 2 * V + 6 * N; break;
            case 7: adc_launch_arm_sum2(P, w, w.volA, w.volB, 0, w.sup_v, ln.st, &e->launches); bytes = 2 * V + 6 * N; break;
            case 8: adc_launch_arm_sum(P, w, w.volA, w.volB, 0, w.sup_v, ln.st, &e->launches); bytes = 2 * V + 6 * N; break;
            case 9: adc_launch_arm_sum(P, w, w.volA, w.volB, 1, nullptr, ln.st, &e->launches); bytes = 2 * V + 4 * N; break;
            case 10:    // source: volA's bytes taken as the wave's raw volumes (the kernel's traffic does not depend on the values)
                adc_launch_cost_ingest(P, w, w.volA, e->cost_layout, e->cost_dtype, w.volB, ln.st, &e->launches);
                bytes = N * P.dm.D * (double)adc_cost_elem_bytes(e->cost_dtype) + N * P.dm.Dp * 4.0;
                break;
            case 11:    // volA's volumes exported into volB (N*D elements of at most 4 bytes fit in N*Dp floats)
                adc_launch_cost_export(P, w, w.volA, w.volB, e->export_layout, e->export_dtype, ln.st, &e->launches);
                bytes = N * P.dm.Dp * 4.0 + N * P.dm.D * (double)adc_cost_elem_bytes(e->export_dtype);
                break;
            case 12:    // both confidence maps of volA into volB (2*N floats of a pair fit in its N*Dp, Dp >= 4)
                adc_launch_confidence(P, w, w.volA, w.volB, w.volB + (size_t)e->S * P.dm.N, ln.st, &e->launches);
                bytes = N * P.dm.Dp * 4.0 + 2 * 4.0 * N;
                break;
            case 13: {  // volA's bytes taken as the wave's tight images (at most 2*4*N bytes a pair: they fit in its N*Dp floats)
                AdcImageGeom g = adc_image_tight(e->img_format, P.dm.W, P.dm.H);
                const long long foot = g.image_stride;
                g.image_stride = 2 * foot;
                const uint8_t* src = reinterpret_cast<const uint8_t*>(w.volA);
                ingest_views(e, w.S, src, src + foot, g, nullptr, w.bgr, ln.st);
                bytes = 2.0 * adc_image_read_bytes(e->img_format, P.dm.W, P.dm.H) + 2 * 3.0 * N;
                break;
            }
            case 14: {  // volA's bytes taken as the wave's tight raw frames, resampled through the engine's maps or resized
                if (e->rect_type < 0) return fail(ADC_ERR_ARG, "adc_profile_kernel: no rectification is set (adc_set_rectification)");
                AdcImageGeom g = adc_image_tight(e->rect_format, e->rect_src_w, e->rect_src_h);
                const long long foot = g.image_stride;
                if (2 * foot > P.dm.vol_stride * 4)
                    return fail(ADC_ERR_UNSUPPORTED, "adc_profile_kernel: a pair's raw frames (%lld bytes) exceed its share of a lane volume", 2 * foot);
                g.image_stride = 2 * foot;
                const AdcRectGeom rg = rect_geom(e);
                const uint8_t* src = reinterpret_cast<const uint8_t*>(w.volA);
                ingest_views(e, w.S, src, src + foot, g, &rg, w.bgr, ln.st);
                bytes = 2.0 * adc_image_read_bytes(e->rect_format, e->rect_src_w, e->rect_src_h) + 2 * 3.0 * N +
                        (adc_is_resize(e->rect_type) ? 0.0 : 2 * 8.0 * N / e->S);
                break;
            }
            case 15:    // the cost computed from the wave's images and census words, summed as iteration 0's H pass into volA
                if (!adc_launch_cost_arm_sum_h(P, w, w.volA, nullptr, ln.st, &e->launches))
                    return fail(ADC_ERR_UNSUPPORTED, "fused cost and horizontal arm sums not applicable");
                bytes = V + 24 * N + (double)arm_line_rec(P.dm.W, P.dm.H, 1, 0) * arm_rec_words(P.L1) * 4.0;   // + horizontal records (all before the vertical axis's first)
                break;
            case 16:    // the -y pass fused with the WTA: volA's volumes in, disp_l and the right view's records into volB
            case 17: {  // the records in volB folded into disp_r
                const long long plane = so_wta_plane(P.dm.W, P.dm.H, P.dm.D, P.dm.Dp);
                if (SO_WTA_FIELDS * plane > P.dm.vol_stride)
                    return fail(ADC_ERR_UNSUPPORTED, "adc_profile_kernel: the WTA records do not fit in a pair's volume");
                const double recs = 4.0 * SO_WTA_FIELDS * P.dm.H * (double)so_wta_row_records(P.dm.W, P.dm.D, P.dm.Dp, P.dm.dmin);
                if (kernel_id == 16) {
                    if (adc_launch_scanline_wta(P, w, w.volA, w.volB, ln.st, &e->launches)) return fail(ADC_ERR_UNSUPPORTED, "scanline");
                    bytes = V + 6 * N + recs + 4 * N;
                } else {
                    adc_launch_wta_merge(P, w, w.volB, ln.st, &e->launches);
                    bytes = recs + 4 * N;
                }
                break;
            }
            default: return fail(ADC_ERR_ARG, "adc_profile_kernel: unknown kernel id %d", kernel_id);
        }
    }
    CK(cudaEventRecord(e1, ln.st));
    CK(cudaStreamSynchronize(ln.st));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    *avg_ms = ms / reps;
    if (algorithmic_bytes) *algorithmic_bytes = bytes * e->S;
    return ADC_OK;
}

// ---- debug taps -----------------------------------------------------------------------------
int adc_debug_run(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, int32_t last_stage) {
    const char* fn = "adc_debug_run";
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (!img_left || !img_right) return fail(ADC_ERR_ARG, "%s: NULL image", fn);
    if (last_stage < 0 || last_stage >= ADC_STAGE_COUNT) return fail(ADC_ERR_ARG, "%s: bad stage", fn);
    MatchReq q;
    q.final_map = false;
    q.debug_stage = last_stage;
    return match_host(e, fn, q, img_left, img_right, nullptr);
}

int adc_debug_run_cost(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, const void* cost, int32_t layout,
                       int32_t dtype, int32_t last_stage) {
    const char* fn = "adc_debug_run_cost";
    int rc = check_cost(fn, true, layout, dtype);
    if (rc) return rc;
    if (!e) return fail(ADC_ERR_ARG, "%s: engine is NULL", fn);
    if (!img_left || !img_right || !cost) return fail(ADC_ERR_ARG, "%s: NULL image or cost", fn);
    if (last_stage < 0 || last_stage >= ADC_STAGE_COUNT) return fail(ADC_ERR_ARG, "%s: bad stage", fn);
    MatchReq q;
    q.cost = CostSrc{cost, layout, dtype};
    q.final_map = false;
    q.debug_stage = last_stage;
    return match_host(e, fn, q, img_left, img_right, nullptr);
}

int adc_debug_counters(adc_engine* e, int32_t out[16]) {
    if (!e || !out) return fail(ADC_ERR_ARG, "adc_debug_counters: bad arguments");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpy(out, e->lanes[0].w.counters, 16 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return ADC_OK;
}

size_t adc_debug_get(adc_engine* e, int32_t tap, void* dst, size_t cap) {
    if (!e) { fail(ADC_ERR_ARG, "adc_debug_get: engine is NULL"); return 0; }
    if (cudaSetDevice(e->cfg.device) != cudaSuccess) return 0;
    const AdcDims& dm = e->P.dm;
    const Lane& ln = e->lanes[0];
    const size_t N = (size_t)dm.N;
    const void* src = nullptr;
    size_t bytes = 0;
    switch (tap) {
        case ADC_TAP_GRAY_L: src = ln.w.gray; bytes = N; break;
        case ADC_TAP_GRAY_R: src = ln.w.gray + N; bytes = N; break;
        case ADC_TAP_CENSUS_L: src = ln.w.census; bytes = N * 8; break;
        case ADC_TAP_CENSUS_R: src = ln.w.census + N; bytes = N * 8; break;
        case ADC_TAP_ARMS: src = ln.w.arms; bytes = N * 4; break;
        case ADC_TAP_SUPCNT_H: src = ln.w.sup_h; bytes = N * 2; break;
        case ADC_TAP_SUPCNT_V: src = ln.w.sup_v; bytes = N * 2; break;
        case ADC_TAP_DISP_L: src = ln.w.disp_l; bytes = N * 4; break;
        case ADC_TAP_DISP_R: src = ln.w.disp_r; bytes = N * 4; break;
        case ADC_TAP_VOL_INIT:
        case ADC_TAP_VOL_AGGR: {
            const float* v = tap == ADC_TAP_VOL_INIT ? e->dbg_init : e->dbg_aggr;
            bytes = N * dm.D * sizeof(float);
            if (dst && cap >= bytes && !v) {
                if (tap == ADC_TAP_VOL_AGGR && e->dbg_so_wta)
                    fail(ADC_ERR_ARG, "adc_debug_get: no such volume: the last run's final scanline pass took the WTA as its "
                                      "epilogue (fused scanline + WTA) and stored no optimised volume");
                else
                    fail(ADC_ERR_ARG, "adc_debug_get: no such volume: no run yet, or the last run computed the cost inside the aggregation");
                return 0;
            }
            if (!dst || cap < bytes || !v) return bytes;
            // strip the Dp padding: [N][Dp] -> [N][D]
            if (cudaMemcpy2D(dst, (size_t)dm.D * 4, v, (size_t)dm.Dp * 4, (size_t)dm.D * 4, N, cudaMemcpyDeviceToHost) != cudaSuccess) {
                fail(ADC_ERR_CUDA, "adc_debug_get: copy failed: %s", cudaGetErrorString(cudaGetLastError()));
                return 0;
            }
            return bytes;
        }
        case ADC_TAP_MISMATCHES:
        case ADC_TAP_OCCLUSIONS: {
            // the lists are the pixels labelled 1 / 2, in raster order (the reference builds them by a
            // raster scan and only ever erases from them)
            std::vector<uint8_t> lab(N);
            if (cudaMemcpy(lab.data(), ln.w.label, N, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
            const uint8_t want = tap == ADC_TAP_MISMATCHES ? 1 : 2;
            size_t cnt = 0;
            for (size_t i = 0; i < N; i++) cnt += lab[i] == want;
            bytes = cnt * 8;
            if (!dst || cap < bytes) return bytes;
            int32_t* o = static_cast<int32_t*>(dst);
            for (size_t i = 0; i < N; i++)
                if (lab[i] == want) { *o++ = (int32_t)(i % dm.W); *o++ = (int32_t)(i / dm.W); }
            return bytes;
        }
        default: fail(ADC_ERR_ARG, "adc_debug_get: unknown tap %d", tap); return 0;
    }
    if (!dst || cap < bytes) return bytes;
    if (cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) {
        fail(ADC_ERR_CUDA, "adc_debug_get: copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        return 0;
    }
    return bytes;
}

}  // extern "C"
