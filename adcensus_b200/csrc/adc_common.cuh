// adc_common.cuh -- shared declarations for the sm_90a AD-Census kernels.
//
// Data layout in HBM (per wave of S stereo pairs; every array is [S][...], pair index outermost):
//   bgr      u8  [S][2][H][W][3]   left, right packed BGR: copied as the caller passes them, or written by the view
//                                  ingestion kernel (k_image.cuh) from another format, pitch or source geometry
//   gray     u8  [S][2][H][W]
//   census   u64 [S][2][H][W]
//   volA/B   f32 [S][H][W][Dp]     the two cost volumes, d fastest, Dp = D rounded up to 4 so that
//                                  every pixel's disparity vector is a whole number of 128-bit words
//   arms     u8x4[S][H][W]         left,right,top,bottom (cross_aggregator.h:17-20)
//   sup_h/v  u16 [S][H][W]
//   dmap     u8  [S][4][H][W]      colour-difference maps used by the scanline optimiser
//   disp_*   f32 [S][H][W]
//   label    u8  [S][H][W]         0 = valid, 1 = mismatch list, 2 = occlusion list
#pragma once
#include <cuda.h>     // CUtensorMap and its enums only
#include <cuda_runtime.h>
#include <stdint.h>

#include "img_format.h"

#define ADC_INVALID_F (__int_as_float(0x7f800000))  // +inf  (adcensus_types.h:33)
#define ADC_LARGE_F 99999.0f                         // adcensus_types.h:35
#define ADC_CNT 16                                   // ints of per-pair counters

struct AdcDims {
    int W, H, D, Dp;        // Dp: padded disparity stride (multiple of 4)
    int dmin, dmax;
    int N;                  // W*H
    long long vol_stride;   // floats per pair volume = N*Dp
};

// Everything a kernel may need from ADCensusOption plus derived constants, passed by value.
struct AdcParams {
    AdcDims dm;
    int L1, L2, t1, t2;          // cross arm parameters (L1 already clamped to 255)
    float p1, p2, p1_4, p2_4, p1_10, p2_10;  // so_p1/so_p2 and their /4, /10 quotients (IEEE, host-computed)
    int tso;
    int irv_ts; float irv_th;
    float lr_thres;
    int max_search;              // max(|dmax|,|dmin|)
    int dbg;                     // adc_config.debug_flags (test hooks, ADC_DBG_* in adcensus_b200.h)
};

__device__ __forceinline__ int adc_colour_dist(uchar3 a, uchar3 b) {
    int d0 = abs((int)a.x - (int)b.x), d1 = abs((int)a.y - (int)b.y), d2 = abs((int)a.z - (int)b.z);
    return max(d0, max(d1, d2));
}

__device__ __forceinline__ uchar3 adc_load_bgr(const uint8_t* __restrict__ img, int idx) {
    const uint8_t* p = img + 3ll * idx;
    return make_uchar3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}

// order-preserving float -> uint key (any sign), for REDUX-based warp minima
__device__ __forceinline__ unsigned adc_f2key(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float adc_key2f(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Parabola through (best-1, best, best+1), ADCensusStereo.cpp:234-240 (k_wta.cu, k_scanline.cu).  Explicit _rn
// intrinsics keep nvcc from contracting c1 + c2 - 2*min into an FMA.
__device__ __forceinline__ float adc_subpixel(float c1, float c2, float cmin, int best) {
    const float denom = __fsub_rn(__fadd_rn(c1, c2), __fmul_rn(2.0f, cmin));
    if (denom != 0.0f) return __fadd_rn((float)best, __fdiv_rn(__fsub_rn(c1, c2), __fmul_rn(denom, 2.0f)));
    return (float)best;
}

// Function attributes and __device__ / __constant__ symbols exist once per device: one-time set-up is keyed by the
// current device (one process may own engines on several GPUs, driven from several threads: the flags are atomics, and
// a thread that loses the race may run the kernel before the winner's attribute call has returned -- so every caller
// that finds the flag unset performs the (idempotent) set-up itself, and the flag is only published afterwards).
#include <atomic>
struct AdcOnce { std::atomic<int> done[64]; };
inline bool adc_once_needed(AdcOnce& o) {
    int dev = 0;
    cudaGetDevice(&dev);
    return o.done[dev & 63].load(std::memory_order_acquire) == 0;
}
inline void adc_once_done(AdcOnce& o) {
    int dev = 0;
    cudaGetDevice(&dev);
    o.done[dev & 63].store(1, std::memory_order_release);
}

// SMs of the current device (grid sizes of the grid-stride and look-ahead launches scale with it)
inline int adc_sm_count() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 1;
}

// TMA descriptors (CUtensorMap, 128 bytes each) of a lane's two cost volumes for the axes of the double passes that take
// the TMA form (arm_sum2_form, ca_plan.h); the other axis's are zero and never read
struct alignas(64) AdcArmTmaps { unsigned char map[2][2][128]; };
// TMA descriptors of the scanline passes, per axis (0: +-x, 1: +-y): the two volumes and the penalty records, with the boxes
// of that axis's launch plan (T steps per ring slot, NS slots per warp, dynamic shared memory per CTA; so_plan.h)
struct alignas(64) AdcSoTmaps { unsigned char cost[2][2][128]; unsigned char rec[2][128]; int T[2], NS[2]; unsigned smem[2]; };
// cuTensorMapEncodeTiled, fetched through the runtime (no link-time libcuda dependency); NULL when the driver lacks it
typedef CUresult (*AdcTmapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
AdcTmapEncodeFn adc_tmap_encoder();

// ---- launchers (defined in the k_*.cu files; all asynchronous on `st`) -------------------------
struct AdcWave {            // device pointers of one wave (S pairs)
    int S;                  // active pairs in this launch
    uint8_t* bgr;           // [S][2][N*3]
    unsigned* bgrx;         // [S][2][N] the same pixels packed B | G<<8 | R<<16 (one 32-bit load per pixel)
    uint8_t* gray;          // [S][2][N]
    unsigned long long* census; // [S][2][N]
    float* volA; float* volB;
    uchar4* arms;
    const AdcArmTmaps* arm_tm;   // host memory, owned by the lane: tensor maps of the aggregation double passes
    unsigned* arm_rec;      // [S][window records of both axes] which of a group's four outputs takes which tap (k_aggregate.cu)
    uint16_t* sup_h; uint16_t* sup_v;
    uint8_t* dmap;          // [S][4][N]: 0 = left-horizontal, 1 = left-vertical, 2 = right-horizontal, 3 = right-vertical
    float* disp_l; float* disp_r; float* disp_t;
    uint8_t* label; uint8_t* flag;
    int* pend;              // [S][2][N] mismatch / occlusion pixel lists (raster order)
    int* vlist;             // [S][2][N] the sub-lists region voting works on (pixels that can still be filled)
    int* counters;          // [S][ADC_CNT]: 0,1 list sizes; 2 voting rounds; 3 voting evaluations; 4.. flags/queues
    int* rowcnt;            // [S][2][H] per-row list counts / offsets
    unsigned* so_bitrows;   // [S][4][H][row words] mirrored per-row bit vectors of the right image (scanline optimiser)
    unsigned* so_rec;       // [S][4][N][rec words] per-pixel penalty records of the four pass directions
    const AdcSoTmaps* so_tm;     // host memory, owned by the lane: tensor maps of the scanline passes
    int* vote_work;         // [S][N]     region voting: slots whose histogram changed, to derive this round
    int2* vote_chg;         // [S][N]     region voting: change records of the current round / fills of a commit
    uchar2* vote_alr;       // [S][N]     region voting: horizontal arms only (left, right)
    uchar2* vote_atbT;      // [S][W][H]  region voting: vertical arms (top, bottom), transposed (a column is contiguous)
    int* vote_pslotT;       // [S][W][H]  region voting: histogram slot of a pending pixel, -1 otherwise (transposed)
    uint16_t* vote_val;     // [S][N]     region voting: current vote per slot (one byte used unless D > 254 or L1 > 127)
    uint8_t* vote_dirtyb;   // [S][N]     region voting: slot's histogram changed since its last derive
    int* vote_state;        // [S][N]     region voting: disparity index of a valid pixel, -1 invalid, -(slot+2) pending
    int* vote_off;          // [S][N+1]   region voting: adjacency list lengths -> offsets -> fill cursors (CSR by target slot)
    unsigned* vote_hist;    // [S][vol_stride] region voting: histograms + forward lists + adjacency (= volB, idle after the last scanline pass)
    const float* lut_ad;    // [766]  (1 - exp(-(s/3)/lambda_ad)) + 1, host libm expf
    const float* lut_cen;   // [64]   exp(-h/lambda_census)
    const double* ray_sin; const double* ray_cos; // [16] host libm sin/cos of the accumulated angles
    const short2* ray_off;  // [16][max_search] (dx,dy) = (lround(m*cos), lround(m*sin)); NULL if not verified exact
};

void adc_launch_gray_census(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
void adc_launch_cost(const AdcParams& P, const AdcWave& w, float* vol, cudaStream_t st, unsigned long long* launches);
// cost-input mode (k_ingest.cu): the wave's caller volumes at `src` (pair stride N*D elements, layout ADC_COST_HWD /
// ADC_COST_DHW, element type ADC_COST_F32 / F16 / BF16) -> `vol`, clamped to the documented value domain
void adc_launch_cost_ingest(const AdcParams& P, const AdcWave& w, const void* src, int layout, int dtype, float* vol,
                            cudaStream_t st, unsigned long long* launches);
size_t adc_cost_elem_bytes(int dtype);
// volume export (k_ingest.cu): the wave's [S][N][Dp] f32 volume `vol` -> `dst` (pair stride N*D elements, layout
// ADC_COST_HWD / ADC_COST_DHW, element type ADC_COST_F32 / F16 / BF16 rounded to nearest even); dst aligned to its element
void adc_launch_cost_export(const AdcParams& P, const AdcWave& w, const float* vol, void* dst, int layout, int dtype,
                            cudaStream_t st, unsigned long long* launches);
// The engine's internal form of a view's remap table (k_rectify.cu): one uint2 per output pixel, .x = (u16)x0 |
// (u16)y0 << 16, .y = ax | ay << 5 (DESIGN.md section 14).
struct AdcRectGeom {
    const uint2* map[2];   // left, right: [H][W] each (nullptr for a resize)
    int src_w, src_h;      // raw frame size
    int type;              // the geometry: ADC_REMAP_* (through map) or ADC_RESIZE_* (factors checked against dm.W x dm.H)
};
IMG_HD constexpr bool adc_is_resize(int type) { return type == ADC_RESIZE_AREA || type == ADC_RESIZE_LINEAR_EXACT; }
// a view's adc_remap (map1 / map2 with byte pitches, device-readable, ADC_REMAP_F32 / ADC_REMAP_FIXED) -> out [H][W]
void adc_launch_remap_convert(const AdcDims& dm, int map_type, const void* map1, long long pitch1, const void* map2,
                              long long pitch2, uint2* out, cudaStream_t st);
// image ingestion (k_image.cu): S pairs of views at left / right (pair i at byte i*image_stride, format ADC_IMG_*,
// pitches resolved: no zero defaults left; the formats, their geometry and adc_image_tight are in img_format.h) ->
// bgr as packed BGR [S][2][N*3] (a wave's w.bgr, or a caller's views).  r == nullptr: views of the engine's size, read
// in place; otherwise raw src_w x src_h frames, resampled through r's maps or resized.  One launch of at most
// adc_view_ingest_max_pairs(dm) pairs.
void adc_launch_view_ingest(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                            const AdcRectGeom* r, uint8_t* bgr, cudaStream_t st, unsigned long long* launches);
int adc_view_ingest_max_pairs(const AdcDims& dm);
// reprojection to 3-D (k_reproject.cu): n maps of dm.N pixels at disp -> the outputs whose pointer is not NULL (map i
// at pixel i*N of each), Q row-major; s16_invalid = the DISP_S16 value of a +inf pixel.  One launch.
struct AdcReprojQ { double q[16]; };
void adc_launch_reproject(const AdcDims& dm, long long n, const float* disp, const AdcReprojQ& Q, float* points,
                          float* depth, int16_t* s16, int16_t s16_invalid, cudaStream_t st, unsigned long long* launches);
// point clouds (k_cloud.cu): the kept pixels of n maps of dm.N pixels at disp (finite d, finite point, z_min <= Z <=
// z_max), compacted in raster order: map i's first `capacity` points at point i*capacity of points / colors (R, G, B of
// the pixel of bgr + i*bgr_stride; NULL = none) / pixels (NULL = none), its full count at counts[i].  `work` holds
// adc_point_cloud_work_bytes(dm, n) bytes, 8-byte aligned and zeroed in stream order before the launch.  One launch.
struct AdcCloudOut {
    float* points;
    uint8_t* colors;
    int32_t* pixels;
    int32_t* counts;
    long long capacity;
};
size_t adc_point_cloud_work_bytes(const AdcDims& dm, long long n);
void adc_launch_point_cloud(const AdcDims& dm, long long n, const float* disp, const AdcReprojQ& Q, const uint8_t* bgr,
                            long long bgr_stride, float z_min, float z_max, const AdcCloudOut& out, void* work,
                            cudaStream_t st, unsigned long long* launches);
// speckle removal (k_speckle.cu): the rules resolved on the host.  S16: missing = (int)v == nv_i, connected =
// |a - b| <= md_i in int, written (int16)nv_i.  F32: missing = v == nv_f, connected = fabsf(a - b) <= md_f (the largest
// float not above max_diff), written nv_f.  A component of at most max_size pixels is removed.
struct AdcSpeckle {
    int nv_i, md_i;
    float nv_f, md_f;
    int max_size;
};
// n maps of dm.N pixels at maps (int16, or float when f32), filtered in place; work = n*N int32 parents, then n*N
// uint32 sizes.  Four launches.
void adc_launch_speckles(const AdcDims& dm, long long n, bool f32, void* maps, void* work, const AdcSpeckle& p,
                         cudaStream_t st, unsigned long long* launches);
// previews (k_preview.cu): n maps of dm.N pixels at maps -> n frames of dst_w x dst_h at dst (frame i at byte
// i*image_stride, format ADC_IMG_BGR / BGRA / RGBA / GRAY / NV12 / NV21 / I420 / YV12, pitches resolved).  work
// non-NULL = MINMAX: 2*n uint32 zeroed in stream order before the call, (alpha, beta) unused; NULL = FIXED with the
// float (alpha, beta).  inv_x / inv_y = 1.0 / ((double)dst_w / W), 1.0 / ((double)dst_h / H).  Two launches (MINMAX)
// or one.
struct AdcPreviewArgs {
    uint8_t* dst;
    unsigned* work;
    long long row_pitch, plane_pitch, image_stride;
    double inv_x, inv_y;
    float alpha, beta;
    int format, colormap, dst_w, dst_h;
    uint8_t invalid[3];
};
void adc_launch_preview(const AdcDims& dm, long long n, const float* maps, const AdcPreviewArgs& a, cudaStream_t st,
                        unsigned long long* launches);
void adc_launch_diffmaps(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
void adc_launch_arms(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
// one 1-D pass of the cross aggregation: horizontal (dir=0) or vertical (dir=1) ordered sums,
// optionally divided by the support count `sup` (second pass of an iteration)
void adc_launch_arm_sum(const AdcParams& P, const AdcWave& w, const float* src, float* dst, int dir,
                        const uint16_t* sup, cudaStream_t st, unsigned long long* launches);
// two consecutive passes along the same axis (second pass of an iteration, divided by `sup_mid`, then the first pass of the
// next iteration) with the intermediate kept in shared memory, in the form arm_sum2_form picks (ca_plan.h); src = w.volA
// or w.volB
void adc_launch_arm_sum2(const AdcParams& P, const AdcWave& w, const float* src, float* dst, int dir,
                         const uint16_t* sup_mid, cudaStream_t st, unsigned long long* launches);
// the AD-census cost computed in place of the cost volume and summed as the first horizontal pass (no division) into
// `dst`; cost_out (nullable) also receives the cost volume, padding disparities included, as adc_launch_cost writes it.
// false = not applicable for these parameters (ca_plan.h), nothing launched
bool adc_cost_arm_sum_h_available(const AdcParams& P);
bool adc_launch_cost_arm_sum_h(const AdcParams& P, const AdcWave& w, float* dst, float* cost_out, cudaStream_t st,
                               unsigned long long* launches);
size_t adc_arm_rec_bytes(const AdcDims& dm, int L1);   // window records of one pair
// tensor maps of the double passes' TMA-form axes over a lane of capacity S (false: they cannot be encoded)
bool adc_arm_tmaps_encode(const AdcParams& P, int S, float* volA, float* volB, AdcArmTmaps* out);
size_t adc_arm_overread_floats(const AdcDims& dm);     // padding the arena keeps behind the two volumes
void adc_launch_so_bitrows(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
size_t adc_so_rec_bytes(const AdcDims& dm);
size_t adc_so_bitrow_bytes(const AdcDims& dm);
// tensor maps and launch plans of the scanline passes over a lane of capacity S (false: they cannot be encoded)
bool adc_so_tmaps_encode(const AdcParams& P, int S, float* volA, float* volB, unsigned* so_rec, AdcSoTmaps* out);
// one scanline pass: (sx,sy) in {(1,0),(-1,0),(0,1),(0,-1)}, src = w.volA or w.volB; non-zero: not launched
int adc_launch_scanline(const AdcParams& P, const AdcWave& w, const float* src, float* dst, int sx, int sy,
                        cudaStream_t st, unsigned long long* launches);
int adc_launch_wta(const AdcParams& P, const AdcWave& w, const float* vol, cudaStream_t st, unsigned long long* launches);
// the last scanline pass (-y) fused with the WTA (so_wta_fused, so_plan.h): src = w.volB's optimised-so-far volume; writes
// disp_l and the right view's partial records to rec; k_wta_merge folds them into disp_r
int adc_launch_scanline_wta(const AdcParams& P, const AdcWave& w, const float* src, float* rec, cudaStream_t st,
                            unsigned long long* launches);
int adc_launch_wta_merge(const AdcParams& P, const AdcWave& w, const float* rec, cudaStream_t st, unsigned long long* launches);
// cost-curve confidence (k_confidence.cu): per pixel of the wave's volume `vol`, c1 = C(d1) -> min_cost and c1 / c2 ->
// peak_ratio (either may be NULL; pair i at element i*N, 4-byte aligned)
void adc_launch_confidence(const AdcParams& P, const AdcWave& w, const float* vol, float* min_cost, float* peak_ratio,
                           cudaStream_t st, unsigned long long* launches);
void adc_launch_outlier(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
void adc_launch_build_lists(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
// the voting lists (w.vlist, counters 10/11): the listed pixels whose cross region can ever pass the vote
void adc_launch_active_lists(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
// region voting (k_vote.cu): fills pixels of disp_l / disp_t, then rebuilds the outlier lists; uses w.volB as storage
void adc_launch_voting(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches);
// k = 0: mismatch list, k = 1: occlusion list; reads disp_l, writes disp_t
void adc_launch_interp_list(const AdcParams& P, const AdcWave& w, int k, cudaStream_t st, unsigned long long* launches);
void adc_launch_discontinuity(const AdcParams& P, const AdcWave& w, const float* vol, cudaStream_t st, unsigned long long* launches);
// in-place-equivalent 3x3 median: reads `in`, writes `out` (different buffers); non-zero if H is too large
// output side of the demo (k_render.cu): 8-bit normalised map + JET colouring; (x,y,d,r,g,b) cloud of the valid pixels
int adc_launch_render(const AdcDims& dm, const float* d_disp, unsigned* d_mm, uint8_t* d_gray, uint8_t* d_jet, float* d_mm_out,
                      cudaStream_t st, unsigned long long* launches);
void adc_launch_cloud(const AdcParams& P, const AdcWave& w1, const float* d_disp, const uint8_t* d_bgr, float* d_cloud,
                      cudaStream_t st, unsigned long long* launches);
int adc_launch_median(const AdcParams& P, const AdcWave& w, const float* in, float* out, cudaStream_t st,
                      unsigned long long* launches);
