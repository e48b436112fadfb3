/* include/adcensus_b200.h -- the drop-in boundary of the H100-native AD-Census engine.
 *
 * A plain C ABI (extern "C", raw pointers and sizes, no torch / CUDA types) over the sm_90a
 * kernels in adcensus_b200/csrc.  The reference (ethan-li-coding/AD-Census) has no FFI of its
 * own: its boundary is the C++ class ADCensusStereo (ADCensusStereo.h:14-95) compiled into the
 * caller.  include/ADCensusStereo.h in this repo is the header-compatible shim of that class and
 * is implemented purely in terms of the functions declared here; INTEGRATION.md shows how an
 * existing caller of the reference switches over.
 *
 * Each entry point names the reference interface it stands in for.
 */
#ifndef ADCENSUS_B200_H_
#define ADCENSUS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Byte-identical to the reference's ADCensusOption (adcensus_types.h:45-75): 60 bytes, align 4.
 * A pointer to the reference's struct may be passed wherever adc_option is expected.
 *
 * Accepted domain.  adc_create fails with ADC_ERR_ARG, naming the field, for:
 *   - max_disparity - min_disparity <= 0 (the reference's Initialize returns false);
 *   - bounds whose max - min or abs() overflows int32, or whose candidate columns x - d or x + d (0 <= x < width)
 *     overflow int32: signed overflow in the reference's cost and right-view WTA loops;
 *   - lambda_ad < 1 or lambda_census < 1: at 0 the cost divides by zero (NaN on every flat patch); below, costs fall
 *     under zero and reach -inf once exp overflows;
 *   - so_p1 or so_p2 negative or not finite: path costs reach -inf or NaN, and the sub-pixel disparities NaN.
 * Every other value of every field is accepted and computed as the reference computes it, for example cross_L1 < 0
 * (no arms) or > 255 (limited to 255), cross_t1 <= 0 (no arms), cross_L2 < 0 or >= cross_L1, so_tso <= 0 (every
 * step in the smallest penalty class), any irv_ts, and irv_th or lrcheck_thres negative, infinite or NaN (every
 * comparison with NaN is false: no region vote succeeds, no left/right difference exceeds it). */
typedef struct adc_option {
    int32_t min_disparity;   /* offset  0 */
    int32_t max_disparity;   /*         4   (exclusive) */
    int32_t lambda_ad;       /*         8 */
    int32_t lambda_census;   /*        12 */
    int32_t cross_L1;        /*        16 */
    int32_t cross_L2;        /*        20 */
    int32_t cross_t1;        /*        24 */
    int32_t cross_t2;        /*        28 */
    float   so_p1;           /*        32 */
    float   so_p2;           /*        36 */
    int32_t so_tso;          /*        40 */
    int32_t irv_ts;          /*        44 */
    float   irv_th;          /*        48 */
    float   lrcheck_thres;   /*        52 */
    uint8_t do_lr_check;     /*        56   (C++ bool in the reference) */
    uint8_t do_filling;      /*        57 */
    uint8_t do_discontinuity_adjustment; /* 58 */
    uint8_t reserved_;       /*        59   padding byte, ignored */
} adc_option;

typedef struct adc_engine adc_engine; /* opaque; owns the device arena, streams and tables */

/* error codes (0 = success).  adc_last_error() gives the text for the calling thread. */
enum {
    ADC_OK = 0,
    ADC_ERR_ARG = 1,          /* null pointer / non-positive size / empty disparity range: the cases where
                                 the reference's Initialize/Match return false (ADCensusStereo.cpp:31,38,71,74);
                                 an option outside the domain stated at adc_option */
    ADC_ERR_CUDA = 2,         /* a CUDA runtime call failed */
    ADC_ERR_UNSUPPORTED = 3,  /* configuration outside what the kernels implement (see DESIGN.md) */
    ADC_ERR_NOMEM = 4         /* device or pinned-host allocation failed */
};

/* Engine tuning knobs; zero-initialise for defaults. */
typedef struct adc_config {
    int32_t device;          /* CUDA device ordinal */
    int32_t wave_pairs;      /* stereo pairs processed by one batched kernel launch (default: auto) */
    int32_t lanes;           /* concurrent waves in flight, one stream each (default: auto) */
    int32_t debug_flags;     /* test hooks, 0 in production: force the alternate code paths that otherwise only unusual
                                parameters reach, so that the parity tests can run every shipped kernel (ADC_DBG_*) */
    int32_t reserved[12];    /* must be zero */
} adc_config;

enum {
    ADC_DBG_NO_RAY_TABLE = 1,     /* interpolation evaluates lround(y + m*sin) in double per step instead of the verified integer table */
    ADC_DBG_VOTE_ENUM = 2,        /* region voting finds the affected histograms by enumeration instead of adjacency lists */
    ADC_DBG_VOTE_GLOBAL_STATE = 4,/* region voting keeps its per-slot state in global instead of shared memory */
    ADC_DBG_UNFUSED_AGG = 8,      /* aggregation as eight single passes instead of five (three of them fused double passes) */
    ADC_DBG_UNFUSED_SO_WTA = 32,  /* the last scanline pass stores the optimised volume and the WTA reads it back, also where
                                     the pass would take the WTA as its epilogue */
    ADC_DBG_FUSED_SO_WTA = 64,    /* the last scanline pass takes the WTA as its epilogue wherever nothing else reads the
                                     optimised volume and its partial records fit in a pair's volume, also where the
                                     records' traffic would not pay for it */
    ADC_DBG_POISON = 16           /* every byte of a lane's device arena is set to the pattern ADC_DBG_POISON_BYTE gives, on
                                     the lane's stream: at adc_create instead of zeros; at the start of every wave of a batch
                                     call, after the lane has joined the caller's stream and before the wave's inputs
                                     arrive; in the one-pair host calls (and adc_debug_run*) before the pair is uploaded;
                                     in adc_render_disparity and adc_disparity_cloud before their uploads.  The device
                                     staging of the one-pair host calls is filled too, whenever a call takes it.  So a
                                     kernel that reads memory its wave or call did not write meets the pattern, not zeros or
                                     a plausible earlier pair.  Not filled: what explicit calls set and later calls rely
                                     on -- the cost and ray tables, the integer ray offsets, the tensor maps, the
                                     rectification maps (adc_set_rectification), the right-view map adc_get_right_disparity
                                     returns and the pinned host staging.  A test hook: the fills cost bandwidth */
};
/* The pattern byte of ADC_DBG_POISON (bits 8-15 of debug_flags): 0xFF makes floats NaN and integers -1, 0x7F floats
 * 3.4e38 and integers large and positive, 0x01 every byte label a mismatch. */
#define ADC_DBG_POISON_BYTE(b) (((b) & 0xff) << 8)

/* stands in for: ADCensusOption::ADCensusOption() defaults (adcensus_types.h:67-74) */
void adc_default_option(adc_option* opt);

/* Sizes the kernels implement; the reference has no such limits (it only rejects non-positive sizes).  A configuration
 * outside them fails at adc_create / Initialize with ADC_ERR_UNSUPPORTED -- never later, in adc_match. */
#define ADC_MAX_DISPARITY_RANGE 256   /* max_disparity - min_disparity */
#define ADC_MAX_HEIGHT 4096
#define ADC_MAX_WIDTH 10000           /* also bounds width + disparity range */

/* stands in for: ADCensusStereo::Initialize(width, height, option) (ADCensusStereo.h:25,
 * ADCensusStereo.cpp:21-67).  cfg may be NULL.  Fails (ADC_ERR_ARG) exactly where Initialize
 * returns false: width<=0, height<=0, max_disparity-min_disparity<=0, and for an option outside the domain stated at
 * adc_option, checked before any device work; fails with ADC_ERR_UNSUPPORTED beyond the limits above. */
int adc_create(int32_t width, int32_t height, const adc_option* opt, const adc_config* cfg, adc_engine** out);

/* stands in for: ADCensusStereo::~ADCensusStereo / Release (ADCensusStereo.cpp:15-19,312-316) */
void adc_destroy(adc_engine* e);

/* stands in for: ADCensusStereo::Match(img_left, img_right, disp_left) (ADCensusStereo.h:33,
 * ADCensusStereo.cpp:69-132).  Packed BGR u8 [H][W][3] host images (main.cpp:61-76), caller-
 * allocated float32 [H][W] host output, +inf = invalid.  Synchronous. */
int adc_match(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, float* disp_left);

/* The right-view disparity map of the most recent adc_match call: what the reference computes into its private
 * disp_right_ (ADCensusStereo::ComputeDisparityRight, ADCensusStereo.cpp:245-310) for the left-right check and never
 * hands out -- float32 [H][W], sub-pixel, not refined (a minimum at either end of the range is the integer disparity).
 * Host pointer.  The one-pair host entries with a final map (adc_match, adc_match_cost and, with disp, the volumes,
 * outputs, images and rectified ones) count as adc_match calls here; batch calls, synchronous or not, pipelined or not,
 * made since do not change the map this returns.  SURVEY.md 8(f) rank 4. */
int adc_get_right_disparity(adc_engine* e, float* disp_right);

/* Batched Match over n independent pairs (the data-parallel form of the call above; the
 * reference would loop Match).  Pointers are host pointers; pinned buffers are copied
 * asynchronously straight from/to the caller's memory, pageable ones go through an internal
 * pinned staging ring.  Synchronous: returns when every disp_left[i] is complete. */
int adc_match_batch(adc_engine* e, int32_t n, const uint8_t* const* img_left,
                    const uint8_t* const* img_right, float* const* disp_left);

/* Same, contiguous host arrays: left/right [n][H][W][3], disp [n][H][W]. */
int adc_match_batch_strided(adc_engine* e, int32_t n, const uint8_t* left, const uint8_t* right, float* disp);

/* Same, but the arrays already live in device memory (HBM-resident form used for the
 * kernel-only throughput figure).  Work is enqueued on the engine's streams, fork/joined on
 * `stream` (a cudaStream_t passed as void*, NULL = legacy default stream) and NOT synchronised:
 * the caller brackets it with its own events. */
int adc_match_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                           float* d_disp, void* stream);

/* Asynchronous host-buffer form for callers that pipeline their own I/O: buffers must be pinned
 * (adc_host_alloc or cudaHostAlloc / cudaHostRegister).  Enqueues H2D, compute and D2H, joined on
 * `stream`, without synchronising. */
int adc_match_batch_pinned_async(adc_engine* e, int32_t n, const uint8_t* left, const uint8_t* right,
                                 float* disp, void* stream);

/* Streaming use (SURVEY.md 8f rank 1): by default every async batch call makes `stream` wait for all of its work, so
 * two calls in a row drain the engine in between (the last waves of a call end in latency-bound refinement kernels with
 * nothing left to overlap them with).  In pipelined mode a batch call returns without that join: the next call's first
 * waves start on the lanes that are already free, and the caller makes its stream wait once, with adc_join, before it
 * touches any result.  Inputs are still consumed in stream order of the call; outputs of a call are complete only
 * after adc_join (or adc_synchronize).  Has no effect on the synchronous entry points. */
int adc_set_pipelined(adc_engine* e, int32_t on);
int adc_join(adc_engine* e, void* stream);

/* ---- matching from a caller-supplied cost volume ------------------------------------------------
 * The entry points below replace stage 1 (gray, census, AD-census cost) by the caller's own matching cost -- from a
 * network, another census variant, a fusion of cues -- and run everything after it unchanged: cross-based aggregation,
 * scanline optimisation, left/right WTA with the parabola, LR check, region voting, interpolation, discontinuity
 * adjustment and the median.  The images are still required: the cross arms, the scanline penalties and the refinement
 * read them.
 *
 * Layout of one pair's volume, contiguous, d = disparity - min_disparity in [0, D), D = max_disparity - min_disparity:
 *   ADC_COST_HWD  [H][W][D]  element (y * W + x) * D + d        (the reference's cost_init_ layout)
 *   ADC_COST_DHW  [D][H][W]  element (d * H + y) * W + x        (a network's [N, D, H, W] cost tensor, one pair)
 * Pairs follow each other with a stride of H*W*D elements.  Element types: ADC_COST_F32, ADC_COST_F16 (IEEE half) and
 * ADC_COST_BF16 (bfloat16), converted to float exactly.
 * Value domain, applied to every element on the way in: NaN, +inf and values >= ADC_COST_MAX become ADC_COST_MAX;
 * negative values, -0.0 and -inf become +0.0.  (The engine treats columns outside the image as cost 99999, never the
 * minimum; aggregation and scanline optimisation never exceed their largest input by more than rounding, so inputs up
 * to 65536 keep that ordering.  -0.0 would let equal minima tie-break differently from the reference's comparisons.)
 * Lower cost = better match, as in the AD-census cost.  lambda_ad and lambda_census are ignored, but must be >= 1;
 * every other option applies.  After a cost call, adc_get_right_disparity, adc_last_stage_ms (out[0] = uploads + ingestion),
 * adc_launch_count and the VOL_* / DISP_* / list debug taps behave as after the image calls; the GRAY_* / CENSUS_* taps
 * are not meaningful.  An unknown layout or element type, or a NULL pointer, fails with ADC_ERR_ARG before any
 * device work. */
enum { ADC_COST_HWD = 0, ADC_COST_DHW = 1 };
enum { ADC_COST_F32 = 0, ADC_COST_F16 = 1, ADC_COST_BF16 = 2 };
#define ADC_COST_MAX 65536.0f

/* adc_match with the cost volume of the pair given: host pointers (images as for adc_match, `cost` one pair's volume),
 * synchronous. */
int adc_match_cost(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right,
                   const void* cost, int32_t layout, int32_t dtype, float* disp_left);

/* adc_match_batch_device with one cost volume per pair: d_cost holds n volumes in device memory (pair i at element
 * i*H*W*D), read straight from there by the ingestion kernel of each wave.  Stream, fork/join and pipelined-mode
 * behaviour (adc_set_pipelined / adc_join) as for adc_match_batch_device; the caller's buffers must stay untouched
 * until the work is joined. */
int adc_match_cost_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                const void* d_cost, int32_t layout, int32_t dtype, float* d_disp, void* stream);

/* ---- exporting the cost volumes ------------------------------------------------------------------
 * The entry points below hand out up to three volumes of every pair next to (or instead of) the disparity map:
 *   ADC_VOL_COST  the matching cost: the reference's cost_init_ after ComputeCost; with a caller's cost (d_cost / cost
 *                 non-NULL), the ingested volume after the value domain above
 *   ADC_VOL_AGGR  the cross-aggregated cost after the 4 iterations: cost_aggr_ after Aggregate
 *   ADC_VOL_OPT   the scanline-optimised cost after the 4 passes, the volume the WTA reads: cost_aggr_ after Optimize
 * in the layouts and element types of cost input (ADC_COST_HWD / ADC_COST_DHW, ADC_COST_F32 / F16 / BF16), pair i of
 * `dst` at element i*H*W*D, the padding disparities and the right view never included.  f32 is the engine's values bit
 * for bit; f16 is IEEE round-to-nearest-even (values >= 65520 become +inf: torch's .half(), numpy's astype(float16));
 * bf16 is round-to-nearest-even.  The volumes hold no NaN.  Each volume is written by one extra pass over it, enqueued
 * where the volume is live; the disparity map of a call that exports is bit-identical to the same call without export.
 * disp NULL = volumes only: the pipeline stops after the latest exported stage (no WTA, no refinement).
 * Fails with ADC_ERR_ARG before any device work, naming the field: n_outs outside 0..3; outs NULL with n_outs > 0; a
 * stage requested twice; an unknown stage, layout or dtype; a NULL dst (on the device entry also a dst not aligned to its
 * element size); a non-zero reserved; n_outs == 0 with disp NULL; an unknown cost layout or dtype when a cost is given. */
enum { ADC_VOL_COST = 0, ADC_VOL_AGGR = 1, ADC_VOL_OPT = 2 };
typedef struct adc_volume_out {
    void*   dst;      /* n volumes of H*W*D elements, pair i at element i*H*W*D */
    int32_t stage;    /* ADC_VOL_* */
    int32_t layout;   /* ADC_COST_HWD / ADC_COST_DHW */
    int32_t dtype;    /* ADC_COST_F32 / ADC_COST_F16 / ADC_COST_BF16 */
    int32_t reserved; /* must be zero */
} adc_volume_out;

/* adc_match_batch_device / adc_match_cost_batch_device plus volume export.  d_cost NULL = the AD-census cost
 * (cost_layout / cost_dtype ignored).  d_disp NULL = stop after the latest exported stage.  Device pointers; stream,
 * fork/join and pipelined-mode behaviour as for adc_match_batch_device. */
int adc_match_volumes_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                   const void* d_cost, int32_t cost_layout, int32_t cost_dtype, float* d_disp,
                                   const adc_volume_out* outs, int32_t n_outs, void* stream);
/* One pair, host pointers (images, optional cost, optional disp, outs[i].dst), synchronous.  The volumes pass through
 * device staging that the engine allocates on first use, grows when a call needs more and frees in adc_destroy
 * (ADC_ERR_NOMEM, before any work, if that allocation fails).  With disp: adc_last_stage_ms (each export counted in the
 * stage that produced its volume) and adc_get_right_disparity behave as after adc_match; after a volumes-only call
 * (disp NULL) neither is meaningful. */
int adc_match_volumes(adc_engine* e, const uint8_t* left, const uint8_t* right, const void* cost, int32_t cost_layout,
                      int32_t cost_dtype, float* disp, const adc_volume_out* outs, int32_t n_outs);

/* ---- per-pixel side maps ---------------------------------------------------------------------------
 * The entry points below hand out, for every pair and in the same pipeline pass, up to five [H][W] maps next to (or
 * instead of) the final disparity map and the exported volumes (pair i at element i*H*W of its destination):
 *   ADC_MAP_WTA_LEFT    f32  the left map right after the WTA, before any refinement: disp_left_ after ComputeDisparity
 *   ADC_MAP_WTA_RIGHT   f32  the right-view map: disp_right_ (what adc_get_right_disparity gives for one pair)
 *   ADC_MAP_OUTLIERS    u8   0 = kept, 1 = mismatch, 2 = occlusion, as the LR check classified the pixel BEFORE region
 *                            voting (the pixels of mismatches_ / occlusions_ after OutlierDetection); all 0 when
 *                            do_lr_check is off
 *   ADC_MAP_MIN_COST    f32  c1 = C(d1)
 *   ADC_MAP_PEAK_RATIO  f32  c1 / c2 in [0, 1]; 0 = unique minimum, 1 = ambiguous
 * Confidence definitions.  C is the scanline-optimised volume, the one the WTA reads and ADC_VOL_OPT exports; d runs
 * over [0, D).
 *   d1 = the smallest d where C(d) is minimal.  This is the index the left WTA picks: it scans with a strict '>' from
 *        99999, and every cost is below that.  It is defined for every pixel, including pixels whose WTA value is
 *        Invalid because d1 lies at either end of the range.
 *   c2 = min of C(d) over |d - d1| >= 2.  The immediate neighbours are excluded, as in OpenCV's uniqueness check.
 *   PEAK_RATIO = c1 / c2, an IEEE round-to-nearest f32 division (__fdiv_rn).  It is 1.0f when no d with |d - d1| >= 2
 *        exists (D <= 2, or D = 3 with d1 = 1) or when c2 == 0; in that case c1 == 0 too, because the costs are
 *        non-negative.
 * The WTA maps and the confidence are enqueued right after the WTA (counted in its stage by adc_last_stage_ms), the
 * outlier map right after the LR check (counted in refinement).  The confidence costs one extra read of the optimised
 * volume; the other maps are copies.  The final map of a call with side maps is bit-identical to the same call without.
 * disp NULL = no final map: the pipeline stops after the latest requested output (the WTA for the WTA and confidence
 * maps, the LR check for ADC_MAP_OUTLIERS, the stage of the latest exported volume), so no voting, interpolation or
 * median runs.
 * Fails with ADC_ERR_ARG before any device work, naming the field: every rule of the volume entries above for vols /
 * n_vols; n_maps outside 0..5; maps NULL with n_maps > 0; a kind requested twice or unknown; a NULL dst; a non-zero
 * reserved; on the device entry an f32 map's dst not 4-byte aligned (u8 maps may start at any byte); no map, no volume
 * and no disp. */
enum { ADC_MAP_WTA_LEFT = 0, ADC_MAP_WTA_RIGHT = 1, ADC_MAP_OUTLIERS = 2, ADC_MAP_MIN_COST = 3, ADC_MAP_PEAK_RATIO = 4 };
typedef struct adc_map_out {
    void*   dst;      /* n maps of H*W elements (f32, or u8 for ADC_MAP_OUTLIERS), pair i at element i*H*W */
    int32_t kind;     /* ADC_MAP_* */
    int32_t reserved; /* must be zero */
} adc_map_out;

/* adc_match_volumes_batch_device plus side maps: one pipeline pass gives the final map (d_disp), the exported volumes
 * (vols) and the maps (maps), any of them optional but not all.  Device pointers; stream, fork/join and pipelined-mode
 * behaviour as for adc_match_batch_device. */
int adc_match_outputs_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                   const void* d_cost, int32_t cost_layout, int32_t cost_dtype, float* d_disp,
                                   const adc_volume_out* vols, int32_t n_vols,
                                   const adc_map_out* maps, int32_t n_maps, void* stream);
/* One pair, host pointers, synchronous; volumes and maps pass through the device staging of adc_match_volumes.  With
 * disp: adc_last_stage_ms and adc_get_right_disparity behave as after adc_match; without, neither is meaningful. */
int adc_match_outputs(adc_engine* e, const uint8_t* left, const uint8_t* right, const void* cost,
                      int32_t cost_layout, int32_t cost_dtype, float* disp,
                      const adc_volume_out* vols, int32_t n_vols, const adc_map_out* maps, int32_t n_maps);

/* ---- image input formats ----------------------------------------------------------------------------
 * The entry points below read the caller's images in place, in any of these u8 formats, with any row, plane and image
 * pitch, instead of requiring packed BGR with rows exactly 3*W bytes and pairs exactly 3*H*W bytes apart:
 *   ADC_IMG_BGR         3 bytes per pixel, packed, B G R       (OpenCV, the reference's main.cpp)
 *   ADC_IMG_RGB         3 bytes per pixel, packed, R G B       (PIL / imageio / numpy loaders, channels-last torch)
 *   ADC_IMG_BGRA        4 bytes per pixel, packed, B G R A     (OpenCV 4-channel Mat, ZED SDK)
 *   ADC_IMG_RGBA        4 bytes per pixel, packed, R G B A     (PIL RGBA, GL / capture buffers)
 *   ADC_IMG_GRAY        1 byte per pixel, one plane            (mono stereo cameras)
 *   ADC_IMG_RGB_PLANAR  1 byte per pixel in each of three planes R, G, B   (torchvision [N, 3, H, W])
 * Semantics: an image in any format is matched exactly as if the caller had packed the same pixels as BGR u8 and called
 * the corresponding packed-BGR entry point.  The channel order is resolved, alpha is ignored, and a gray pixel v is the
 * BGR pixel (v, v, v).  A gray image therefore goes through the engine's gray conversion like any other: the reference's
 * fp64 luma of (v, v, v), truncated, is not always v (gray(128, 128, 128) = 127), and the AD term and the arm / scanline
 * colour distances see three equal channels.
 * Geometry (shared by both views; each view has its own base pointer).  Offsets are bytes, 64-bit:
 *   pixel (x, y) of pair i, packed / gray:  base + i*image_stride + y*row_pitch + x*bytes_per_pixel
 *   channel c (0 = R, 1 = G, 2 = B) of a planar pixel:  base + i*image_stride + c*plane_pitch + y*row_pitch + x
 * Zero-initialised means tight packed BGR, i.e. the packed-BGR entry points' contract.  Rules: none of the pitches may be
 * negative; row_pitch (0 = tight: W * bytes per pixel, W for gray / planar) must be at least W * bytes per pixel;
 * plane_pitch must be 0 for every format but ADC_IMG_RGB_PLANAR, where 0 = H * row_pitch and it must be at least
 * H * row_pitch; image_stride (0 = tight: the view's footprint) must be at least the view's footprint, H * row_pitch or,
 * planar, 3 * plane_pitch; reserved must be zero.  Base pointers and pitches may have any byte alignment (a side-by-side
 * right view starts W * 4 bytes into a BGRA frame; a crop starts at an arbitrary x).  The engine reads only the pixels
 * themselves: nothing past the last pixel of a view's last row, and never an alpha byte.
 * Rule violations fail with ADC_ERR_ARG naming the field: the rules that need no image size before the engine is
 * checked, the size-dependent ones before any device work.
 * Cost: tight packed BGR takes the packed-BGR entry points' copies; every other format or geometry runs one ingestion
 * kernel per wave that writes the wave's packed BGR in one pass.  The Bayer, YUV and high-bit-depth formats (below) are
 * formats of this list, with the geometry rules stated there. */
enum { ADC_IMG_BGR = 0, ADC_IMG_RGB = 1, ADC_IMG_BGRA = 2, ADC_IMG_RGBA = 3, ADC_IMG_GRAY = 4, ADC_IMG_RGB_PLANAR = 5 };
/* Bayer mosaics: raw 8-bit colour-filter frames, 1 byte per pixel in one plane (geometry and rules as for ADC_IMG_GRAY),
 * demosaiced on the way in.  The name gives the colours of the view's OWN top-left 2x2 block, row 0 then row 1, as
 * GenICam's pixel formats do; a crop that starts at an odd x or y has a different pattern, and both views share one.
 *   ADC_IMG_BAYER_RGGB  R G / G B   GenICam BayerRG8   OpenCV COLOR_BayerRGGB2BGR = legacy COLOR_BayerBG2BGR (46)
 *   ADC_IMG_BAYER_GRBG  G R / B G   GenICam BayerGR8   OpenCV COLOR_BayerGRBG2BGR = legacy COLOR_BayerGB2BGR (47)
 *   ADC_IMG_BAYER_BGGR  B G / G R   GenICam BayerBG8   OpenCV COLOR_BayerBGGR2BGR = legacy COLOR_BayerRG2BGR (48)
 *   ADC_IMG_BAYER_GBRG  G B / R G   GenICam BayerGB8   OpenCV COLOR_BayerGBRG2BGR = legacy COLOR_BayerGR2BGR (49)
 * Beware OpenCV's legacy names: they name the second row's second and third pixels, so COLOR_BayerBG2BGR is the RGGB
 * sensor, not BGGR.
 * Semantics: a Bayer view is matched exactly as if the caller had run cv::cvtColor(view, <the code above>) (bilinear;
 * OpenCV's result is the same with and without IPP) and passed the result as packed BGR; through the rectified entries,
 * cvtColor on the raw frame, then cv::remap as described there.  The demosaic of a W x H view:
 *   if W < 3 or H < 3, every pixel is (0, 0, 0);
 *   otherwise pixel (x, y) is the interior rule at (clamp(x, 1, W - 2), clamp(y, 1, H - 2)) -- the border rows and
 *   columns, corners included, repeat their inner neighbours.  Interior rule, the site's colour from the pattern at
 *   (y mod 2, x mod 2), N / S / W / E / NW / ... the raw neighbours:
 *     the site's own colour is its raw value;
 *     at an R or B site: G = (N + S + W + E + 2) >> 2, the other of R / B = (NW + NE + SW + SE + 2) >> 2;
 *     at a G site: the colour of its left and right neighbours = (W + E + 1) >> 1, that of the ones above and below
 *     = (N + S + 1) >> 1.
 * Only the view's own pixels are read. */
enum { ADC_IMG_BAYER_RGGB = 16, ADC_IMG_BAYER_GRBG = 17, ADC_IMG_BAYER_BGGR = 18, ADC_IMG_BAYER_GBRG = 19 };
/* YUV video and camera frames, converted on the way in:
 *   ADC_IMG_NV12  Y plane, then one plane of interleaved U V   OpenCV COLOR_YUV2BGR_NV12 (91)   (NVDEC, V4L2, Jetson)
 *   ADC_IMG_NV21  Y plane, then one plane of interleaved V U   OpenCV COLOR_YUV2BGR_NV21 (93)   (Android)
 *   ADC_IMG_YUYV  packed 4:2:2, macropixel Y0 U Y1 V           OpenCV COLOR_YUV2BGR_YUYV (116) = _YUY2   (UVC, ZED)
 *   ADC_IMG_UYVY  packed 4:2:2, macropixel U Y0 V Y1           OpenCV COLOR_YUV2BGR_UYVY (108) = _Y422
 *   ADC_IMG_YVYU  packed 4:2:2, macropixel Y0 V Y1 U           OpenCV COLOR_YUV2BGR_YVYU (118)
 *   ADC_IMG_I420  Y plane, then a U plane, then a V plane      OpenCV COLOR_YUV2BGR_I420 (128) = _IYUV   (FFmpeg
 *                                                              yuv420p, PyAV, GStreamer I420, libcamera YUV420)
 *   ADC_IMG_YV12  Y plane, then a V plane, then a U plane      OpenCV COLOR_YUV2BGR_YV12 (132)
 *   ADC_IMG_P016  16-bit little-endian words: Y plane, then one plane of interleaved U V (NVDEC's high-bit-depth
 *                 surface, FFmpeg p016le; also P010 and P012, whose samples are MSB-aligned in the same words)
 * Colour encoding: any of these codes may be OR-ed with ADC_IMG_YUV_BT709 (ITU-R BT.709 instead of BT.601) and
 * ADC_IMG_YUV_FULL_RANGE (Y, U, V over 0..255, JPEG / JFIF, instead of limited range).  No flag is BT.601 limited range.
 * A flag on a format that is not YUV, or any other bit above 0xff, fails with ADC_ERR_ARG naming img->format, before
 * the engine is checked.
 * Conversion, per pixel from its own Y and the U, V of its chroma sample, all in int32 with arithmetic shifts,
 * u = U - 128, v = V - 128, sat = clamp to 0..255:
 *   limited range (OpenCV's 20-bit rule), y' = max(0, Y - 16) * 1220542, h = 1 << 19:
 *     R = sat((y' + h + Rv*v) >> 20),  G = sat((y' + h + Gu*u + Gv*v) >> 20),  B = sat((y' + h + Bu*u) >> 20)
 *   full range (OpenCV's 14-bit rule):
 *     R = sat(Y + ((Rv*v + 8192) >> 14)),  G = sat(Y + ((Gu*u + Gv*v + 8192) >> 14)),  B = sat(Y + ((Bu*u + 8192) >> 14))
 *                                      Rv        Gu       Gv       Bu
 *   BT.601 limited (no flag)       1673527   -409993  -852492  2116026   = cv::cvtColor(frame, COLOR_YUV2BGR_<F>)
 *   BT.709 limited                 1879825   -223607  -558796  2215014   = round(k * 2^20) of the exact BT.709
 *                                                                          coefficients (Kr 0.2126, Kb 0.0722) times
 *                                                                          255/224
 *   BT.601 full range                22987     -5636   -11698    29049   = cv::cvtColor(ycrcb, COLOR_YCrCb2BGR) on
 *                                                                          the pixels (Y, V, U)
 *   BT.709 full range                25802     -3069    -7670    30402   = round(k * 2^14) of the exact coefficients
 * Every intermediate fits in int32.  The BT.709 rules are within +-1 of the floating-point BT.709 matrix, rounded and
 * saturated (limited range: for Y >= 16; below, Y - 16 clamps at 0 as in the BT.601 rule).  BT.601 limited range
 * expands Y = 16..235 to 0..255: Y = U = V = 128 gives (130, 130, 130), and Y = U = V = 0 gives (0, 154, 0); the luma
 * term of both limited-range rules is the same, so a grey pixel converts alike under BT.601 and BT.709.
 * P016: every word is first reduced to 8 bits with the high-bit-depth rule at s = 8, to8(v) = min(255, (v + 127 +
 * ((v >> 8) & 1)) >> 8) (convertTo(CV_8U, 1.0 / 256)), then the 8-bit rule of the frame's encoding applies.
 * Geometry (offsets in bytes, 64-bit; each view has its own base; image_stride as for every format):
 *   NV12 / NV21: luma of pixel (x, y) at base + i*image_stride + y*row_pitch + x; its chroma pair at
 *     base + i*image_stride + plane_pitch + (y >> 1)*row_pitch + 2*(x >> 1), U first for NV12, V first for NV21.
 *     row_pitch: 0 = 2*ceil(W/2) (W rounded up to even), and at least that -- a chroma row of an odd-width view is one
 *     byte wider than its luma row.  plane_pitch: 0 = H * row_pitch, and at least that (an NVDEC surface of height
 *     Hs has plane_pitch = pitch * Hs).  Footprint: plane_pitch + ceil(H/2)*row_pitch.  plane_pitch is measured from the
 *     view's own base, so the right half of a side-by-side NV12 frame of even W is simply base + W; a top-bottom NV12
 *     pair cannot be expressed with one shared plane_pitch.
 *   I420 / YV12: luma of pixel (x, y) at base + i*image_stride + y*row_pitch + x.  The chroma planes have row pitch
 *     row_pitch / 2, so row_pitch must be even (ADC_ERR_ARG naming it otherwise, before the engine is checked); the
 *     first (U for I420, V for YV12) starts at plane_pitch, the second ceil(H/2)*(row_pitch/2) bytes after the first,
 *     and the sample of (x, y) is at (y >> 1)*(row_pitch/2) + (x >> 1) within its plane.  row_pitch: 0 = 2*ceil(W/2),
 *     and at least that.  plane_pitch: 0 = H * row_pitch, and at least that.  Footprint: plane_pitch +
 *     ceil(H/2)*row_pitch.  With tight pitches on an even frame this is OpenCV's (H*3/2, W) I420 Mat and FFmpeg's
 *     contiguous yuv420p buffer.  A side-by-side I420 pair cannot be expressed with one shared plane_pitch: the
 *     chroma rows of each half are not row_pitch / 2 apart.
 *   P016: NV12's geometry in 16-bit words: luma word of (x, y) at base + i*image_stride + y*row_pitch + 2*x; its
 *     chroma pair at base + i*image_stride + plane_pitch + (y >> 1)*row_pitch + 4*(x >> 1), U first.  row_pitch: 0 =
 *     4*ceil(W/2), and at least that; plane_pitch: 0 = H * row_pitch, and at least that.  Footprint: plane_pitch +
 *     ceil(H/2)*row_pitch.  On the device entries both base pointers, row_pitch, plane_pitch and image_stride must be
 *     even (ADC_ERR_ARG naming the argument otherwise, before the engine is checked); the host entries take any
 *     alignment, they upload the rows tightly.
 *   YUYV / UYVY / YVYU: pixel (x, y) is the Y0 (x even) or Y1 (x odd) of the macropixel at
 *     base + i*image_stride + y*row_pitch + 4*(x >> 1), with that macropixel's U and V.  row_pitch: 0 = 4*ceil(W/2),
 *     and at least that.  plane_pitch must be 0.  Footprint: H * row_pitch.
 * Semantics: a W x H view is matched exactly as if the caller had taken any even-sized frame holding the view at its
 * top-left, converted it with the rule above (without flags: cv::cvtColor(frame, COLOR_YUV2BGR_<F>); P016:
 * convertTo(CV_8U, 1.0 / 256), then COLOR_YUV2BGR_NV12), cropped the result to W x H and passed that as packed BGR
 * (for even sizes: the conversion of the view itself).  Chroma is sited at even positions relative to the view's own
 * (0, 0), so a crop of a larger frame must start at an even x (and, for 4:2:0, an even y): that is the caller's
 * responsibility, as the pattern is for the Bayer formats.  Through the rectified entries the whole src_width x
 * src_height frame is converted with its encoding first and that BGR frame is resampled; a neighbour outside the frame
 * is BGR (0, 0, 0), not the conversion of YUV (0, 0, 0).  Only the view's own samples are read: nothing past the last
 * chroma byte or word of a 4:2:0 view, nothing past ceil(W/2) bytes of an I420 / YV12 chroma row, nothing past
 * 4*ceil(W/2) bytes of a packed 4:2:2 row.
 * Out of scope: BT.2020 and HDR transfer functions, planar and semi-planar 4:2:2 and 4:4:4 (I422, NV16), packed 10-bit
 * (v210, Y210), side-by-side I420. */
enum { ADC_IMG_NV12 = 32, ADC_IMG_NV21 = 33, ADC_IMG_YUYV = 34, ADC_IMG_UYVY = 35, ADC_IMG_YVYU = 36 };
enum { ADC_IMG_I420 = 38, ADC_IMG_YV12 = 39, ADC_IMG_P016 = 40 };
enum { ADC_IMG_YUV_BT709 = 0x100, ADC_IMG_YUV_FULL_RANGE = 0x200 };
/* High-bit-depth mono and Bayer frames, as GigE Vision / USB3 Vision cameras deliver them, reduced to 8 bits on the way
 * in.  The names are the GenICam PFNC pixel formats; five containers, each as mono and as the four Bayer patterns:
 *   ADC_IMG_MONO10   ADC_IMG_BAYER_{RG,GR,BG,GB}10    Mono10 / BayerRG10 ...: one sample per little-endian uint16,
 *                                                     LSB-aligned, 10 significant bits; a tight row is 2*W bytes
 *   ADC_IMG_MONO12   ADC_IMG_BAYER_{RG,GR,BG,GB}12    Mono12 / BayerRG12 ...: the same, 12 significant bits
 *   ADC_IMG_MONO16   ADC_IMG_BAYER_{RG,GR,BG,GB}16    Mono16 / BayerRG16 ...: the same, 16 bits.  Also the format for
 *                                                     10- / 12-bit data delivered MSB-aligned in 16-bit words
 *   ADC_IMG_MONO10P  ADC_IMG_BAYER_{RG,GR,BG,GB}10P   Mono10p / BayerRG10p ...: 4 samples in 5 bytes; a tight row is
 *                                                     ceil(10*W / 8) bytes
 *   ADC_IMG_MONO12P  ADC_IMG_BAYER_{RG,GR,BG,GB}12P   Mono12p / BayerRG12p ...: 2 samples in 3 bytes; a tight row is
 *                                                     ceil(12*W / 8) bytes
 * The Bayer names follow the 8-bit block's convention, the colours of the view's OWN top-left 2x2 block, and map onto
 * the same four OpenCV codes: RG = ADC_IMG_BAYER_RGGB = COLOR_BayerRGGB2BGR = legacy COLOR_BayerBG2BGR (46), GR = _GRBG
 * = legacy COLOR_BayerGB2BGR (47), BG = _BGGR = legacy COLOR_BayerRG2BGR (48), GB = _GBRG = legacy COLOR_BayerGR2BGR
 * (49).  The same warning applies: OpenCV's legacy names are not the sensor's, COLOR_BayerBG2BGR is the RG sensor.
 * Sample of pixel x of a row (b = 10, 12 or 16 the depth):
 *   16-bit containers: v = the x-th uint16 of the row, the whole word; bits above b are NOT masked off.
 *   10p / 12p: the row is a little-endian bit stream that starts at the row's first byte (rows are not packed across
 *     their ends); with o = x*b and k = o >> 3:  v = ((row[k] | row[k+1] << 8) >> (o & 7)) & (2^b - 1).  A field always
 *     spans exactly two bytes, and for x = W - 1 byte k + 1 is the last byte of the tight row.  (12p: byte0 = p0[7:0],
 *     byte1 = p0[11:8] | p1[3:0] << 4, byte2 = p1[11:4].)
 * Depth reduction, one rule for every format, s = b - 8 (2, 4 or 8):
 *   to8(v) = min(255, (v + 2^(s-1) - 1 + ((v >> s) & 1)) >> s)
 * which is round_half_even(v / 2^s) saturated: cv::Mat::convertTo(dst, CV_8U, 1.0 / (1 << s)).  A 10- or 12-bit word with
 * bits set above its depth therefore saturates to 255, as OpenCV treats the uint16 array.
 * Semantics:
 *   mono: the view is matched exactly as if the caller had unpacked it to CV_16UC1, run convertTo(CV_8U, 2^-s) and passed
 *     the result as ADC_IMG_GRAY.
 *   Bayer: as if the caller had unpacked it to CV_16UC1, run cv::cvtColor(raw16, <the code above>) at full depth (the
 *     interior rule and border clamp stated under ADC_IMG_BAYER_* on the 16-bit values; W < 3 or H < 3 gives all-zero
 *     views), then convertTo(CV_8U, 2^-s) on the three channels, and passed that as packed BGR.  Demosaic first, reduce
 *     second: the other order differs in the last bit.
 *   through the rectified entries: the whole src_width x src_height frame is converted that way first and the 8-bit BGR
 *     frame is resampled as described there; a neighbour outside the frame is BGR 0.
 * Geometry (both views share it): sample x of row y of pair i is read from the row at base + i*image_stride +
 * y*row_pitch.  plane_pitch must be 0; row_pitch: 0 = the tight row above, and at least that; image_stride: 0 =
 * H * row_pitch, and at least that.  16-bit containers on the device entries: both base pointers, row_pitch and
 * image_stride must be even, so that the words are aligned (ADC_ERR_ARG naming the argument otherwise, before the
 * engine is checked); the host entries take any pointer and pitch, they upload the rows tightly.  10p / 12p: any byte
 * alignment; a crop or the right half of a side-by-side frame must start on a byte boundary of the stream (x a multiple
 * of 4 for 10p, of 2 for 12p) and, for Bayer, at an even x and y or with the correspondingly different pattern: the
 * caller's responsibility, as for the 8-bit mosaics.  Only the view's own samples are read: nothing past 2*W bytes of a
 * 16-bit row, nothing past ceil(b*W / 8) bytes of a packed row.
 * Out of scope: big-endian words, 14-bit formats, the legacy GigE Vision Mono12Packed / Bayer**12Packed nibble order,
 * 16-bit colour images. */
enum {
    ADC_IMG_MONO10 = 64, ADC_IMG_BAYER_RG10 = 65, ADC_IMG_BAYER_GR10 = 66, ADC_IMG_BAYER_BG10 = 67, ADC_IMG_BAYER_GB10 = 68,
    ADC_IMG_MONO12 = 69, ADC_IMG_BAYER_RG12 = 70, ADC_IMG_BAYER_GR12 = 71, ADC_IMG_BAYER_BG12 = 72, ADC_IMG_BAYER_GB12 = 73,
    ADC_IMG_MONO16 = 74, ADC_IMG_BAYER_RG16 = 75, ADC_IMG_BAYER_GR16 = 76, ADC_IMG_BAYER_BG16 = 77, ADC_IMG_BAYER_GB16 = 78,
    ADC_IMG_MONO10P = 79, ADC_IMG_BAYER_RG10P = 80, ADC_IMG_BAYER_GR10P = 81, ADC_IMG_BAYER_BG10P = 82, ADC_IMG_BAYER_GB10P = 83,
    ADC_IMG_MONO12P = 84, ADC_IMG_BAYER_RG12P = 85, ADC_IMG_BAYER_GR12P = 86, ADC_IMG_BAYER_BG12P = 87, ADC_IMG_BAYER_GB12P = 88
};
typedef struct adc_image_desc {
    int32_t format;        /* ADC_IMG_* (including ADC_IMG_BAYER_*, the YUV and the high-bit-depth formats; a YUV
                              format OR-ed with ADC_IMG_YUV_BT709 / ADC_IMG_YUV_FULL_RANGE) */
    int32_t reserved;      /* must be zero */
    int64_t row_pitch;     /* bytes from one row to the next; 0 = tight (W * bytes per pixel; W for gray / Bayer / planar;
                              2*ceil(W/2) for NV12 / NV21 / I420 / YV12; 4*ceil(W/2) for P016 and YUYV / UYVY /
                              YVYU; 2*W for the 16-bit
                              containers; ceil(10*W/8) for 10p, ceil(12*W/8) for 12p) */
    int64_t plane_pitch;   /* RGB_PLANAR: bytes from one channel plane to the next, 0 = H * row_pitch; NV12 / NV21 /
                              P016: bytes from the luma plane to the chroma plane, I420 / YV12: to the first chroma
                              plane, 0 = H * row_pitch; other formats: must be 0 */
    int64_t image_stride;  /* bytes from pair i's view to pair i+1's view, 0 = tight (H * row_pitch, or 3 * plane_pitch;
                              plane_pitch + ceil(H/2) * row_pitch for NV12 / NV21 / I420 / YV12 / P016) */
} adc_image_desc;          /* 32 bytes */

/* adc_match_outputs_batch_device with the images described by `img` (NULL = tight packed BGR, the same call as
 * adc_match_outputs_batch_device).  Device pointers; stream, fork/join and pipelined-mode behaviour, cost input, volume
 * export, side maps and their argument rules as for adc_match_outputs_batch_device.  A NULL descriptor, or one that
 * describes tight packed BGR, issues exactly the launches of adc_match_outputs_batch_device; any other adds one
 * ingestion launch per wave.  The caller's images must stay untouched until the work is joined. */
int adc_match_images_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                  const adc_image_desc* img, const void* d_cost, int32_t cost_layout, int32_t cost_dtype,
                                  float* d_disp, const adc_volume_out* vols, int32_t n_vols,
                                  const adc_map_out* maps, int32_t n_maps, void* stream);
/* One pair, host pointers, synchronous: adc_match_outputs with the images described by `img` (image_stride is not used),
 * e.g. an OpenCV gray Mat's data and step.  Each view's pixels are uploaded into device memory the engine already owns
 * (the lane volume that stage 1 writes) and converted there.  With disp: adc_last_stage_ms (out[0] = uploads + ingestion
 * + stage 1) and adc_get_right_disparity behave as after adc_match. */
int adc_match_images(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img,
                     const void* cost, int32_t cost_layout, int32_t cost_dtype, float* disp,
                     const adc_volume_out* vols, int32_t n_vols, const adc_map_out* maps, int32_t n_maps);

/* ---- rectification on the way in ---------------------------------------------------------------------
 * The rectified entry points take raw camera frames and resample each view through a per-view remap table (as from
 * cv::initUndistortRectifyMap) while they ingest it: one gather pass per view writes the wave's packed BGR, and
 * everything after that is the pipeline of the image entry points.
 * Semantics: a raw pair matched through adc_match_rectified* gives exactly what this two-step path gives -- the final
 * map, the exported volumes and the side maps, bit for bit:
 *   cv::remap(view, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) on each view, then the same call through
 *   adc_match_outputs* with the rectified images packed as BGR.
 * Channels are resampled independently; formats are resolved as for adc_match_images (gray v -> (v, v, v)), which
 * commutes with the resampling.  A Bayer mosaic is demosaiced over the whole src_width x src_height frame first (the
 * rule under ADC_IMG_BAYER_*, with its clamp at the frame's edges; frames narrower or lower than 3 pixels give all-zero
 * views), and that BGR frame is resampled; so is a YUV frame (each neighbour converted from its own luma and chroma,
 * a neighbour outside the frame BGR 0) and a high-bit-depth frame (demosaiced at full depth and reduced to 8 bits
 * first).  For each output pixel, with (X, Y) its source coordinate in 1/32 pixel and (ax, ay)
 * the 5-bit fractions:
 *   ADC_REMAP_F32 (map1 = float x [H][W], map2 = float y [H][W], CV_32FC1 each):
 *     X = round_half_even(x * 32) saturated to int32, where NaN and values outside int32 give INT_MIN;
 *     x0 = sat_int16(X >> 5) (arithmetic shift), ax = X & 31; likewise Y, y0, ay.
 *   ADC_REMAP_FIXED (map1 = int16 (x, y) pairs [H][W][2], CV_16SC2; map2 = uint16 [H][W], CV_16UC1, as from
 *   initUndistortRectifyMap(..., CV_16SC2) or cv::convertMaps):
 *     (x0, y0) = map1; a = map2 & 1023, ax = a & 31, ay = a >> 5 (the high bits of map2 are ignored).
 *   out = (sum over dx, dy in {0, 1} of w * s + 512) >> 10, with w = (dx ? ax : 32 - ax) * (dy ? ay : 32 - ay) and s
 *   the source byte at (x0 + dx, y0 + dy), or 0 for a neighbour outside the src_width x src_height frame.
 * Every map is [H][W] over the engine's output size; each map's rows may be pitched (bytes, 0 = tight).  The maps of
 * an F32 set and the map2 of a FIXED set are as cv::remap takes them; both map types are pinned to what cv::remap does
 * with that map (initUndistortRectifyMap's CV_16SC2 output is not convertMaps of its float output everywhere).
 *
 * Resizing on the way in: the same entries take frames of another size than W x H when the geometry set is a resize,
 * map_type ADC_RESIZE_AREA or ADC_RESIZE_LINEAR_EXACT (no maps).  Each raw view is converted to 8-bit packed BGR at
 * src_width x src_height with its format's rule, exactly as above (demosaic, YUV rule, depth reduction, gray ->
 * (v, v, v)), and that frame is resized to W x H; the final map, the exported volumes and the side maps are bit for bit
 * those of cv::resize(bgr, (W, H), interpolation = INTER_AREA / INTER_LINEAR_EXACT) followed by adc_match_images* on
 * the result as tight packed BGR.  Channels are resized independently:
 *   ADC_RESIZE_AREA (cv::INTER_AREA at integer factors, downscaling only): src_width = kx * W, src_height = ky * H,
 *     kx * ky <= 4096, and each factor k exact in double as OpenCV computes it, 1.0 / ((double)W / src_width) == kx
 *     and likewise ky.  That holds for 3456 of the factors 1..4096; the other 640 (49, 93, 98, 99, 103, ...) are
 *     rejected, because OpenCV then takes its general area path, which rounds differently.  For every accepted pair,
 *     with s the integer sum of an output pixel's kx x ky source block and n = kx * ky: out = (s + 2) >> 2 for
 *     kx = ky = 2; otherwise out = round_half_even((float)s * (1.0f / n)) saturated to 255, both products in IEEE
 *     float (1 x 1, unequal factors such as 2 x 3, and every other accepted factor).
 *   ADC_RESIZE_LINEAR_EXACT (cv::INTER_LINEAR_EXACT, any sizes, up or down), separable; per axis with n_src -> n_dst
 *     and d the output index: f = (d + 0.5) * scale - 0.5 with scale = 1.0 / ((double)n_dst / n_src), all in IEEE
 *     double without fused multiply-add (scale is OpenCV's, the inverse of its inv_scale; (double)n_src / n_dst
 *     differs from it in the last bit for some sizes, e.g. 49 -> 256, and then so can the output), i = floor(f),
 *     c1 = round_half_even((f - i) * 256), c0 = 256 - c1; i < 0 gives i = 0, c1 = 0 and i >= n_src - 1 gives
 *     i = n_src - 1, c1 = 0 (the border replicates; nothing outside the frame is read).  Per row
 *     h = p[i] * c0x + p[i + 1] * c1x, and out = (h(y0) * c0y + h(y0 + 1) * c1y + 2^15) >> 16.
 * cv::INTER_LINEAR itself is not offered: OpenCV's 8-bit path mixes vector and scalar rounding, so no one rule gives
 * its results.  adc_match_rectified* and adc_ingest_views(rectified = 1) follow whichever geometry is set, maps or a
 * resize; adc_profile_kernel id 14 times the resize ingestion while a resize is set. */
enum { ADC_REMAP_F32 = 0, ADC_REMAP_FIXED = 1 };
enum { ADC_RESIZE_AREA = 16, ADC_RESIZE_LINEAR_EXACT = 17 };
typedef struct adc_remap {
    const void* map1;      /* F32: float x [H][W]; FIXED: int16 (x, y) [H][W][2] */
    const void* map2;      /* F32: float y [H][W]; FIXED: uint16 [H][W] */
    int64_t map1_pitch;    /* bytes from one row of map1 to the next, 0 = tight (W * 4) */
    int64_t map2_pitch;    /* bytes from one row of map2 to the next, 0 = tight (W * 4, FIXED: W * 2) */
} adc_remap;               /* 32 bytes */
typedef struct adc_rectification {
    int32_t src_width;     /* raw frame size, each 1..32767 (OpenCV's coordinates are int16) */
    int32_t src_height;
    int32_t map_type;      /* ADC_REMAP_*, or ADC_RESIZE_* with every view's maps NULL and pitches 0 */
    int32_t reserved;      /* must be zero */
    adc_remap view[2];     /* left, right */
} adc_rectification;       /* 80 bytes */

/* Sets (r != NULL) or clears (r == NULL) the engine's rectification.  Both views' maps are copied and converted into
 * device memory the engine owns (8 bytes per output pixel and view; the caller's maps may be freed on return).  Map
 * pointers may be host memory (pageable or pinned) or device memory; device maps must be complete when the call is
 * made.  Synchronous: before the maps are replaced the device is synchronised, so that every earlier call, pipelined
 * or not, runs with the maps that were set when it was made.  Rules (each violation fails with ADC_ERR_ARG naming the
 * field; those that need no output size before the engine is checked): src_width and src_height in 1..32767;
 * map_type one of ADC_REMAP_* or ADC_RESIZE_*; reserved zero; for maps, no map pointer NULL; pitches not negative
 * and, when not 0, at least a row's bytes; map pointers and pitches aligned to their element (4 bytes for float, 2 for
 * int16 / uint16).  For a resize every map pointer is NULL and every pitch 0, checked before the engine; after it, for
 * ADC_RESIZE_AREA, src_width a multiple of W and src_height a multiple of H (naming the field; W x H itself is the
 * factor 1 x 1), each factor exact in double (1.0 / ((double)W / src_width) == kx, naming r->src_width; likewise
 * r->src_height) and kx * ky <= 4096.  A resize allocates nothing.  A failed allocation fails with ADC_ERR_NOMEM
 * before anything changes.  adc_destroy frees the maps. */
int adc_set_rectification(adc_engine* e, const adc_rectification* r);

/* adc_match_images_batch_device / adc_match_images on raw frames: `img` (NULL = tight packed BGR) describes the raw
 * views, and its size-dependent rules are checked against src_width x src_height instead of W x H.  Each view is
 * resampled through the maps set with adc_set_rectification (semantics above) by one ingestion launch per wave, in
 * place of the image ingestion; cost input, volume export, side maps, streams and pipelined mode as for the image entry
 * points.  Without a rectification set they fail with ADC_ERR_ARG.  The host entry uploads the raw views tightly into
 * the lane volume that stage 1 writes when they fit there, and otherwise into the device staging the exported volumes
 * use (allocated on first use, grown when needed), so it runs for every source size adc_set_rectification accepts. */
int adc_match_rectified_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                     const adc_image_desc* img, const void* d_cost, int32_t cost_layout,
                                     int32_t cost_dtype, float* d_disp, const adc_volume_out* vols, int32_t n_vols,
                                     const adc_map_out* maps, int32_t n_maps, void* stream);
int adc_match_rectified(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img,
                        const void* cost, int32_t cost_layout, int32_t cost_dtype, float* disp,
                        const adc_volume_out* vols, int32_t n_vols, const adc_map_out* maps, int32_t n_maps);

/* ---- reprojection to 3-D ------------------------------------------------------------------------------
 * The entry points below turn f32 [H][W] disparity maps of the engine's size (the engine's final maps, +inf = invalid,
 * or any other) into up to three outputs in one pass, with the 4x4 row-major double matrix Q that cv::stereoRectify
 * returns next to the rectification maps:
 *   ADC_REPROJ_POINTS    f32 [H][W][3]  cv::reprojectImageTo3D(disp, Q, handleMissingValues = false), bit for bit (CV_32FC3)
 *   ADC_REPROJ_DEPTH     f32 [H][W]     the third coordinate of ADC_REPROJ_POINTS, bit for bit (a third of the bytes)
 *   ADC_REPROJ_DISP_S16  int16 [H][W]   the StereoBM / StereoSGBM encoding "disparity * 16" that cv::filterSpeckles,
 *                                       cv::validateDisparity and ximgproc's WLS filter take
 * Semantics of pixel (x, y) with value d; every operation is one IEEE double operation, round to nearest, no fused
 * multiply-add:
 *   h_i = (((+0.0 + Q[i][0]*x) + Q[i][1]*y) + Q[i][2]*d) + Q[i][3]      i = 0..3; x, y, d as double
 *   P_c = (float)((double)(float)h_c * (1.0 / h_3))                     c = 0, 1, 2
 * which is OpenCV's: each coordinate is rounded to float twice (Vec3f /= double multiplies by the reciprocal), and the
 * +0.0 start turns a -0 first product into +0.  With a stereoRectify Q, column 2 of rows 0..2 is zero, so an invalid
 * (+inf) pixel gives 0 * inf = NaN in all three coordinates, exactly as OpenCV does; that is also the NaN-as-missing
 * convention of organised point clouds (PCL, Open3D).  NaN payloads are not specified.  One exception, OpenCV's too:
 * P_2 = 10000.0f where d is exactly FLT_MAX, whatever Q is (reprojectImageTo3D's bigZ for |d - minDisparity| <=
 * FLT_EPSILON, where minDisparity is FLT_MAX without handleMissingValues).
 * DISP_S16: d = +inf gives (min_disparity - 1) * 16 saturated to int16 (the StereoMatcher invalid value, with the
 * engine's min_disparity); any other d gives cv::saturate_cast<short>(d * 16) as on x86: t = d * 16 rounded half to
 * even, saturated to [-32768, 32767] when it fits in int32, and -32768 otherwise, for NaN and for -inf.
 * Fails with ADC_ERR_ARG naming the field, every rule before the engine is checked: n_outs outside 1..3; outs NULL; a
 * kind unknown or requested twice; a NULL dst; a non-zero reserved; a NULL map or Q; a negative n; on the device entry
 * also a map or a POINTS / DEPTH dst not 4-byte aligned, or a DISP_S16 dst not 2-byte aligned. */
enum { ADC_REPROJ_POINTS = 0, ADC_REPROJ_DEPTH = 1, ADC_REPROJ_DISP_S16 = 2 };
typedef struct adc_reproject_out {
    void*   dst;      /* n outputs of H*W pixels of the kind, map i at pixel i*H*W */
    int32_t kind;     /* ADC_REPROJ_* */
    int32_t reserved; /* must be zero */
} adc_reproject_out;  /* 16 bytes */

/* n maps in device memory (map i at element i*H*W) to the requested outputs in device memory, one kernel launch
 * enqueued on `stream` (a cudaStream_t, NULL = legacy default stream), not synchronised.  Q is passed to the kernel by
 * value: the caller may free it on return.  No engine buffer is touched, so the call may run next to the engine's batch
 * calls.  The maps must be complete in `stream`'s order: in pipelined mode, after adc_join on that stream.  A second
 * stream that waits with adc_join keeps the next batch call from waiting for the reprojection (INTEGRATION.md). */
int adc_reproject_batch_device(adc_engine* e, int32_t n, const float* d_disp, const double Q[16],
                               const adc_reproject_out* outs, int32_t n_outs, void* stream);
/* One map, host pointers, synchronous.  The map and the outputs pass through the device staging of adc_match_volumes
 * (allocated on first use, grown when needed; ADC_ERR_NOMEM before any work if that fails).  Like adc_render_disparity,
 * not concurrently with another call on the same engine. */
int adc_reproject(adc_engine* e, const float* disp, const double Q[16], const adc_reproject_out* outs, int32_t n_outs);

/* ---- speckle removal ----------------------------------------------------------------------------------
 * cv::filterSpeckles(img, new_val, max_size, max_diff) on [H][W] maps of the engine's size, in place, for two map types:
 *   ADC_SPECKLE_S16  int16 maps (CV_16SC1: the ADC_REPROJ_DISP_S16 output, StereoSGBM's maps), OpenCV's plain C++ path
 *   ADC_SPECKLE_F32  f32 maps (the engine's own final maps, +inf = invalid); OpenCV has no f32 counterpart
 * A pixel is missing if its value equals new_val.  Two 4-neighbours are connected if neither is missing and their
 * difference is at most max_diff.  Every connected component of at most max_size pixels has all its pixels set to
 * new_val; missing pixels are left as they are.  Components do not depend on a scan order, so the result is exact.
 * S16: new_val and max_diff are turned into ints with cvRound (round half to even as x86's cvtsd2si does, INT_MIN for
 *   NaN and for anything outside int32); the missing test compares the pixel promoted to int with that int, the
 *   differences are taken in int, and the value written is (int16)new_val, which wraps (new_val = 40000 marks nothing
 *   as missing and writes -25536).  max_diff < 0 connects nothing; max_size <= 0 removes nothing.
 *   OpenCV's IPP path (on in the pip wheel) differs in one corner: it wraps cvRound(max_diff) and cvRound(new_val) to
 *   int16 first, so when either lies outside [-32768, 32767] the two paths may give different maps (max_diff 32768 ..
 *   2^31-1 connect nothing under IPP, 65536 connects only equal values, 70000 differences up to 4464, 1e10 and NaN
 *   round to INT_MIN, which IPP wraps to 0; new_val = 40000 makes the pixels equal to -25536 missing under IPP).  The
 *   engine follows the plain path, which every build without IPP computes; with both inside int16, as in every
 *   realistic call, the two agree.
 * F32: nv = (float)new_val rounded to nearest; a pixel is missing if v == nv (IEEE); two pixels are connected if
 *   neither is missing and (double)fabsf(a - b) <= max_diff, with a - b one float subtraction rounded to nearest.  A
 *   NaN pixel never connects (it is removed when max_size >= 1), -inf next to -inf gives NaN and does not connect;
 *   new_val = +inf makes the engine's invalid pixels the missing ones.  max_diff must not be NaN.
 * Fails with ADC_ERR_ARG naming the field: params NULL, params.type unknown, params.reserved not zero, a NaN max_diff
 * on F32, a NULL map, a negative n; on the device entry also maps not 2-byte (S16) or 4-byte (F32) aligned, or the
 * workspace not 4-byte aligned -- all of them before the engine is checked; then (device entry) a workspace smaller
 * than adc_speckle_workspace_bytes for n maps, or NULL while n > 0. */
enum { ADC_SPECKLE_S16 = 0, ADC_SPECKLE_F32 = 1 };
typedef struct adc_speckle_params {
    int32_t type;      /* ADC_SPECKLE_* */
    int32_t max_size;  /* OpenCV's maxSpeckleSize: components of at most this many pixels are removed */
    double  new_val;   /* the missing value, and the value written */
    double  max_diff;  /* the largest difference between connected neighbours */
    int64_t reserved;  /* must be zero */
} adc_speckle_params;  /* 32 bytes */

/* *out = the device workspace n maps need: 8 bytes per pixel (n * H * W * 8). */
int adc_speckle_workspace_bytes(const adc_engine* e, int32_t n, size_t* out);
/* n maps in device memory (map i at element i*H*W) filtered in place, using only the caller's workspace d_work of
 * work_bytes bytes: four kernel launches enqueued on `stream` (a cudaStream_t, NULL = legacy default stream) whatever the
 * content, not synchronised, no host round trip.  No engine buffer is touched, so the call may run next to the engine's
 * batch calls; the maps must be complete in `stream`'s order (in pipelined mode, after adc_join on that stream). */
int adc_filter_speckles_batch_device(adc_engine* e, int32_t n, void* d_maps, const adc_speckle_params* params,
                                     void* d_work, size_t work_bytes, void* stream);
/* One map, host pointer, filtered in place, synchronous.  The map and the workspace pass through the device staging of
 * adc_match_volumes (allocated on first use, grown when needed; ADC_ERR_NOMEM before any work if that fails).  Not
 * concurrently with another call on the same engine. */
int adc_filter_speckles(adc_engine* e, void* map, const adc_speckle_params* params);

/* ---- the views as the engine matches them ----------------------------------------------------------------
 * The packed BGR views that stage 1 of a match reads, handed to the caller: n pairs described by `img` (NULL = tight
 * packed BGR), plain (rectified = 0, what adc_match_images* ingests) or resampled through the maps set with
 * adc_set_rectification (rectified = 1, what adc_match_rectified* ingests), written as packed BGR u8 [n][2][H][W][3]:
 * pair i's left view at byte i*6*H*W, its right view 3*H*W bytes after it.  The bytes are exactly those the image or
 * rectified entries feed to stage 1 for the same arguments, so every rule of those entries carries over: formats,
 * geometry, alignment, the demosaic, YUV and depth-reduction rules, cv::remap, and BGR 0 outside the frame.  Passing
 * d_views back to adc_match_images_batch_device as tight packed BGR therefore matches exactly what the raw-format call
 * matches, and d_views with a stride of 6*H*W colours adc_point_cloud_batch_device's points by the left view.
 * Fails with ADC_ERR_ARG naming the field: the image entries' rules on img (before the engine is checked, and on the
 * device entry the 16-bit alignment rule), rectified not 0 or 1, views NULL, then (after the engine check) a negative
 * n, a NULL view with n > 0, the size-dependent rules of img against W x H (plain) or the raw frame size (rectified),
 * and, rectified, no rectification set.  d_views needs no alignment.
 * The device entry enqueues ceil(n / 65535) ingestion launches (one per 65535 pairs) on `stream` (a cudaStream_t,
 * NULL = legacy default stream), not synchronised; the caller's views must stay untouched until they complete.  It touches no engine buffer but the rectification maps, which adc_set_rectification replaces only
 * after synchronising the device, so it may run next to the engine's batch calls. */
int adc_ingest_views_batch_device(adc_engine* e, int32_t n, const uint8_t* d_left, const uint8_t* d_right,
                                  const adc_image_desc* img, int32_t rectified, uint8_t* d_views, void* stream);
/* One pair, host pointers (image_stride is not used), synchronous: views = [2][H][W][3].  The raw views and the output
 * pass through the device staging of adc_match_volumes (allocated on first use, grown when needed; ADC_ERR_NOMEM
 * before any work if that fails); one ingestion launch.  Not concurrently with another call on the same engine. */
int adc_ingest_views(adc_engine* e, const uint8_t* left, const uint8_t* right, const adc_image_desc* img,
                     int32_t rectified, uint8_t* views);

/* ---- point clouds -------------------------------------------------------------------------------------------
 * The valid points of f32 [H][W] disparity maps of the engine's size, compacted in raster order, with their colours:
 * what cv::reprojectImageTo3D followed by boolean indexing gives (OpenCV's samples/python/stereo_match.py), in one pass
 * and without a host round trip.  Let P be ADC_REPROJ_POINTS of pixel (x, y) with value d (the reprojection formula
 * above, bit for bit).  The pixel is kept iff d is finite, P_x, P_y and P_z are finite, and z_min <= P_z <= z_max as
 * IEEE float comparisons (z_min > z_max keeps nothing; +-inf bounds keep every finite Z).  A non-finite d never has a
 * finite point (with Q[i][2] = 0 the product 0 * inf is NaN), so the d-finite term states the rule without changing the
 * result for any Q; an invalid (+inf) pixel is never kept.  Kept pixels
 * are written in raster order, each with P (f32 x, y, z), then (R, G, B) = (bgr[2], bgr[1], bgr[0]) of pixel (x, y) of
 * that map's colour image, then y*W + x.  When a map keeps more than `capacity` pixels only the first `capacity` are
 * written, nothing past them is touched, and counts[i] still holds the full number.  Kept points are finite, so every
 * output compares bit for bit (no NaN payloads).  In numpy:
 *   P = cv2.reprojectImageTo3D(disp, Q)
 *   keep = np.isfinite(disp) & np.isfinite(P).all(-1) & (P[..., 2] >= z_min) & (P[..., 2] <= z_max)
 *   points, colors, pixels = P[keep], cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)[keep], np.flatnonzero(keep)
 * Colour: packed BGR u8 [H][W][3] per map, bgr_stride bytes from one map's image to the next (0 = 3*H*W): the images
 * the maps were matched from, e.g. adc_ingest_views_batch_device's views with stride 6*H*W (the left views). */
typedef struct adc_cloud_out {
    float*   points;    /* f32 [capacity][3] per map, map i's points at point i*capacity (required) */
    uint8_t* colors;    /* u8 [capacity][3] R, G, B per map, or NULL; non-NULL iff a colour image is given */
    int32_t* pixels;    /* int32 [capacity] per map, y*W + x of each point, or NULL */
    int32_t* counts;    /* int32 [n]: the points each map keeps, the true number even beyond capacity (required) */
    int64_t  capacity;  /* points per map in the destinations, 1..H*W */
    int64_t  reserved;  /* must be zero */
} adc_cloud_out;        /* 48 bytes */

/* *out = the device workspace adc_point_cloud_batch_device needs for n maps: 8 * (1 + n * ceil(H*W / 2048)) bytes, 0 for
 * n = 0. */
int adc_point_cloud_workspace_bytes(const adc_engine* e, int32_t n, size_t* out);
/* n maps in device memory (map i at element i*H*W), colour images d_bgr (or NULL) and the destinations of `out` in
 * device memory, using only the caller's workspace d_work of work_bytes bytes, which the call initialises itself: one
 * cudaMemsetAsync of the workspace and one kernel launch enqueued on `stream` (a cudaStream_t, NULL = legacy default
 * stream) for any n and any content, not synchronised, no host round trip.  The kernel is a single pass: each tile of
 * 2048 pixels computes its points once, and finds its place in the map's output by a decoupled look-back over the
 * map's earlier tiles.  Q is passed by value: the caller may free it on return.  No engine buffer is touched, so the
 * call may run next to the engine's batch calls; the maps must be complete in `stream`'s order (in pipelined mode,
 * after adc_join on that stream).
 * Fails with ADC_ERR_ARG naming the field, before the engine is checked: out NULL; out->points, out->counts, the map or
 * Q NULL; out->colors and the colour image not both given or both NULL; capacity below 1; a non-zero reserved; z_min or
 * z_max NaN; a negative n or bgr_stride; on the device entry the map, out->points, out->pixels or out->counts not
 * 4-byte aligned, or d_work not 8-byte aligned; then capacity above H*W, work_bytes below
 * adc_point_cloud_workspace_bytes for n maps, d_work NULL while n > 0.  n == 0 is a no-op. */
int adc_point_cloud_batch_device(adc_engine* e, int32_t n, const float* d_disp, const double Q[16], const uint8_t* d_bgr,
                                 int64_t bgr_stride, float z_min, float z_max, const adc_cloud_out* out, void* d_work,
                                 size_t work_bytes, void* stream);
/* One map, host pointers (bgr [H][W][3] or NULL; out's arrays and counts[0]), synchronous.  The map, the image, the
 * workspace and the outputs pass through the device staging of adc_match_volumes (allocated on first use, grown when
 * needed; ADC_ERR_NOMEM before any work if that fails); only the min(count, capacity) kept points are copied back.
 * Not concurrently with another call on the same engine. */
int adc_point_cloud(adc_engine* e, const float* disp, const double Q[16], const uint8_t* bgr, float z_min, float z_max,
                    const adc_cloud_out* out);

void* adc_host_alloc(size_t bytes);  /* pinned host memory (cudaHostAlloc) */
void  adc_host_free(void* p);
int   adc_synchronize(adc_engine* e);

/* number of kernel launches issued by this engine since creation (bench.py's gpu_launches) */
uint64_t adc_launch_count(const adc_engine* e);
/* per-stage device milliseconds of the most recent adc_match call (CUDA events):
 * out[0..5] = cost, aggregation, scanline, wta, refine, output copy -- the six figures the
 * reference prints from Match (ADCensusStereo.cpp:88-129).  Where the aggregation is fused (the default) and the cost
 * is AD-census, the matching cost is computed inside the first aggregation pass: out[0] then covers gray + census only
 * and the cost computation is counted in out[1]. */
int adc_last_stage_ms(const adc_engine* e, float out[6]);
/* resolved configuration (wave_pairs, lanes, ...) */
int adc_get_config(const adc_engine* e, adc_config* out);

/* Times one kernel of the pipeline in isolation on the engine's own stream (CUDA events), over one
 * wave of wave_pairs pairs: kernel_id 0 = cost volume, 1 = horizontal arm sum, 2 = vertical arm sum
 * with division, 3 = scanline pass along x, 4 = scanline pass along y, 5 = WTA left+right, 6 / 7 = the fused
 * vertical / horizontal double pass of the aggregation (divide + sum, intermediate in shared memory), 8 = horizontal
 * arm sum with division, 9 = vertical arm sum without division, 10 = cost-volume ingestion (layout and element type of
 * the engine's last cost call, ADC_COST_DHW / ADC_COST_F32 if there was none; N*D*sizeof(element) + N*Dp*4 bytes per
 * pair, Dp = D rounded up to a multiple of 4), 11 = volume export (layout and element type of the engine's last export
 * call, ADC_COST_DHW / ADC_COST_F32 if there was none; N*Dp*4 + N*D*sizeof(element) bytes per pair), 12 = confidence
 * (MIN_COST and PEAK_RATIO of the left view; N*Dp*4 + 2*4*N bytes per pair), 13 = image ingestion (format of the
 * engine's last adc_match_images* call, ADC_IMG_RGB_PLANAR if there was none, tight pitches; the source bytes of both
 * views + 2*3*N written per pair), 14 = rectified ingestion (format of the engine's last adc_match_rectified* call,
 * ADC_IMG_BGR if there was none, tight raw frames; needs a rectification set; per pair the bytes of both raw frames +
 * 2*3*N written, plus both views' internal maps, 2*8*N, once per wave; while a resize is set the resize ingestion, per
 * pair the bytes of both raw frames + 2*3*N written, no maps), 15 = the AD-census cost computed inside the first
 * horizontal arm sum, which the fused pipeline runs in place of ids 0 and 1 (per pair one volume written, 24*N bytes of
 * packed pixels and census words read, plus the horizontal window records), 16 = the scanline pass along -y with the WTA
 * as its epilogue, which the pipeline runs in place of ids 4 and 5 where nothing else reads the optimised volume (per pair
 * one volume read, disp_l and the right view's partial records written), 17 = the fold of those records into the
 * right-view map (records read, disp_r written).
 * algorithmic_bytes (optional) receives the bytes one launch must move (SURVEY.md section 8d). */
int adc_profile_kernel(adc_engine* e, int32_t kernel_id, int32_t reps, float* avg_ms, double* algorithmic_bytes);

/* Output side of the reference's demo program (main.cpp, outside ADCensusStereo itself; SURVEY.md 8f):
 *   adc_render_disparity = ShowDisparityMap / SaveDisparityMap (main.cpp:147-207): the 8-bit image
 *       uchar((|d| - min) / (max - min) * 255) with min / max over the valid pixels (0 where d is Invalid_Float),
 *       and that image through cv::COLORMAP_JET as packed BGR.  gray8 [W*H], jet_bgr [W*H*3], min_max [2]; any
 *       of the three may be NULL.  The file encoding (PNG) stays with the caller.
 *   adc_disparity_cloud = SaveDisparityCloud (main.cpp:209-230): one record (x, y, |d|, r, g, b) as six floats per
 *       valid pixel in raster order; `cloud` must hold W*H*6 floats, *n_points receives the record count.  The
 *       text formatting ("%f %f %f %d %d %d") stays with the caller.
 * Host pointers; the engine's lane 0 is used, so not concurrently with adc_match on the same engine. */
int adc_render_disparity(adc_engine* e, const float* disp, uint8_t* gray8, uint8_t* jet_bgr, float* min_max);
int adc_disparity_cloud(adc_engine* e, const uint8_t* img_left, const float* disp, float* cloud, int32_t* n_points);

const char* adc_last_error(void);
const char* adc_version(void);

/* ---- debug taps (parity tests) -------------------------------------------------------------
 * adc_debug_run executes the production pipeline on ONE pair up to and including `last_stage` and leaves every
 * buffer live (a run that stops between two aggregation iterations, AGG1..AGG3, takes the eight single aggregation
 * passes instead of the fused same-axis passes, whose intermediate never reaches memory); adc_debug_get copies a buffer out in the
 * reference's layout ([H][W][D] with d fastest for the volumes).  Stage and tap ids follow the
 * reference's structure: stages are the steps of Match / Aggregate / Optimize / Refine, taps are
 * the private members a parity test wants to see (cost_computor.h:80-91, cross_aggregator.h:88-102,
 * ADCensusStereo.h:88-92, multistep_refiner.h:96-99).
 * After a call that ran all four scanline passes, VOL_AGGR is the SO4 volume where the last pass stored it: after
 * adc_debug_run*, and after a match call that exports the OPT volume, asks for a MIN_COST or PEAK_RATIO map, runs the
 * discontinuity adjustment, runs on an engine with ADC_DBG_UNFUSED_SO_WTA, or whose shape the fused pass does not pay
 * for.  After any other match call (Cone under the default options, for one) that pass took the WTA as its epilogue
 * and stored no volume, and VOL_AGGR fails with ADC_ERR_ARG.  VOL_INIT does not depend on that choice. */
enum {
    ADC_STAGE_COST = 0, ADC_STAGE_ARMS = 1,
    ADC_STAGE_AGG1 = 2, ADC_STAGE_AGG2 = 3, ADC_STAGE_AGG3 = 4, ADC_STAGE_AGG4 = 5,
    ADC_STAGE_SO1 = 6, ADC_STAGE_SO2 = 7, ADC_STAGE_SO3 = 8, ADC_STAGE_SO4 = 9,
    ADC_STAGE_WTA = 10, ADC_STAGE_OUTLIER = 11, ADC_STAGE_VOTE = 12, ADC_STAGE_INTERP = 13,
    ADC_STAGE_DISC = 14, ADC_STAGE_MEDIAN = 15, ADC_STAGE_COUNT = 16
};
enum {
    ADC_TAP_GRAY_L = 0, ADC_TAP_GRAY_R = 1,       /* u8  [H][W] */
    ADC_TAP_CENSUS_L = 2, ADC_TAP_CENSUS_R = 3,   /* u64 [H][W] */
    ADC_TAP_VOL_INIT = 4, ADC_TAP_VOL_AGGR = 5,   /* f32 [H][W][D]  (reference cost_init_ / cost_aggr_) */
    ADC_TAP_ARMS = 6,                             /* u8  [H][W][4]  left,right,top,bottom */
    ADC_TAP_SUPCNT_H = 7, ADC_TAP_SUPCNT_V = 8,   /* u16 [H][W] */
    ADC_TAP_DISP_L = 9, ADC_TAP_DISP_R = 10,      /* f32 [H][W] */
    ADC_TAP_MISMATCHES = 11, ADC_TAP_OCCLUSIONS = 12, /* i32 [n][2] (x,y), list order */
    ADC_TAP_COUNT = 13
};
int adc_debug_run(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right, int32_t last_stage);
/* adc_debug_run with a caller-supplied cost volume (host pointer, layouts and domain as for adc_match_cost) */
int adc_debug_run_cost(adc_engine* e, const uint8_t* img_left, const uint8_t* img_right,
                       const void* cost, int32_t layout, int32_t dtype, int32_t last_stage);
/* region-voting statistics of pair 0 of the last run: out[0],out[1] = remaining mismatch / occlusion
 * list sizes, out[2] = fixed-point rounds, out[3] = vote evaluations, out[4..8] = microseconds spent building the
 * adjacency lists / in the whole voting kernel / deriving / pushing / collecting, out[9] = forward-list entries
 * reserved, out[10],out[11] = voting list sizes, out[12] = vote changes, out[13] = 1 when the adjacency lists were
 * used (0: the inverse regions were enumerated), out[14] = adjacency entries, out[15] = forward-list room */
int adc_debug_counters(adc_engine* e, int32_t out[16]);
/* returns the tap's size in bytes (also when dst is NULL or cap is too small), 0 on error */
size_t adc_debug_get(adc_engine* e, int32_t tap, void* dst, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* ADCENSUS_B200_H_ */
