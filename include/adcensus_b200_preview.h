/* include/adcensus_b200_preview.h -- previews: the engine's maps rendered as 8-bit frames for a display or a video
 * encoder, on the GPU, bit-exact with OpenCV.
 *
 * The output side of a stereo camera pipeline, kept apart from the matching ABI of adcensus_b200.h: nothing here is
 * part of a match, no entry point below touches an engine buffer, and a caller that never shows or records a map
 * never needs this header.  It adds entry points to the same library (libadcensus_b200.so) and takes the engine,
 * adc_image_desc and the ADC_IMG_* codes of adcensus_b200.h, which it includes.
 */
#ifndef ADCENSUS_B200_PREVIEW_H_
#define ADCENSUS_B200_PREVIEW_H_

#include "adcensus_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- previews ---------------------------------------------------------------------------------------------
 * f32 [H][W] maps of the engine's size (final maps, the WTA and confidence side maps, ADC_REPROJ_DEPTH, or any other)
 * rendered as 8-bit frames a display or a video encoder takes, at any size.  For every map m the frame is bit for bit
 *   g   = cv2.normalize(m, None, 0, 255, NORM_MINMAX, CV_8U, mask = isfinite(m))    (ADC_PREVIEW_MINMAX)
 *         m.convertTo(CV_8U, alpha, beta)                                           (ADC_PREVIEW_FIXED)
 *   bgr = cv2.applyColorMap(g, colormap) (or (g, g, g) for ADC_COLORMAP_NONE), invalid pixels set to invalid_bgr
 *   out = cv2.cvtColor(cv2.resize(bgr, (dst_width, dst_height), interpolation = INTER_NEAREST), COLOR_BGR2<format>)
 * Rules, step by step:
 *   1. A pixel is valid when it is finite: the engine's +inf and the NaN depth of an invalid disparity are invalid.
 *   2. (scale, shift), in IEEE double without fused multiply-add: MINMAX takes cv::normalize's, with smin / smax the
 *      minimum and maximum of the valid pixels: scale = 255 * (smax - smin > DBL_EPSILON ? 1 / (smax - smin) : 0),
 *      shift = 0 - smin * scale.  A map with no valid pixel has scale = shift = 0 (cv::minMaxIdx over an empty mask
 *      gives 0 and 0), which changes nothing: every pixel is invalid.  A constant map gives g = 0.  FIXED takes
 *      (alpha, beta) as given; a negative alpha inverts (near = warm for depth with alpha = -255 / z_far, beta = 255).
 *   3. g = sat_u8(t) with t = round_half_even(fmaf(m, (float)scale, (float)shift)): one fused multiply-add in float,
 *      rounded once; sat_u8 clamps to 0..255, except that a t outside int32 (including +-inf) gives 0, as x86's
 *      cvtps2dq makes it INT_MIN before the saturating packs.  This is OpenCV's cvt32f8u as its AVX2 and AVX-512
 *      dispatch computes it (v_fma in the vector loop, a contracted multiply-add in the scalar tail), the dispatch the
 *      pip wheels take on an AVX2 CPU; a build or CPU whose best dispatch is the SSE baseline rounds m * scale before
 *      adding shift, and its g may then differ by one for a few values per map.
 *   4. bgr = the 256-entry table of cv::applyColorMap(arange(256), colormap) at g, or (g, g, g); invalid pixels
 *      invalid_bgr.
 *   5. INTER_NEAREST, per axis with n_src -> n_dst (n_src = W or H): the destination index d reads source index
 *      min(floor(d * (1.0 / ((double)n_dst / n_src))), n_src - 1), in IEEE double.  The normalisation of step 2 uses the
 *      engine-size map, so the resize only picks pixels.
 *   6. Format, per output pixel (B, G, R), integer arithmetic:
 *        ADC_IMG_BGR / BGRA / RGBA  the pixel, A = 255 (COLOR_BGR2BGRA / COLOR_BGR2RGBA)
 *        ADC_IMG_GRAY               (9798 R + 19235 G + 3735 B + 2^14) >> 15 (COLOR_BGR2GRAY)
 *        ADC_IMG_I420 / YV12        Y = sat_u8((269484 R + 528482 G + 102760 B + 2^19 + (16 << 20)) >> 20) for every
 *                                   pixel; per 2x2 block, from its top-left pixel alone,
 *                                   U = sat_u8((-155188 R - 305135 G + 460324 B + 2^19 + (128 << 20)) >> 20),
 *                                   V = sat_u8((460324 R - 385875 G - 74448 B + 2^19 + (128 << 20)) >> 20)
 *                                   (COLOR_BGR2YUV_I420 / COLOR_BGR2YUV_YV12: BT.601, limited range)
 *        ADC_IMG_NV12 / NV21        the I420 samples with U and V interleaved in that order (V first for NV21)
 *      4:2:0 formats need an even dst_width and dst_height, as OpenCV does.
 * adc_render_disparity keeps the reference demo's rule, which differs: it takes |d|, starts min / max at +-W, divides,
 * and truncates; a preview keeps the sign, multiplies by OpenCV's scale and rounds half to even.
 * Destination: an adc_image_desc over the dst_width x dst_height frame, formats ADC_IMG_BGR, BGRA, RGBA, GRAY, NV12,
 * NV21, I420 and YV12 without ADC_IMG_YUV_* flags, with the pitches, zero defaults and rules of the input frames
 * (row_pitch, plane_pitch = the offset of the (first) chroma plane, image_stride from frame i to frame i + 1).  A frame
 * may thus be written into an encoder surface as it is, or beside another view in a side-by-side frame (a pointer
 * offset and a pitch); only the frame's own bytes are written, and any alignment is accepted (aligned rows are stored
 * in whole words).  NULL = tight packed BGR.
 * Fails with ADC_ERR_ARG naming the field.  Before the engine is checked: p NULL; an unknown colormap, range or format,
 * or a format flag; non-zero reserved bytes (p and the descriptor); a NaN or infinite alpha / beta, or non-zero ones
 * under MINMAX; dst_width / dst_height outside 0..32767, or odd for a 4:2:0 format; a negative pitch, or an odd
 * row_pitch for I420 / YV12; NULL maps or dst; a negative n; on the device entry maps not 4-byte aligned or d_work not
 * 4-byte aligned.  After it: an engine-size (0) dimension that is odd for a 4:2:0 format, the pitches against the
 * frame size (as for input frames), and on the device entry a work_bytes below adc_preview_workspace_bytes with
 * MINMAX, or d_work NULL with MINMAX and n > 0.  FIXED needs no workspace. */
enum { ADC_PREVIEW_MINMAX = 0, ADC_PREVIEW_FIXED = 1 };
enum { ADC_COLORMAP_NONE = -1 };   /* gray (g, g, g); 0..21 are cv::ColormapTypes, COLORMAP_AUTUMN .. COLORMAP_DEEPGREEN */
#define ADC_COLORMAP_COUNT 22
typedef struct adc_preview_params {
    int32_t colormap;        /* ADC_COLORMAP_NONE or 0..21, the value of cv::COLORMAP_* */
    int32_t range;           /* ADC_PREVIEW_MINMAX or ADC_PREVIEW_FIXED */
    double  alpha, beta;     /* FIXED: convertTo's scale and shift; MINMAX: 0 */
    int32_t dst_width;       /* frame size, 0 = the engine's W / H; otherwise resized with INTER_NEAREST */
    int32_t dst_height;
    uint8_t invalid_bgr[3];  /* colour of invalid pixels, B, G, R */
    uint8_t reserved_[5];    /* must be zero */
    int64_t reserved;        /* must be zero */
} adc_preview_params;        /* 48 bytes */

/* *out = the device workspace adc_preview_batch_device needs for n maps with MINMAX: 8 * n bytes. */
int adc_preview_workspace_bytes(const adc_engine* e, int32_t n, size_t* out);
/* n maps in device memory (map i at element i*H*W) rendered into n frames at d_dst (frame i at byte i*image_stride),
 * using only the caller's workspace (MINMAX; the call initialises it itself): MINMAX enqueues one cudaMemsetAsync of
 * the workspace, one min / max launch and one colour launch, FIXED one colour launch, on `stream` (a cudaStream_t,
 * NULL = legacy default stream), whatever n and the content, not synchronised, no host round trip.  No engine buffer
 * is touched, so the call may run next to the engine's batch calls; the maps must be complete in `stream`'s order (in
 * pipelined mode, after adc_join on that stream).  n == 0 is a no-op. */
int adc_preview_batch_device(adc_engine* e, int32_t n, const float* d_maps, const adc_preview_params* p, void* d_dst,
                             const adc_image_desc* dst, void* d_work, size_t work_bytes, void* stream);
/* One map, host pointers (`dst` laid out by `desc`, image_stride unused), synchronous.  The map, the workspace and the
 * frame pass through the device staging of adc_match_volumes (allocated on first use, grown when needed; ADC_ERR_NOMEM
 * before any work if that fails), and only the frame's rows are copied back.  Not concurrently with another call on the
 * same engine. */
int adc_preview(adc_engine* e, const float* map, const adc_preview_params* p, void* dst, const adc_image_desc* desc);

#ifdef __cplusplus
}
#endif
#endif /* ADCENSUS_B200_PREVIEW_H_ */
