// img_format.h -- the image input formats (ADC_IMG_*, include/adcensus_b200.h): which codes exist, their family, the
// parameters each family's reader takes, and the geometry and descriptor rules of a view.  The one place that knows
// them: engine.cu asks it for the descriptor checks and the host staging, the dispatch of the ingestion kernel
// (k_image.cu) and its instantiations are generated from its list, and the readers (k_image.cuh) take
// their constants from it.  Plain C++ with no CUDA dependency, so g++ compiles it as well as nvcc.
#pragma once

#include "../../include/adcensus_b200.h"

#ifdef __CUDACC__
#define IMG_HD __host__ __device__
#else
#define IMG_HD
#endif

// Every format once, by family.  The family decides the reader and the translation unit that instantiates its
// kernels: packed and planar u8 pixels (k_image.cu), 8-bit Bayer mosaics (k_bayer.cu), YUV frames
// (k_yuv.cu; k_yuv_video.cu and k_yuv_encodings.cu for the newer containers and the encoding flags) and the
// high-bit-depth mono and Bayer frames (k_rawdepth.cu).
#define ADC_IMG_PACKED_FORMATS(X) \
    X(ADC_IMG_BGR) X(ADC_IMG_RGB) X(ADC_IMG_BGRA) X(ADC_IMG_RGBA) X(ADC_IMG_GRAY) X(ADC_IMG_RGB_PLANAR)
#define ADC_IMG_BAYER_FORMATS(X) X(ADC_IMG_BAYER_RGGB) X(ADC_IMG_BAYER_GRBG) X(ADC_IMG_BAYER_BGGR) X(ADC_IMG_BAYER_GBRG)
#define ADC_IMG_YUV_FORMATS(X) X(ADC_IMG_NV12) X(ADC_IMG_NV21) X(ADC_IMG_YUYV) X(ADC_IMG_UYVY) X(ADC_IMG_YVYU)
#define ADC_IMG_YUV_VIDEO_FORMATS(X) X(ADC_IMG_I420) X(ADC_IMG_YV12) X(ADC_IMG_P016)
#define ADC_IMG_RAWDEPTH_FORMATS(X)                                                                                    \
    X(ADC_IMG_MONO10) X(ADC_IMG_BAYER_RG10) X(ADC_IMG_BAYER_GR10) X(ADC_IMG_BAYER_BG10) X(ADC_IMG_BAYER_GB10)          \
    X(ADC_IMG_MONO12) X(ADC_IMG_BAYER_RG12) X(ADC_IMG_BAYER_GR12) X(ADC_IMG_BAYER_BG12) X(ADC_IMG_BAYER_GB12)          \
    X(ADC_IMG_MONO16) X(ADC_IMG_BAYER_RG16) X(ADC_IMG_BAYER_GR16) X(ADC_IMG_BAYER_BG16) X(ADC_IMG_BAYER_GB16)          \
    X(ADC_IMG_MONO10P) X(ADC_IMG_BAYER_RG10P) X(ADC_IMG_BAYER_GR10P) X(ADC_IMG_BAYER_BG10P) X(ADC_IMG_BAYER_GB10P)     \
    X(ADC_IMG_MONO12P) X(ADC_IMG_BAYER_RG12P) X(ADC_IMG_BAYER_GR12P) X(ADC_IMG_BAYER_BG12P) X(ADC_IMG_BAYER_GB12P)
#define ADC_IMG_FORMATS(X)                                                                                             \
    ADC_IMG_PACKED_FORMATS(X) ADC_IMG_BAYER_FORMATS(X) ADC_IMG_YUV_FORMATS(X) ADC_IMG_YUV_VIDEO_FORMATS(X)             \
    ADC_IMG_RAWDEPTH_FORMATS(X)

// The codes of a YUV container F with a colour encoding flag (ADC_IMG_YUV_BT709, ADC_IMG_YUV_FULL_RANGE, both), each
// its own kernel instantiation (k_yuv_encodings.cu for the formats of k_yuv.cu, k_yuv_video.cu for the others), and
// every code a kernel is instantiated for: the formats without a flag, then the YUV formats with one.
#define IMG_YUV_FLAGGED(X, F) \
    X(F | ADC_IMG_YUV_BT709) X(F | ADC_IMG_YUV_FULL_RANGE) X(F | ADC_IMG_YUV_BT709 | ADC_IMG_YUV_FULL_RANGE)
#define ADC_IMG_YUV_FLAGGED_FORMATS(X)                                                                                 \
    IMG_YUV_FLAGGED(X, ADC_IMG_NV12) IMG_YUV_FLAGGED(X, ADC_IMG_NV21) IMG_YUV_FLAGGED(X, ADC_IMG_YUYV)                   \
    IMG_YUV_FLAGGED(X, ADC_IMG_UYVY) IMG_YUV_FLAGGED(X, ADC_IMG_YVYU)
#define ADC_IMG_YUV_VIDEO_FLAGGED_FORMATS(X) \
    IMG_YUV_FLAGGED(X, ADC_IMG_I420) IMG_YUV_FLAGGED(X, ADC_IMG_YV12) IMG_YUV_FLAGGED(X, ADC_IMG_P016)
#define ADC_IMG_CODES(X) ADC_IMG_FORMATS(X) ADC_IMG_YUV_FLAGGED_FORMATS(X) ADC_IMG_YUV_VIDEO_FLAGGED_FORMATS(X)

enum { IMG_UNKNOWN, IMG_PACKED, IMG_BAYER, IMG_YUV, IMG_RAWDEPTH };

// A format code is a container (bits 0..7) and, for the YUV containers only, the colour encoding flags (bits 8, 9).
// Everything below but img_code_ok takes a code that passed img_code_ok and looks at its container alone, except
// img_encoding.
IMG_HD constexpr int img_base(int f) { return f & 0xff; }
IMG_HD constexpr int img_encoding(int f) { return f >> 8 & 3; }   // bit 0: BT.709, bit 1: full range

#define IMG_CASE(F) case F:
IMG_HD constexpr int img_family(int f) {
    switch (img_base(f)) {
        ADC_IMG_PACKED_FORMATS(IMG_CASE) return IMG_PACKED;
        ADC_IMG_BAYER_FORMATS(IMG_CASE) return IMG_BAYER;
        ADC_IMG_YUV_FORMATS(IMG_CASE) ADC_IMG_YUV_VIDEO_FORMATS(IMG_CASE) return IMG_YUV;
        ADC_IMG_RAWDEPTH_FORMATS(IMG_CASE) return IMG_RAWDEPTH;
        default: return IMG_UNKNOWN;
    }
}
#undef IMG_CASE

// 0: a known container with no flags or a YUV container with encoding flags; 1: an unknown container or a bit set above
// the flags (negative codes included); 2: a flag on a container that is not YUV.
IMG_HD constexpr int img_code_error(int f) {
    return (f & ~0x3ff) || img_family(f) == IMG_UNKNOWN ? 1 : f > 0xff && img_family(f) != IMG_YUV ? 2 : 0;
}

// ---- family parameters ----

// YUV 4:2:0: a luma plane and one interleaved chroma plane (NV12, NV21; P016 in 16-bit words), or a luma plane and two
// chroma planes of half its row pitch (I420, YV12).  The other YUV formats are packed 4:2:2 macropixels.
IMG_HD constexpr bool img_yuv_planar(int f) { return img_base(f) == ADC_IMG_I420 || img_base(f) == ADC_IMG_YV12; }
IMG_HD constexpr bool img_yuv420(int f) {
    return img_base(f) == ADC_IMG_NV12 || img_base(f) == ADC_IMG_NV21 || img_base(f) == ADC_IMG_P016 || img_yuv_planar(f);
}

// High bit depth: the code is ADC_IMG_MONO10 + 5 * container + colour.  Container 0 / 1 / 2 = one sample per
// little-endian 16-bit word with 10 / 12 / 16 significant bits, 3 / 4 = the PFNC 10p / 12p bit streams; colour 0 = mono,
// 1..4 = the Bayer patterns in the order of ADC_IMG_BAYER_RGGB ... _GBRG.
IMG_HD constexpr int img_container(int f) { return (f - ADC_IMG_MONO10) / 5; }
IMG_HD constexpr int img_bits(int f) { return img_container(f) == 2 ? 16 : img_container(f) % 3 == 0 ? 10 : 12; }
// The formats with one sample per little-endian 16-bit word, which the kernels load whole: the 16-bit containers and
// P016.
IMG_HD constexpr bool img_words(int f) {
    return (img_family(f) == IMG_RAWDEPTH && img_container(f) <= 2) || img_base(f) == ADC_IMG_P016;
}

// Mosaics: an 8-bit Bayer code is its own pattern and keeps its samples as they are; a high-bit-depth Bayer code has
// the pattern of its colour and reduces its samples by shift = bits - 8.  `r_site` is the position of the pattern's R
// site in its 2 x 2 block (bit 0: its column, bit 1: its row).
IMG_HD constexpr bool img_mosaic(int f) {
    return img_family(f) == IMG_BAYER || (img_family(f) == IMG_RAWDEPTH && (f - ADC_IMG_MONO10) % 5 != 0);
}
IMG_HD constexpr int img_pattern(int f) {
    return img_family(f) == IMG_BAYER ? f : ADC_IMG_BAYER_RGGB + (f - ADC_IMG_MONO10) % 5 - 1;
}
IMG_HD constexpr int img_shift(int f) { return img_family(f) == IMG_BAYER ? 0 : img_bits(f) - 8; }
IMG_HD constexpr int img_r_site(int pattern) {
    return pattern == ADC_IMG_BAYER_RGGB ? 0 : pattern == ADC_IMG_BAYER_GRBG ? 1 : pattern == ADC_IMG_BAYER_GBRG ? 2 : 3;
}

// ---- geometry and descriptor rules ----

// The tight row pitch of a w pixel wide view (of each plane of a planar image, of the luma plane of NV12 / NV21), and
// the rule's name in error messages.
IMG_HD constexpr long long img_row_pitch(int f, long long w) {
    switch (img_family(f)) {
        case IMG_YUV: return (img_yuv420(f) && !img_words(f) ? 2 : 4) * ((w + 1) / 2);
        case IMG_RAWDEPTH: return img_words(f) ? 2 * w : (img_bits(f) * w + 7) / 8;
        default: return (f == ADC_IMG_BGR || f == ADC_IMG_RGB ? 3 : f == ADC_IMG_BGRA || f == ADC_IMG_RGBA ? 4 : 1) * w;
    }
}
inline const char* img_row_rule(int f) {
    switch (img_family(f)) {
        case IMG_YUV: return img_yuv420(f) && !img_words(f) ? "2 * ceil(W / 2)" : "4 * ceil(W / 2)";
        case IMG_RAWDEPTH: return img_words(f) ? "2 * W" : img_bits(f) == 10 ? "ceil(10 * W / 8)" : "ceil(12 * W / 8)";
        default: return "W * bytes per pixel";
    }
}

// Planes of a view: the R, G and B planes of a planar image, plane_pitch apart; the luma and chroma planes of NV12 /
// NV21 / P016, the chroma plane at plane_pitch; the luma and the two chroma planes of I420 / YV12, the first chroma
// plane at plane_pitch and the second right after it; one for every other format.  Only a format with more than one
// may be given a non-zero plane_pitch.  Plane c of an h row view has h rows, but ceil(h / 2) for a 4:2:0 chroma plane,
// and rows row_pitch apart, but row_pitch / 2 for an I420 / YV12 chroma plane.
IMG_HD constexpr int img_planes(int f) {
    return f == ADC_IMG_RGB_PLANAR || img_yuv_planar(f) ? 3 : img_yuv420(f) ? 2 : 1;
}
IMG_HD constexpr long long img_plane_rows(int f, int c, long long h) { return c && img_yuv420(f) ? (h + 1) / 2 : h; }
IMG_HD constexpr long long img_plane_row_pitch(int f, int c, long long row_pitch) {
    return c && img_yuv_planar(f) ? row_pitch / 2 : row_pitch;
}
IMG_HD constexpr long long img_plane_offset(int f, int c, long long h, long long row_pitch, long long plane_pitch) {
    return c == 2 && img_yuv_planar(f) ? plane_pitch + (h + 1) / 2 * (row_pitch / 2) : c * plane_pitch;
}

// The footprint of an h row view into *foot, false when it overflows: h * row_pitch for one plane; for a planar image
// 3 * plane_pitch, the last plane's padding included; for 4:2:0 plane_pitch and the ceil(h / 2) chroma rows of
// row_pitch bytes (one interleaved plane, or the two planes of half the pitch).
inline bool img_footprint(int f, long long h, long long row_pitch, long long plane_pitch, long long* foot) {
    if (img_yuv420(f)) {
        long long chroma = 0;
        return !__builtin_mul_overflow(img_plane_rows(f, 1, h), row_pitch, &chroma) &&
               !__builtin_add_overflow(plane_pitch, chroma, foot);
    }
    if (f == ADC_IMG_RGB_PLANAR) return !__builtin_mul_overflow(3ll, plane_pitch, foot);
    return !__builtin_mul_overflow(h, row_pitch, foot);
}

// A view's geometry: format, row pitch, plane pitch (0 for one plane) and the bytes from one pair's view to the next.
struct AdcImageGeom {
    int format;
    long long row_pitch, plane_pitch, image_stride;
};

// The tight layout of a w x h view in `format`: tight rows, planes back to back, and the footprint in image_stride.
inline AdcImageGeom adc_image_tight(int format, long long w, long long h) {
    const long long rp = img_row_pitch(format, w), plane = h * rp;
    long long foot = plane;
    img_footprint(format, h, rp, plane, &foot);
    return AdcImageGeom{format, rp, img_planes(format) > 1 ? plane : 0, foot};
}

// The bytes of a w x h view the ingestion kernels read: the tight footprint without the padding sample of odd-width
// 4:2:0 luma rows.
inline long long adc_image_read_bytes(int format, long long w, long long h) {
    if (img_yuv420(format)) return (img_words(format) ? 2 : 1) * (w * h + 2 * ((w + 1) / 2) * ((h + 1) / 2));
    return adc_image_tight(format, w, h).image_stride;
}
