"""ctypes binding of the C ABI (include/adcensus_b200.h) and the Python mirror of the reference's
ADCensusStereo class.  Every call goes through libadcensus_b200.so; nothing is computed in Python."""
from __future__ import annotations

import ctypes
from pathlib import Path

import numpy as np

Invalid_Float = float("inf")  # reference adcensus_types.h:33

STAGES = ["COST", "ARMS", "AGG1", "AGG2", "AGG3", "AGG4", "SO1", "SO2", "SO3", "SO4",
          "WTA", "OUTLIER", "VOTE", "INTERP", "DISC", "MEDIAN"]
STAGE = {n: i for i, n in enumerate(STAGES)}
TAPS = ["GRAY_L", "GRAY_R", "CENSUS_L", "CENSUS_R", "VOL_INIT", "VOL_AGGR", "ARMS", "SUPCNT_H",
        "SUPCNT_V", "DISP_L", "DISP_R", "MISMATCHES", "OCCLUSIONS"]
TAP = {n: i for i, n in enumerate(TAPS)}
_TAP_DTYPE = {"GRAY_L": np.uint8, "GRAY_R": np.uint8, "CENSUS_L": np.uint64, "CENSUS_R": np.uint64,
              "VOL_INIT": np.float32, "VOL_AGGR": np.float32, "ARMS": np.uint8, "SUPCNT_H": np.uint16,
              "SUPCNT_V": np.uint16, "DISP_L": np.float32, "DISP_R": np.float32,
              "MISMATCHES": np.int32, "OCCLUSIONS": np.int32}


class ADCensusOption(ctypes.Structure):
    """Mirror of the reference's ADCensusOption (adcensus_types.h:45-75): same fields, order,
    types and defaults; 60 bytes, passed to the C ABI as-is."""
    _fields_ = [("min_disparity", ctypes.c_int32), ("max_disparity", ctypes.c_int32),
                ("lambda_ad", ctypes.c_int32), ("lambda_census", ctypes.c_int32),
                ("cross_L1", ctypes.c_int32), ("cross_L2", ctypes.c_int32),
                ("cross_t1", ctypes.c_int32), ("cross_t2", ctypes.c_int32),
                ("so_p1", ctypes.c_float), ("so_p2", ctypes.c_float),
                ("so_tso", ctypes.c_int32), ("irv_ts", ctypes.c_int32),
                ("irv_th", ctypes.c_float), ("lrcheck_thres", ctypes.c_float),
                ("do_lr_check", ctypes.c_bool), ("do_filling", ctypes.c_bool),
                ("do_discontinuity_adjustment", ctypes.c_bool), ("_reserved", ctypes.c_uint8)]

    def __init__(self, **kw):
        super().__init__(0, 64, 10, 30, 34, 17, 20, 6, 1.0, 3.0, 15, 20, 0.4, 1.0, True, True, False, 0)
        for k, v in kw.items():
            if k not in dict(self._fields_):
                raise AttributeError(f"ADCensusOption has no field {k!r}")
            setattr(self, k, v)


assert ctypes.sizeof(ADCensusOption) == 60


class _Config(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int32), ("wave_pairs", ctypes.c_int32), ("lanes", ctypes.c_int32),
                ("debug_flags", ctypes.c_int32), ("reserved", ctypes.c_int32 * 12)]


# adc_config.debug_flags (test hooks)
DBG_NO_RAY_TABLE, DBG_VOTE_ENUM, DBG_VOTE_GLOBAL_STATE, DBG_UNFUSED_AGG, DBG_POISON = 1, 2, 4, 8, 16
DBG_UNFUSED_SO_WTA, DBG_FUSED_SO_WTA = 32, 64


def poison_flags(byte: int) -> int:
    """debug_flags that fill every lane arena with `byte` before each wave and call (ADC_DBG_POISON with
    ADC_DBG_POISON_BYTE(byte))."""
    return DBG_POISON | ((int(byte) & 0xff) << 8)

# cost-input mode (adc_match_cost*): volume layouts, element types and the value domain's ceiling
COST_HWD, COST_DHW = 0, 1
COST_F32, COST_F16, COST_BF16 = 0, 1, 2
COST_MAX = 65536.0
COST_LAYOUTS = {"hwd": COST_HWD, "dhw": COST_DHW}
COST_DTYPES = {"f32": COST_F32, "f16": COST_F16, "bf16": COST_BF16}

# volume export (adc_match_volumes*): which volume a request names
VOL_COST, VOL_AGGR, VOL_OPT = 0, 1, 2
VOL_STAGES = {"cost": VOL_COST, "aggr": VOL_AGGR, "opt": VOL_OPT}
_VOL_NP = {COST_F32: np.float32, COST_F16: np.float16, COST_BF16: np.uint16}


class VolumeOut(ctypes.Structure):
    """adc_volume_out: one exported volume (destination, ADC_VOL_* stage, layout, element type)."""
    _fields_ = [("dst", ctypes.c_void_p), ("stage", ctypes.c_int32), ("layout", ctypes.c_int32),
                ("dtype", ctypes.c_int32), ("reserved", ctypes.c_int32)]


# per-pixel side maps (adc_match_outputs*): which map a request names, and its element type
MAP_WTA_LEFT, MAP_WTA_RIGHT, MAP_OUTLIERS, MAP_MIN_COST, MAP_PEAK_RATIO = 0, 1, 2, 3, 4
MAP_KINDS = {"wta_left": MAP_WTA_LEFT, "wta_right": MAP_WTA_RIGHT, "outliers": MAP_OUTLIERS, "min_cost": MAP_MIN_COST,
             "peak_ratio": MAP_PEAK_RATIO}
_MAP_NP = {MAP_WTA_LEFT: np.float32, MAP_WTA_RIGHT: np.float32, MAP_OUTLIERS: np.uint8, MAP_MIN_COST: np.float32,
           MAP_PEAK_RATIO: np.float32}


class MapOut(ctypes.Structure):
    """adc_map_out: one requested side map (destination, ADC_MAP_* kind)."""
    _fields_ = [("dst", ctypes.c_void_p), ("kind", ctypes.c_int32), ("reserved", ctypes.c_int32)]


# image input formats (adc_match_images*): u8 pixels, packed or planar, matched exactly as the same pixels packed as BGR
IMG_BGR, IMG_RGB, IMG_BGRA, IMG_RGBA, IMG_GRAY, IMG_RGB_PLANAR = 0, 1, 2, 3, 4, 5
IMG_FORMATS = {"bgr": IMG_BGR, "rgb": IMG_RGB, "bgra": IMG_BGRA, "rgba": IMG_RGBA, "gray": IMG_GRAY,
               "rgb_planar": IMG_RGB_PLANAR}
IMG_CHANNELS = {IMG_BGR: 3, IMG_RGB: 3, IMG_BGRA: 4, IMG_RGBA: 4, IMG_GRAY: 1, IMG_RGB_PLANAR: 1}   # bytes per pixel (plane)
# Bayer mosaics, 1 byte per pixel, demosaiced as cv2.cvtColor does; the name is the view's own top-left 2x2 block
# (GenICam BayerRG8 = "bayer_rggb" = OpenCV's legacy COLOR_BayerBG2BGR)
IMG_BAYER_RGGB, IMG_BAYER_GRBG, IMG_BAYER_BGGR, IMG_BAYER_GBRG = 16, 17, 18, 19
BAYER_FORMATS = {"bayer_rggb": IMG_BAYER_RGGB, "bayer_grbg": IMG_BAYER_GRBG, "bayer_bggr": IMG_BAYER_BGGR,
                 "bayer_gbrg": IMG_BAYER_GBRG}
# YUV frames, converted as cv2.cvtColor(frame, COLOR_YUV2BGR_<name>) does (BT.601 limited range): NV12 / NV21 are a Y
# plane and an interleaved chroma plane at plane_pitch (video decoders), the others packed 4:2:2 (UVC cameras)
IMG_NV12, IMG_NV21, IMG_YUYV, IMG_UYVY, IMG_YVYU = 32, 33, 34, 35, 36
YUV_FORMATS = {"nv12": IMG_NV12, "nv21": IMG_NV21, "yuyv": IMG_YUYV, "uyvy": IMG_UYVY, "yvyu": IMG_YVYU}
# the YUV containers of video decoders: I420 / YV12 (a Y plane, then U and V planes, resp. V and U, of half the row
# pitch: FFmpeg yuv420p, PyAV, OpenCV's (H*3/2, W) I420 Mat) and P016 (NV12's layout in little-endian 16-bit words, the
# samples MSB-aligned: NVDEC's 10- / 12- / 16-bit surface, FFmpeg p016le / p010le)
IMG_I420, IMG_YV12, IMG_P016 = 38, 39, 40
YUV_VIDEO_FORMATS = {"i420": IMG_I420, "yv12": IMG_YV12, "p016": IMG_P016}
# colour encoding flags, OR-ed into the code of any YUV format (YUV_FORMATS, YUV_VIDEO_FORMATS); no flag is BT.601
# limited range.  In a format name the encoding follows the container after a slash: "p016/bt709", "nv12/bt601_full".
IMG_YUV_BT709, IMG_YUV_FULL_RANGE = 0x100, 0x200
YUV_ENCODINGS = {"bt601": 0, "bt709": IMG_YUV_BT709, "bt601_full": IMG_YUV_FULL_RANGE,
                 "bt709_full": IMG_YUV_BT709 | IMG_YUV_FULL_RANGE}
# high-bit-depth mono and Bayer frames under their GenICam PFNC names, reduced to 8 bits as cv2.convertScaleAbs(v,
# alpha=2**-(bits - 8)) does (Bayer: after cv2.cvtColor on the uint16 mosaic): one sample per little-endian uint16 with
# 10, 12 or 16 significant bits ("u16"), or the 10p / 12p bit streams ("p": 4 samples in 5 bytes, 2 in 3)
IMG_MONO10, IMG_BAYER_RG10, IMG_BAYER_GR10, IMG_BAYER_BG10, IMG_BAYER_GB10 = 64, 65, 66, 67, 68
IMG_MONO12, IMG_BAYER_RG12, IMG_BAYER_GR12, IMG_BAYER_BG12, IMG_BAYER_GB12 = 69, 70, 71, 72, 73
IMG_MONO16, IMG_BAYER_RG16, IMG_BAYER_GR16, IMG_BAYER_BG16, IMG_BAYER_GB16 = 74, 75, 76, 77, 78
IMG_MONO10P, IMG_BAYER_RG10P, IMG_BAYER_GR10P, IMG_BAYER_BG10P, IMG_BAYER_GB10P = 79, 80, 81, 82, 83
IMG_MONO12P, IMG_BAYER_RG12P, IMG_BAYER_GR12P, IMG_BAYER_BG12P, IMG_BAYER_GB12P = 84, 85, 86, 87, 88
# name -> (code, significant bits, container)
RAW_DEPTH_FORMATS = {f"{colour}{suffix}": (IMG_MONO10 + 5 * k + c, bits, container)
                     for k, (suffix, bits, container) in enumerate((("10", 10, "u16"), ("12", 12, "u16"), ("16", 16, "u16"),
                                                                    ("10p", 10, "p"), ("12p", 12, "p")))
                     for c, colour in enumerate(("mono", "bayer_rg", "bayer_gr", "bayer_bg", "bayer_gb"))}
_RAW_DEPTH = {code: (bits, container) for code, bits, container in RAW_DEPTH_FORMATS.values()}


class ImageDesc(ctypes.Structure):
    """adc_image_desc: format (IMG_*) and byte pitches of the images of one call; zero pitches mean tight."""
    _fields_ = [("format", ctypes.c_int32), ("reserved", ctypes.c_int32), ("row_pitch", ctypes.c_int64),
                ("plane_pitch", ctypes.c_int64), ("image_stride", ctypes.c_int64)]


assert ctypes.sizeof(ImageDesc) == 32


def image_desc(format="bgr", row_pitch=0, plane_pitch=0, image_stride=0) -> ImageDesc:
    """An ImageDesc from a format name or IMG_* code and byte pitches (0 = tight)."""
    return ImageDesc(_img_format(format), 0, int(row_pitch), int(plane_pitch), int(image_stride))


_IMG_NAMES = {**IMG_FORMATS, **BAYER_FORMATS, **YUV_FORMATS, **YUV_VIDEO_FORMATS,
              **{k: v[0] for k, v in RAW_DEPTH_FORMATS.items()}}
_YUV_CODES = set(YUV_FORMATS.values()) | set(YUV_VIDEO_FORMATS.values())


def _img_format(v) -> int:
    """The code of a format name ("i420", or a YUV container and an encoding: "i420/bt709") or IMG_* code."""
    if isinstance(v, str):
        name, _, enc = v.partition("/")
        if name not in _IMG_NAMES or (enc and (enc not in YUV_ENCODINGS or _IMG_NAMES[name] not in _YUV_CODES)):
            raise ValueError(f"unknown image format {v!r} (one of {sorted(_IMG_NAMES)}; a YUV format may be followed by "
                             f"/ and one of {sorted(YUV_ENCODINGS)})")
        return _IMG_NAMES[name] | YUV_ENCODINGS.get(enc, 0)
    return int(v)


def _image_view_desc(a: np.ndarray, fmt: int, H: int, W: int) -> ImageDesc:
    """The descriptor of one numpy view of an image: [H][W][C] (packed), [H][W] (gray, Bayer), [3][H][W] (planar R,
    G, B), [H + ceil(H/2)][2*ceil(W/2)] (NV12 / NV21: the luma rows, then the chroma rows; OpenCV's (H*3/2, W) Mat for
    even sizes; the same shape in uint16 words for P016), [H][2*ceil(W/2)][2] (4:2:2, OpenCV's CV_8UC2), uint16 [H][W]
    (the 16-bit containers) or [H][ceil(bits*W/8)] (10p / 12p: each row's bytes) with the pixels / channels of a row
    contiguous; the pitches come from the view's strides, so slices of a larger frame (crops, side-by-side halves) need
    no copy.  I420 / YV12: [H + ceil(H/2)][2*ceil(W/2)] as well (the luma rows, then the U and V planes, each
    ceil(H/2) rows of ceil(W/2) bytes), with contiguous rows: a chroma plane's rows are half a luma row apart, which a
    slice of a wider array does not hold.  A YUV format may carry the encoding flags (IMG_YUV_BT709, ...)."""
    base = fmt & 0xff if (fmt & 0xff) in _YUV_CODES else fmt
    bits, container = _RAW_DEPTH.get(fmt, (8, None))
    if base == IMG_P016:
        container = "u16"
    dtype = np.uint16 if container == "u16" else np.uint8
    if a.dtype != dtype:
        raise ValueError(f"images of format {fmt} must be {np.dtype(dtype)}, got {a.dtype}")
    C = IMG_CHANNELS.get(fmt, 1)
    if base in (IMG_NV12, IMG_NV21, IMG_P016, IMG_I420, IMG_YV12):
        shape, inner, pitches = (H + (H + 1) // 2, 2 * ((W + 1) // 2)), (a.itemsize,), (0, a.strides[0], H * a.strides[0])
        if base in (IMG_I420, IMG_YV12) and a.strides[0] != shape[1]:
            raise ValueError(f"an I420 / YV12 image needs contiguous rows (row stride {shape[1]}), got {a.strides}")
    elif container == "u16":
        shape, inner, pitches = (H, W), (2,), (0, a.strides[0], 0)
    elif container == "p":
        shape, inner, pitches = (H, (bits * W + 7) // 8), (1,), (0, a.strides[0], 0)
    elif fmt == IMG_RGB_PLANAR:
        shape, inner, pitches = (3, H, W), (1,), (0, a.strides[1], a.strides[0])
    elif fmt == IMG_GRAY or fmt in BAYER_FORMATS.values():
        shape, inner, pitches = (H, W), (1,), (0, a.strides[0], 0)
    elif base in YUV_FORMATS.values():
        shape, inner, pitches = (H, 2 * ((W + 1) // 2), 2), (2, 1), (0, a.strides[0], 0)
    else:
        shape, inner, pitches = (H, W, C), (C, 1), (0, a.strides[0], 0)
    if a.shape != shape:
        raise ValueError(f"expected an image of shape {shape} for format {fmt}, got {a.shape}")
    if tuple(a.strides[-len(inner):]) != inner or min(a.strides) < 0:
        raise ValueError(f"the pixels of an image row must be contiguous (strides {a.strides})")
    return ImageDesc(fmt, 0, pitches[1], pitches[2], 0)


def _image_pair_desc(left: np.ndarray, right: np.ndarray, fmt: int, H: int, W: int) -> ImageDesc:
    """The one descriptor of a left and a right numpy view (_image_view_desc), which need the same strides."""
    desc = _image_view_desc(left, fmt, H, W)
    if _image_view_desc(right, fmt, H, W).row_pitch != desc.row_pitch or \
            (fmt == IMG_RGB_PLANAR and right.strides != left.strides):
        raise ValueError(f"left and right must have the same strides, got {left.strides} and {right.strides}")
    return desc


# rectification on the way in (adc_set_rectification, adc_match_rectified*): remap tables as cv2.initUndistortRectifyMap
# returns them, float32 x / y planes or int16 (x, y) pairs + uint16 fractions
REMAP_F32, REMAP_FIXED = 0, 1
# resizing on the way in: the same entries over frames of another size, resized as cv2.resize with INTER_AREA (integer
# downscale factors) or INTER_LINEAR_EXACT
RESIZE_AREA, RESIZE_LINEAR_EXACT = 16, 17
RESIZE_INTERPOLATIONS = {"area": RESIZE_AREA, "linear_exact": RESIZE_LINEAR_EXACT}


class Remap(ctypes.Structure):
    """adc_remap: one view's map1 / map2 (host or device pointers) and their row pitches in bytes (0 = tight)."""
    _fields_ = [("map1", ctypes.c_void_p), ("map2", ctypes.c_void_p), ("map1_pitch", ctypes.c_int64),
                ("map2_pitch", ctypes.c_int64)]


class Rectification(ctypes.Structure):
    """adc_rectification: raw frame size, REMAP_* map type and both views' maps, or a RESIZE_* type and no maps."""
    _fields_ = [("src_width", ctypes.c_int32), ("src_height", ctypes.c_int32), ("map_type", ctypes.c_int32),
                ("reserved", ctypes.c_int32), ("view", Remap * 2)]


assert ctypes.sizeof(Remap) == 32 and ctypes.sizeof(Rectification) == 80


def _map_plane(a, H: int, W: int, pair: bool):
    """(pointer, row pitch in bytes, dtype name) of one remap plane: a numpy array or a torch tensor (CPU or CUDA) of
    shape [H][W] ([H][W][2] for the int16 pairs) whose rows are contiguous; the pitch comes from the row stride."""
    if hasattr(a, "data_ptr"):   # torch
        if not a.is_cuda:
            a = a.numpy()
        else:
            name = str(a.dtype).replace("torch.", "")
            es = a.element_size()
            shape, strides, ptr = tuple(a.shape), tuple(x * es for x in a.stride()), a.data_ptr()
    if isinstance(a, np.ndarray):
        name, es = a.dtype.name, a.dtype.itemsize
        shape, strides, ptr = a.shape, a.strides, a.ctypes.data
    want = (H, W, 2) if pair else (H, W)
    if shape != want:
        raise ValueError(f"expected a map of shape {want}, got {shape}")
    inner = (2 * es, es) if pair else (es,)
    if tuple(strides[1:]) != inner or strides[0] < 0:
        raise ValueError(f"the elements of a map row must be contiguous (strides {strides})")
    return ptr, strides[0], name


def _remap(maps, H: int, W: int):
    """(map type, Remap) of one view's (map1, map2) as cv2.initUndistortRectifyMap returns them: float32 [H][W] x and
    y, or int16 [H][W][2] and uint16 [H][W] (int16 accepted for a CUDA tensor, as the same bits)."""
    map1, map2 = maps
    pair = len(getattr(map1, "shape", ())) == 3
    p1, q1, t1 = _map_plane(map1, H, W, pair)
    p2, q2, t2 = _map_plane(map2, H, W, False)
    if not pair and (t1, t2) == ("float32", "float32"):
        return REMAP_F32, Remap(p1, p2, q1, q2)
    if pair and t1 == "int16" and t2 in ("uint16", "int16"):
        return REMAP_FIXED, Remap(p1, p2, q1, q2)
    raise ValueError(f"maps must be float32 [H][W] x2 or int16 [H][W][2] + uint16 [H][W], got {t1} and {t2}")


# reprojection to 3-D (adc_reproject*): which output a request names, and its element type
REPROJ_POINTS, REPROJ_DEPTH, REPROJ_DISP_S16 = 0, 1, 2
REPROJ_KINDS = {"points": REPROJ_POINTS, "depth": REPROJ_DEPTH, "disp_s16": REPROJ_DISP_S16}
_REPROJ_NP = {REPROJ_POINTS: np.float32, REPROJ_DEPTH: np.float32, REPROJ_DISP_S16: np.int16}


class ReprojectOut(ctypes.Structure):
    """adc_reproject_out: one requested reprojection output (destination, ADC_REPROJ_* kind)."""
    _fields_ = [("dst", ctypes.c_void_p), ("kind", ctypes.c_int32), ("reserved", ctypes.c_int32)]


assert ctypes.sizeof(ReprojectOut) == 16


def _q_matrix(Q):
    """ctypes double[16] of a 4x4 array-like, converted to float64 as cv::Mat::convertTo(CV_64F) does."""
    q = np.asarray(Q)
    if q.shape != (4, 4):
        raise ValueError(f"Q must be a 4x4 matrix, got shape {q.shape}")
    return (ctypes.c_double * 16)(*q.astype(np.float64).reshape(-1).tolist())


# speckle removal (adc_filter_speckles*): the map type, and the params struct
SPECKLE_S16, SPECKLE_F32 = 0, 1
SPECKLE_TYPES = {"s16": SPECKLE_S16, "f32": SPECKLE_F32}


class SpeckleParams(ctypes.Structure):
    """adc_speckle_params: map type (ADC_SPECKLE_*), max_size, new_val, max_diff, reserved (zero)."""
    _fields_ = [("type", ctypes.c_int32), ("max_size", ctypes.c_int32), ("new_val", ctypes.c_double),
                ("max_diff", ctypes.c_double), ("reserved", ctypes.c_int64)]


assert ctypes.sizeof(SpeckleParams) == 32


# previews (adc_preview*): colormap names -> cv2.COLORMAP_* values ("none" = gray), the range rules, the output formats
COLORMAP_NONE = -1
COLORMAPS = {"none": COLORMAP_NONE, "autumn": 0, "bone": 1, "jet": 2, "winter": 3, "rainbow": 4, "ocean": 5, "summer": 6,
             "spring": 7, "cool": 8, "hsv": 9, "pink": 10, "hot": 11, "parula": 12, "magma": 13, "inferno": 14,
             "plasma": 15, "viridis": 16, "cividis": 17, "twilight": 18, "twilight_shifted": 19, "turbo": 20,
             "deepgreen": 21}
PREVIEW_MINMAX, PREVIEW_FIXED = 0, 1
PREVIEW_FORMATS = {"bgr": IMG_BGR, "bgra": IMG_BGRA, "rgba": IMG_RGBA, "gray": IMG_GRAY, "nv12": IMG_NV12,
                   "nv21": IMG_NV21, "i420": IMG_I420, "yv12": IMG_YV12}


class PreviewParams(ctypes.Structure):
    """adc_preview_params: colormap (COLORMAPS value), range (PREVIEW_*), alpha / beta (FIXED), frame size (0 = the
    engine's), the colour of invalid pixels (B, G, R) and reserved zeros."""
    _fields_ = [("colormap", ctypes.c_int32), ("range", ctypes.c_int32), ("alpha", ctypes.c_double),
                ("beta", ctypes.c_double), ("dst_width", ctypes.c_int32), ("dst_height", ctypes.c_int32),
                ("invalid_bgr", ctypes.c_uint8 * 3), ("reserved_", ctypes.c_uint8 * 5), ("reserved", ctypes.c_int64)]


assert ctypes.sizeof(PreviewParams) == 48


def preview_params(colormap="turbo", value_range=None, size=None, invalid=(0, 0, 0)) -> PreviewParams:
    """A PreviewParams from a colormap name or value, value_range None (MINMAX over the valid pixels) or (alpha, beta)
    (FIXED: convertTo's scale and shift), size None (the engine's) or (width, height), and the invalid colour (B, G, R)."""
    cm = _code(COLORMAPS, colormap, "colormap") if isinstance(colormap, str) else int(colormap)
    w, h = (0, 0) if size is None else (int(size[0]), int(size[1]))
    rng, a, b = (PREVIEW_MINMAX, 0.0, 0.0) if value_range is None else \
        (PREVIEW_FIXED, float(value_range[0]), float(value_range[1]))
    return PreviewParams(cm, rng, a, b, w, h, (ctypes.c_uint8 * 3)(*[int(v) for v in invalid]))


def preview_shape(format, width: int, height: int):
    """The numpy shape of one tight preview frame: [h][w][3] BGR, [h][w][4] BGRA / RGBA, [h][w] gray, [h * 3 / 2][w]
    for the 4:2:0 formats (OpenCV's I420 / YV12 Mat, NV12 / NV21 alike)."""
    f = _code(PREVIEW_FORMATS, format, "preview format") if isinstance(format, str) else int(format)
    return {IMG_BGR: (height, width, 3), IMG_BGRA: (height, width, 4), IMG_RGBA: (height, width, 4),
            IMG_GRAY: (height, width)}.get(f, (height * 3 // 2, width))


class CloudOut(ctypes.Structure):
    """adc_cloud_out: the destinations of a point cloud (points, colors or None, pixels or None, counts), the points
    per map they hold (capacity) and a reserved zero."""
    _fields_ = [("points", ctypes.c_void_p), ("colors", ctypes.c_void_p), ("pixels", ctypes.c_void_p),
                ("counts", ctypes.c_void_p), ("capacity", ctypes.c_int64), ("reserved", ctypes.c_int64)]


assert ctypes.sizeof(CloudOut) == 48


class AdcError(RuntimeError):
    pass


def lib_path() -> Path:
    return Path(__file__).resolve().parent / "lib" / "libadcensus_b200.so"


_lib = None


def load_library() -> ctypes.CDLL:
    """Loads libadcensus_b200.so.  Raises if it has not been built: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not p.exists():
        raise AdcError(f"{p} is missing: build it with adcensus_b200.build_library() "
                       "(nvcc, sm_90a).  This package has no CPU fallback.")
    L = ctypes.CDLL(str(p))
    vp, i32, u8p, f32p = ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p
    L.adc_default_option.argtypes = [ctypes.POINTER(ADCensusOption)]
    L.adc_create.argtypes = [i32, i32, ctypes.POINTER(ADCensusOption), ctypes.POINTER(_Config), ctypes.POINTER(vp)]
    L.adc_create.restype = ctypes.c_int
    L.adc_destroy.argtypes = [vp]
    L.adc_destroy.restype = None
    L.adc_match.argtypes = [vp, u8p, u8p, f32p]
    L.adc_get_right_disparity.argtypes = [vp, f32p]
    L.adc_match_batch.argtypes = [vp, i32, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.adc_match_batch_strided.argtypes = [vp, i32, u8p, u8p, f32p]
    L.adc_match_batch_device.argtypes = [vp, i32, u8p, u8p, f32p, vp]
    L.adc_match_batch_pinned_async.argtypes = [vp, i32, u8p, u8p, f32p, vp]
    L.adc_host_alloc.argtypes = [ctypes.c_size_t]
    L.adc_host_alloc.restype = vp
    L.adc_host_free.argtypes = [vp]
    L.adc_host_free.restype = None
    L.adc_synchronize.argtypes = [vp]
    L.adc_launch_count.argtypes = [vp]
    L.adc_launch_count.restype = ctypes.c_uint64
    L.adc_last_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float * 6)]
    L.adc_get_config.argtypes = [vp, ctypes.POINTER(_Config)]
    L.adc_profile_kernel.argtypes = [vp, i32, i32, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)]
    L.adc_set_pipelined.argtypes = [vp, i32]
    L.adc_join.argtypes = [vp, vp]
    L.adc_render_disparity.argtypes = [vp, f32p, u8p, u8p, f32p]
    L.adc_disparity_cloud.argtypes = [vp, u8p, f32p, f32p, ctypes.POINTER(ctypes.c_int32)]
    L.adc_last_error.restype = ctypes.c_char_p
    L.adc_version.restype = ctypes.c_char_p
    L.adc_debug_run.argtypes = [vp, u8p, u8p, i32]
    L.adc_match_cost.argtypes = [vp, u8p, u8p, vp, i32, i32, f32p]
    L.adc_match_cost_batch_device.argtypes = [vp, i32, u8p, u8p, vp, i32, i32, f32p, vp]
    L.adc_debug_run_cost.argtypes = [vp, u8p, u8p, vp, i32, i32, i32]
    L.adc_match_volumes.argtypes = [vp, u8p, u8p, vp, i32, i32, f32p, ctypes.POINTER(VolumeOut), i32]
    L.adc_match_volumes_batch_device.argtypes = [vp, i32, u8p, u8p, vp, i32, i32, f32p, ctypes.POINTER(VolumeOut), i32, vp]
    L.adc_match_outputs.argtypes = [vp, u8p, u8p, vp, i32, i32, f32p, ctypes.POINTER(VolumeOut), i32,
                                    ctypes.POINTER(MapOut), i32]
    L.adc_match_outputs_batch_device.argtypes = [vp, i32, u8p, u8p, vp, i32, i32, f32p, ctypes.POINTER(VolumeOut), i32,
                                                 ctypes.POINTER(MapOut), i32, vp]
    L.adc_match_images.argtypes = [vp, u8p, u8p, ctypes.POINTER(ImageDesc), vp, i32, i32, f32p,
                                   ctypes.POINTER(VolumeOut), i32, ctypes.POINTER(MapOut), i32]
    L.adc_match_images_batch_device.argtypes = [vp, i32, u8p, u8p, ctypes.POINTER(ImageDesc), vp, i32, i32, f32p,
                                                ctypes.POINTER(VolumeOut), i32, ctypes.POINTER(MapOut), i32, vp]
    L.adc_set_rectification.argtypes = [vp, ctypes.POINTER(Rectification)]
    L.adc_match_rectified.argtypes = [vp, u8p, u8p, ctypes.POINTER(ImageDesc), vp, i32, i32, f32p,
                                      ctypes.POINTER(VolumeOut), i32, ctypes.POINTER(MapOut), i32]
    L.adc_match_rectified_batch_device.argtypes = [vp, i32, u8p, u8p, ctypes.POINTER(ImageDesc), vp, i32, i32, f32p,
                                                   ctypes.POINTER(VolumeOut), i32, ctypes.POINTER(MapOut), i32, vp]
    L.adc_reproject.argtypes = [vp, f32p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ReprojectOut), i32]
    L.adc_reproject_batch_device.argtypes = [vp, i32, f32p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ReprojectOut),
                                             i32, vp]
    L.adc_speckle_workspace_bytes.argtypes = [vp, i32, ctypes.POINTER(ctypes.c_size_t)]
    L.adc_filter_speckles.argtypes = [vp, vp, ctypes.POINTER(SpeckleParams)]
    L.adc_filter_speckles_batch_device.argtypes = [vp, i32, vp, ctypes.POINTER(SpeckleParams), vp, ctypes.c_size_t, vp]
    L.adc_ingest_views.argtypes = [vp, u8p, u8p, ctypes.POINTER(ImageDesc), i32, u8p]
    L.adc_ingest_views_batch_device.argtypes = [vp, i32, u8p, u8p, ctypes.POINTER(ImageDesc), i32, u8p, vp]
    L.adc_point_cloud_workspace_bytes.argtypes = [vp, i32, ctypes.POINTER(ctypes.c_size_t)]
    L.adc_point_cloud.argtypes = [vp, f32p, ctypes.POINTER(ctypes.c_double), u8p, ctypes.c_float, ctypes.c_float,
                                  ctypes.POINTER(CloudOut)]
    L.adc_point_cloud_batch_device.argtypes = [vp, i32, f32p, ctypes.POINTER(ctypes.c_double), u8p, ctypes.c_int64,
                                               ctypes.c_float, ctypes.c_float, ctypes.POINTER(CloudOut), vp,
                                               ctypes.c_size_t, vp]
    L.adc_preview_workspace_bytes.argtypes = [vp, i32, ctypes.POINTER(ctypes.c_size_t)]
    L.adc_preview.argtypes = [vp, f32p, ctypes.POINTER(PreviewParams), vp, ctypes.POINTER(ImageDesc)]
    L.adc_preview_batch_device.argtypes = [vp, i32, f32p, ctypes.POINTER(PreviewParams), vp, ctypes.POINTER(ImageDesc),
                                           vp, ctypes.c_size_t, vp]
    L.adc_debug_get.argtypes = [vp, i32, vp, ctypes.c_size_t]
    L.adc_debug_get.restype = ctypes.c_size_t
    L.adc_debug_counters.argtypes = [vp, ctypes.POINTER(ctypes.c_int32 * 16)]
    _lib = L
    return L


def _check(rc: int):
    if rc != 0:
        raise AdcError(f"adcensus_b200 error {rc}: {load_library().adc_last_error().decode()}")


def _img(a, shape) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.shape != shape:
        raise ValueError(f"expected packed BGR uint8 array of shape {shape}, got {a.shape}")
    return a


def _code(table, v, what):
    if isinstance(v, str):
        if v not in table:
            raise ValueError(f"unknown cost {what} {v!r} (one of {sorted(table)})")
        return table[v]
    return int(v)


def _volume_outs(outs):
    """ctypes array of adc_volume_out from (ptr, stage, layout, dtype) tuples (names or ADC_* codes)."""
    arr = (VolumeOut * max(1, len(outs)))()
    for i, (ptr, stage, layout, dtype) in enumerate(outs):
        arr[i] = VolumeOut(ptr, _code(VOL_STAGES, stage, "volume stage"), _code(COST_LAYOUTS, layout, "layout"),
                           _code(COST_DTYPES, dtype, "dtype"), 0)
    return arr


def _map_outs(maps):
    """ctypes array of adc_map_out from (ptr, kind) tuples (names or ADC_MAP_* codes)."""
    arr = (MapOut * max(1, len(maps)))()
    for i, (ptr, kind) in enumerate(maps):
        arr[i] = MapOut(ptr, _code(MAP_KINDS, kind, "map kind"), 0)
    return arr


def _device_cost(d_cost, layout, dtype):
    """(pointer or None, layout code, dtype code): the cost arguments of a device batch entry."""
    return d_cost or None, _code(COST_LAYOUTS, layout, "layout"), _code(COST_DTYPES, dtype, "dtype")


def _reproject_outs(outs):
    """ctypes array of adc_reproject_out from (ptr, kind) tuples (names or ADC_REPROJ_* codes)."""
    arr = (ReprojectOut * max(1, len(outs)))()
    for i, (ptr, kind) in enumerate(outs):
        arr[i] = ReprojectOut(ptr, _code(REPROJ_KINDS, kind, "reprojection kind"), 0)
    return arr


class Engine:
    """Thin object wrapper over adc_create/.../adc_destroy."""

    def __init__(self, width: int, height: int, option: ADCensusOption | None = None, device: int = 0,
                 wave_pairs: int = 0, lanes: int = 0, debug_flags: int = 0):
        self._L = load_library()
        self.width, self.height = int(width), int(height)
        self.option = option or ADCensusOption()
        self.D = self.option.max_disparity - self.option.min_disparity
        cfg = _Config(device=device, wave_pairs=wave_pairs, lanes=lanes, debug_flags=debug_flags)
        h = ctypes.c_void_p()
        _check(self._L.adc_create(self.width, self.height, ctypes.byref(self.option), ctypes.byref(cfg), ctypes.byref(h)))
        self._h = h
        got = _Config()
        self._L.adc_get_config(self._h, ctypes.byref(got))
        self.wave_pairs, self.lanes, self.device = got.wave_pairs, got.lanes, got.device
        self.rect_src_size = None   # (width, height) of the raw frames while a rectification is set

    def close(self):
        if getattr(self, "_h", None):
            self._L.adc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- Match ----------------------------------------------------------------------------
    def match(self, left, right) -> np.ndarray:
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        disp = np.empty((self.height, self.width), np.float32)
        _check(self._L.adc_match(self._h, left.ctypes.data, right.ctypes.data, disp.ctypes.data))
        return disp

    def right_disparity(self) -> np.ndarray:
        """Right-view map of the most recent match() (the reference's private disp_right_)."""
        disp = np.empty((self.height, self.width), np.float32)
        _check(self._L.adc_get_right_disparity(self._h, disp.ctypes.data))
        return disp

    # ---- matching from a caller's cost volume (adc_match_cost*) -------------------------------
    def _cost(self, cost, layout, dtype):
        """(contiguous numpy volume, layout code, dtype code) for a host cost volume of one pair.  numpy has no bfloat16:
        a bf16 volume is passed as its uint16 bit patterns with dtype="bf16"."""
        lay = _code(COST_LAYOUTS, layout, "layout")
        cost = np.ascontiguousarray(cost)
        if dtype is None:
            dt = {np.dtype(np.float32): COST_F32, np.dtype(np.float16): COST_F16}.get(cost.dtype)
            if dt is None:
                raise ValueError(f"cost volume must be float32 or float16 (or uint16 bits with dtype='bf16'), got {cost.dtype}")
        else:
            dt = _code(COST_DTYPES, dtype, "dtype")
            if cost.dtype != _VOL_NP.get(dt):
                raise ValueError(f"dtype {dtype!r} expects a numpy {np.dtype(_VOL_NP.get(dt, np.float32)).name} array, got {cost.dtype}")
        H, W, D = self.height, self.width, self.D
        want = (H, W, D) if lay == COST_HWD else (D, H, W)
        if cost.shape != want:
            raise ValueError(f"expected a cost volume of shape {want} for layout {layout!r}, got {cost.shape}")
        return cost, lay, dt

    def _outputs(self, maps, volumes, layout, dtype, cost, cost_layout, cost_dtype, disparity):
        """The arrays a host entry with outputs fills, and its C arguments after the views: (disp or None, {name: array}
        of the requested volumes and maps, (cost, cost_layout, cost_dtype, disp, vols, n_vols, maps, n_maps)).  The
        arguments hold the cost volume and the arrays until the call."""
        maps = [maps] if isinstance(maps, (str, int)) else list(maps)
        volumes = [volumes] if isinstance(volumes, (str, int)) else list(volumes)
        lay, dt = _code(COST_LAYOUTS, layout, "layout"), _code(COST_DTYPES, dtype, "dtype")
        H, W, D = self.height, self.width, self.D
        shape = (H, W, D) if lay == COST_HWD else (D, H, W)
        out = {s: np.empty(shape, _VOL_NP.get(dt, np.float32)) for s in volumes}
        vouts = _volume_outs([(out[s].ctypes.data, s, lay, dt) for s in volumes])
        for m in maps:
            out[m] = np.empty((H, W), _MAP_NP.get(_code(MAP_KINDS, m, "map kind"), np.float32))
        mouts = _map_outs([(out[m].ctypes.data, m) for m in maps])
        c, clay, cdt = (None, 0, 0) if cost is None else self._cost(cost, cost_layout, cost_dtype)
        disp = np.empty((H, W), np.float32) if disparity else None
        return disp, out, (None if c is None else c.ctypes, clay, cdt, None if disp is None else disp.ctypes, vouts,
                           len(volumes), mouts, len(maps))

    def match_cost(self, left, right, cost, layout="hwd", dtype=None) -> np.ndarray:
        """Match with the given matching cost instead of the AD-census cost: `cost` is one pair's volume, float32 or
        float16, [H][W][D] (layout "hwd") or [D][H][W] ("dhw"); lower = better.  Values are clamped to [0, COST_MAX]."""
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        cost, lay, dt = self._cost(cost, layout, dtype)
        disp = np.empty((self.height, self.width), np.float32)
        _check(self._L.adc_match_cost(self._h, left.ctypes.data, right.ctypes.data, cost.ctypes.data, lay, dt, disp.ctypes.data))
        return disp

    def match_cost_batch_device(self, n: int, d_left: int, d_right: int, d_cost: int, d_disp: int,
                                layout="dhw", dtype="f32", stream: int = 0):
        """Device pointers (ints): n pairs of images, n cost volumes of H*W*D elements each (layout "hwd" / "dhw", dtype
        "f32" / "f16" / "bf16"), n maps out; enqueued on `stream` without synchronising, like match_batch_device."""
        _check(self._L.adc_match_cost_batch_device(self._h, n, d_left, d_right, *_device_cost(d_cost, layout, dtype), d_disp,
                                                   stream))

    # ---- exporting the cost volumes (adc_match_volumes*) --------------------------------------
    def match_volumes(self, left, right, stages, layout="hwd", dtype="f32", cost=None, cost_layout="hwd", cost_dtype=None,
                      disparity=True):
        """(disparity map or None, {stage: volume}) of one pair.  `stages`: one or more of "cost", "aggr", "opt" (the
        matching cost, the cross-aggregated cost, the scanline-optimised cost).  Volumes come back [H][W][D] ("hwd") or
        [D][H][W] ("dhw") as float32, float16 or -- numpy has no bfloat16 -- uint16 bit patterns for "bf16".  `cost`: a
        caller's matching cost instead of the AD-census cost, as for match_cost.  disparity=False stops the pipeline after
        the latest requested volume."""
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        stages = dict.fromkeys([stages] if isinstance(stages, (str, int)) else stages)   # a stage named twice: one volume
        disp, vols, args = self._outputs((), stages, layout, dtype, cost, cost_layout, cost_dtype, disparity)
        _check(self._L.adc_match_volumes(self._h, left.ctypes.data, right.ctypes.data, *args[:6]))
        return disp, vols

    def match_volumes_batch_device(self, n: int, d_left: int, d_right: int, outs, d_disp: int = 0, d_cost: int = 0,
                                   cost_layout="dhw", cost_dtype="f32", stream: int = 0):
        """Device pointers (ints): n pairs of images, optional n cost volumes, optional n maps (d_disp 0 = volumes only);
        `outs` a list of (ptr, stage, layout, dtype), each ptr n volumes of H*W*D elements.  Enqueued on `stream` without
        synchronising, like match_batch_device."""
        _check(self._L.adc_match_volumes_batch_device(self._h, n, d_left, d_right,
                                                      *_device_cost(d_cost, cost_layout, cost_dtype), d_disp or None,
                                                      _volume_outs(outs), len(outs), stream))

    # ---- per-pixel side maps, with or without volumes (adc_match_outputs*) -----------------------
    def match_outputs(self, left, right, maps=(), volumes=(), layout="hwd", dtype="f32", cost=None, cost_layout="hwd",
                      cost_dtype=None, disparity=True):
        """(disparity map or None, {name: array}) of one pair from one pipeline pass.  `maps`: any of "wta_left",
        "wta_right" (float32 [H][W], the WTA's maps before refinement), "outliers" (uint8 [H][W], 0 kept / 1 mismatch /
        2 occlusion before region voting), "min_cost", "peak_ratio" (float32 [H][W], the cost-curve confidence).
        `volumes`: any of "cost", "aggr", "opt" in `layout` / `dtype`, as for match_volumes.  `cost`: a caller's matching
        cost, as for match_cost.  disparity=False stops the pipeline after the latest requested output."""
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        disp, out, args = self._outputs(maps, volumes, layout, dtype, cost, cost_layout, cost_dtype, disparity)
        _check(self._L.adc_match_outputs(self._h, left.ctypes.data, right.ctypes.data, *args))
        return disp, out

    def match_outputs_batch_device(self, n: int, d_left: int, d_right: int, maps=(), volumes=(), d_disp: int = 0,
                                   d_cost: int = 0, cost_layout="dhw", cost_dtype="f32", stream: int = 0):
        """Device pointers (ints): n pairs of images, optional n cost volumes, optional n maps (d_disp 0 = no final map);
        `maps` a list of (ptr, kind), each ptr n maps of H*W elements (float32, uint8 for "outliers"); `volumes` a list
        of (ptr, stage, layout, dtype) as for match_volumes_batch_device.  Enqueued on `stream` without synchronising,
        like match_batch_device."""
        _check(self._L.adc_match_outputs_batch_device(self._h, n, d_left, d_right,
                                                      *_device_cost(d_cost, cost_layout, cost_dtype), d_disp or None,
                                                      _volume_outs(volumes), len(volumes), _map_outs(maps), len(maps),
                                                      stream))

    # ---- image input formats (adc_match_images*) -----------------------------------------------
    def match_images(self, left, right, format="bgr", maps=(), volumes=(), layout="hwd", dtype="f32", cost=None,
                     cost_layout="hwd", cost_dtype=None, disparity=True):
        """match_outputs for images in any IMG_* format, read in place: `left` / `right` are uint8 numpy views of shape
        [H][W][3 or 4] (bgr, rgb, bgra, rgba), [H][W] (gray, bayer_*), [3][H][W] (rgb_planar),
        [H + ceil(H/2)][2*ceil(W/2)] (nv12, nv21) or [H][2*ceil(W/2)][2] (yuyv, uyvy, yvyu), uint16 views [H][W]
        (mono10 / 12 / 16, bayer_rg10 ...) or uint8 views [H][ceil(bits*W/8)] of the rows' bytes (mono10p, bayer_rg12p
        ...: what a camera SDK's buffer is to numpy), [H + ceil(H/2)][2*ceil(W/2)] uint8 (i420, yv12, contiguous rows)
        or uint16 (p016), whose rows may be pitched,
        e.g. frame[:, :W] and frame[:, W:] of a side-by-side frame or a crop; both views need the same strides.
        The result is what match_outputs gives for the same pixels packed as BGR (for a Bayer mosaic: for
        cv2.cvtColor(view, COLOR_Bayer*2BGR), the pattern being the view's own top-left 2x2 block; for a YUV frame: for
        cv2.cvtColor(frame, COLOR_YUV2BGR_*) cropped to W x H, or its BT.709 / full-range rule for a format name with
        an encoding such as "p016/bt709" (include/adcensus_b200.h); for a high-bit-depth frame: for the unpacked uint16
        samples, demosaiced if Bayer, through cv2.convertScaleAbs(v, alpha=2**-(bits - 8)))."""
        return self._match_views(self._L.adc_match_images, self.height, self.width, left, right, format, maps, volumes,
                                 layout, dtype, cost, cost_layout, cost_dtype, disparity)

    def _match_views(self, call, vh, vw, left, right, format, maps, volumes, layout, dtype, cost, cost_layout,
                     cost_dtype, disparity):
        """The host entries that take views in an IMG_* format: adc_match_images (views of H x W) and
        adc_match_rectified (raw frames of vh x vw)."""
        desc = _image_pair_desc(left, right, _img_format(format), vh, vw)
        disp, out, args = self._outputs(maps, volumes, layout, dtype, cost, cost_layout, cost_dtype, disparity)
        _check(call(self._h, left.ctypes.data, right.ctypes.data, ctypes.byref(desc), *args))
        return disp, out

    def match_images_batch_device(self, n: int, d_left: int, d_right: int, image=None, maps=(), volumes=(),
                                  d_disp: int = 0, d_cost: int = 0, cost_layout="dhw", cost_dtype="f32", stream: int = 0):
        """match_outputs_batch_device for images described by `image` (an ImageDesc, e.g. from image_desc(); None = tight
        packed BGR): device pointers (ints) to the first pair's left and right view, pair i at i * image_stride bytes.
        Enqueued on `stream` without synchronising, like match_batch_device."""
        _check(self._L.adc_match_images_batch_device(self._h, n, d_left, d_right,
                                                     None if image is None else ctypes.byref(image),
                                                     *_device_cost(d_cost, cost_layout, cost_dtype), d_disp or None,
                                                     _volume_outs(volumes), len(volumes), _map_outs(maps), len(maps),
                                                     stream))

    # ---- rectification on the way in (adc_set_rectification, adc_match_rectified*) --------------------
    def set_rectification(self, left_maps, right_maps=None, src_size=None):
        """Sets the remap tables the rectified entries resample each raw view through: `left_maps` / `right_maps` are
        (map1, map2) exactly as cv2.initUndistortRectifyMap returns them for this engine's (width, height) -- float32
        [H][W] x and y, or int16 [H][W][2] and uint16 [H][W] -- as numpy arrays or CUDA tensors (row pitches from the
        strides); `src_size` = (width, height) of the raw frames.  The maps are copied: the caller's may be freed.
        set_rectification(None) clears them."""
        if left_maps is None:
            _check(self._L.adc_set_rectification(self._h, None))
            self.rect_src_size = None
            return
        sw, sh = (int(v) for v in src_size)
        t0, left = _remap(left_maps, self.height, self.width)
        t1, right = _remap(right_maps, self.height, self.width)
        if t0 != t1:
            raise ValueError("both views' maps must be of the same type")
        r = Rectification(sw, sh, t0, 0, (Remap * 2)(left, right))
        _check(self._L.adc_set_rectification(self._h, ctypes.byref(r)))
        self.rect_src_size = (sw, sh)

    def set_resize(self, src_size, interpolation="area"):
        """Sets a resize as the geometry of the rectified entries: raw frames of src_size = (width, height) are converted
        to BGR with their format's rule and resized to this engine's (width, height) as cv2.resize does with
        INTER_AREA (interpolation "area": integer downscale factors that are exact in double as OpenCV computes them,
        at most 4096 source pixels an output pixel) or
        INTER_LINEAR_EXACT ("linear_exact": any sizes), bit for bit.  It replaces maps set with set_rectification, and
        set_rectification(None) clears it.  match_rectified*, ingest_views(rectified=True) then take such frames."""
        sw, sh = (int(v) for v in src_size)
        t = RESIZE_INTERPOLATIONS.get(interpolation) if isinstance(interpolation, str) else int(interpolation)
        if t is None:
            raise ValueError(f"unknown interpolation {interpolation!r} (one of {sorted(RESIZE_INTERPOLATIONS)})")
        _check(self._L.adc_set_rectification(self._h, ctypes.byref(Rectification(sw, sh, t, 0))))
        self.rect_src_size = (sw, sh)

    def match_rectified(self, left, right, format="bgr", maps=(), volumes=(), layout="hwd", dtype="f32", cost=None,
                        cost_layout="hwd", cost_dtype=None, disparity=True):
        """match_images for raw frames: `left` / `right` are uint8 numpy views of the src_size frames given to
        set_rectification, in any IMG_* format and pitch, resampled through the maps on the way in.  The result is what
        match_outputs gives for cv2.remap(view, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) of each view packed as
        BGR; with a resize set (set_resize), for cv2.resize(view, (width, height), interpolation=...) instead."""
        if self.rect_src_size is None:
            raise AdcError("no rectification is set (set_rectification)")
        sw, sh = self.rect_src_size
        return self._match_views(self._L.adc_match_rectified, sh, sw, left, right, format, maps, volumes, layout, dtype,
                                 cost, cost_layout, cost_dtype, disparity)

    def match_rectified_batch_device(self, n: int, d_left: int, d_right: int, image=None, maps=(), volumes=(),
                                     d_disp: int = 0, d_cost: int = 0, cost_layout="dhw", cost_dtype="f32",
                                     stream: int = 0):
        """match_images_batch_device for raw frames: `image` (an ImageDesc, None = tight packed BGR) describes the raw
        views of the src_size given to set_rectification; pair i at i * image_stride bytes.  Enqueued on `stream`
        without synchronising, like match_batch_device."""
        _check(self._L.adc_match_rectified_batch_device(self._h, n, d_left, d_right,
                                                        None if image is None else ctypes.byref(image),
                                                        *_device_cost(d_cost, cost_layout, cost_dtype), d_disp or None,
                                                        _volume_outs(volumes), len(volumes), _map_outs(maps), len(maps),
                                                        stream))

    # ---- reprojection to 3-D (adc_reproject*) ---------------------------------------------------------
    def reproject(self, disp, Q, outputs=("points",)):
        """{name: array} of one disparity map (float32 [H][W], +inf = invalid) and the 4x4 matrix Q of
        cv2.stereoRectify: "points" float32 [H][W][3] (cv2.reprojectImageTo3D(disp, Q) bit for bit), "depth" float32
        [H][W] (its Z), "disp_s16" int16 [H][W] (the StereoSGBM "disparity * 16" encoding, invalid pixels
        (min_disparity - 1) * 16)."""
        H, W = self.height, self.width
        disp = np.ascontiguousarray(disp, np.float32)
        if disp.shape != (H, W):
            raise ValueError(f"expected a disparity map of shape {(H, W)}, got {disp.shape}")
        outputs = [outputs] if isinstance(outputs, (str, int)) else list(outputs)
        shape = {REPROJ_POINTS: (H, W, 3), REPROJ_DEPTH: (H, W), REPROJ_DISP_S16: (H, W)}
        out = {}
        for name in outputs:
            k = _code(REPROJ_KINDS, name, "reprojection kind")
            out[name] = np.empty(shape.get(k, (H, W)), _REPROJ_NP.get(k, np.float32))
        arr = _reproject_outs([(out[name].ctypes.data, name) for name in outputs])
        _check(self._L.adc_reproject(self._h, disp.ctypes.data, _q_matrix(Q), arr, len(outputs)))
        return out

    def reproject_batch_device(self, n: int, d_disp: int, Q, outs, stream: int = 0):
        """Device pointers (ints): n maps of H*W float32 at d_disp; `outs` a list of (ptr, kind), each ptr n outputs of
        H*W pixels (points: 3 float32, depth: float32, disp_s16: int16).  One launch enqueued on `stream` without
        synchronising; in pipelined mode the maps must be joined on `stream` first."""
        arr = _reproject_outs(outs)
        _check(self._L.adc_reproject_batch_device(self._h, n, d_disp, _q_matrix(Q), arr, len(outs), stream))

    # ---- speckle removal (adc_filter_speckles*) -------------------------------------------------------
    def speckle_invalid(self, map_type):
        """The engine's invalid value of a map type: +inf for f32, (min_disparity - 1) * 16 for s16 (StereoSGBM's)."""
        return float("inf") if _code(SPECKLE_TYPES, map_type, "speckle map type") == SPECKLE_F32 else \
            float((self.option.min_disparity - 1) * 16)

    def speckle_workspace_bytes(self, n: int) -> int:
        """Bytes of device workspace that filter_speckles_batch_device needs for n maps (8 per pixel)."""
        out = ctypes.c_size_t()
        _check(self._L.adc_speckle_workspace_bytes(self._h, n, ctypes.byref(out)))
        return int(out.value)

    def filter_speckles(self, map, max_size: int, max_diff: float, new_val=None) -> np.ndarray:
        """cv2.filterSpeckles(map, new_val, max_size, max_diff) of one [H][W] map on the GPU, returned as a filtered copy.
        int16 maps follow OpenCV's plain path (new_val and max_diff through cvRound), float32 maps the f32 rules of the
        header.  new_val None = speckle_invalid(type): +inf for float32, (min_disparity - 1) * 16 for int16."""
        a = np.asarray(map)
        if a.dtype not in (np.int16, np.float32):
            raise ValueError(f"speckle maps are int16 or float32, got {a.dtype}")
        if a.shape != (self.height, self.width):
            raise ValueError(f"expected a map of shape {(self.height, self.width)}, got {a.shape}")
        t = SPECKLE_S16 if a.dtype == np.int16 else SPECKLE_F32
        out = np.array(a, order="C", copy=True)
        nv = self.speckle_invalid(t) if new_val is None else new_val
        p = SpeckleParams(t, int(max_size), float(nv), float(max_diff), 0)
        _check(self._L.adc_filter_speckles(self._h, out.ctypes.data, ctypes.byref(p)))
        return out

    def filter_speckles_batch_device(self, n: int, d_maps: int, map_type, max_size: int, max_diff: float, new_val,
                                     d_work: int, work_bytes: int, stream: int = 0):
        """Device pointers (ints): n maps of H*W elements (map_type "s16" = int16, "f32" = float32) at d_maps filtered in
        place, with work_bytes >= speckle_workspace_bytes(n) of workspace at d_work.  Four launches enqueued on `stream`
        without synchronising; in pipelined mode the maps must be joined on `stream` first.  new_val None =
        speckle_invalid(map_type)."""
        t = _code(SPECKLE_TYPES, map_type, "speckle map type")
        nv = self.speckle_invalid(t) if new_val is None else new_val
        p = SpeckleParams(t, int(max_size), float(nv), float(max_diff), 0)
        _check(self._L.adc_filter_speckles_batch_device(self._h, n, d_maps, ctypes.byref(p), d_work, work_bytes, stream))

    # ---- the views as the engine matches them (adc_ingest_views*) ---------------------------------------
    def ingest_views(self, left, right, format="bgr", rectified=False) -> np.ndarray:
        """uint8 [2][H][W][3]: the packed BGR left and right views that match_images (rectified=False) or
        match_rectified (rectified=True) feed to stage 1 for the same views, in the shapes those entries take."""
        fmt = _img_format(format)
        if rectified and self.rect_src_size is None:
            raise AdcError("no rectification is set (set_rectification)")
        vw, vh = self.rect_src_size if rectified else (self.width, self.height)
        desc = _image_pair_desc(left, right, fmt, vh, vw)
        views = np.empty((2, self.height, self.width, 3), np.uint8)
        _check(self._L.adc_ingest_views(self._h, left.ctypes.data, right.ctypes.data, ctypes.byref(desc),
                                        1 if rectified else 0, views.ctypes.data))
        return views

    def ingest_views_batch_device(self, n: int, d_left: int, d_right: int, d_views: int, image=None, rectified=False,
                                  stream: int = 0):
        """Device pointers (ints): n pairs described by `image` (an ImageDesc, None = tight packed BGR), plain or through
        the rectification, written to d_views as packed BGR [n][2][H][W][3].  One launch per 65535 pairs (fewer for
        an engine of more than 2^27 pixels) enqueued on `stream` without synchronising."""
        _check(self._L.adc_ingest_views_batch_device(self._h, n, d_left, d_right,
                                                     None if image is None else ctypes.byref(image),
                                                     1 if rectified else 0, d_views, stream))

    # ---- point clouds (adc_point_cloud*) ------------------------------------------------------------------
    def point_cloud(self, disp, Q, bgr=None, z_range=(-np.inf, np.inf), pixels=False):
        """The valid points of one disparity map (float32 [H][W]) in raster order: points float32 [k][3], plus colors
        uint8 [k][3] (R, G, B of `bgr`, a packed BGR [H][W][3] image) and pixels int32 [k] (y*W + x) when requested --
        cv2.reprojectImageTo3D(disp, Q)[keep] with keep = finite d, finite point, z_range[0] <= Z <= z_range[1].
        Returns points alone, or a tuple (points[, colors][, pixels])."""
        H, W = self.height, self.width
        disp = np.ascontiguousarray(disp, np.float32)
        if disp.shape != (H, W):
            raise ValueError(f"expected a disparity map of shape {(H, W)}, got {disp.shape}")
        img = None if bgr is None else _img(bgr, (H, W, 3))
        N = H * W
        pts = np.empty((N, 3), np.float32)
        cols = np.empty((N, 3), np.uint8) if img is not None else None
        pix = np.empty(N, np.int32) if pixels else None
        count = np.zeros(1, np.int32)
        out = CloudOut(pts.ctypes.data, None if cols is None else cols.ctypes.data, None if pix is None else pix.ctypes.data,
                       count.ctypes.data, N, 0)
        _check(self._L.adc_point_cloud(self._h, disp.ctypes.data, _q_matrix(Q), None if img is None else img.ctypes.data,
                                       float(z_range[0]), float(z_range[1]), ctypes.byref(out)))
        k = int(count[0])
        res = [pts[:k].copy()] + ([cols[:k].copy()] if cols is not None else []) + ([pix[:k].copy()] if pixels else [])
        return res[0] if len(res) == 1 else tuple(res)

    def point_cloud_workspace_bytes(self, n: int) -> int:
        """Bytes of device workspace that point_cloud_batch_device needs for n maps."""
        out = ctypes.c_size_t()
        _check(self._L.adc_point_cloud_workspace_bytes(self._h, n, ctypes.byref(out)))
        return int(out.value)

    def point_cloud_batch_device(self, n: int, d_disp: int, Q, d_points: int, d_counts: int, capacity: int,
                                 d_work: int, work_bytes: int, d_bgr: int = 0, bgr_stride: int = 0, d_colors: int = 0,
                                 d_pixels: int = 0, z_range=(-np.inf, np.inf), stream: int = 0):
        """Device pointers (ints): n maps of H*W float32 at d_disp; map i's first `capacity` kept points at point
        i*capacity of d_points (float32 x3), d_colors (uint8 R, G, B of d_bgr + i*bgr_stride, 0 = 3*H*W) and d_pixels
        (int32), its full count at d_counts[i]; work_bytes >= point_cloud_workspace_bytes(n) of workspace at d_work.  A
        memset and one launch enqueued on `stream` without synchronising; in pipelined mode the maps must be joined on
        `stream` first."""
        out = CloudOut(d_points, d_colors or None, d_pixels or None, d_counts, int(capacity), 0)
        _check(self._L.adc_point_cloud_batch_device(self._h, n, d_disp, _q_matrix(Q), d_bgr or None, int(bgr_stride),
                                                    float(z_range[0]), float(z_range[1]), ctypes.byref(out), d_work,
                                                    work_bytes, stream))

    # ---- previews (adc_preview*) ---------------------------------------------------------------------------
    def preview(self, map, colormap="turbo", value_range=None, size=None, format="bgr", invalid=(0, 0, 0)) -> np.ndarray:
        """One float32 [H][W] map (final map, side map, depth; non-finite = invalid) rendered as a tight 8-bit frame of
        preview_shape(format, *size): cv2.normalize(NORM_MINMAX over the valid pixels; value_range (alpha, beta) =
        convertTo(CV_8U, alpha, beta) instead) -> cv2.applyColorMap(colormap; "none" = gray) -> invalid pixels set to
        `invalid` (B, G, R) -> cv2.resize(size = (width, height), INTER_NEAREST; None = the engine's size) ->
        cv2.cvtColor(COLOR_BGR2<format>), bit for bit."""
        H, W = self.height, self.width
        m = np.ascontiguousarray(map, np.float32)
        if m.shape != (H, W):
            raise ValueError(f"expected a map of shape {(H, W)}, got {m.shape}")
        p = preview_params(colormap, value_range, size, invalid)
        f = _code(PREVIEW_FORMATS, format, "preview format") if isinstance(format, str) else int(format)
        out = np.empty(preview_shape(f, p.dst_width or W, p.dst_height or H), np.uint8)
        _check(self._L.adc_preview(self._h, m.ctypes.data, ctypes.byref(p), out.ctypes.data,
                                   ctypes.byref(ImageDesc(f, 0, 0, 0, 0))))
        return out

    def preview_workspace_bytes(self, n: int) -> int:
        """Bytes of device workspace that preview_batch_device needs for n maps with MINMAX (8 per map)."""
        out = ctypes.c_size_t()
        _check(self._L.adc_preview_workspace_bytes(self._h, n, ctypes.byref(out)))
        return int(out.value)

    def preview_batch_device(self, n: int, d_maps: int, d_dst: int, image=None, colormap="turbo", value_range=None,
                             size=None, invalid=(0, 0, 0), d_work: int = 0, work_bytes: int = 0, stream: int = 0):
        """Device pointers (ints): n float32 maps of H*W at d_maps rendered as preview() renders them into n frames at
        d_dst described by `image` (an ImageDesc of a preview format, e.g. image_desc("nv12", row_pitch=...), None =
        tight BGR); MINMAX needs work_bytes >= preview_workspace_bytes(n) at d_work.  A memset and two launches
        (MINMAX) or one launch (FIXED) enqueued on `stream` without synchronising; in pipelined mode the maps must be
        joined on `stream` first."""
        p = preview_params(colormap, value_range, size, invalid)
        _check(self._L.adc_preview_batch_device(self._h, n, d_maps, ctypes.byref(p), d_dst,
                                                None if image is None else ctypes.byref(image), d_work or None,
                                                work_bytes, stream))

    def match_batch(self, lefts, rights) -> np.ndarray:
        """lefts/rights: arrays [n][H][W][3] (or sequences of images).  Host memory in, host memory out."""
        lefts = np.ascontiguousarray(lefts, np.uint8)
        rights = np.ascontiguousarray(rights, np.uint8)
        n = lefts.shape[0]
        if lefts.shape != (n, self.height, self.width, 3) or rights.shape != lefts.shape:
            raise ValueError("expected [n][H][W][3] uint8 arrays")
        disp = np.empty((n, self.height, self.width), np.float32)
        _check(self._L.adc_match_batch_strided(self._h, n, lefts.ctypes.data, rights.ctypes.data, disp.ctypes.data))
        return disp

    def match_batch_ptrs(self, lefts, rights):
        """Pointer-array form (adc_match_batch): independent per-pair buffers."""
        n = len(lefts)
        ls = [_img(a, (self.height, self.width, 3)) for a in lefts]
        rs = [_img(a, (self.height, self.width, 3)) for a in rights]
        ds = [np.empty((self.height, self.width), np.float32) for _ in range(n)]
        arr = ctypes.c_void_p * n
        _check(self._L.adc_match_batch(self._h, n, arr(*[a.ctypes.data for a in ls]),
                                       arr(*[a.ctypes.data for a in rs]), arr(*[a.ctypes.data for a in ds])))
        return ds

    def match_batch_device(self, n: int, d_left: int, d_right: int, d_disp: int, stream: int = 0):
        """Device pointers (ints), enqueued on `stream` (cudaStream_t as int) without synchronising."""
        _check(self._L.adc_match_batch_device(self._h, n, d_left, d_right, d_disp, stream))

    def match_batch_pinned_async(self, n: int, left_ptr: int, right_ptr: int, disp_ptr: int, stream: int = 0):
        _check(self._L.adc_match_batch_pinned_async(self._h, n, left_ptr, right_ptr, disp_ptr, stream))

    def synchronize(self):
        _check(self._L.adc_synchronize(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._L.adc_launch_count(self._h))

    def last_stage_ms(self):
        out = (ctypes.c_float * 6)()
        _check(self._L.adc_last_stage_ms(self._h, ctypes.byref(out)))
        return list(out)

    PROFILE_KERNELS = {"cost_volume": 0, "arm_sum_h": 1, "arm_sum_v_div": 2, "scanline_x": 3, "scanline_y": 4, "wta": 5,
                       "arm_sum2_v": 6, "arm_sum2_h": 7, "arm_sum_h_div": 8, "arm_sum_v": 9, "cost_ingest": 10,
                       "cost_export": 11, "confidence": 12, "image_ingest": 13,
                       "rectify": 14, "cost_arm_sum_h": 15, "scanline_y_wta": 16, "wta_merge": 17}

    def profile_kernel(self, name: str, reps: int = 5):
        """(mean ms per launch over one wave, algorithmic bytes per launch) of one pipeline kernel."""
        ms, by = ctypes.c_float(), ctypes.c_double()
        _check(self._L.adc_profile_kernel(self._h, self.PROFILE_KERNELS[name], reps, ctypes.byref(ms), ctypes.byref(by)))
        return ms.value, by.value

    # ---- streaming: consecutive async batch calls without a drain in between -------------------
    def set_pipelined(self, on: bool = True):
        _check(self._L.adc_set_pipelined(self._h, 1 if on else 0))

    def join(self, stream: int = 0):
        """Makes `stream` wait for everything submitted so far (required before results are read in pipelined mode)."""
        _check(self._L.adc_join(self._h, stream))

    # ---- output side of the reference's demo (main.cpp:147-230) -------------------------------
    def render_disparity(self, disp: np.ndarray):
        """(gray8 [H][W], jet_bgr [H][W][3], (min, max)): SaveDisparityMap's two images (main.cpp:180-207)."""
        disp = np.ascontiguousarray(disp, np.float32).reshape(self.height, self.width)
        gray = np.empty((self.height, self.width), np.uint8)
        jet = np.empty((self.height, self.width, 3), np.uint8)
        mm = np.empty(2, np.float32)
        _check(self._L.adc_render_disparity(self._h, disp.ctypes.data, gray.ctypes.data, jet.ctypes.data, mm.ctypes.data))
        return gray, jet, (float(mm[0]), float(mm[1]))

    def disparity_cloud(self, left: np.ndarray, disp: np.ndarray) -> np.ndarray:
        """[n][6] float32 records (x, y, |d|, r, g, b) of the valid pixels in raster order (main.cpp:209-230)."""
        left = _img(left, (self.height, self.width, 3))
        disp = np.ascontiguousarray(disp, np.float32).reshape(self.height, self.width)
        cloud = np.empty((self.height * self.width, 6), np.float32)
        n = ctypes.c_int32(0)
        _check(self._L.adc_disparity_cloud(self._h, left.ctypes.data, disp.ctypes.data, cloud.ctypes.data, ctypes.byref(n)))
        return cloud[:n.value].copy()

    # ---- debug taps -------------------------------------------------------------------------
    def debug_run(self, left, right, last_stage: str):
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        _check(self._L.adc_debug_run(self._h, left.ctypes.data, right.ctypes.data, STAGE[last_stage]))

    def debug_run_cost(self, left, right, cost, layout, last_stage: str, dtype=None):
        left = _img(left, (self.height, self.width, 3))
        right = _img(right, (self.height, self.width, 3))
        cost, lay, dt = self._cost(cost, layout, dtype)
        _check(self._L.adc_debug_run_cost(self._h, left.ctypes.data, right.ctypes.data, cost.ctypes.data, lay, dt,
                                          STAGE[last_stage]))

    def counters(self):
        out = (ctypes.c_int32 * 16)()
        _check(self._L.adc_debug_counters(self._h, ctypes.byref(out)))
        return list(out)

    def tap(self, name: str) -> np.ndarray:
        tid = TAP[name]
        nbytes = self._L.adc_debug_get(self._h, tid, None, 0)
        buf = np.empty(nbytes, np.uint8)
        if nbytes:
            got = self._L.adc_debug_get(self._h, tid, buf.ctypes.data, nbytes)
            if got != nbytes:
                raise AdcError(f"adc_debug_get({name}) failed: {self._L.adc_last_error().decode()}")
        a = buf.view(_TAP_DTYPE[name])
        if name in ("VOL_INIT", "VOL_AGGR"):
            return a.reshape(self.height, self.width, self.D)
        if name == "ARMS":
            return a.reshape(self.height, self.width, 4)
        if name in ("MISMATCHES", "OCCLUSIONS"):
            return a.reshape(-1, 2)
        return a.reshape(self.height, self.width)


class ADCensusStereo:
    """Python mirror of the reference class (ADCensusStereo.h:14-95): Initialize / Match / Reset
    with the reference's bool-returning error behaviour."""

    def __init__(self):
        self._engine = None
        self.last_error = ""

    def Initialize(self, width: int, height: int, option: ADCensusOption) -> bool:
        self.Release()
        try:
            self._engine = Engine(width, height, option)
        except (AdcError, ValueError) as e:
            self.last_error = str(e)
            self._engine = None
            return False
        return True

    def Match(self, img_left, img_right, disp_left: np.ndarray | None = None):
        """Returns False (like the reference) when not initialised or when an image is None;
        otherwise fills/returns the float32 disparity map."""
        if self._engine is None or img_left is None or img_right is None:
            return False
        out = self._engine.match(img_left, img_right)
        if disp_left is not None:
            np.copyto(disp_left.reshape(out.shape), out)
            return True
        return out

    def Reset(self, width: int, height: int, option: ADCensusOption) -> bool:
        self.Release()
        return self.Initialize(width, height, option)

    def Release(self):
        if self._engine is not None:
            self._engine.close()
        self._engine = None
