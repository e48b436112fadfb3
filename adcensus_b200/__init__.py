"""adcensus_b200 -- H100-native AD-Census stereo matching behind the reference's ADCensusStereo API.

The compute path is the hand-written sm_90a CUDA library ``adcensus_b200/lib/libadcensus_b200.so``
(sources in ``adcensus_b200/csrc``), reached through its C ABI (``include/adcensus_b200.h``).
This package is the Python mirror of the reference's interface for that path
(``ADCensusOption`` and ``ADCensusStereo.Initialize / Match / Reset``, reference
``adcensus_types.h:45-75`` and ``ADCensusStereo.h:14-95``).  There is no CPU fallback: importing
works anywhere, but creating an engine without the CUDA library or without a GPU raises.
"""
from .engine import (ADCensusOption, ADCensusStereo, AdcError, Engine, STAGE, TAP, lib_path,  # noqa: F401
                     load_library, Invalid_Float, COST_HWD, COST_DHW, COST_F32, COST_F16, COST_BF16, COST_MAX,
                     VOL_COST, VOL_AGGR, VOL_OPT, MAP_WTA_LEFT, MAP_WTA_RIGHT, MAP_OUTLIERS, MAP_MIN_COST,
                     MAP_PEAK_RATIO, IMG_BGR, IMG_RGB, IMG_BGRA, IMG_RGBA, IMG_GRAY, IMG_RGB_PLANAR, ImageDesc,
                     IMG_BAYER_RGGB, IMG_BAYER_GRBG, IMG_BAYER_BGGR, IMG_BAYER_GBRG, BAYER_FORMATS, IMG_NV12, IMG_NV21,
                     IMG_YUYV, IMG_UYVY, IMG_YVYU, YUV_FORMATS, image_desc, REMAP_F32, REMAP_FIXED, Remap,
                     Rectification, REPROJ_POINTS, REPROJ_DEPTH,
                     REPROJ_DISP_S16, REPROJ_KINDS, ReprojectOut, SPECKLE_S16,
                     SPECKLE_F32, SPECKLE_TYPES, SpeckleParams, CloudOut)
from .engine import (IMG_MONO10, IMG_BAYER_RG10, IMG_BAYER_GR10, IMG_BAYER_BG10, IMG_BAYER_GB10, IMG_MONO12,
                     IMG_BAYER_RG12, IMG_BAYER_GR12, IMG_BAYER_BG12, IMG_BAYER_GB12, IMG_MONO16,
                     IMG_BAYER_RG16, IMG_BAYER_GR16, IMG_BAYER_BG16, IMG_BAYER_GB16,
                     IMG_MONO10P, IMG_BAYER_RG10P, IMG_BAYER_GR10P, IMG_BAYER_BG10P,
                     IMG_BAYER_GB10P, IMG_MONO12P, IMG_BAYER_RG12P, IMG_BAYER_GR12P,
                     IMG_BAYER_BG12P, IMG_BAYER_GB12P, RAW_DEPTH_FORMATS)  # noqa: F401
from .engine import (IMG_I420, IMG_YV12, IMG_P016, YUV_VIDEO_FORMATS, IMG_YUV_BT709, IMG_YUV_FULL_RANGE,  # noqa: F401
                     YUV_ENCODINGS)
from .engine import RESIZE_AREA, RESIZE_LINEAR_EXACT, RESIZE_INTERPOLATIONS  # noqa: F401
from .engine import (COLORMAPS, COLORMAP_NONE, PREVIEW_MINMAX, PREVIEW_FIXED, PREVIEW_FORMATS,  # noqa: F401
                     PreviewParams, preview_params, preview_shape)
from .build import build_library  # noqa: F401

__all__ = ["ADCensusOption", "ADCensusStereo", "AdcError", "Engine", "STAGE", "TAP", "lib_path",
           "load_library", "build_library", "Invalid_Float", "COST_HWD", "COST_DHW", "COST_F32", "COST_F16", "COST_BF16",
           "COST_MAX", "VOL_COST", "VOL_AGGR", "VOL_OPT", "MAP_WTA_LEFT", "MAP_WTA_RIGHT", "MAP_OUTLIERS", "MAP_MIN_COST",
           "MAP_PEAK_RATIO", "IMG_BGR", "IMG_RGB", "IMG_BGRA", "IMG_RGBA", "IMG_GRAY", "IMG_RGB_PLANAR", "ImageDesc",
           "IMG_BAYER_RGGB", "IMG_BAYER_GRBG", "IMG_BAYER_BGGR", "IMG_BAYER_GBRG", "BAYER_FORMATS",
           "IMG_NV12", "IMG_NV21", "IMG_YUYV", "IMG_UYVY", "IMG_YVYU", "YUV_FORMATS",
           "IMG_MONO10", "IMG_BAYER_RG10", "IMG_BAYER_GR10", "IMG_BAYER_BG10", "IMG_BAYER_GB10", "IMG_MONO12",
           "IMG_BAYER_RG12", "IMG_BAYER_GR12", "IMG_BAYER_BG12", "IMG_BAYER_GB12", "IMG_MONO16",
           "IMG_BAYER_RG16", "IMG_BAYER_GR16", "IMG_BAYER_BG16", "IMG_BAYER_GB16", "IMG_MONO10P",
           "IMG_BAYER_RG10P", "IMG_BAYER_GR10P", "IMG_BAYER_BG10P", "IMG_BAYER_GB10P", "IMG_MONO12P",
           "IMG_BAYER_RG12P", "IMG_BAYER_GR12P", "IMG_BAYER_BG12P", "IMG_BAYER_GB12P", "RAW_DEPTH_FORMATS",
           "IMG_I420", "IMG_YV12", "IMG_P016", "YUV_VIDEO_FORMATS", "IMG_YUV_BT709", "IMG_YUV_FULL_RANGE", "YUV_ENCODINGS",
           "image_desc", "REMAP_F32", "REMAP_FIXED", "Remap", "Rectification", "REPROJ_POINTS", "REPROJ_DEPTH",
           "REPROJ_DISP_S16", "REPROJ_KINDS", "ReprojectOut", "SPECKLE_S16", "SPECKLE_F32", "SPECKLE_TYPES",
           "SpeckleParams", "CloudOut", "RESIZE_AREA", "RESIZE_LINEAR_EXACT", "RESIZE_INTERPOLATIONS",
           "COLORMAPS", "COLORMAP_NONE", "PREVIEW_MINMAX", "PREVIEW_FIXED", "PREVIEW_FORMATS", "PreviewParams",
           "preview_params", "preview_shape"]
