"""numpy restatement of the point-cloud entries (adc_point_cloud*, include/adcensus_b200.h): the pixels of a disparity map
whose value is finite, whose cv2.reprojectImageTo3D point is finite and whose Z lies in [z_min, z_max], in raster order,
with their points, R, G, B and pixel indices."""
import numpy as np

import reproject_testlib as RP


def keep(disp: np.ndarray, Q, z_min=-np.inf, z_max=np.inf):
    """(points float32 [H][W][3], keep bool [H][W]): finite d, finite point, z_min <= Z <= z_max compared in float32."""
    P = RP.points(disp, Q)
    with np.errstate(invalid="ignore"):
        k = np.isfinite(disp) & np.isfinite(P).all(-1) & (P[..., 2] >= np.float32(z_min)) & (P[..., 2] <= np.float32(z_max))
    return P, k


def cloud(disp: np.ndarray, Q, bgr=None, z_min=-np.inf, z_max=np.inf):
    """(points float32 [k][3], colors uint8 [k][3] R, G, B or None, pixels int32 [k] = y*W + x)."""
    P, k = keep(disp, Q, z_min, z_max)
    colors = None if bgr is None else np.ascontiguousarray(np.asarray(bgr)[..., ::-1][k])
    return P[k], colors, np.flatnonzero(k).astype(np.int32)
