"""Writes tests/golden/golden_cloud_cases.npz: disparity maps, Q matrices, z ranges, colour images and the point clouds
that live cv2.reprojectImageTo3D plus numpy masking give for them, so that the point-cloud tests need no OpenCV on the
GPU host.  The file is written with fixed zip timestamps, so regenerating it gives the same bytes.

Cases (keys "<name>/disp" f32 [H][W], "<name>/Q" f64 [4][4], "<name>/z" f32 [2] = (z_min, z_max), "<name>/bgr" u8
[H][W][3], "<name>/points" f32 [k][3], "<name>/colors" u8 [k][3] R, G, B, "<name>/pixels" int32 [k]):
  rand_*     random Q at extreme scales (1e-30 .. 1e30, +-0 entries), maps with +-inf, NaN, +-0, subnormals, +-3e38;
  rig_*      cv2.stereoRectify Q with and without CALIB_ZERO_DISPARITY on engine-like maps, with z ranges of +-inf,
             equal bounds at a point's Z, bounds that cut exactly at points' Z, and z_min > z_max;
  colzero_*  a Q whose column 2 is zero in every row, so that d enters no coordinate: +-inf and NaN pixels still have
             no finite point (0 * inf is NaN) and are dropped;
  line_*     1 x 1, 1 x N and N x 1 maps;
  all_*, none_*, last_*  every pixel kept, none kept, only the last pixel kept.

    python tools/make_golden_cloud.py [out.npz]
"""
import io
import sys
import zipfile
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden_reproject as MG  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_cloud_cases.npz"
INF = np.float32(np.inf)


def cv_cloud(disp, Q, bgr, z):
    P = cv2.reprojectImageTo3D(disp, Q)
    with np.errstate(invalid="ignore"):
        keep = np.isfinite(disp) & np.isfinite(P).all(-1) & (P[..., 2] >= z[0]) & (P[..., 2] <= z[1])
    return P[keep], cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)[keep], np.flatnonzero(keep).astype(np.int32)


def cases():
    rng = np.random.default_rng(20261016)
    out = {}

    def img(H, W):
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)

    full = np.array([-INF, INF], np.float32)
    for i in range(10):
        H, W = (int(v) for v in rng.integers(1, 40, 2))
        out[f"rand_{i}"] = (MG.random_disp(rng, H, W), MG.random_Q(rng), full, img(H, W))
    for i, (W, H, dmin) in enumerate([(48, 32, 0), (33, 21, -4), (40, 24, 2)]):
        for name, zero in (("zero", True), ("free", False)):
            d = MG.engine_disp(rng, H, W, dmin)
            Q = MG.rig_Q(W, H, zero)
            P = cv2.reprojectImageTo3D(d, Q)
            zs = np.sort(P[..., 2][np.isfinite(P).all(-1) & np.isfinite(d)])
            a, b = zs[len(zs) // 4], zs[3 * len(zs) // 4]
            for zname, z in (("inf", full), ("eq", [a, a]), ("cut", [a, b]), ("neg", [b, a]), ("half", [-INF, a])):
                out[f"rig_{name}_{i}_{zname}"] = (d, Q, np.array(z, np.float32), img(H, W))
    for i in range(2):
        Q = MG.random_Q(rng)
        Q[:, 2] = 0.0
        Q[3, 3] = 1.0
        out[f"colzero_{i}"] = (MG.random_disp(rng, 17, 23), Q, full, img(17, 23))
    for name, (H, W) in (("1x1", (1, 1)), ("1xN", (1, 600)), ("Nx1", (37, 1))):
        out[f"line_{name}"] = (MG.random_disp(rng, H, W), MG.rig_Q(max(W, 2), max(H, 2), False), full, img(H, W))
    W, H = 45, 29
    d = (1 + rng.integers(0, 4 * 60, (H, W)) / 4.0).astype(np.float32)
    out["all_0"] = (d, MG.rig_Q(W, H, True), full, img(H, W))
    out["none_0"] = (np.full((H, W), np.inf, np.float32), MG.rig_Q(W, H, True), full, img(H, W))
    out["none_1"] = (d, MG.rig_Q(W, H, True), np.array([1.0, -1.0], np.float32), img(H, W))
    last = np.full((H, W), np.inf, np.float32)
    last[-1, -1] = 17.25
    out["last_0"] = (last, MG.rig_Q(W, H, False), full, img(H, W))
    return out


def arrays():
    res = {}
    for name, (disp, Q, z, bgr) in cases().items():
        pts, cols, pix = cv_cloud(disp, Q, bgr, z)
        res.update({f"{name}/disp": disp, f"{name}/Q": Q, f"{name}/z": z, f"{name}/bgr": bgr, f"{name}/points": pts,
                    f"{name}/colors": cols, f"{name}/pixels": pix})
    return res


def write_npz(path, arrs):
    """np.savez_compressed with fixed timestamps, so that the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrs):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrs[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(f"{k}.npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)


def main(path=OUT):
    arrs = arrays()
    for name in {k.split("/")[0] for k in arrs}:
        n = len(arrs[f"{name}/pixels"])
        N = arrs[f"{name}/disp"].size
        assert (name.startswith("all") and n == N) or (name.startswith("none") and n == 0) or \
            (name.startswith("last") and list(arrs[f"{name}/pixels"]) == [N - 1]) or name.split("_")[0] not in (
                "all", "none", "last"), name
    write_npz(path, arrs)
    print(f"wrote {path}: {len(arrs) // 7} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
