#!/usr/bin/env python
"""High-bit-depth camera frames on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident,
pipelined), in one process so that every figure comes from the same run:

  python tools/bench_rawdepth.py [--steps 5 --warmup 3 --rounds 3]

* rg12p / rg12 / mono12p : adc_match_images_batch_device on Cone synthesised at 12 bits (the 8-bit samples x 16 plus
                 seeded low bits) as BayerRG12p, BayerRG12 and Mono12p frames, tight rows
* rg12p_bgr / mono12p_bgr : adc_match_batch_device on the same frames converted beforehand (unpack, cv2.cvtColor on
                 uint16, cv2.convertScaleAbs), packed BGR on the device: the yardsticks (BayerRG12 holds the samples of
                 BayerRG12p, so rg12p_bgr is its yardstick too)
* rect_rg12p   : adc_match_rectified_batch_device on raw 640 x 480 BayerRG12p frames (Cone resized and synthesised),
                 rectified through initUndistortRectifyMap maps (CV_16SC2) of rectify_testlib's made-up rig
* rect_bgr_raw : adc_match_rectified_batch_device on the same raw frames converted beforehand, [N, 480, 640, 3]
  The seven are timed in alternating windows (`--rounds`); the medians are reported.
* host         : the same raw BayerRG12p frames through a numpy unpack, cv2.cvtColor, cv2.convertScaleAbs and cv2.remap
                 on the host (both views of every pair, 16 OpenCV threads) followed by adc_match_batch on the rectified
                 images: wall clock over one batch, after a warm-up batch.
* kernels      : the plain ingestion kernel (adc_profile_kernel id 13) for BayerRG12p, BayerRG10p, BayerRG12, Mono12p and
                 8-bit BayerRG8, and the rectified one (id 14) for BayerRG12p and BGR, over one wave (CUDA events), each
                 next to a device-to-device cudaMemcpyAsync (torch copy_) that moves as many bytes (read + write) as the
                 kernel's algorithmic bytes (per view the tight rows read and 3N written; plus both views' maps once per
                 wave for id 14).
Every map is checked bit for bit against the packed-BGR maps of the converted images (and the host path's).  The card's
name and power limit are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import statistics
import sys

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import rawdepth_testlib as X
import rectify_testlib as R


def unpack12p(rows, W):
    """uint16 [H][W] of Mono12p / Bayer12p rows, W even: the host path's unpack, three bytes to two samples."""
    t = rows.reshape(rows.shape[0], -1, 3).astype(np.uint16)
    out = np.empty((rows.shape[0], W), np.uint16)
    out[:, 0::2] = t[..., 0] | (t[..., 1] & 15) << 8
    out[:, 1::2] = t[..., 1] >> 4 | t[..., 2] << 4
    return out


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n, raw=True)
    h, w, _ = left.shape
    sw, sh = 640, 480
    D = 64
    rng = np.random.default_rng(12)

    rg12p = [X.encode(img, "bayer_rg12p", rng) for img in (left, right)]
    rg12 = [X.samples(f, "bayer_rg12p", w, h) for f in rg12p]
    mono12p = [X.encode(img, "mono12p", rng) for img in (left, right)]
    rg_dec = [X.cv_decode(cv2, f, "bayer_rg12p", w, h) for f in rg12p]
    mono_dec = [X.cv_decode(cv2, f, "mono12p", w, h) for f in mono12p]
    raw = [X.encode(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), "bayer_rg12p", rng) for img in (left, right)]
    raw_bgr = [X.cv_decode(cv2, r, "bayer_rg12p", sw, sh) for r in raw]
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    d = {"rg12p": [rep(x) for x in rg12p], "rg12": [rep(x) for x in rg12], "mono12p": [rep(x) for x in mono12p],
         "rg12p_bgr": [rep(x) for x in rg_dec], "mono12p_bgr": [rep(x) for x in mono_dec],
         "rect_rg12p": [rep(x) for x in raw], "rect_bgr_raw": [rep(x) for x in raw_bgr]}
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in d}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()

    def images(name, fmt):
        def call(_):
            eng.match_images_batch_device(n, d[name][0].data_ptr(), d[name][1].data_ptr(), image=A.image_desc(fmt),
                                          d_disp=out[name].data_ptr(), stream=st.cuda_stream)
        call.__name__ = name
        return call

    def packed_bgr(name):
        def call(_):
            eng.match_batch_device(n, d[name][0].data_ptr(), d[name][1].data_ptr(), out[name].data_ptr(), st.cuda_stream)
        call.__name__ = name
        return call

    def rectified(name, fmt):
        def call(_):
            eng.match_rectified_batch_device(n, d[name][0].data_ptr(), d[name][1].data_ptr(), image=A.image_desc(fmt),
                                             d_disp=out[name].data_ptr(), stream=st.cuda_stream)
        call.__name__ = name
        return call

    paths = (images("rg12p", "bayer_rg12p"), packed_bgr("rg12p_bgr"), images("rg12", "bayer_rg12"),
             images("mono12p", "mono12p"), packed_bgr("mono12p_bgr"), rectified("rect_rg12p", "bayer_rg12p"),
             rectified("rect_bgr_raw", "bgr"))
    ms = B.windows(eng, st, paths, args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # host path: unpack + cvtColor + convertScaleAbs + remap of every view on 16 threads, then adc_match_batch
    convert = lambda x: cv2.convertScaleAbs(cv2.cvtColor(unpack12p(x, sw), cv2.COLOR_BayerBG2BGR), alpha=1 / 16)  # noqa: E731
    lefts, rights = [raw[0]] * n, [raw[1]] * n

    def host():
        return eng.match_batch_ptrs([B.remap(convert(x), maps[0]) for x in lefts],
                                    [B.remap(convert(x), maps[1]) for x in rights])

    host_s, host_maps = B.host_seconds(host, args.rounds, threads=16)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {"rg12p_vs_rg12p_bgr": got["rg12p"].tobytes() == got["rg12p_bgr"].tobytes(),
              "rg12_vs_rg12p_bgr": got["rg12"].tobytes() == got["rg12p_bgr"].tobytes(),
              "mono12p_vs_mono12p_bgr": got["mono12p"].tobytes() == got["mono12p_bgr"].tobytes(),
              "rect_rg12p_vs_rect_bgr_raw": got["rect_rg12p"].tobytes() == got["rect_bgr_raw"].tobytes(),
              "rect_rg12p_vs_host": all(got["rect_rg12p"][i].tobytes() == host_maps[i].tobytes() for i in range(n)),
              "rg12p_vs_single_pair": all(got["rg12p"][i].tobytes() == eng.match(rg_dec[0], rg_dec[1]).tobytes()
                                          for i in (0, n - 1))}

    rg10p = [X.from_samples(v >> 2, "bayer_rg10p") for v in rg12]
    rg8 = [(v >> 4).astype(np.uint8) for v in rg12]
    kernels = B.kernels_vs_copy(eng, (
            ("image_ingest_rg12p", "image_ingest", lambda: eng.match_images(rg12p[0], rg12p[1], format="bayer_rg12p")),
            ("image_ingest_rg10p", "image_ingest", lambda: eng.match_images(rg10p[0], rg10p[1], format="bayer_rg10p")),
            ("image_ingest_rg12", "image_ingest", lambda: eng.match_images(rg12[0], rg12[1], format="bayer_rg12")),
            ("image_ingest_mono12p", "image_ingest", lambda: eng.match_images(mono12p[0], mono12p[1], format="mono12p")),
            ("image_ingest_rg8", "image_ingest", lambda: eng.match_images(rg8[0], rg8[1], format="bayer_rggb")),
            ("rectify_rg12p", "rectify", lambda: eng.match_rectified(raw[0], raw[1], format="bayer_rg12p")),
            ("rectify_bgr", "rectify", lambda: eng.match_rectified(raw_bgr[0], raw_bgr[1]))), reps=50, dev=dev)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    calls = {"rg12p": "adc_match_images_batch_device (BayerRG12p, tight rows of 675 bytes)",
             "rg12p_bgr": "adc_match_batch_device (the same frames converted beforehand, packed BGR)",
             "rg12": "adc_match_images_batch_device (BayerRG12, the same samples in 16-bit words)",
             "mono12p": "adc_match_images_batch_device (Mono12p)",
             "mono12p_bgr": "adc_match_batch_device (the same frames converted beforehand, packed BGR)",
             "rect_rg12p": "adc_match_rectified_batch_device (640x480 raw BayerRG12p, CV_16SC2 maps)",
             "rect_bgr_raw": "adc_match_rectified_batch_device (the same raw frames converted beforehand, BGR)"}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            **{k: {"value": rate[k], "call": c} for k, c in calls.items()},
            "host_unpack_cvtcolor_scale_remap": {
                "value": host_rate, "opencv": cv2.__version__,
                "call": "numpy unpack + cv2.cvtColor + cv2.convertScaleAbs + cv2.remap on the host (both views, 16 threads) "
                        "+ adc_match_batch"},
            "rg12p_vs_rg12p_bgr": round(rate["rg12p"] / rate["rg12p_bgr"], 4),
            "rg12_vs_rg12p_bgr": round(rate["rg12"] / rate["rg12p_bgr"], 4),
            "mono12p_vs_mono12p_bgr": round(rate["mono12p"] / rate["mono12p_bgr"], 4),
            "rect_rg12p_vs_rect_bgr_raw": round(rate["rect_rg12p"] / rate["rect_bgr_raw"], 4),
            "rect_rg12p_vs_host": round(rate["rect_rg12p"] / host_rate, 2),
            "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "kernels": kernels,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
