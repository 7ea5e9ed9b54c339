"""Cost of the camera-coloured and IMU-frame publishers (publish_frame_world_color, laserMapping.cpp:310-392, with
imageCallback :250-276; publish_frame_body, :1543-1558) on the device against the host path they replace.

Workload: a synthetic Livox HAP scan ray-cast in a city (about 222k points), undistorted through flb_frontend_process,
and its 0.5 m VoxelGrid; a forward camera (fx = fy = 900, principal point at the image centre) and a seeded random
720 x 1280 bgr8 frame.  Device rows call the C ABI directly with preallocated host buffers; the host rows download the
cloud (flb_frontend_download_undistorted / _down) and run the CPU oracle's sequential loop on one core
(tests/cpp/color_oracle.cpp, a restatement without OpenCV's per-point Mat temporaries, so a lower bound on the
reference's cost), and imageCallback's pixel-by-pixel copy.  Host clock around calls that end in a synchronisation;
medians with p10-p90.  The GPU name and power limit are read in the same run.  Writes one JSON document to stdout and to
--out.

  python tools/color_bench.py --reps 50 --out /tmp/color_bench.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from better_fastlio2_b200 import capi, synth  # noqa: E402
from tests import color_oracle as co  # noqa: E402

W, H = co.W_MAX, co.H_MAX


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:
        limit = None
    return name, limit


def stats(ms):
    a = np.asarray(ms, np.float64)
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90)),
            "n": int(len(a))}


def bench(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return stats(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = gpu_info()

    rng = np.random.default_rng(3)
    world = synth.city_world(half_extent=150, seed=3)
    st_true = synth.trajectory_state(0)
    body = synth.scan_from_pose(world, st_true, synth.lidar_dirs("hap", rng), rng)
    xyz, inten, cur = synth.raw_scan_with_times(body, rng)
    poses, end = synth.imu_pose_sequence(st_true, rng)
    pts48 = np.ascontiguousarray(capi.pack_pointtype(xyz, inten, cur))
    poses = np.ascontiguousarray(poses, np.float64)
    end = np.ascontiguousarray(end, np.float64)
    st = np.ascontiguousarray(st_true, np.float64)
    ex, ki = co.forward_camera(t=(0.04, -0.03, 0.12))
    img = np.random.default_rng(4).integers(0, 256, (H, W, 3), dtype=np.uint8)

    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 20, max_blocks=1 << 16)
    ses = capi.Session(tree, max_scan_points=1 << 18, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 18)
    n_down = fe.process_ptr(pts48.ctypes.data, len(pts48), poses, end, 0.5)
    fe.set_camera(ex, ki)
    fe.upload_image(img)
    L = capi.lib()
    cap = fe.cap
    out_xyzi = np.empty((cap, 4), np.float32)
    out_bgra = np.empty(cap, np.uint32)
    n = C.c_int(0)
    p = capi._p

    def colorize(which):
        capi._chk(L.flb_frontend_points_colorize(fe.h, which, p(st), p(out_xyzi), p(out_bgra), cap, C.byref(n)))
        return n.value

    def upload():
        capi._chk(L.flb_frontend_camera_image(fe.h, C.c_void_p(img.ctypes.data), H, W, 3 * W))
        ses.sync()

    def to_imu():
        capi._chk(L.flb_frontend_points_to_imu(fe.h, p(st), p(out_xyzi), cap, C.byref(n)))

    und, _, _ = fe.download_undistorted()
    down, _ = fe.download_down()
    kept = {"dense": colorize(1), "voxel": colorize(0)}
    # the device result is the oracle's (checked here once, bit for bit, so the timed rows compute the same thing)
    for which, cloud in ((1, und), (0, down)):
        k = colorize(which)
        o = co.colorize(ex, ki, img, cloud, st)
        assert k == len(o[2]) and np.array_equal(out_xyzi[:k], o[0]) and np.array_equal(out_bgra[:k], o[1])

    res = {"gpu": name, "power_limit_w": limit, "reps": a.reps, "warmup": a.warmup, "host_reps": a.host_reps,
           "workload": "synthetic Livox HAP scan ray-cast in a city, undistorted; forward camera fx = fy = 900, 1280 x 720 bgr8",
           "timing": "host wall clock around calls that end in a synchronisation; medians with p10-p90 over the timed calls",
           "host_path": "download of the cloud + the CPU oracle's sequential loop on one core (no OpenCV Mat temporaries: a "
                        "lower bound on the reference); the image row is imageCallback's pixel-by-pixel copy",
           "points": {"dense": len(und), "voxel": int(n_down)}, "kept": kept, "rows": {}}
    R = res["rows"]
    R["colorize_dense_device"] = bench(lambda: colorize(1), a.reps, a.warmup)
    R["colorize_voxel_device"] = bench(lambda: colorize(0), a.reps, a.warmup)
    R["upload_image_device"] = bench(upload, a.reps, a.warmup)
    R["to_imu_device"] = bench(to_imu, a.reps, a.warmup)

    OL = co.lib()
    M16, K12 = np.ascontiguousarray(ex, np.float64), np.ascontiguousarray(ki, np.float64)
    h_xyzi = np.empty((cap, 4), np.float32)
    h_bgra = np.empty(cap, np.uint32)
    h_idx = np.empty(cap, np.int32)
    dl_xyzi = np.empty((cap, 4), np.float32)
    dl_cur = np.empty(cap, np.float32)
    host_img = np.empty((H, W, 3), np.uint8)

    def host_colorize(which):
        if which == 1:
            capi._chk(L.flb_frontend_download_undistorted(fe.h, p(dl_xyzi), p(dl_cur), None, cap, C.byref(n)))
        else:
            capi._chk(L.flb_frontend_download_down(fe.h, p(dl_xyzi), p(dl_cur), cap, C.byref(n)))
        OL.orc_colorize(M16.ctypes.data, K12.ctypes.data, W, H, host_img.ctypes.data, dl_xyzi.ctypes.data, n.value, st.ctypes.data,
                        h_xyzi.ctypes.data, h_bgra.ctypes.data, h_idx.ctypes.data)

    def host_image():
        OL.orc_copy_image(img.ctypes.data, 3 * W, W, H, host_img.ctypes.data)

    def host_to_imu():
        capi._chk(L.flb_frontend_download_undistorted(fe.h, p(dl_xyzi), p(dl_cur), None, cap, C.byref(n)))
        OL.orc_to_imu(dl_xyzi.ctypes.data, n.value, st.ctypes.data, h_xyzi.ctypes.data)

    R["colorize_dense_host"] = bench(lambda: host_colorize(1), a.host_reps, 1)
    R["colorize_voxel_host"] = bench(lambda: host_colorize(0), a.host_reps, 1)
    R["image_copy_host"] = bench(host_image, a.host_reps, 1)
    R["to_imu_host"] = bench(host_to_imu, a.host_reps, 1)
    fe.close()
    ses.close()
    tree.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
