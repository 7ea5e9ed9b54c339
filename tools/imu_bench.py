"""Per-scan cost of the IMU forward propagation: on the device (flb_imu_process) vs the host stand-in (the CPU oracle's
propagation on one core + the IMUpose upload + undistortion + voxel filter through the host-fed front-end calls).

For each sensor (hdl64, hap) and IMU rate (200 Hz, 1 kHz), a drive of driver records (synth.driver_records) with an IMU
stream (synth.imu_samples) runs through both arms; each scan is preprocessed on the device, then
  device arm: flb_imu_process(leaf) -> flb_scan_step
  host arm:   oracle propagation (tests/cpp/imu_oracle.cpp, dense, g++ -O2, one core) -> flb_frontend_undistort ->
              flb_frontend_voxel_filter -> flb_scan_step
and reports per-scan medians: flb_imu_process wall and device time, the propagation kernel alone (torch.profiler, a
separate pass), the host propagation, and scans/s from driver records + IMU span to the posterior for both arms.  The
reference node's own Eigen propagation is not measured here (the oracle is a dense restatement without Eigen).

    python tools/imu_bench.py --scans 40 --warmup 5 --out profiles/imu_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from better_fastlio2_b200 import capi, synth  # noqa: E402
from tests import imu_oracle as io  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        out = f"unavailable: {e}"
    return out


def drive(model, rate, n, seed=1):
    rng = np.random.default_rng(seed)
    world = synth.city_world(half_extent=200, seed=seed)
    irng = np.random.default_rng(seed + 100)
    scans = []
    for k in range(n):
        beg, end = 0.1 * k, 0.1 * k + 0.1
        pos, R, _, _ = synth.imu_trajectory(beg)
        st = synth.make_state(pos=pos, rot=synth.quat_from_rotvec([0, 0, np.arctan2(R[1, 0], R[0, 0])]), offT=(0, 0, 0))
        rec = synth.driver_records(model, world, st, rng, max_range=80.0)
        scans.append((rec, synth.imu_samples(beg, end, rate, irng), beg, end))
    st0 = synth.make_state(pos=synth.imu_trajectory(0.0)[0], rot=(0, 0, 0, 1), offT=(0, 0, 0), vel=(10.0, 0, 0))
    body0 = synth.scan_from_pose(world, st0, synth.lidar_dirs("hdl64" if model == "hdl64" else "hap", rng), rng, max_range=80.0)
    return scans, synth.body_to_world_np(st0, synth.voxel_downsample(body0, 0.2)), st0


def pre_cfg(model):
    if model == "hdl64":
        return capi.preprocess_config(capi.VELO16, n_scans=64, time_unit=capi.SEC, blind=2.0)
    return capi.preprocess_config(capi.LIVOX, n_scans=4, time_unit=capi.NS, blind=2.0)


def run_arm(arm, model, scans, map_pts, st0, leaf, warmup, profile=False):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 22, max_blocks=1 << 19)
    tree.Build(map_pts)
    ses = capi.Session(tree, max_scan_points=1 << 18, max_iterations=4)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 19)
    imu = capi.Imu(fe)
    o = io.OracleImu()
    cfg = pre_cfg(model)
    x, P = st0.copy(), synth.default_cov()
    t_scan, t_call, t_dev, t_host, n_pts, n_imu = [], [], [], [], [], []
    for k, (rec, samples, beg, end) in enumerate(scans):
        t0 = time.perf_counter()
        n_raw, _ = fe.preprocess(rec, cfg)
        if arm == "device":
            t1 = time.perf_counter()
            xp, Pp, r = imu.process(samples, beg, end, x, P, leaf)
            t2 = time.perf_counter()
            status = r.status
        else:
            t1 = time.perf_counter()
            status, xp, Pp, poses = o.process(samples, beg, end, x, P)
            t2 = time.perf_counter()
            if status == 2:
                fe.undistort(poses, xp)
                fe.voxel_filter(leaf)
        if status != 2:
            x, P = xp, Pp
            continue
        x, P, _ = ses.scan_step(None, None, xp, Pp)
        t3 = time.perf_counter()
        if k >= warmup:
            t_scan.append(t3 - t0)
            t_call.append(t2 - t1)
            n_pts.append(n_raw)
            n_imu.append(len(samples))
            if arm == "device":
                t_dev.append(r.gpu_ms * 1e-3)
            else:
                t_host.append(t2 - t1)
    kern = profile_kernel(fe, scans, st0) if profile and arm == "device" else None
    imu.close()
    fe.close()
    ses.close()
    tree.close()
    med = lambda a: float(np.median(a)) * 1e3 if a else None   # noqa: E731
    return dict(scans=len(t_scan), raw_points_median=int(np.median(n_pts)), imu_samples_median=int(np.median(n_imu)),
                scan_ms_median=med(t_scan), scans_per_s=len(t_scan) / float(np.sum(t_scan)),
                propagation_call_ms_median=med(t_call), imu_process_device_ms_median=med(t_dev),
                host_propagation_ms_median=med(t_host), propagation_kernel_ms=kern)


def profile_kernel(fe, scans, st0):
    """Duration of k_imu_propagate alone from torch.profiler's CUDA activity records, in a pass of its own over the same
    IMU spans (a fresh processor, empty scans)."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        imu = capi.Imu(fe)
        fe.upload(np.zeros((0, 12), np.float32))
        x, P = st0.copy(), synth.default_cov()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for rec, samples, beg, end in scans:
                x, P, r = imu.process(samples, beg, end, x, P)
        imu.close()
        times = [ev.device_time_total for ev in prof.events() if "k_imu_propagate" in ev.name]
        return float(np.median(times)) * 1e-3 if times else None
    except Exception as e:   # noqa: BLE001
        return f"not measured: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() <= 0:
        raise SystemExit("no CUDA device: this benchmark measures the GPU path and has no CPU fallback")
    res = dict(gpu=gpu_info(), scans=a.scans, warmup=a.warmup, leaf=a.leaf, rows=[],
               not_measured=["the reference node's own Eigen predict chain (the host arm runs the dense oracle restatement)",
                             "sync_packages and the driver callbacks"])
    for model in ("hdl64", "hap"):
        for rate in (200.0, 1000.0):
            scans, mp, st0 = drive(model, rate, a.scans + 1)
            dev = run_arm("device", model, scans, mp, st0, a.leaf, a.warmup, profile=True)
            host = run_arm("host", model, scans, mp, st0, a.leaf, a.warmup)
            row = dict(model=model, imu_rate_hz=rate, device=dev, host=host)
            print(json.dumps(row), flush=True)
            res["rows"].append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
