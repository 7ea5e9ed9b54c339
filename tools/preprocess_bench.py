#!/usr/bin/env python
"""Driver records -> posterior on one GPU, with Preprocess::process on the device (flb_frontend_preprocess), next to
the path it replaces (host preprocessing, then 48-byte PointType records uploaded with flb_frontend_upload).

Per sensor (HDL-64 Velodyne with and without per-point time, Ouster 64x1024, Livox HAP-style CustomMsg) it reports:
  preprocess_device_ms     CUDA events around flb_frontend_preprocess on the session stream (H2D copy + kernels)
  preprocess_call_ms       host clock around the same call (ends in its one synchronisation)
  to_feats_down_ms         host clock: preprocess + undistort + VoxelGrid (feats_down_body left on the device)
  scans_per_s              driver records -> posterior: the above + flb_scan_step, over the timed steps
  h2d_bytes_per_scan       the driver message vs the PointType path's n_kept * 48 bytes
  host_path                the same chain with the CPU preprocessing (the oracle restatement, one host core) and
                           the PointType upload: oracle_preprocess_ms, to_feats_down_ms, scans_per_s
The GPU name and power limit are read in the same run.  Writes one JSON document to stdout and to --out.

  python tools/preprocess_bench.py --steps 40 --out /tmp/preprocess_bench.json
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
from tests import preprocess_cases as pc  # noqa: E402
from tests import preprocess_oracle as po  # noqa: E402

SENSORS = [("hdl64_time", "hdl64", True), ("hdl64_no_time", "hdl64", False), ("os64", "os64", True), ("hap_livox", "hap", True)]
LEAF = 0.5


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    limit = None
    try:
        import pynvml
        pynvml.nvmlInit()
        limit = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1e3
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            limit = float(out.splitlines()[0])
        except Exception:
            limit = None
    return name, limit


def run_sensor(label, model, with_time, steps, warmup, n_sweeps, world, map_pts):
    import torch
    cfg = dict(pc.SENSOR_CFG[model])
    rng = np.random.default_rng(11)
    sweeps = []
    for k in range(n_sweeps):
        st = synth.trajectory_state(k)
        rec = synth.driver_records(model, world, st, rng, with_time=with_time)
        poses, end = synth.imu_pose_sequence(st, rng)
        sweeps.append((rec, poses, end, synth.perturb_state(st, rng, sig_pos=0.02, sig_rot_deg=0.2)))
    cap = max(len(s[0]) for s in sweeps)
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 22, max_blocks=1 << 19)
    tree.Build(map_pts)
    ses = capi.Session(tree, max_scan_points=cap, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=cap)
    stream = torch.cuda.ExternalStream(ses.stream_ptr())
    P = synth.default_cov()

    def device_path(i):
        rec, poses, end, prior = sweeps[i % n_sweeps]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        n, last = fe.preprocess(rec, cfg)
        e1.record(stream)
        t1 = time.perf_counter()
        fe.undistort(poses, end)
        fe.voxel_filter(LEAF)
        t2 = time.perf_counter()
        ses.scan_step(None, None, prior, P)
        t3 = time.perf_counter()
        e1.synchronize()
        return dict(dev=e0.elapsed_time(e1), call=(t1 - t0) * 1e3, down=(t2 - t0) * 1e3, step=(t3 - t0), n=n,
                    bytes=rec.nbytes)

    def host_path(i):
        rec, poses, end, prior = sweeps[i % n_sweeps]
        t0 = time.perf_counter()
        xyzi, cur, last = po.preprocess(rec, cfg)
        t1 = time.perf_counter()
        fe.upload(capi.pack_pointtype(xyzi[:, :3], xyzi[:, 3], cur))
        fe.undistort(poses, end)
        fe.voxel_filter(LEAF)
        t2 = time.perf_counter()
        ses.scan_step(None, None, prior, P)
        t3 = time.perf_counter()
        return dict(orc=(t1 - t0) * 1e3, down=(t2 - t0) * 1e3, step=(t3 - t0), n=len(xyzi))

    for i in range(warmup):
        device_path(i)
        host_path(i)
    dev, host = [], []
    for i in range(steps):   # the two paths alternate, so drift on the shared host hits both alike
        dev.append(device_path(i))
        host.append(host_path(i))
    fe.close()
    ses.close()
    tree.close()
    med = lambda rows, k: float(np.median([r[k] for r in rows]))   # noqa: E731
    return {
        "sensor": label, "records_per_scan": int(np.mean([len(s[0]) for s in sweeps])),
        "record_bytes": int(sweeps[0][0].dtype.itemsize), "points_kept_per_scan": int(np.mean([r["n"] for r in dev])),
        "preprocess_device_ms": med(dev, "dev"), "preprocess_call_ms": med(dev, "call"), "to_feats_down_ms": med(dev, "down"),
        "scans_per_s": len(dev) / sum(r["step"] for r in dev),
        "h2d_bytes_per_scan": int(np.mean([r["bytes"] for r in dev])),
        "host_path": {"oracle_preprocess_ms": med(host, "orc"), "to_feats_down_ms": med(host, "down"),
                      "scans_per_s": len(host) / sum(r["step"] for r in host),
                      "h2d_bytes_per_scan": int(np.mean([r["n"] for r in host])) * capi.POINT_STRIDE},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sweeps", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() <= 0:
        raise SystemExit("preprocess_bench: no CUDA device (nothing is measured without one)")
    name, limit = gpu_info()
    rng = np.random.default_rng(7)
    world = synth.city_world(half_extent=200, seed=7)
    map_pts = synth.sample_surface_map(world, (30, 0, 0), 110, 0.2, rng)
    res = {"gpu": name, "power_limit_w": limit, "steps": a.steps, "warmup": a.warmup, "leaf": LEAF, "sensors": []}
    for label, model, with_time in SENSORS:
        res["sensors"].append(run_sensor(label, model, with_time, a.steps, a.warmup, a.sweeps, world, map_pts))
        print(json.dumps(res["sensors"][-1]), file=sys.stderr, flush=True)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
