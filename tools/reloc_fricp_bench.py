#!/usr/bin/env python
"""Relocalisation registration on one GPU: flb_keyframes_fricp (regMode 4, Fast and Robust ICP) next to a host path.

Workload (synthetic): body-frame key frames ray-cast in the city world, a prior session of key frames along a street and
a live scan of one of its places (another noise draw) displaced from its prior pose by 0.5 m / 2 degrees:
  hdl64_3      a dense HDL-64 /cloud_registered scan against searchNum 3 dense prior key frames
  hap_3        the same with Livox HAP scans
  hdl64_ds_1   the HDL-64 scan 0.5 m voxel-filtered against searchNum 1
For each it reports the device call (median and p10-p90 of a host clock around the synchronising call), its stages and
iterations, the device time per iteration, the share of a call spent before the first iteration (index build, 7-NN
median and the other set-up, from max_icp = 0 calls alternated with the full ones) and the bytes it copies device to host.
The host path is the CPU oracle (tests/cpp/fricp_oracle.cpp, one core, a k-d tree like the reference's nanoflann), which
stands in for the reference's Eigen build: it is run with max_icp = 1 and 12 (two short stages), the difference gives its
time per iteration and the rest its set-up, and it is scaled to the device call's iteration count.  The GPU name and power limit are read in the same run.  Writes one JSON
document to stdout and to --out.

  python tools/reloc_fricp_bench.py --reps 10 --out /tmp/reloc_fricp_bench.json
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
from tests import fricp_oracle as fo  # noqa: E402

STEP_BYTES, MEDIAN_BYTES, SETUP_BYTES = 8 * 17, 8 * 2, 4 * 16 + 8 * 8 + 4 * 7


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


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def p6(R, t):
    return np.array([t[0], t[1], t[2], np.arctan2(R[2, 1], R[2, 2]), -np.arcsin(R[2, 0]), np.arctan2(R[1, 0], R[0, 0])], np.float32)


def voxel(pts, leaf):
    k = np.floor(pts[:, :3] / leaf).astype(np.int64)
    _, inv = np.unique(k, axis=0, return_inverse=True)
    out = np.zeros((inv.max() + 1, 4))
    np.add.at(out, inv.reshape(-1), pts)
    return (out / np.bincount(inv.reshape(-1))[:, None]).astype(np.float32)


def case(model, n_near, leaf, reps):
    world = synth.city_world(half_extent=200.0, seed=5)
    rng = np.random.default_rng(1)
    kfs, poses = [], []
    for j in range(n_near):
        st = synth.trajectory_state(6 * j)
        dirs = synth.lidar_dirs(model, np.random.default_rng(20 + j))
        kfs.append(synth.scan_from_pose(world, st, dirs, np.random.default_rng(j), max_range=100.0, min_range=1.0).astype(np.float32))
        R = synth.quat_to_mat(st[3:7]) @ synth.quat_to_mat(st[7:11])
        poses.append((R, st[0:3] + synth.quat_to_mat(st[3:7]) @ st[11:14]))
    a = n_near // 2
    st = synth.trajectory_state(6 * a)
    live = synth.scan_from_pose(world, st, synth.lidar_dirs(model, np.random.default_rng(20 + a)), np.random.default_rng(99),
                                max_range=100.0, min_range=1.0).astype(np.float32)
    live = np.column_stack([live, rng.integers(0, 256, len(live))]).astype(np.float32)
    if leaf > 0:
        live = voxel(live, leaf)
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(k) for k in kfs) + 16, n_near + 1)
    for c in kfs:
        kf.append(capi.pack_pointtype(c))
    ids = np.arange(n_near, dtype=np.int32)
    poses6 = np.stack([p6(*p) for p in poses])
    init = p6(*poses[a]) + np.array([0.4, -0.3, 0.0, 0.0, 0.0, np.deg2rad(2.0)], np.float32)

    def call(max_icp=100):
        return kf.fricp(live, ids, poses6, src_pose6=init, mode=4, max_icp=max_icp)

    for _ in range(2):   # warm-up of both shapes
        call()
        call(0)
    full, setup = [], []
    for _ in range(reps):   # alternating
        ms, g = timed(call)
        full.append(ms)
        setup.append(timed(lambda: call(0))[0])
    g0 = call(0)
    it = g["iterations"]
    per_it = (np.median(full) - np.median(setup)) / max(it, 1)
    d2h = SETUP_BYTES + 2 * MEDIAN_BYTES + STEP_BYTES * (it + g["rejections"] + 2 * g["stages"] + 1)
    # host path: the oracle on one core, short runs, scaled to the device call's iterations
    src = fo._p4(live)
    tgt = kf.assemble(ids, poses6=poses6)[0]
    from oracle import pyoracle
    pyoracle.build()
    s = pyoracle.transform_cloud_rpy(src, init)
    fo.lib()   # compiled on first use: not part of the timing
    t1, (o1, _, _, _) = timed(lambda: fo.fricp(s, tgt, mode=4, max_icp=1, nu_alpha=1e-9))
    t4, (o4, _, _, _) = timed(lambda: fo.fricp(s, tgt, mode=4, max_icp=12, nu_alpha=1e-9))
    host_it = (t4 - t1) / max(o4["iterations"] - o1["iterations"], 1)
    t_setup = t1 - host_it * o1["iterations"]
    kf.close()
    tree.close()
    return {"n_source": int(len(live)), "n_target": int(g["n_target"]), "call": stats(full), "setup_call": stats(setup),
            "setup_share": float(np.median(setup) / np.median(full)), "stages": g["stages"], "iterations": it,
            "rejections": g["rejections"], "device_ms_per_iteration": float(per_it), "d2h_bytes": int(d2h),
            "setup_stages": g0["stages"],
            "host_oracle": {"setup_ms": t_setup, "ms_per_iteration": host_it, "scaled_call_ms": t_setup + host_it * it}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "reloc_fricp_bench.json"))
    a = ap.parse_args()
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit_w": limit, "mode": 4, "cases": {}}
    for key, model, n, leaf in (("hdl64_3", "hdl64", 3, 0.0), ("hap_3", "hap", 3, 0.0), ("hdl64_ds_1", "hdl64", 1, 0.5)):
        res["cases"][key] = case(model, n, leaf, a.reps)
        print(key, json.dumps(res["cases"][key]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
