#!/usr/bin/env python
"""Loop-closure ICP on one GPU: flb_keyframes_icp next to the host path it replaces.

Workload (synthetic): body-frame key frames ray-cast in the city world (8 distinct scans per sensor, cycled), a loop
sub-map pair of the same key frames where the current pass is displaced by a known motion (0.9 m, 3 degrees):
  hdl64_10   HDL-64, historyKeyframeSearchNum 10 (21 key frames per sub-map)
  hap_10     Livox HAP, searchNum 10 (21 key frames per sub-map)
  hap_1      Livox HAP, searchNum 1 (3 key frames per sub-map)
For each it reports the device call (median and p10-p90 of a host clock around the synchronising call), its iterations
and time per iteration, the share of one call spent building the target index (a max_iterations = 0 call, which runs
the index build, one iteration and the fitness pass, against the full call), the bytes it copies device to host, and
the host path beside it: assemble + download of both sub-maps, then the CPU oracle's ICP (tests/cpp/icp_oracle.cpp) on
one core, which stands in for PCL (not available here), capped at --host-iters iterations.  The GPU name and power
limit are read in the same run.  Writes one JSON document to stdout and to --out.

  python tools/loop_icp_bench.py --reps 10 --out /tmp/loop_icp_bench.json
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
from tests import icp_oracle as io  # noqa: E402

N_DISTINCT = 8
SUMS_BYTES, BOUNDS_BYTES = 8 * 17, 4 * 7   # an iteration's (and the fitness pass's) reduction record; the target box + count


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


def rotz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-iters", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() <= 0:
        raise SystemExit("loop_icp_bench: no CUDA device (nothing is measured without one)")
    name, limit = gpu_info()
    rng = np.random.default_rng(3)
    world = synth.city_world(half_extent=400.0, seed=3)
    scans = {}
    for model in ("hap", "hdl64"):
        scans[model] = []
        for j in range(N_DISTINCT):
            dirs = synth.lidar_dirs(model, np.random.default_rng(100 + j))
            xyz = synth.scan_from_pose(world, synth.trajectory_state(10 * j), dirs, rng, max_range=100.0, min_range=2.0)
            scans[model].append(np.column_stack([xyz, rng.integers(0, 256, len(xyz))]).astype(np.float32))
    R, t = rotz(np.deg2rad(3.0)), np.array([0.9, -0.6, 0.05])
    Ri, ti = R.T, -R.T @ t
    res = {"gpu": name, "power_limit_w": limit, "reps": a.reps, "warmup": a.warmup,
           "workload": f"synthetic key frames ({N_DISTINCT} ray-cast scans per sensor, cycled), loop pair displaced by 0.9 m / 3 deg",
           "timing": "host wall clock around calls that end in a synchronisation; medians with p10-p90 over the timed calls",
           "host_path": "flb_keyframes_assemble of both sub-maps (downloaded) + the CPU oracle's ICP on one core, standing in "
                        "for PCL (not available); capped at host_iters iterations",
           "cases": {}}
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    for case, model, search in (("hdl64_10", "hdl64", 10), ("hap_10", "hap", 10), ("hap_1", "hap", 1)):
        n_kf = 2 * search + 1
        clouds = [scans[model][k % N_DISTINCT] for k in range(n_kf)]
        store = capi.KeyFrameStore(tree, sum(len(c) for c in clouds), n_kf)
        for c in clouds:
            store.append(capi.pack_pointtype(c[:, :3], c[:, 3]))
        prev_T, cur_T = [], []
        for k in range(n_kf):
            A = np.column_stack([rotz(0.02 * (k - search)), [0.8 * (k - search), 0.1 * (k - search), 0.0]])
            prev_T.append(A.astype(np.float32).reshape(12))
            cur_T.append(np.column_stack([Ri @ A[:, :3], Ri @ A[:, 3] + ti]).astype(np.float32).reshape(12))
        ids = np.arange(n_kf, dtype=np.int32)
        prev_T, cur_T = np.stack(prev_T), np.stack(cur_T)
        call = lambda **kw: store.icp(ids, ids, src_affines=cur_T, tgt_affines=prev_T, **kw)  # noqa: E731
        full, first = [], []
        for i in range(a.warmup + a.reps):   # full calls and index-build calls alternate
            tf, g = timed(call)
            t0, _ = timed(lambda: call(max_iterations=0))
            if i >= a.warmup:
                full.append(tf)
                first.append(t0)
        it = g["iterations"]
        med_full, med_first = float(np.median(full)), float(np.median(first))
        per_iter = (med_full - med_first) / max(it - 1, 1)
        index_ms = max(med_first - 2 * per_iter, 0.0)   # one iteration + the fitness pass, which is an iteration's 1-NN
        T = g["final_transformation"].astype(np.float64)
        n_sub = int(g["n_source"])

        def host():
            src, _ = store.assemble(ids, affines=cur_T)
            tgt, _ = store.assemble(ids, affines=prev_T)
            return io.icp(src, tgt, max_iterations=min(it, a.host_iters))
        th, (o, _, _, _) = timed(host)
        res["cases"][case] = {
            "key_frames_per_submap": n_kf, "points_per_submap": [n_sub, int(g["n_target"])],
            "device_call": dict(stats(full), d2h_bytes=SUMS_BYTES * (it + 1) + BOUNDS_BYTES),
            "iterations": it, "state": g["state_name"], "fitness_score": g["fitness_score"],
            "device_ms_per_iteration": per_iter,
            "device_max_iterations_0_call": stats(first),
            "index_build_share_of_call": index_ms / med_full,
            "error_vs_truth_cm": float(np.abs(T[:3, 3] - t).max() * 100),
            "host_assemble_download_oracle_icp": {"ms": th, "iterations": o["iterations"], "ms_per_iteration_incl_tree": th / max(o["iterations"], 1),
                                                  "d2h_bytes": 20 * 2 * n_sub},
        }
        print(json.dumps({case: res["cases"][case]}), file=sys.stderr, flush=True)
        store.release_scratch()
        store.close()
    tree.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
