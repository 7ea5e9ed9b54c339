#!/usr/bin/env python
"""Scan Context descriptors on one GPU: flb_keyframes_scan_context / _scan_contexts next to the host path they replace.

Workload (synthetic): body-frame key frames ray-cast in the city world, Livox HAP (120 x 25 deg, 240 000 rays) and
HDL-64 (64 x 1875 rays), 8 distinct scans of each cycled through the key frames.  In one run it reports:
  loop_attempt   performLoopClosure's gate (laserMapping.cpp:916-940) for two loop sub-maps of 2 * 10 + 1 key frames
                 (historyKeyframeSearchNum = 10), one affine per key frame, the identity for the key frame itself:
                   device  two flb_keyframes_scan_context calls
                   host    two flb_keyframes_assemble calls (dense, downloaded) + the oracle's makeScancontext of each
                           on one host core
                 with the bytes each path copies device to host
  saver          the key-frame saver (:2501-2505) over 200 HAP key frames: one flb_keyframes_scan_contexts call against
                 the oracle's makeScancontext of the same clouds on one host core (download not counted)
Timing is host wall clock around calls that end in a synchronisation; medians with p10-p90.  The GPU name and power
limit are read in the same run.  Writes one JSON document to stdout and to --out.

  python tools/scan_context_bench.py --reps 10 --out /tmp/scan_context_bench.json
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
from tests import scan_context_oracle as sco  # noqa: E402

N_DISTINCT = 8
SEARCH_NUM = 10
KEY_BYTES = 20 * 60 * 4   # one descriptor as copied to the host: 1200 uint32 keys, turned into doubles there


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


def affine(p6):
    """pcl::getTransformation as a 4x4 float64 matrix."""
    x, y, z, roll, pitch, yaw = [float(v) for v in p6]
    A, B, C, D, E, F = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    return np.array([[A * C, A * D * F - B * E, B * F + A * D * E, x], [B * C, A * E + B * D * F, B * D * E - A * F, y],
                     [-D, C * F, C * E, z], [0, 0, 0, 1]])


def loop_selection(key, poses):
    """loopFindNearKeyframes: ids key-10 .. key+10 and keyTrans^-1 * keyNearTrans (the identity for key itself)."""
    ids, T = [], []
    for i in range(-SEARCH_NUM, SEARCH_NUM + 1):
        k = key + i
        if 0 <= k < len(poses):
            ids.append(k)
            T.append(np.eye(3, 4) if i == 0 else (np.linalg.inv(affine(poses[key])) @ affine(poses[k]))[:3])
    return np.array(ids, np.int32), np.stack(T).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--save-keyframes", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() <= 0:
        raise SystemExit("scan_context_bench: no CUDA device (nothing is measured without one)")
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
    res = {"gpu": name, "power_limit_w": limit, "reps": a.reps, "warmup": a.warmup,
           "workload": f"synthetic key frames ({N_DISTINCT} ray-cast scans per sensor, cycled), body frame",
           "timing": "host wall clock around calls that end in a synchronisation; medians with p10-p90 over the timed calls",
           "loop_attempt": {}}
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)

    # ---------------------------------------------------------------------------------------------- one loop attempt
    n_kf = 4 * SEARCH_NUM + 4
    poses = np.array([[0.8 * k, 0.1 * k, 0.0, 0.0, 0.0, 0.02 * k] for k in range(n_kf)], np.float32)
    for model in ("hap", "hdl64"):
        clouds = [scans[model][k % N_DISTINCT] for k in range(n_kf)]
        store = capi.KeyFrameStore(tree, sum(len(c) for c in clouds), n_kf)
        for c in clouds:
            store.append(capi.pack_pointtype(c[:, :3], c[:, 3]))
        cur, prev = loop_selection(n_kf - 1 - SEARCH_NUM, poses), loop_selection(SEARCH_NUM, poses)
        n_sub = [int(sum(len(clouds[k]) for k in s[0])) for s in (cur, prev)]
        dev_ms, host_ms = [], []
        for i in range(a.warmup + a.reps):   # the two paths alternate, so drift on the shared host hits both alike
            td, (dc, dp) = timed(lambda: (store.scan_context(cur[0], affines=cur[1]), store.scan_context(prev[0], affines=prev[1])))

            def host():
                out = []
                for ids, T in (cur, prev):
                    xyzi, _ = store.assemble(ids, affines=T)
                    out.append(sco.scan_context(xyzi, 1.5)[0])
                return out
            th, (hc, hp) = timed(host)
            if i >= a.warmup:
                dev_ms.append(td)
                host_ms.append(th)
        _, _, mask_c = sco.scan_context(store.assemble(cur[0], affines=cur[1])[0], 1.5)
        same = bool(np.array_equal(dc[~mask_c], hc[~mask_c]))
        res["loop_attempt"][model] = {
            "key_frames_per_submap": int(len(cur[0])), "points_per_submap": n_sub,
            "device_two_scan_context": dict(stats(dev_ms), d2h_bytes=2 * KEY_BYTES),
            "host_assemble_download_makeScancontext": dict(stats(host_ms), d2h_bytes=20 * sum(n_sub)),
            "descriptors_agree_off_atan_sensitive_bins": same}
        print(json.dumps({model: res["loop_attempt"][model]}), file=sys.stderr, flush=True)
        store.close()

    # ---------------------------------------------------------------------------------------------- saver
    K = a.save_keyframes
    clouds = [scans["hap"][k % N_DISTINCT] for k in range(K)]
    n_save = int(sum(len(c) for c in clouds))
    sv = capi.KeyFrameStore(tree, n_save, K)
    for c in clouds:
        sv.append(capi.pack_pointtype(c[:, :3], c[:, 3]))
    ids = np.arange(K, dtype=np.int32)
    ms = []
    for i in range(a.warmup + a.reps):
        t, d = timed(lambda: sv.scan_contexts(ids))
        if i >= a.warmup:
            ms.append(t)
    t0 = time.perf_counter()
    host = [sco.scan_context(c, 1.5) for c in clouds]
    host_ms = (time.perf_counter() - t0) * 1e3
    same = all(np.array_equal(d[j][~host[j][2]], host[j][0][~host[j][2]]) for j in range(K))
    res["saver"] = {"key_frames": K, "points": n_save, "device_scan_contexts": dict(stats(ms), d2h_bytes=K * KEY_BYTES),
                    "host_makeScancontext_one_core_ms": host_ms, "host_note": "once, over the same clouds already on the host",
                    "descriptors_agree_off_atan_sensitive_bins": bool(same),
                    "map_scratch_bytes_after": sv.info()["map_scratch_bytes"]}
    sv.release_scratch()
    sv.close()
    tree.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
