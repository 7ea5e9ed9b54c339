#!/usr/bin/env python
"""Key-frame clouds on one GPU: the device key-frame store (flb_keyframes) next to the host-cloud path it replaces.

Workload (synthetic, cfg3-style): Livox HAP scans (120 x 25 deg, 240 000 rays, ray-cast in the city world) as body-frame
key frames.  In one run it reports:
  rebuild            recontructIKdTree of the 40 key frames within 10 m, leaf 0.2 (laserMapping.cpp:612-669):
                       host_clouds  flb_map_reconstruct_keyframes on 48-byte PointType records (uploaded every call)
                       store        flb_map_reconstruct_from_keyframes on the stored clouds
                     both alternate in the timed loop; wall clock per call (each call ends in a synchronisation)
  append             one key frame: flb_keyframes_append_frontend (device to device, timed to a stream synchronise) and
                     flb_keyframes_append from host records
  save_map           flb_keyframes_assemble over a few hundred key frames (saveMapService): dense (GlobalMap.pcd) and
                     VoxelGrid 0.7 m (mappingSurfLeafSize + 0.2, filterGlobalMap.pcd), results copied to the host
  h2d_bytes_per_call computed from shapes (records + segment table)
  cpu                the CPU restatement of the rebuild's data path (oracle transformPointCloud + pcl::VoxelGrid, one
                     core), once, for context
The GPU name and power limit are read in the same run.  Writes one JSON document to stdout and to --out.

  python tools/keyframe_bench.py --reps 10 --out /tmp/keyframe_bench.json
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

KF_SEG_BYTES = 72        # sizeof(KfSeg): the per-key-frame row of the assembly's segment table
N_DISTINCT = 8           # distinct ray-cast scans, cycled through the key frames
REBUILD_KF, RADIUS, LEAF = 40, 10.0, 0.2
SAVE_LEAF = 0.7


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


def pose6(st):
    R = synth.quat_to_mat(st[3:7])
    return [st[0], st[1], st[2], np.arctan2(R[2, 1], R[2, 2]), -np.arcsin(R[2, 0]), np.arctan2(R[1, 0], R[0, 0])]


def stats(ms):
    a = np.asarray(ms, np.float64)
    return {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max()),
            "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90)), "n": int(len(a))}


def timed(fn, sync):
    t0 = time.perf_counter()
    r = fn()
    sync()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--save-keyframes", type=int, default=200)
    ap.add_argument("--no-cpu", action="store_true", help="skip the one-core CPU restatement")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() <= 0:
        raise SystemExit("keyframe_bench: no CUDA device (nothing is measured without one)")
    import torch
    name, limit = gpu_info()
    sync = torch.cuda.synchronize

    rng = np.random.default_rng(3)
    world = synth.city_world(half_extent=400.0, seed=3)
    scans = []
    for j in range(N_DISTINCT):
        dirs = synth.lidar_dirs("hap", np.random.default_rng(100 + j))
        scans.append(synth.scan_from_pose(world, synth.trajectory_state(10 * j), dirs, rng, max_range=100.0, min_range=2.0))
    recs = [capi.pack_pointtype(s, rng.integers(0, 256, len(s)).astype(np.float32), np.linspace(0, 100, len(s), dtype=np.float32))
            for s in scans]
    pts_per_kf = float(np.mean([len(s) for s in scans]))
    print(f"[keyframe_bench] {name}, {N_DISTINCT} HAP scans of ~{pts_per_kf:.0f} points", file=sys.stderr, flush=True)

    # ---------------------------------------------------------------------------------------------- sub-map rebuild
    # 40 key frames 0.25 m apart: all within the 10 m search radius of the newest one
    poses = np.array([pose6(synth.trajectory_state(k, speed=2.5)) for k in range(REBUILD_KF)], np.float32)
    assert np.linalg.norm(poses[:, :3] - poses[-1, :3], axis=1).max() <= RADIUS
    kf_recs = [recs[k % N_DISTINCT] for k in range(REBUILD_KF)]
    n_sub = int(sum(len(r) for r in kf_recs))
    ta = capi.KDTree(voxel_size=0.1, max_points=32 << 20, max_blocks=4 << 20)
    tb = capi.KDTree(voxel_size=0.1, max_points=32 << 20, max_blocks=4 << 20)
    store = capi.KeyFrameStore(tb, n_sub, REBUILD_KF)
    for r in kf_recs:
        store.append(r)
    ids = np.arange(REBUILD_KF, dtype=np.int32)
    host_ms, store_ms = [], []
    for i in range(a.warmup + a.reps):   # the two paths alternate, so drift on the shared host hits both alike
        th, fa = timed(lambda: capi.reconstruct_keyframes(ta, kf_recs, poses, LEAF), sync)
        ts, fb = timed(lambda: store.reconstruct(ids, poses, LEAF), sync)
        if i >= a.warmup:
            host_ms.append(th)
            store_ms.append(ts)
    same = bool(np.array_equal(fa, fb) and ta.validnum() == tb.validnum())
    rebuild = {"key_frames": REBUILD_KF, "points_in": n_sub, "leaf": LEAF, "feats_from_map": int(len(fb)),
               "host_clouds": dict(stats(host_ms), h2d_bytes_per_call=n_sub * capi.POINT_STRIDE + REBUILD_KF * KF_SEG_BYTES),
               "store": dict(stats(store_ms), h2d_bytes_per_call=REBUILD_KF * KF_SEG_BYTES),
               "outputs_bit_identical": same}
    print(json.dumps(rebuild), file=sys.stderr, flush=True)
    store.close()
    ta.close()

    # ---------------------------------------------------------------------------------------------- append
    ses = capi.Session(tb, max_scan_points=1 << 18)
    cap = max(len(r) for r in recs)
    fe = capi.FrontEnd(ses, max_raw_points=cap)
    n_app = a.warmup + a.reps
    st_app = capi.KeyFrameStore(tb, 2 * n_app * cap, 2 * n_app)
    fe_ms, host_app_ms = [], []
    for i in range(n_app):
        r = recs[i % N_DISTINCT]
        fe.upload(r)
        sync()
        t1, _ = timed(lambda: st_app.append_frontend(fe), ses.sync)
        t2, _ = timed(lambda: st_app.append(r), ses.sync)
        if i >= a.warmup:
            fe_ms.append(t1)
            host_app_ms.append(t2)
    append = {"points_per_key_frame": pts_per_kf,
              "from_frontend": dict(stats(fe_ms), h2d_bytes_per_call=0),
              "from_host_records": dict(stats(host_app_ms), h2d_bytes_per_call=int(pts_per_kf) * capi.POINT_STRIDE),
              "device_bytes_per_point": 20}
    st_app.close()
    fe.close()
    ses.close()

    # ---------------------------------------------------------------------------------------------- save map
    K = a.save_keyframes
    save_poses = np.array([pose6(synth.trajectory_state(k)) for k in range(K)], np.float32)   # 1 m apart
    n_save = int(sum(len(recs[k % N_DISTINCT]) for k in range(K)))
    sv = capi.KeyFrameStore(tb, n_save, K)
    for k in range(K):
        sv.append(recs[k % N_DISTINCT])
    all_ids = np.arange(K, dtype=np.int32)
    save = {"key_frames": K, "points_in": n_save, "store_device_bytes": sv.info()["device_bytes"]}
    for label, leaf in (("dense", 0.0), ("filtered", SAVE_LEAF)):
        ms = []
        for i in range(1 + a.reps // 2):
            t, (xyzi, cur) = timed(lambda: sv.assemble(all_ids, poses6=save_poses, leaf=leaf), sync)
            if i >= 1:
                ms.append(t)
        save[label] = dict(stats(ms), leaf=leaf, points_out=int(len(xyzi)), h2d_bytes_per_call=K * KF_SEG_BYTES,
                           d2h_bytes_per_call=int(len(xyzi)) * 20)
        del xyzi, cur
    save["map_scratch_bytes_after"] = sv.info()["map_scratch_bytes"]   # what the readers keep with the map until released
    sv.release_scratch()
    print(json.dumps(save), file=sys.stderr, flush=True)
    sv.close()
    tb.close()

    res = {"gpu": name, "power_limit_w": limit, "reps": a.reps, "warmup": a.warmup,
           "workload": f"synthetic Livox HAP key frames ({N_DISTINCT} ray-cast scans cycled), body frame",
           "rebuild": rebuild, "append": append, "save_map": save,
           "timing": "host wall clock around each call, which ends in a device synchronise; medians over the timed calls"}

    # ---------------------------------------------------------------------------------------------- CPU restatement
    if not a.no_cpu:
        from oracle import pyoracle as po
        po.build()
        p4 = [np.column_stack([r[:, 0:3], r[:, 8]]).astype(np.float32) for r in kf_recs]
        t0 = time.perf_counter()
        sub = np.concatenate([po.transform_cloud_rpy(p, poses[k]) for k, p in enumerate(p4)])
        t1 = time.perf_counter()
        o, _, _ = po.voxel_grid(sub, LEAF, order="pcl")
        t2 = time.perf_counter()
        res["cpu"] = {"what": "rebuild data path restated on one host core (oracle transformPointCloud + pcl::VoxelGrid), once; "
                              "the ikd-Tree build is not included",
                      "transform_ms": (t1 - t0) * 1e3, "voxel_grid_ms": (t2 - t1) * 1e3, "points_out": int(len(o))}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
