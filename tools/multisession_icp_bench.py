#!/usr/bin/env python
"""Inter-session registration on one GPU: flb_keyframes_icp_batch (every pair of a round in lockstep) next to the same
pairs as one call each, and a host stand-in.

Workload (synthetic): two sessions of the same street, ray-cast in the city world.  The central session has N key frames
(body-frame clouds, poses along the trajectory); the query session has another noise draw of the same N places, its
clouds displaced by a known rigid motion and its central-frame poses drifted by a few cm.  All SC pairs (query key frame s
alone vs central key frames s-2 .. s+2, every key frame at the zero pose, loopFindNearKeyframesLocalCoord) and all RS
pairs (the same selections at the key frames' poses, loopFindNearKeyframesCentralCoord) of one IncreMapping::run, at leaf
0.2 with doICPVirtualRelative's settings (30 m, 10 iterations, 1e-6, 1e-6):
  hdl64   N = 50 places of dense HDL-64 scans (100 key frames), 100 pairs
  hap     N = 50 places of Livox HAP scans (100 key frames), 100 pairs
For each it reports the batched call and the same pairs as one call each (n_pairs = 1): medians and p10-p90 of a host
clock around the synchronising call, alternating; the rounds and synchronisations; and the host stand-in on one core:
the assembly downloaded from the store, the CPU oracle's VoxelGrid and the CPU oracle's ICP (tests/cpp/icp_oracle.cpp,
an exact k-d tree), timed on a few pairs and scaled to all pairs (PCL is not part of the build).  The GPU name and power
limit are read in the same run.  Writes one JSON document to stdout and to --out.

  python tools/multisession_icp_bench.py --reps 5 --out /tmp/multisession_icp_bench.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from better_fastlio2_b200 import capi, synth  # noqa: E402
from reloc_fricp_bench import gpu_info, p6, stats, timed  # noqa: E402
from tests import icp_oracle as io  # noqa: E402
from tests.icp_cases import rot  # noqa: E402

CFG = dict(max_correspondence_distance=30.0, max_iterations=10, transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6)
LEAF = 0.2
N_PLACES = 50
HOST_PAIRS = 3


def sessions(model, n):
    world = synth.city_world(half_extent=400.0, seed=8)
    rng = np.random.default_rng(2)
    R, t = rot((0.003, -0.004, np.deg2rad(1.5))), np.array([0.35, -0.25, 0.03])
    central, query, poses, qposes = [], [], [], []
    for j in range(n):
        st = synth.trajectory_state(3 * j)
        dirs = synth.lidar_dirs(model, np.random.default_rng(300 + j))
        central.append(synth.scan_from_pose(world, st, dirs, rng, max_range=100.0, min_range=1.0).astype(np.float32))
        q = synth.scan_from_pose(world, st, dirs, rng, max_range=100.0, min_range=1.0).astype(np.float64)
        query.append(((q - t) @ R).astype(np.float32))
        Rw = synth.quat_to_mat(st[3:7]) @ synth.quat_to_mat(st[7:11])
        tw = st[0:3] + synth.quat_to_mat(st[3:7]) @ st[11:14]
        poses.append(p6(Rw, tw))
        drift = rot((0.0, 0.0, np.deg2rad(0.2 * ((j % 3) - 1))))
        qposes.append(p6(Rw @ R @ drift, tw + Rw @ t + np.array([0.05, -0.03, 0.0]) * ((j % 3) - 1)))
    return central, query, poses, qposes


def pairs_of(n, poses, qposes):
    zero = [0.0] * 6
    near = [[k for k in range(s - 2, s + 3) if 0 <= k < n] for s in range(n)]
    sc = [([n + s], [zero], near[s], [zero] * len(near[s])) for s in range(n)]
    rs = [([n + s], [qposes[s]], near[s], [poses[k] for k in near[s]]) for s in range(n)]
    return sc + rs


def case(model, reps):
    central, query, poses, qposes = sessions(model, N_PLACES)
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(c) for c in central + query) + 16, 2 * N_PLACES)
    for c in central + query:
        kf.append(capi.pack_pointtype(c))
    pairs = pairs_of(N_PLACES, poses, qposes)

    def batched():
        return kf.icp_batch(pairs, leaf=LEAF, **CFG)

    def each():
        return [kf.icp_batch([p], leaf=LEAF, **CFG) for p in pairs]

    res, st = batched()
    singles = each()
    assert all(a["final_transformation"].tobytes() == b[0][0]["final_transformation"].tobytes() for a, b in zip(res, singles))
    each_syncs = [sum(b[1][k] for b in singles) for k in ("setup_syncs", "iteration_syncs")]
    for _ in range(2):   # warm-up of every shape
        batched()
        each()
    t_batch, t_each = [], []
    for _ in range(reps):   # alternating
        t_batch.append(timed(batched)[0])
        t_each.append(timed(each)[0])
    # the host stand-in on a few pairs of each kind, scaled to all pairs
    from oracle import pyoracle
    pyoracle.build()
    io.icp(np.zeros((4, 4), np.float32), np.zeros((4, 4), np.float32))   # compiled on first use: not part of the timing
    host = {"assemble_download_ms": [], "voxel_grid_ms": [], "icp_ms": []}
    pick = list(range(HOST_PAIRS)) + list(range(N_PLACES, N_PLACES + HOST_PAIRS))
    for p in pick:
        si, sp, ti, tp = pairs[p]
        clouds = []
        for ids, ps in ((si, sp), (ti, tp)):
            ms, (c, _) = timed(lambda: kf.assemble(ids, poses6=np.asarray(ps, np.float32).reshape(-1, 6)))
            host["assemble_download_ms"].append(ms)
            ms, f = timed(lambda: pyoracle.voxel_grid(c, LEAF))
            host["voxel_grid_ms"].append(ms)
            clouds.append(np.asarray(f[0] if isinstance(f, tuple) else f, np.float32))
        ms, _ = timed(lambda: io.icp(clouds[0], clouds[1], **CFG))
        host["icp_ms"].append(ms)
    per_pair = {k: float(np.sum(v) / len(pick)) for k, v in host.items()}
    kf.close()
    tree.close()
    states = {}
    for r in res:
        states[r["state_name"]] = states.get(r["state_name"], 0) + 1
    return {"n_pairs": len(pairs), "n_keyframes": 2 * N_PLACES, "leaf": LEAF,
            "mean_source_points": float(np.mean([r["n_source"] for r in res])),
            "mean_target_points": float(np.mean([r["n_target"] for r in res])), "states": states,
            "iterations": [r["iterations"] for r in res], "batched": stats(t_batch), "one_call_each": stats(t_each),
            "speedup_vs_one_call_each": float(np.median(t_each) / np.median(t_batch)), "batched_stats": st,
            "one_call_each_syncs": {"setup_syncs": each_syncs[0], "iteration_syncs": each_syncs[1]},
            "host_one_core": {"pairs_timed": len(pick), "per_pair_ms": per_pair,
                              "scaled_all_pairs_ms": float(sum(per_pair.values()) * len(pairs))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "multisession_icp_bench.json"))
    a = ap.parse_args()
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit_w": limit, "icp": CFG, "cases": {}}
    for key in ("hdl64", "hap"):
        res["cases"][key] = case(key, a.reps)
        print(key, json.dumps(res["cases"][key]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
