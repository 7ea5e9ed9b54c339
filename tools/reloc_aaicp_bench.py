#!/usr/bin/env python
"""Relocalisation AA-ICP on one GPU: flb_keyframes_aaicp (regMode 1, Registeration's ICP::Parameters) next to a host path.

Workload (synthetic, the one of tools/reloc_fricp_bench.py): body-frame key frames ray-cast in the city world, a prior
session of key frames along a street and a live scan of one of its places (another noise draw) displaced from its prior
pose by 0.5 m / 2 degrees:
  hdl64_3      a dense HDL-64 /cloud_registered scan against searchNum 3 dense prior key frames
  hap_3        the same with Livox HAP scans
  hdl64_ds_1   the HDL-64 scan 0.5 m voxel-filtered against searchNum 1
For each it reports the device call (median and p10-p90 of a host clock around the synchronising call), its iterations
(the loop index at exit), passes, accepted Anderson steps, resets and history length, the time per pass (the full call
minus a max_icp = 0 call, over the passes), the host's Anderson time per pass (the Euler / QR / mixing work, timed
inside the CPU oracle's run of the same registration, whose host algebra is the library's written out again), the host
synchronisations and the bytes copied device to host.  The host path is the CPU oracle (orc_aaicp in tests/cpp/aaicp_oracle.cpp, one core, an exact k-d
tree), which stands in for the reference's Eigen build: its set-up and its first iteration are timed from short runs
(medians of 3 with max_icp 0 and 1) and scaled to the device call's passes.  The GPU name and power limit are read in the
same run.  Writes one JSON document to stdout and to --out.

  python tools/reloc_aaicp_bench.py --reps 10 --out /tmp/reloc_aaicp_bench.json
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
from reloc_fricp_bench import gpu_info, p6, stats, timed, voxel  # noqa: E402
from tests import aaicp_oracle as ao  # noqa: E402
from tests.fricp_oracle import _p4  # noqa: E402

SETUP_BYTES, PASS_BYTES = 3 * 4 * 7 + 8 * 8, 8 * 17   # three bounds records and the means; one step record per pass


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

    def call(**kw):
        return kf.aaicp(live, ids, poses6, src_pose6=init, **kw)

    g, log = call(log=True)
    passes = len(log)
    for _ in range(2):   # warm-up of every shape
        call()
        call(max_icp=0)
    full, setup = [], []
    for _ in range(reps):   # alternating
        full.append(timed(call)[0])
        setup.append(timed(lambda: call(max_icp=0))[0])
    per_pass = (np.median(full) - np.median(setup)) / max(passes, 1)
    # host path: the oracle on one core, short runs, scaled to the device call's passes
    src = _p4(live)
    tgt = kf.assemble(ids, poses6=poses6)[0]
    from oracle import pyoracle
    pyoracle.build()
    s = pyoracle.transform_cloud_rpy(src, init)
    ao.aaicp(s[:10], tgt[:10], max_icp=1)   # compiled on first use: not part of the timing
    t0 = np.median([timed(lambda: ao.aaicp(s, tgt, max_icp=0))[0] for _ in range(3)])
    t1 = np.median([timed(lambda: ao.aaicp(s, tgt, max_icp=1))[0] for _ in range(3)])
    o, _, _, olog = ao.aaicp(s, tgt, norm=(g["scale"], g["mu_source"], g["mu_target"]))
    anderson = o["anderson_ms"] / max(len(olog), 1)
    kf.close()
    tree.close()
    return {"n_source": int(len(live)), "n_target": int(g["n_target"]), "call": stats(full),
            "setup_call": stats(setup), "setup_share": float(np.median(setup) / np.median(full)), "iterations": g["iterations"],
            "passes": passes, "accepted": g["accepted"], "resets": g["resets"], "history": g["history"],
            "ms_per_pass": float(per_pass), "anderson_host_ms_per_pass": float(anderson),
            "oracle_path": {"iterations": o["iterations"], "accepted": o["accepted"], "resets": o["resets"]}, "syncs": g["syncs"],
            "d2h_bytes": int(SETUP_BYTES + PASS_BYTES * passes + 8), "energy": g["energy"],
            "host_oracle": {"setup_ms": float(t0), "pass_ms": float(t1 - t0), "scaled_call_ms": float(t0 + (t1 - t0) * passes)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "reloc_aaicp_bench.json"))
    a = ap.parse_args()
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit_w": limit, "mode": 1, "cases": {}}
    for key, model, n, leaf in (("hdl64_3", "hdl64", 3, 0.0), ("hap_3", "hap", 3, 0.0), ("hdl64_ds_1", "hdl64", 1, 0.5)):
        res["cases"][key] = case(model, n, leaf, a.reps)
        print(key, json.dumps(res["cases"][key]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
