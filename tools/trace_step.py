#!/usr/bin/env python
"""Device-side timeline of one graph-launched scan step (needs the DEBUG library: tools/trace_build.sh, FLB_LIB=...).

  FLB_LIB=better_fastlio2_b200/libfastlio_b200_trace.so python tools/trace_step.py [--steps 20] [--out file.json]

Prints, per kernel and pass, the mean start / end (us after k_esikf_begin started) over the steps, the clock-cycle
phases inside k_esikf_post, and when the first pass's unresolved k-NN queries are published by the stencil kernel and
picked up by the exact kernel.  The timeline comes from %globaltimer stamps taken by the kernels themselves, so it shows
the real critical path of the CUDA-graph execution (launch gaps, side-stream overlap) without a profiler attached.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

NAMES = {0: "esikf_begin", 1: "esikf_pre", 2: "knn_stencil", 3: "knn_exact_pick", 4: "residual", 5: "esikf_post", 6: "classify",
         7: "touch_blocks", 8: "ds_scatter", 9: "ds_apply", 10: "append_points", 11: "relocate_chains"}
PHASES = ["start", "partials reduced", "matrices staged", "inverse", "gain+dx", "boxplus(+J)", "cov/state written"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--pairs", type=int, default=10, help="also time PAIRS of steps in flight together (inter-step gap)")
    args = ap.parse_args()
    import torch
    from better_fastlio2_b200 import capi
    L = capi.lib()
    if not hasattr(L, "flb_debug_trace_read"):
        raise SystemExit("not a trace build: run tools/trace_build.sh and set FLB_LIB")
    n_scans = args.warmup + args.steps
    work = bench.make_workload(20, n_scans)
    tree = capi.KDTree(voxel_size=bench.DS, max_points=16 << 20, max_blocks=2 << 20, device=0)
    bench.build_map(tree, work["map"])
    nmax = max(len(s) for s in work["scans"])
    ses = capi.Session(tree, max_scan_points=max(131072, nmax), max_iterations=bench.MAX_ITER, filter_size_map_min=bench.DS)
    fov = capi.make_fov(cube_len=1000.0, det_range=100.0)
    dev = []
    for s in work["scans"]:
        b4 = np.zeros((len(s), 4), np.float32)
        b4[:, :3] = s
        dev.append(torch.from_numpy(b4).to("cuda:0"))
    torch.cuda.synchronize()
    NS, NP = 128, 96
    tr = (C.c_ulonglong * (2 * NS))()
    ph = (C.c_longlong * NP)()
    dbg = (C.c_ulonglong * 128)()
    dbg_sum = np.zeros(128, np.float64)
    dbg_max = np.zeros(128, np.float64)

    def step(k):
        ses.scan_set_device(dev[k].data_ptr(), len(work["scans"][k]))
        st = work["priors"][k].copy()
        P = work["P"].copy()
        return ses.scan_step_ptr(fov, None, 0, 0, st, P)

    for k in range(args.warmup):
        step(k)
    L.flb_debug_trace_read(tr, ph, dbg)
    rows = {}
    phases = {}
    pre_ph = []
    total = []
    for k in range(args.warmup, n_scans):
        step(k)
        L.flb_debug_trace_read(tr, ph, dbg)
        d = np.array(dbg, dtype=np.float64)
        dbg_sum += d
        dbg_max = np.maximum(dbg_max, d)
        t = np.array(tr, dtype=np.uint64).reshape(NS, 2)
        t0 = int(t[0, 0])
        last = 0
        for slot in range(NS):
            a, b = int(t[slot, 0]), int(t[slot, 1])
            if a == 0xFFFFFFFFFFFFFFFF:
                continue
            sa = (a - t0) * 1e-3
            sb = (b - t0) * 1e-3 if b else float("nan")
            rows.setdefault(slot, []).append((sa, sb))
            if b:
                last = max(last, b - t0)
        total.append(last * 1e-3)
        p = np.array(ph, dtype=np.int64).reshape(8, 12)
        if p[6, 0] and p[6, 6]:
            pre_ph.append([p[6, j] - p[6, 0] for j in range(7)])
        for pas in range(1, 5):
            if p[pas, 0] and p[pas, 6]:
                phases.setdefault(pas, []).append([(p[pas, j] - p[pas, 0]) if p[pas, j] else -1 for j in range(7)])
    out = {"steps": args.steps, "timeline_us": [], "post_phases_cycles": {}, "last_kernel_end_us_mean": float(np.mean(total))}
    print(f"# mean over {args.steps} steps; us after k_esikf_begin started; last kernel end {np.mean(total):.1f} us")
    print("# knn_exact_pick: the exact k-NN kernel runs beside the stencil kernel; start = its first work-list pick-up, "
          "end = its last warp's exit")
    print(f"{'kernel':<16}{'pass':>5}{'start':>10}{'end':>10}{'dur':>9}{'ran':>6}")
    for slot in sorted(rows, key=lambda s: np.mean([r[0] for r in rows[s]])):
        r = np.array(rows[slot])
        ran = r[~np.isnan(r[:, 1])]
        sa = float(np.mean(r[:, 0]))
        sb = float(np.mean(ran[:, 1])) if len(ran) else float("nan")
        dur = float(np.mean(ran[:, 1] - ran[:, 0])) if len(ran) else float("nan")
        print(f"{NAMES.get(slot // 8, slot // 8):<16}{slot % 8:>5}{sa:>10.1f}{sb:>10.1f}{dur:>9.1f}{len(ran):>6}")
        out["timeline_us"].append({"kernel": NAMES.get(slot // 8, str(slot // 8)), "pass": slot % 8, "start": sa, "end": sb,
                                   "dur": dur, "ran": int(len(ran))})
    print("# k_esikf_post phases (clock cycles after kernel start, thread 0)")
    for pas in sorted(phases):
        m = np.mean(np.array(phases[pas], dtype=np.float64), axis=0)
        print(f"pass {pas}: " + ", ".join(f"{PHASES[j]}={m[j]:.0f}" for j in range(1, 7)))
        out["post_phases_cycles"][str(pas)] = {PHASES[j]: float(m[j]) for j in range(1, 7)}
    if pre_ph:
        m = np.mean(np.array(pre_ph, dtype=np.float64), axis=0)
        names = ["", "state / covariance staged", "boxminus + Jacobians", "covariance projected", "projection stored", "inverse", "Q written"]
        print("# k_esikf_pre, pass 1 (clock cycles after kernel start, thread 0): " + ", ".join(f"{names[j]}={m[j]:.0f}" for j in range(1, 7)))
        out["pre_phases_cycles"] = {names[j]: float(m[j]) for j in range(1, 7)}
    S = args.steps
    if dbg_sum[16] > 0:
        nq = dbg_sum[16]
        print("# exact kernel, first pass: "
              f"queries/step={nq / S:.0f} cycles/query={dbg_sum[17] / nq:.0f} max={dbg_max[18]:.0f} "
              f"done after ring1/2/3={dbg_sum[19] / nq:.3f}/{dbg_sum[20] / nq:.3f}/{dbg_sum[21] / nq:.3f} coarse={dbg_sum[25] / nq:.4f} "
              "")
        print("# exact kernel, first pass: share of queries by duration (8192-cycle buckets): " + " ".join(f"{dbg_sum[58 + j] / nq:.3f}" for j in range(6)))
        if dbg_sum[32] > 0:
            print("# exact kernel, cycles/query by phase: " + ", ".join(
                f"{nm}={dbg_sum[i] / nq:.0f}" for nm, i in (("ticket", 32), ("seed loads + block batches (probes, compaction, point loads)", 33),
                                                            ("merges", 36))))
    if dbg_sum[40] > 0:
        nw = dbg_sum[40]
        print(f"# stencil kernel, first pass: warps/step={nw / S:.0f} mean cycles/warp={dbg_sum[41] / nw:.0f} max={dbg_max[42]:.0f}; "
              f"warps with a whole-shell lane={dbg_sum[43] / nw:.3f} (mean cycles {dbg_sum[44] / max(dbg_sum[43], 1):.0f}, "
              f"{dbg_sum[45] / max(dbg_sum[43], 1):.1f} such lanes each); largest per-lane candidate count of a warp: mean={dbg_sum[56] / nw:.1f} max={dbg_max[57]:.0f}")
        print("# stencil kernel, first pass: share of warps by duration (8192-cycle buckets): " +
              " ".join(f"{dbg_sum[48 + j] / nw:.3f}" for j in range(8)))
    for nm, i0 in (("published by the stencil kernel", 64), ("picked up by the exact kernel", 80)):
        h = dbg_sum[i0:i0 + 16]
        if h.sum() > 0:
            print(f"# first pass, unresolved queries {nm}: share by us after the stencil kernel's start (4-us buckets, last = 60+): " +
                  " ".join(f"{v / h.sum():.3f}" for v in h) + f"  ({h.sum() / S:.0f}/step)")
            out.setdefault("worklist_hist_4us", {})[nm] = (h / S).tolist()
    if args.pairs > 0:
        # two steps in flight: device time from the first kernel of step k to the last kernel of step k+1, against twice the
        # single-step span -> what the device loses BETWEEN two graph launches (copies, graph start-up)
        spans = []
        base = args.warmup
        for j in range(args.pairs):
            k0, k1 = base + (2 * j) % args.steps, base + (2 * j + 1) % args.steps
            sa, Pa = work["priors"][k0].copy(), work["P"].copy()
            sb, Pb = work["priors"][k1].copy(), work["P"].copy()
            ses.scan_set_device(dev[k0].data_ptr(), len(work["scans"][k0]))
            ses.scan_step_begin(fov, sa, Pa, True)
            ses.scan_set_device(dev[k1].data_ptr(), len(work["scans"][k1]))
            ses.scan_step_begin(fov, sb, Pb, True)
            ses.scan_step_finish(fov, sa, Pa)
            ses.scan_step_finish(fov, sb, Pb)
            L.flb_debug_trace_read(tr, ph, dbg)
            t = np.array(tr, dtype=np.uint64).reshape(NS, 2)
            ok = t[:, 0] != np.uint64(0xFFFFFFFFFFFFFFFF)
            spans.append((int(t[ok, 1].max()) - int(t[0, 0])) * 1e-3)
        single = float(np.mean(total))
        print(f"# two steps in flight: first kernel of step k -> last kernel of step k+1 = {np.mean(spans):.1f} us; 2 x single span = "
              f"{2 * single:.1f} us; inter-step gap on the device = {np.mean(spans) - 2 * single:.1f} us")
        out["pair_span_us_mean"] = float(np.mean(spans))
    out["dbg_sum"] = dbg_sum.tolist()
    out["dbg_max"] = dbg_max.tolist()
    if args.out:
        json.dump(out, open(args.out, "w"), indent=1)
    ses.close()
    tree.close()


if __name__ == "__main__":
    main()
