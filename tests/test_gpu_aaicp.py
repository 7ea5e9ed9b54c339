"""GPU tests of the relocalisation AA-ICP (flb_keyframes_aaicp, regMode 1) against the sequential CPU oracle (orc_aaicp in
tests/cpp/aaicp_oracle.cpp), on the ray-cast HDL-64 and HAP street scenes of test_gpu_fricp.py.  Given the device's
normalisation, the first pass's matches and residuals are bit-equal to the oracle's and the first Kabsch step lands within
1e-12; whole registrations take the oracle's path (outcome and α count of every iteration) up to its first decision
without a safe margin (1e-9 on the stop and reset tests, 1e-3 on the α bounds, since ill-conditioned Anderson solves
magnify last-bit differences), with the counts, res_trans and the energy checked wherever the whole path matched (1e-6,
or 1000 times the oracle's own one-ulp sensitivity where that is larger); the convergence energy against numpy on the call's own outputs; the store left unchanged; a negative-roll start, an exact
subset, NaN and duplicate points, tiny targets, source sizes around the block and the near kernel's grid stride,
max_icp = 0, repeat calls, one host synchronisation per pass, the scratch, the rejected configs, and a displaced,
outlier-laden scan checked against the oracle's own outcome."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi
from tests import aaicp_oracle as ao
from tests.icp_cases import rot, rot_err
from tests.test_gpu_fricp import EXT, PLACES, _norm, _p6, _target, scene, store  # noqa: F401  (the shared scene fixtures)

pytestmark = pytest.mark.gpu

STOP, THR, ALPHA_MARGIN = 1e-5, 0.05, 1e-3


def _sub(a, k):
    return np.ascontiguousarray(a[::k])


def _prefix(log, stop=STOP, thr=THR, alpha_margin=ALPHA_MARGIN):
    """The rows before the first decision without a safe margin: a stop or reset test within 1e-9 relative of its
    threshold, or an alphas_cond test within alpha_margin (absolute) of its bounds.  α comes from least-squares solves on
    nearly collinear history columns, which magnify the last-bit differences of the fixed-order device sums far beyond
    1e-9, so only a wide α margin makes the α count a decision both sides must share."""
    for k, (e, p, _, _, s2, am) in enumerate(log):
        if k:
            with np.errstate(divide="ignore", invalid="ignore"):
                r = (e - p) / p
            if abs(s2 - stop) <= 1e-9 * stop or (np.isfinite(r) and abs(r - thr) <= 1e-9 * thr) or not am > alpha_margin:
                return k
    return len(log)


def _compare(g, o, what, tol=1e-6):
    assert g["status"] == o["status"] == 0, what
    assert (g["n_source_finite"], g["n_target_finite"]) == (o["n_source_finite"], o["n_target_finite"]), what
    T, U = g["res_trans"], o["res_trans"]
    assert np.abs(T[:3, 3] - U[:3, 3]).max() <= tol and rot_err(T, U[:3, :3]) <= tol, (what, T, U)


def _energy_of(g, gi, s, tgt):
    """Σ |final X0 - Q|² from the call's own res_trans, normalisation and last matches, in numpy: the convergence energy
    AaEnergyOp has to return."""
    sc, ms, mt = g["scale"], g["mu_source"], g["mu_target"]
    R = g["res_trans"][:3, :3]
    t = g["res_trans"][:3, 3] / sc - (mt - R @ ms)
    ok = gi >= 0
    X0 = s[ok, :3].astype(np.float64) / sc - ms
    Q = tgt[gi[ok], :3].astype(np.float64) / sc - mt
    return float((np.linalg.norm(X0 @ R.T + t - Q, axis=1) ** 2).sum())


def _sensitivity(s, tgt, g, o, kw):
    """How far the oracle's own result moves when its input moves by one rounding: the source mean's x nudged by one ulp,
    and the scale by one ulp.  An Anderson run whose path is decided identically can still magnify such a difference by
    orders of magnitude (its least-squares solves on nearly collinear history columns), and the device's fixed-order
    sums differ from the oracle's sequential ones by a few roundings, so the device may land this far from the oracle
    times a factor for that count.  Returns sens_t (m), sens_r (rad) and sens_e (relative energy)."""
    sc, ms, mt = _norm(g)
    dt = dr = de = 0.0
    for norm in ((sc, ms + np.array([np.spacing(ms[0]), 0.0, 0.0]), mt), (sc * (1 + 2.0 ** -52), ms, mt)):
        p = ao.aaicp(s, tgt, norm=norm, **kw)[0]
        dt = max(dt, float(np.abs(p["res_trans"][:3, 3] - o["res_trans"][:3, 3]).max()))
        dr = max(dr, rot_err(p["res_trans"], o["res_trans"][:3, :3]))
        de = max(de, abs(p["energy"] - o["energy"]) / max(o["energy"], 1e-300))
    return {"sens_t": dt, "sens_r": dr, "sens_e": de}


def _case(store, oracle, src, ids, p6, init6=None, ext=EXT, **kw):
    g, gi, gr, glog = store.aaicp(src, ids, p6, tgt_pre_pose6=ext, src_pose6=init6, correspondences=True, log=True, **kw)
    s = src if init6 is None else oracle.transform_cloud_rpy(src, init6)
    tgt = _target(oracle, store, ids, p6, ext)
    o, oi, orr, olog = ao.aaicp(s, tgt, norm=_norm(g), **kw)
    if len(olog) > 1 and o["status"] == 0:
        o.update(_sensitivity(s, tgt, g, o, kw))
    if len(glog) and g["status"] == 0:   # the matched branch of the energy op, against the call's own outputs
        e = _energy_of(g, gi, s, tgt)
        assert abs(g["energy"] - e) <= 1e-9 * e + 1e-24 * len(gi), (g["energy"], e)   # floor: rounding of an exact fit
    return g, gi, gr, glog, o, oi, orr, olog


def _follows(g, glog, o, olog, what, posed=True):
    """On a well-posed registration the device's log (outcome and α count of every iteration) equals the oracle's over
    the rows before the first decision without a safe margin (_prefix), with energies within 1e-6 relative there.  Where
    the whole path matched, iterations, accepted, resets and history are the oracle's, and res_trans and the energy land
    within 1e-6 m / 1e-6 rad / 1e-6 relative of its, or within 1000 times the oracle's own one-ulp sensitivity
    (_sensitivity) where that is larger; elsewhere res_trans lands within the stop criterion (|Δt| <= stop * scale in the
    caller's units, the rotation within stop rad)."""
    j = min(_prefix(olog), len(glog), len(olog))
    same = len(glog) == len(olog) and np.array_equal(glog[:, 2:4], olog[:, 2:4])
    T, U = g["res_trans"], o["res_trans"]
    dt, dr = np.abs(T[:3, 3] - U[:3, 3]).max(), rot_err(T, U[:3, :3])
    de = float(np.max(np.abs(glog[:j, 0] - olog[:j, 0]) / np.maximum(olog[:j, 0], 1e-300))) if j else 0.0
    print(f"[aaicp path] {what}: {len(glog)} / {len(olog)} passes, compared rows {j}, same whole path {same}, "
          f"energy rel diff over them {de:.2e}, final energy rel diff {abs(g['energy'] - o['energy']) / max(o['energy'], 1e-300):.2e}, "
          f"|dt| {dt:.2e} m, |dR| {dr:.2e}")
    assert g["status"] == o["status"] == 0 and np.isfinite(T).all(), what
    if not posed:
        return
    assert np.array_equal(glog[:j, 2:4], olog[:j, 2:4]), (what, j, glog[:, 2:4].tolist(), olog[:, 2:4].tolist())
    assert de <= 1e-6, (what, de)
    if same:
        assert (g["iterations"], g["accepted"], g["resets"], g["history"]) == \
               (o["iterations"], o["accepted"], o["resets"], o["history"]), what
        # 1e-6 m / 1e-6 rad, or 1000 times the oracle's own movement under a one-ulp input change where that is larger
        tol_t, tol_r = max(1e-6, 1e3 * o.get("sens_t", 0.0)), max(1e-6, 1e3 * o.get("sens_r", 0.0))
        tol_e = max(1e-6, 1e3 * o.get("sens_e", 0.0))
        print(f"[aaicp path] {what}: one-ulp oracle sensitivity {o.get('sens_t', 0.0):.2e} m / {o.get('sens_r', 0.0):.2e} rad "
              f"/ {o.get('sens_e', 0.0):.2e} energy")
        assert dt <= tol_t and dr <= tol_r, (what, dt, dr, tol_t, tol_r)
        assert abs(g["energy"] - o["energy"]) <= tol_e * o["energy"] + 1e-300, (what, g["energy"], o["energy"], tol_e)
    else:
        assert dt <= STOP * g["scale"] and dr <= STOP, (what, T, U)


def test_first_pass_and_first_step(scene, store, oracle):
    kfs, poses = scene
    for what, places in PLACES.items():
        ids = np.array([2 * k for k in places], np.int32)
        p6 = np.stack([_p6(*poses[k]) for k in places])
        a = places[len(places) // 2]
        init = _p6(*poses[a]) + np.array([0.4, -0.3, 0.05, 0.0, 0.0, 0.03], np.float32)
        for off in (np.zeros(6, np.float32), np.array([60.0, -90.0, 35.0, 0, 0, 0.3], np.float32)):   # the second: 20-150 m away
            w = f"{what} off={off[:3]}"
            g, gi, gr, glog, o, oi, orr, olog = _case(store, oracle, kfs[2 * a + 1], ids, p6, init + off, max_icp=1)
            assert np.array_equal(gi, oi), (w, np.nonzero(gi != oi)[0][:5])
            assert np.array_equal(gr.view(np.uint64), orr.view(np.uint64)), w
            assert g["iterations"] == o["iterations"] == 1 and glog[0, 2] == olog[0, 2] == -1, w
            _compare(g, o, w, tol=1e-12)
            assert abs(glog[0, 0] - olog[0, 0]) <= 1e-12 * olog[0, 0], w
            assert abs(g["energy"] - o["energy"]) <= 1e-9 * o["energy"], (w, g["energy"], o["energy"])   # after the re-seat
            print(f"[aaicp first step] {w}: {g['n_source']} -> {g['n_target']} points, "
                  f"|dT| {np.abs(g['res_trans'] - o['res_trans']).max():.2e}")


@pytest.mark.parametrize("what,far", [("HDL-64", False), ("HAP", False), ("mixed", False), ("HDL-64", True), ("mixed", True)])
def test_registration_follows_the_oracle(scene, store, oracle, what, far):
    kfs, poses = scene
    places = PLACES[what]
    ids = np.array([2 * k for k in places], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in places])
    a = places[len(places) // 2]
    init = _p6(*poses[a]) + np.array([0.5, -0.4, 0.0, 0.0, 0.0, np.deg2rad(2.0)], np.float32)
    if far:
        init = init + np.array([60.0, -90.0, 35.0, 0, 0, 0.3], np.float32)
    snap = [store.download(k) for k in range(len(kfs))]
    g, _, _, glog, o, _, _, olog = _case(store, oracle, _sub(kfs[2 * a + 1], 8), ids, p6, init)
    for k, (p, c) in enumerate(snap):   # the store is unchanged
        q, d = store.download(k)
        assert np.array_equal(q.view(np.uint32), p.view(np.uint32)) and np.array_equal(d.view(np.uint32), c.view(np.uint32))
    _follows(g, glog, o, olog, f"{what} far={far}")
    print(f"[aaicp] {what} far={far}: {g['iterations']} iterations, {g['accepted']} accepted, {g['resets']} resets, history "
          f"{g['history']}")


def test_negative_roll_start_and_exact_subset(scene, store, oracle):
    kfs, poses = scene
    ids = np.array([0, 2], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in (0, 1)])
    # the correction D has a negative roll: eulerAngles returns its first angle near π, the other two reflected
    D, Dt = rot((-0.03, 0.01, 0.02)), np.array([0.2, -0.1, 0.05])
    R0, t0 = poses[0]
    init = _p6(D.T @ R0, D.T @ (t0 - Dt))   # D^-1 applied to the key frame's pose
    g, _, _, glog, o, _, _, olog = _case(store, oracle, _sub(kfs[1], 8), ids, p6, init)
    _follows(g, glog, o, olog, "negative roll")
    R = g["res_trans"][:3, :3]
    assert np.arctan2(R[2, 1], R[2, 2]) < -0.02 and rot_err(g["res_trans"], D) < 0.02   # the returned correction rolls negatively
    # the source is the target itself: the first energy is exactly 0 on both sides
    one = np.zeros((1, 6), np.float32)
    g, gi, _, glog, o, oi, _, olog = _case(store, oracle, kfs[0], [0], one, ext=None, max_icp=10)
    assert glog[0, 0] == olog[0, 0] == 0.0 and np.array_equal(gi, oi) and (gi == np.arange(len(kfs[0]))).mean() > 0.999
    _compare(g, o, "exact subset", tol=1e-8)
    assert np.abs(g["res_trans"] - np.eye(4)).max() < 1e-9
    print(f"[aaicp exact subset] log {glog[:, :3].tolist()}")


def test_nan_duplicates_and_tiny_targets(scene, oracle):
    kfs, _ = scene
    base = kfs[0]
    tgt = np.concatenate([base[:30000], base[:5000]])   # duplicated target points: the lower index wins
    tgt[::101, 2] = np.nan
    src = base[3:12000].copy()
    src = np.concatenate([src, src[:500]])               # duplicated source points
    src[::53, 0] = np.inf
    src[7::211, 1] = np.nan
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(tgt) + 64, 32)
    kf.append(capi.pack_pointtype(tgt[:, :3], tgt[:, 3]))
    one = np.zeros((1, 6), np.float32)
    shift = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.02], np.float32)
    g, gi, gr, _, o, oi, orr, _ = _case(kf, oracle, src, [0], one, shift, ext=None, max_icp=1)
    assert np.array_equal(gi, oi) and np.array_equal(gr.view(np.uint64), orr.view(np.uint64))
    assert (gi[::53] == -1).all() and (gi[7::211] == -1).all()
    g, _, _, glog, o, _, _, olog = _case(kf, oracle, src, [0], one, shift, ext=None, max_icp=30)
    _follows(g, glog, o, olog, "nan + duplicates")
    for n in range(1, 9):
        k = kf.append(capi.pack_pointtype(base[100:100 + n, :3] * 3.0, base[100:100 + n, 3]))
        _, gi, _, _, _, oi, _, _ = _case(kf, oracle, src[:2000], [k], one, ext=None, max_icp=1)
        assert np.array_equal(gi, oi)
        g, _, _, glog, o, _, _, olog = _case(kf, oracle, src[:2000], [k], one, ext=None, max_icp=10)
        _follows(g, glog, o, olog, f"{n} target points", posed=False)   # a rotation about the few points is free
    k = kf.append(capi.pack_pointtype(np.full((3, 3), np.nan, np.float32)))
    g = kf.aaicp(src[:100], [k], one)
    assert g["status_name"] == "FEW_TARGET" and np.array_equal(g["res_trans"], np.eye(4))
    kf.close()
    tree.close()


def test_source_sizes_at_the_launch_boundaries(scene, oracle):
    import torch
    kfs, _ = scene
    big = np.concatenate(kfs[2:])
    stride = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256   # the near kernel's grid stride
    sizes = [1, 2, 255, 257, stride - 1, stride + 1]
    assert len(big) >= max(sizes), (len(big), stride)
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(kfs[0]) + 64, 4)
    kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
    one = np.zeros((1, 6), np.float32)
    shift = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.02], np.float32)
    for n in sizes:
        g, gi, gr, glog, o, oi, orr, olog = _case(kf, oracle, big[:n], [0], one, shift, ext=None, max_icp=3)
        assert np.array_equal(gi, oi) or g["iterations"] == 0, n
        assert len(glog) == len(olog) and np.array_equal(glog[:, 2:4], olog[:, 2:4]), (n, glog[:, 2:4], olog[:, 2:4])
        _follows(g, glog, o, olog, f"n_source={n}")
    kf.close()
    tree.close()


def test_max_icp_zero_repeat_calls_syncs_scratch_and_rejected_configs(scene, oracle):
    kfs, _ = scene
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(kfs[0]) + 16, 4)
    kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
    one = np.zeros((1, 6), np.float32)
    shift = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.02], np.float32)
    assert kf.info()["map_scratch_bytes"] == 0
    # max_icp = 0: no pass, Q is the zero matrix, the energy is Σ |X0|²
    g, gi, gr, glog, o, _, _, _ = _case(kf, oracle, kfs[1], [0], one, shift, ext=None, max_icp=0)
    assert g["iterations"] == 0 and len(glog) == 0 and (gi == -1).all() and np.isinf(gr).all()
    assert np.array_equal(g["res_trans"][:3, :3], np.eye(3)) and abs(g["energy"] - o["energy"]) <= 1e-12 * o["energy"]
    setup_syncs = g["syncs"] - 1
    r = kf.aaicp(kfs[1], [0], one, src_pose6=shift, max_icp=40, correspondences=True, log=True)
    assert r[0]["syncs"] == setup_syncs + len(r[3]) + 1, (r[0]["syncs"], setup_syncs, len(r[3]))
    assert len(r[3]) == r[0]["iterations"] + (1 if r[0]["iterations"] < 40 else 0)
    assert kf.info()["map_scratch_bytes"] >= 4 * 32 * len(kfs[1])
    r2 = kf.aaicp(kfs[1], [0], one, src_pose6=shift, max_icp=40, correspondences=True, log=True)
    kf.release_scratch()
    assert kf.info()["map_scratch_bytes"] == 0
    r3 = kf.aaicp(kfs[1], [0], one, src_pose6=shift, max_icp=40, correspondences=True, log=True)
    for other in (r2, r3):
        assert all(np.array_equal(np.asarray(r[0][k]), np.asarray(other[0][k])) for k in r[0])
        for a, b in zip(r[1:], other[1:]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    for kw, msg in ((dict(max_icp=-1), "max_icp"), (dict(stop=np.nan), "stop"), (dict(stop=-1e-6), "stop"),
                    (dict(stop=np.inf), "stop"), (dict(error_overflow_threshold=np.nan), "error_overflow_threshold"),
                    (dict(error_overflow_threshold=np.inf), "error_overflow_threshold"),
                    (dict(src_pose6=[0, 0, np.inf, 0, 0, 0]), "finite")):
        with pytest.raises(capi.FlbError, match=msg):
            kf.aaicp(kfs[1], [0], one, **kw)
    with pytest.raises(capi.FlbError, match="regMode 1 is not supported"):
        kf.fricp(kfs[1], [0], one, mode=1)
    with pytest.raises(capi.FlbError, match="out of range"):
        kf.aaicp(kfs[1], [3], one)
    g = kf.aaicp(kfs[1][:0], [0], one)
    assert g["status_name"] == "NO_SOURCE" and g["iterations"] == 0
    kf.close()
    tree.close()


def test_recovery_of_a_displaced_scan_with_outliers(scene, store, oracle):
    kfs, poses = scene
    places = [0, 1, 2]
    ids = np.array([2 * k for k in places], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in places])
    world = np.concatenate([kfs[2 * k + 1][:, :3].astype(np.float64) @ poses[k][0].T + poses[k][1] for k in places])
    rng = np.random.default_rng(9)
    n_out = int(0.15 * len(world))
    lo, hi = world.min(0), world.max(0)
    outl = rng.uniform(lo, hi, size=(n_out, 3))   # stand-ins for dynamic objects
    R, t = rot((0.01, -0.01, np.deg2rad(2.0))), np.array([1.2, -0.9, 0.05])
    t = t / np.linalg.norm(t) * 0.5
    pts = np.concatenate([world, outl])
    src = _sub(((pts - t) @ R).astype(np.float32), 4)   # D^-1 x: the registration should return D = (R, t)
    g, _, _, glog, o, _, _, olog = _case(store, oracle, src, ids, p6, ext=None)
    _follows(g, glog, o, olog, "recovery", posed=False)   # a diverging run: ~100 history columns, its path is chaotic
    T = g["res_trans"]
    err = (np.abs(T[:3, 3] - t).max(), rot_err(T, R))
    oerr = (np.abs(o["res_trans"][:3, 3] - t).max(), rot_err(o["res_trans"], R))
    # the device's outcome is the oracle's: both recover within 2 cm / 0.1 deg, or neither does
    assert (err[0] < 0.02 and err[1] < np.deg2rad(0.1)) == (oerr[0] < 0.02 and oerr[1] < np.deg2rad(0.1)), (err, oerr)
    print(f"[aaicp recovery] 0.5 m / 2 deg, 15 % outliers: {g['iterations']} iterations, {g['accepted']} accepted, "
          f"{g['resets']} resets, {g['syncs']} syncs, error {err[0] * 100:.2f} cm / {np.rad2deg(err[1]):.4f} deg "
          f"(oracle {oerr[0] * 100:.2f} cm / {np.rad2deg(oerr[1]):.4f} deg)")
