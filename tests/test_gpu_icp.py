"""GPU tests of the loop-closure ICP of the key-frame store (flb_keyframes_icp) against the sequential CPU oracle
(tests/cpp/icp_oracle.cpp).  The exact 1-NN is bit-equal to the oracle's; a registration takes the oracle's path (state,
iterations) and lands within 1e-5 m / 1e-5 rad of its transformation (the device sums in double in another fixed order);
the known perturbation of a ray-cast loop pair is recovered."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import icp_oracle as io
from tests.icp_cases import rot, rot_err

pytestmark = pytest.mark.gpu

EYE = np.eye(3, 4, dtype=np.float32).reshape(12)


def _p4(xyz, rng):
    return np.column_stack([xyz, rng.integers(0, 256, len(xyz))]).astype(np.float32)


def _affine(R, t):
    return np.column_stack([R, t]).astype(np.float32).reshape(12)


def _inv(R, t):
    return R.T, -R.T @ t


@pytest.fixture(scope="module")
def scene():
    """Ray-cast key frames along a street: 4 HDL-64 and 2 HAP (80 000 rays) scans, their poses, and a second pass of
    the same places (another noise draw) for the loop's current sub-map."""
    world = synth.city_world(half_extent=150.0, seed=6)
    rng = np.random.default_rng(3)
    kfs, poses = [], []
    for j, model in enumerate(["hdl64", "hdl64", "hdl64", "hdl64", "hap", "hap"]):
        st = synth.trajectory_state(4 * j)
        dirs = synth.lidar_dirs(model, np.random.default_rng(50 + j))
        if model == "hap":
            dirs = dirs[:80000]
        for rep in range(2):   # rep 0: previous pass, rep 1: current pass
            kfs.append(_p4(synth.scan_from_pose(world, st, dirs, np.random.default_rng(10 * j + rep), max_range=100.0,
                                                min_range=1.0), rng))
        R = synth.quat_to_mat(st[3:7]) @ synth.quat_to_mat(st[7:11])
        poses.append((R, st[0:3] + synth.quat_to_mat(st[3:7]) @ st[11:14]))
    return kfs, poses


@pytest.fixture()
def store(scene):
    kfs, _ = scene
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(k) for k in kfs) + (1 << 20), 64)
    for p in kfs:
        kf.append(capi.pack_pointtype(p[:, :3], p[:, 3]))
    yield kf
    kf.close()
    tree.close()


def _loop_pair(scene, places, anchor, P):
    """loopFindNearKeyframes-style selections: previous pass of `places` in the frame of place `anchor`, current pass of
    the same places in that frame displaced by the known motion P = (R, t) (source = P^-1 target)."""
    _, poses = scene
    Ra, ta = _inv(*poses[anchor])
    Ri, ti = _inv(*P)
    prev_ids, prev_T, cur_ids, cur_T = [], [], [], []
    for k in places:
        R, t = poses[k]
        Rr, tr = Ra @ R, Ra @ t + ta
        prev_ids.append(2 * k)
        prev_T.append(EYE if k == anchor else _affine(Rr, tr))
        cur_ids.append(2 * k + 1)
        cur_T.append(_affine(Ri @ Rr, Ri @ tr + ti))
    return (np.array(cur_ids, np.int32), np.stack(cur_T)), (np.array(prev_ids, np.int32), np.stack(prev_T))


def _host_clouds(store, cur, prev, pre, oracle):
    src, _ = store.assemble(cur[0], affines=cur[1])
    tgt, _ = store.assemble(prev[0], affines=prev[1])
    if pre is not None:
        src = oracle.transform_cloud_rpy(src, np.asarray(pre, np.float32))
    return src, tgt


def _snapshot(kf, n):
    return [kf.download(k) for k in range(n)]


def _same_store(kf, snap):
    for k, (p, c) in enumerate(snap):
        q, d = kf.download(k)
        assert np.array_equal(q.view(np.uint32), p.view(np.uint32)) and np.array_equal(d.view(np.uint32), c.view(np.uint32))


def _nn_equal(g, gi, gd, src, tgt, max_dist=200.0, what=""):
    oi, od = io.nearest(src, tgt)
    assert np.array_equal(gi, oi), (what, np.nonzero(gi != oi)[0][:5])
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), what
    assert g["n_correspondences"] == int(((oi >= 0) & (od.astype(np.float64) <= max_dist * max_dist)).sum())


def test_exact_nearest_on_submaps(scene, store, oracle):
    P = (rot((0.01, -0.01, np.deg2rad(2.0))), np.array([0.8, -0.5, 0.05]))
    for places, anchor, what in (([0, 1, 2], 1, "HDL-64"), ([4, 5], 4, "HAP"), ([0, 1, 2, 3, 4, 5], 2, "mixed")):
        cur, prev = _loop_pair(scene, places, anchor, P)
        for pre in (None, [0, 0, 0, 0, 0, -0.7], [60.0, -90.0, 35.0, 0, 0, 0.3]):   # the last: 20-150 m from every target point
            g, gi, gd = store.icp(cur[0], prev[0], src_affines=cur[1], tgt_affines=prev[1], pre_pose6=pre, max_iterations=1,
                                  correspondences=True)
            src, tgt = _host_clouds(store, cur, prev, pre, oracle)
            _nn_equal(g, gi, gd, src, tgt, what=f"{what} pre={pre}")
            assert g["iterations"] == 1 and g["n_source"] == len(src) and g["n_target"] == len(tgt)
            print(f"[icp nn] {what} pre={pre}: {len(src)} -> {len(tgt)} points, median d {np.sqrt(np.median(gd)):.3f} m")


def test_exact_nearest_with_nan_duplicates_and_launch_boundaries(scene, oracle):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kfs, _ = scene
    base = kfs[0]
    tgt = np.concatenate([base[:30000], base[:5000]])            # duplicated target points: the lower index wins
    tgt[::101, 2] = np.nan
    src = base[3:40000].copy()
    src[::53, 0] = np.inf
    src[7::211, 1] = np.nan
    sizes = [0, 1, 2, 3, 2 * sms * 256 - 1, 2 * sms * 256, 2 * sms * 256 + 1, 8 * sms * 256 - 1, 8 * sms * 256, 8 * sms * 256 + 1]
    big = np.concatenate([kfs[2], kfs[3], kfs[6]])
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(tgt) + len(src) + sum(sizes) + 16, 32)
    kf.append(capi.pack_pointtype(tgt[:, :3], tgt[:, 3]))
    kf.append(capi.pack_pointtype(src[:, :3], src[:, 3]))
    for n in sizes:
        assert len(big) >= n
        kf.append(capi.pack_pointtype(big[:n, :3], big[:n, 3]))
    one = EYE[None]
    g, gi, gd = kf.icp([1], [0], src_affines=one, tgt_affines=one, max_iterations=1, correspondences=True)
    _nn_equal(g, gi, gd, src, tgt, what="nan + duplicates")
    dup = gi >= 30000                                            # a copy wins only where the original is NaN
    assert (gi[::53] == -1).all() and dup.sum() > 0 and np.isnan(tgt[gi[dup] - 30000, 2]).all()
    for j, n in enumerate(sizes):
        g, gi, gd = kf.icp([2 + j], [0], src_affines=one, tgt_affines=one, max_iterations=1, correspondences=True)
        _nn_equal(g, gi, gd, big[:n], tgt, what=f"n_source={n}")
        o, _, _, _ = io.icp(big[:n], tgt, max_iterations=1)
        assert (g["state"], g["iterations"], g["converged"]) == (o["state"], o["iterations"], o["converged"]), n
    kf.close()
    tree.close()


CASES = [   # places, anchor, perturbation (rpy, t), SC yaw of the pre-transform, kind, id order
    ([0, 1, 2], 1, ((0.0, 0.0, np.deg2rad(3.0)), (0.9, -0.4, 0.05)), 0.0, "affine", "plain"),
    ([1, 2, 3], 2, ((0.01, -0.005, np.deg2rad(-2.0)), (-0.7, 0.6, 0.1)), 0.0, "affine", "permuted"),
    ([4, 5], 5, ((0.0, 0.01, np.deg2rad(4.0)), (1.0, 0.3, -0.05)), 0.0, "affine", "repeated"),
    ([0, 1, 2], 0, ((0.0, 0.0, np.deg2rad(-3.0)), (0.5, 0.8, 0.0)), np.deg2rad(6.0), "affine", "plain"),
    ([0, 1, 2], 1, ((0.0, 0.0, np.deg2rad(2.5)), (-0.8, -0.5, 0.0)), 0.0, "pose6", "plain"),
]


def _margins(log, cfg):
    """How far each iteration's convergence values stayed from the thresholds (relative)."""
    teps, feps = cfg
    m = []
    for cosa, tr2, mse, prev in log:
        rel = abs(mse - prev) / prev if prev < 1e300 else np.inf
        m.append(min(abs(tr2 - teps) / teps, abs(rel - feps) / feps if np.isfinite(rel) else np.inf))
    return min(m) if m else np.inf


@pytest.mark.parametrize("case", range(len(CASES)))
def test_registration_matches_oracle_and_recovers_the_motion(scene, store, oracle, case):
    places, anchor, (rpy, t), sc_yaw, kind, order = CASES[case]
    R, t = rot(rpy), np.asarray(t)
    cur, prev = _loop_pair(scene, places, anchor, (R, t))
    if order == "permuted":
        p = np.array([2, 0, 1])
        cur, prev = (cur[0][p], cur[1][p]), (prev[0][::-1], prev[1][::-1])
    elif order == "repeated":
        cur, prev = (np.r_[cur[0], cur[0][:1]], np.r_[cur[1], cur[1][:1]]), (np.r_[prev[0], prev[0]], np.r_[prev[1], prev[1]])
    pre = [0, 0, 0, 0, 0, -sc_yaw]
    snap = _snapshot(store, 12)
    if kind == "pose6":   # the previous pass at the key frames' own poses (cloudKeyPoses6D), the current one displaced
        _, poses = scene
        def p6(Rm, tv):
            return [tv[0], tv[1], tv[2], np.arctan2(Rm[2, 1], Rm[2, 2]), -np.arcsin(Rm[2, 0]), np.arctan2(Rm[1, 0], Rm[0, 0])]
        Ri, ti = _inv(R, t)
        prev6 = np.array([p6(*poses[k]) for k in places], np.float32)
        cur6 = np.array([p6(Ri @ poses[k][0], Ri @ poses[k][1] + ti) for k in places], np.float32)
        kw = dict(src_poses6=cur6, tgt_poses6=prev6)
        src = np.concatenate([oracle.transform_cloud_rpy(store.download(2 * k + 1)[0], cur6[j]) for j, k in enumerate(places)])
        tgt = np.concatenate([oracle.transform_cloud_rpy(store.download(2 * k)[0], prev6[j]) for j, k in enumerate(places)])
        src = oracle.transform_cloud_rpy(src, np.asarray(pre, np.float32))
    else:
        kw = dict(src_affines=cur[1], tgt_affines=prev[1])
        src, tgt = _host_clouds(store, cur, prev, pre, oracle)
    ids = (cur[0], prev[0]) if kind != "pose6" else (np.array([2 * k + 1 for k in places], np.int32), np.array([2 * k for k in places], np.int32))
    g = store.icp(ids[0], ids[1], pre_pose6=pre, **kw)
    g2 = store.icp(ids[0], ids[1], pre_pose6=pre, **kw)
    o, _, _, log = io.icp(src, tgt)
    assert (g["state"], g["converged"], g["iterations"]) == (o["state"], o["converged"], o["iterations"]), (g, o)
    T, U = g["final_transformation"].astype(np.float64), o["final_transformation"].astype(np.float64)
    assert np.abs(T[:3, 3] - U[:3, 3]).max() <= 1e-5 and rot_err(T, U[:3, :3]) <= 1e-5, (T, U)
    assert abs(g["fitness_score"] - o["fitness_score"]) <= 1e-6 * o["fitness_score"]
    # the known motion: final * pre = P
    Pre = np.eye(4)
    Pre[:3, :3] = rot((0.0, 0.0, -sc_yaw))
    want = np.eye(4)
    want[:3, :3], want[:3, 3] = R, t
    got = T @ Pre
    assert np.abs(got[:3, 3] - t).max() < 0.02 and rot_err(got, R) < np.deg2rad(0.1), (got, want)
    # determinism: two calls bit-identical
    assert all(np.array_equal(np.asarray(g[k]), np.asarray(g2[k])) for k in g)
    _same_store(store, snap)
    print(f"[icp] case {case} ({kind}, {order}, yaw {np.rad2deg(sc_yaw):.0f} deg): {g['iterations']} iterations, "
          f"{g['state_name']}, fitness {g['fitness_score']:.5f}, |dt| vs oracle {np.abs(T[:3, 3] - U[:3, 3]).max():.2e}, "
          f"error vs truth {np.abs(got[:3, 3] - t).max() * 100:.2f} cm / {np.rad2deg(rot_err(got, R)):.4f} deg, "
          f"threshold margin {_margins(log, (1e-6, 1e-6)):.3g}")


def test_no_correspondences_and_empty_selections(scene, store):
    cur, prev = _loop_pair(scene, [0, 1], 0, (np.eye(3), np.zeros(3)))
    g = store.icp(cur[0], prev[0], src_affines=cur[1], tgt_affines=prev[1], pre_pose6=[0, 0, 500, 0, 0, 0],
                  max_correspondence_distance=1.0)
    assert g["state_name"] == "NO_CORRESPONDENCES" and not g["converged"] and g["iterations"] == 0
    assert np.array_equal(g["final_transformation"], np.eye(4, dtype=np.float32))
    for a, b in (([], prev), (cur, ([], np.zeros((0, 12), np.float32)))):
        ai = a[0] if len(a) else np.zeros(0, np.int32)
        at = a[1] if len(a) else np.zeros((0, 12), np.float32)
        g, gi, _ = store.icp(ai, b[0], src_affines=at, tgt_affines=b[1], correspondences=True)
        assert g["state"] == 0 and g["iterations"] == 0 and g["fitness_score"] == np.finfo(np.float64).max
        assert (gi == -1).all()
    with pytest.raises(capi.FlbError, match="out of range"):
        store.icp([0, 99], [1], src_affines=np.stack([EYE, EYE]), tgt_affines=EYE[None])


def test_scan_step_after_icp_is_identical_and_scratch_is_released(scene):
    rng = np.random.default_rng(7)
    world = synth.city_world(half_extent=120, seed=7)
    st_true = synth.trajectory_state(0)
    body = synth.scan_from_pose(world, st_true, synth.lidar_dirs("vlp16"), rng)
    mp = synth.sample_surface_map(world, (0, 0, 0), 50, 0.2, rng)
    prior = synth.perturb_state(st_true, rng)
    P0 = synth.default_cov()
    kfs, _ = scene
    out = []
    for with_icp in (False, True):
        tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
        tree.Build(mp)
        ses = capi.Session(tree, max_scan_points=len(body), max_iterations=3)
        kf = capi.KeyFrameStore(tree, len(kfs[0]) + len(kfs[1]), 4)
        kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
        kf.append(capi.pack_pointtype(kfs[1][:, :3], kfs[1][:, 3]))
        if with_icp:
            assert kf.info()["map_scratch_bytes"] == 0
            g = kf.icp([1], [0], src_affines=EYE[None], tgt_affines=EYE[None])
            assert g["converged"]
            s1 = kf.info()["map_scratch_bytes"]
            assert s1 >= 20 * (len(kfs[0]) + len(kfs[1]))
        st, P, r = ses.scan_step(None, body, prior, P0)
        out.append((st, P, r.update.effct_feat_num, tree.validnum()))
        if with_icp:
            kf.release_scratch()
            assert kf.info()["map_scratch_bytes"] == 0
            g2 = kf.icp([1], [0], src_affines=EYE[None], tgt_affines=EYE[None])   # the same after the release
            assert all(np.array_equal(np.asarray(g[k]), np.asarray(g2[k])) for k in g)
        kf.close()
        ses.close()
        tree.close()
    (sa, Pa, ma, va), (sb, Pb, mb, vb) = out
    assert ma > 500 and ma == mb and va == vb
    assert np.array_equal(sa, sb) and np.array_equal(Pa, Pb)


def test_full_size_hap_pair(oracle):
    """The bench's HAP size: two sub-maps of 21 key frames (8 ray-cast scans cycled), about 4.7M points each."""
    world = synth.city_world(half_extent=400.0, seed=3)
    rng = np.random.default_rng(3)
    scans = []
    for j in range(8):
        dirs = synth.lidar_dirs("hap", np.random.default_rng(100 + j))
        scans.append(_p4(synth.scan_from_pose(world, synth.trajectory_state(10 * j), dirs, rng, max_range=100.0, min_range=2.0), rng))
    n_kf = 21
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(scans[k % 8]) for k in range(n_kf)) * 2 + 16, 2 * n_kf)
    for k in range(n_kf):
        kf.append(capi.pack_pointtype(scans[k % 8][:, :3], scans[k % 8][:, 3]))
    R, t = rot((0.0, 0.0, np.deg2rad(3.0))), np.array([0.9, -0.6, 0.05])
    prev_T = [_affine(rot((0, 0, 0.02 * k)), [0.8 * (k - 10), 0.1 * (k - 10), 0.0]) for k in range(n_kf)]
    Ri, ti = _inv(R, t)
    cur_T = []
    for a in prev_T:
        A = a.reshape(3, 4).astype(np.float64)
        cur_T.append(_affine(Ri @ A[:, :3], Ri @ A[:, 3] + ti))
    ids = np.arange(n_kf, dtype=np.int32)
    g, gi, gd = kf.icp(ids, ids, src_affines=np.stack(cur_T), tgt_affines=np.stack(prev_T), max_iterations=1, correspondences=True)
    src, _ = kf.assemble(ids, affines=np.stack(cur_T))
    tgt, _ = kf.assemble(ids, affines=np.stack(prev_T))
    assert len(src) > 4_000_000 and len(tgt) > 4_000_000
    _nn_equal(g, gi, gd, src, tgt, what="full size")
    g = kf.icp(ids, ids, src_affines=np.stack(cur_T), tgt_affines=np.stack(prev_T))
    T = g["final_transformation"].astype(np.float64)
    print(f"[icp full size] {len(src)} -> {len(tgt)} points: {g['iterations']} iterations, {g['state_name']}, "
          f"error {np.abs(T[:3, 3] - t).max() * 100:.2f} cm / {np.rad2deg(rot_err(T, R)):.4f} deg")
    assert g["converged"] and np.abs(T[:3, 3] - t).max() < 0.02 and rot_err(T, R) < np.deg2rad(0.1)
    kf.close()
    tree.close()
