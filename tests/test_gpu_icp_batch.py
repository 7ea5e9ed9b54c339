"""GPU tests of the inter-session registration (flb_keyframes_icp_batch) on the ray-cast street scenes of
test_gpu_icp.py.  Two sessions see the same places (two noise draws): the query session's clouds are displaced by a known
rigid motion P, and its central-frame poses carry a small per-pose drift.  The Scan Context pairs register the query key
frame s onto the central key frames t-2 .. t+2 at zero poses (loopFindNearKeyframesLocalCoord); the radius-search pairs do
the same with the key frames' poses (loopFindNearKeyframesCentralCoord).  Every pair must be flb_keyframes_icp's result bit
for bit at leaf 0, follow the CPU oracle on the filtered clouds at leaf 0.2, and not depend on the batch around it."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import icp_oracle as io
from tests.icp_cases import rot, rot_err

pytestmark = pytest.mark.gpu

MODELS = ["hdl64", "hdl64", "hdl64", "hdl64", "hap", "hap"]
P_RPY, P_T = (0.004, -0.006, np.deg2rad(1.5)), np.array([0.35, -0.25, 0.03])   # the query session's displacement
CFG = dict(max_correspondence_distance=30.0, max_iterations=10, transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6)
ZERO = [0.0] * 6


def _p4(xyz, rng):
    return np.column_stack([xyz, rng.integers(0, 256, len(xyz))]).astype(np.float32)


def _p6(R, t):
    return [t[0], t[1], t[2], np.arctan2(R[2, 1], R[2, 2]), -np.arcsin(R[2, 0]), np.arctan2(R[1, 0], R[0, 0])]


def _mat(p6):
    T = np.eye(4)
    T[:3, :3] = rot(p6[3:6])
    T[:3, 3] = p6[:3]
    return T


@pytest.fixture(scope="module")
def sessions():
    """Central key frames 0..5 (body frame, poses `poses`), query key frames 6..11 (another draw of the same places, moved
    by P^-1, so that the query sensor sits at pose * P), 4 full-size HAP scans 12..15 and one all-NaN key frame 16."""
    world = synth.city_world(half_extent=150.0, seed=6)
    rng = np.random.default_rng(3)
    R, t = rot(P_RPY), P_T
    central, query, poses = [], [], []
    for j, model in enumerate(MODELS):
        st = synth.trajectory_state(4 * j)
        dirs = synth.lidar_dirs(model, np.random.default_rng(50 + j))
        if model == "hap":
            dirs = dirs[:80000]
        central.append(_p4(synth.scan_from_pose(world, st, dirs, np.random.default_rng(10 * j), max_range=100.0, min_range=1.0), rng))
        q = _p4(synth.scan_from_pose(world, st, dirs, np.random.default_rng(10 * j + 1), max_range=100.0, min_range=1.0), rng)
        q[:, :3] = ((q[:, :3].astype(np.float64) - t) @ R).astype(np.float32)
        query.append(q)
        Rw = synth.quat_to_mat(st[3:7]) @ synth.quat_to_mat(st[7:11])
        poses.append(np.array(_p6(Rw, st[0:3] + synth.quat_to_mat(st[3:7]) @ st[11:14]), np.float32))
    hap = []
    for j in range(4):
        dirs = synth.lidar_dirs("hap", np.random.default_rng(200 + j))
        hap.append(_p4(synth.scan_from_pose(world, synth.trajectory_state(6 * j), dirs, rng, max_range=100.0, min_range=1.0), rng))
    nan = np.full((500, 4), np.nan, np.float32)
    clouds = central + query + hap + [nan]
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(c) for c in clouds) + 16, 64)
    for c in clouds:
        kf.append(capi.pack_pointtype(c[:, :3], c[:, 3]))
    yield kf, poses, len(clouds)
    kf.close()
    tree.close()


def _query_pose(poses, s, drift):
    """The query key frame's central-frame pose after the optimisation: pose_s * P * drift."""
    D = np.eye(4)
    D[:3, :3] = rot((0.0, 0.0, np.deg2rad(0.3 * drift)))
    D[:3, 3] = (0.08 * drift, -0.05 * drift, 0.0)
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = rot(P_RPY), P_T
    T = _mat(poses[s]) @ P @ D
    return np.array(_p6(T[:3, :3], T[:3, 3]), np.float32)


def _near(t, n=6, search=2):
    return [k for k in range(t - search, t + search + 1) if 0 <= k < n]


def sc_pairs(poses):
    """addSCloops: query key frame s alone vs central t-2 .. t+2, every key frame at the zero pose."""
    return [([6 + s], [ZERO], _near(s), [ZERO] * len(_near(s))) for s in range(6)]


def rs_pairs(poses):
    """addRSloops: query key frame s at its central-frame pose vs central t-2 .. t+2 at their poses."""
    out = []
    for s in range(6):
        drift = (s % 3) - 1
        out.append(([6 + s], [_query_pose(poses, s, drift)], _near(s), [poses[k] for k in _near(s)]))
    return out


def _single(kf, pair, **cfg):
    si, sp, ti, tp = pair
    return kf.icp(np.asarray(si, np.int32), np.asarray(ti, np.int32), src_poses6=np.asarray(sp, np.float32).reshape(-1, 6),
                  tgt_poses6=np.asarray(tp, np.float32).reshape(-1, 6), **cfg)


def _bits(r):
    return (r["state"], r["converged"], r["iterations"], r["n_source"], r["n_target"], r["n_correspondences"],
            r["final_transformation"].tobytes(), np.float64(r["fitness_score"]).tobytes())


def _passes(r):
    return r["iterations"] + (1 if r["state_name"] == "NO_CORRESPONDENCES" else 0)


def _snapshot(kf, n):
    return [kf.download(k) for k in range(n)]


def _same_store(kf, snap):
    for k, (p, c) in enumerate(snap):
        q, d = kf.download(k)
        assert np.array_equal(q.view(np.uint32), p.view(np.uint32)) and np.array_equal(d.view(np.uint32), c.view(np.uint32))


def test_leaf0_every_pair_equals_flb_keyframes_icp_bit_for_bit(sessions):
    kf, poses, n_kf = sessions
    pairs = sc_pairs(poses) + rs_pairs(poses)
    snap = _snapshot(kf, n_kf)
    got, st = kf.icp_batch(pairs, leaf=0.0, **CFG)
    for p, (pair, g) in enumerate(zip(pairs, got)):
        r = _single(kf, pair, **CFG)
        assert _bits(g) == _bits(r), (p, g, r)
        assert g["n_source"] == sum(kf.size(i) for i in pair[0]) and g["n_target"] == sum(kf.size(i) for i in pair[2])
    assert st["rounds"] == 1
    assert st["iteration_syncs"] == max(_passes(g) for g in got) + 1
    assert st["setup_syncs"] == len(pairs)   # leaf 0: one target box per pair, no filter
    _same_store(kf, snap)
    print(f"[icp batch leaf 0] {len(pairs)} pairs: states {[g['state_name'] for g in got]}, stats {st}")


def test_leaf02_follows_the_oracle_and_recovers_the_motion(sessions):
    kf, poses, _ = sessions
    pairs = sc_pairs(poses) + rs_pairs(poses)
    got, st = kf.icp_batch(pairs, leaf=0.2, **CFG)
    first, _ = kf.icp_batch(pairs, leaf=0.2, **dict(CFG, max_iterations=1))
    assert st["rounds"] == 1 and st["setup_syncs"] == 3 * len(pairs)   # two filters and one target box per pair
    assert st["iteration_syncs"] == max(_passes(g) for g in got) + 1
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = rot(P_RPY), P_T
    for p, (pair, g, g1) in enumerate(zip(pairs, got, first)):
        si, sp, ti, tp = pair
        src, _ = kf.assemble(si, poses6=np.asarray(sp, np.float32).reshape(-1, 6), leaf=0.2)
        tgt, _ = kf.assemble(ti, poses6=np.asarray(tp, np.float32).reshape(-1, 6), leaf=0.2)
        assert (g["n_source"], g["n_target"]) == (len(src), len(tgt)), p
        o1, _, _, _ = io.icp(src, tgt, **dict(CFG, max_iterations=1))
        assert g1["n_correspondences"] == o1["n_correspondences"], (p, g1, o1)
        o, _, _, _ = io.icp(src, tgt, **CFG)
        assert (g["state"], g["converged"], g["iterations"]) == (o["state"], o["converged"], o["iterations"]), (p, g, o)
        T, U = g["final_transformation"].astype(np.float64), o["final_transformation"].astype(np.float64)
        assert np.abs(T[:3, 3] - U[:3, 3]).max() <= 1e-5 and rot_err(T, U[:3, :3]) <= 1e-5, (p, T, U)
        assert abs(g["fitness_score"] - o["fitness_score"]) <= 1e-6 * o["fitness_score"], p
        if p < 6:   # SC: the query cloud is P^-1 of the central one, so final = P
            want = P
        else:       # RS: final moves the drifted query pose onto the true one, pose_s * P
            s = p - 6
            want = _mat(poses[s]) @ P @ np.linalg.inv(_mat(_query_pose(poses, s, (s % 3) - 1)))
        err_t, err_r = np.abs(T[:3, 3] - want[:3, 3]).max(), rot_err(T, want[:3, :3])
        print(f"[icp batch leaf 0.2] pair {p}: {len(src)} -> {len(tgt)} points, {g['iterations']} it, {g['state_name']}, "
              f"|dt| vs oracle {np.abs(T[:3, 3] - U[:3, 3]).max():.1e}, error vs truth {err_t * 100:.2f} cm / {np.rad2deg(err_r):.3f} deg")
        if p != 4:   # the HAP place's SC target superposes HDL-64 neighbours at the zero pose: 10 iterations end 17 cm off
            assert err_t < 0.02 and err_r < np.deg2rad(0.3), (p, T, want)


def test_a_pair_does_not_depend_on_its_batch_or_round(sessions):
    kf, poses, _ = sessions
    base = sc_pairs(poses) + rs_pairs(poses)
    mixed = []   # 40 pairs: HDL-64 and HAP places, SC and RS, some with a second central key frame range
    for j in range(40):
        si, sp, ti, tp = base[j % 12]
        if j >= 12:
            ti, tp = list(ti)[: 1 + j % len(ti)], list(tp)[: 1 + j % len(tp)]
        mixed.append((si, sp, ti, tp))
    for leaf in (0.0, 0.2):
        alone = [kf.icp_batch([pr], leaf=leaf, **CFG)[0][0] for pr in mixed]
        batch, st = kf.icp_batch(mixed, leaf=leaf, **CFG)
        perm = np.random.default_rng(5).permutation(len(mixed))
        permuted, _ = kf.icp_batch([mixed[i] for i in perm], leaf=leaf, **CFG)
        for j in range(len(mixed)):
            assert _bits(batch[j]) == _bits(alone[j]), (leaf, j)
        for k, i in enumerate(perm):
            assert _bits(permuted[k]) == _bits(alone[i]), (leaf, i)
        assert st["rounds"] == 1 and st["iteration_syncs"] == max(_passes(g) for g in batch) + 1
    # 16 dense full-size HAP pairs: more summed grid cells than one round holds
    hap = []
    for j in range(16):
        ids = [12 + (j + k) % 4 for k in range(8)]
        p6 = [[0.1 * k, 0.0, 0.0, 0.0, 0.0, 0.01 * k] for k in range(8)]
        hap.append(([12 + j % 4], [[0.3, -0.2, 0.0, 0.0, 0.0, 0.02]], ids, p6))
    batch, st = kf.icp_batch(hap, leaf=0.0, **CFG)
    assert st["rounds"] > 1, st
    for j, pr in enumerate(hap):
        assert _bits(batch[j]) == _bits(kf.icp_batch([pr], leaf=0.0, **CFG)[0][0]), j
        if j < 4:
            assert _bits(batch[j]) == _bits(_single(kf, pr, **CFG)), j
    print(f"[icp batch rounds] 16 HAP pairs of {batch[0]['n_target']} target points: {st}")


def test_mixed_outcomes_in_one_batch(sessions):
    kf, poses, n_kf = sessions
    cfg = dict(max_correspondence_distance=30.0, max_iterations=6, transformation_epsilon=1e-6, euclidean_fitness_epsilon=0.1)
    sc, rs = sc_pairs(poses), rs_pairs(poses)
    far = [poses[k].copy() for k in _near(1)]
    for p6 in far:
        p6[2] += 500.0
    shifted = [([0], [[d, -0.5 * d, 0.0, 0.0, 0.0, 0.1 * d]], [0], [ZERO]) for d in (0.05, 0.2, 1.0)]
    pairs = [
        ([0], [poses[0]], [0], [poses[0]]),                              # the same cloud: TRANSFORM at the first iteration
        ([6], [[6.0, -4.0, 0.0, 0.0, 0.0, 0.3]], [0, 1], [ZERO, ZERO]),   # a large offset: still moving after 6
        ([7], [ZERO], _near(1), far),                                   # the target 500 m away: NO_CORRESPONDENCES
        ([], [], [0, 1], [ZERO, ZERO]),                                  # empty source selection
        ([8], [ZERO], [n_kf - 1], [ZERO]),                              # all-NaN target
    ] + shifted + [sc[2], sc[4], rs[1], rs[3]]                         # residual motions: the fitness test or the limit
    # (the CPU oracle stops the HAP place's SC pair sc[4] with REL_MSE at iteration 5 under this config)
    got, st = kf.icp_batch(pairs, leaf=0.0, **cfg)
    states = [g["state_name"] for g in got]
    print(f"[icp batch mixed] {states}, iterations {[g['iterations'] for g in got]}, stats {st}")
    for j, pr in enumerate(pairs):
        assert _bits(got[j]) == _bits(_single(kf, pr, **cfg)), (j, got[j])
        assert _bits(got[j]) == _bits(kf.icp_batch([pr], leaf=0.0, **cfg)[0][0]), j
    assert states[0] == "TRANSFORM" and got[0]["iterations"] == 1
    assert states[1] == "ITERATIONS" and got[1]["iterations"] == 6
    assert states[2] == "NO_CORRESPONDENCES" and got[2]["iterations"] == 0
    for j in (3, 4):
        assert states[j] == "NOT_CONVERGED" and got[j]["iterations"] == 0 and got[j]["fitness_score"] == np.finfo(np.float64).max
    assert got[4]["n_target"] == 500 and got[3]["n_source"] == 0
    assert states[pairs.index(sc[4])] == "REL_MSE"
    assert st["rounds"] == 1 and st["iteration_syncs"] == max(_passes(g) for g in got) + 1
    # at leaf 0.2 the NaN target filters away: n_target 0, the same empty result
    g4, _ = kf.icp_batch([pairs[4]], leaf=0.2, **cfg)
    assert g4[0]["n_target"] == 0 and g4[0]["state"] == 0
    with pytest.raises(capi.FlbError, match="pair 1: tgt_ids entry 2: key frame 99 out of range"):
        kf.icp_batch([pairs[0], ([0], [ZERO], [0, 99], [ZERO, ZERO])], leaf=0.2, **cfg)


def test_repeat_calls_scratch_release_and_a_scan_step_afterwards(sessions):
    kf, poses, n_kf = sessions
    pairs = sc_pairs(poses)[:3] + rs_pairs(poses)[3:]
    a, _ = kf.icp_batch(pairs, leaf=0.2, **CFG)
    b, _ = kf.icp_batch(pairs, leaf=0.2, **CFG)
    assert all(_bits(x) == _bits(y) for x, y in zip(a, b))
    s1 = kf.info()["map_scratch_bytes"]
    kf.release_scratch()
    assert kf.info()["map_scratch_bytes"] == 0 < s1
    c, _ = kf.icp_batch(pairs, leaf=0.2, **CFG)
    assert all(_bits(x) == _bits(y) for x, y in zip(a, c))

    rng = np.random.default_rng(7)
    world = synth.city_world(half_extent=120, seed=7)
    st_true = synth.trajectory_state(0)
    body = synth.scan_from_pose(world, st_true, synth.lidar_dirs("vlp16"), rng)
    mp = synth.sample_surface_map(world, (0, 0, 0), 50, 0.2, rng)
    prior = synth.perturb_state(st_true, rng)
    P0 = synth.default_cov()
    central = [kf.download(k)[0] for k in (0, 1, 6)]
    out = []
    for with_batch in (False, True):
        tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
        tree.Build(mp)
        ses = capi.Session(tree, max_scan_points=len(body), max_iterations=3)
        store = capi.KeyFrameStore(tree, sum(len(c) for c in central), 4)
        for c in central:
            store.append(capi.pack_pointtype(c[:, :3], c[:, 3]))
        if with_batch:
            g, _ = store.icp_batch([([2], [ZERO], [0, 1], [ZERO, ZERO])], leaf=0.2, **CFG)
            assert g[0]["converged"]
        s, P, r = ses.scan_step(None, body, prior, P0)
        out.append((s, P, r.update.effct_feat_num, tree.validnum()))
        store.close()
        ses.close()
        tree.close()
    (sa, Pa, ma, va), (sb, Pb, mb, vb) = out
    assert ma > 500 and ma == mb and va == vb
    assert np.array_equal(sa, sb) and np.array_equal(Pa, Pb)
