"""GPU tests of the relocalisation registration (flb_keyframes_fricp) against the sequential CPU oracle
(tests/cpp/fricp_oracle.cpp), on ray-cast HDL-64 and HAP key frames along a street.  Given the device's normalisation, the
first correspondence pass (matched target and residual of every source point) and the Welsch scale's first and last value
are bit-equal to the oracle's; whole registrations in modes 0, 2, 3 and 4 take the oracle's path (stages, iterations,
Anderson accept / reject) wherever its decisions have margins above 1e-9 relative, and land within 1e-6 m / 1e-6 rad of its
res_trans; a displaced, outlier-laden scan is recovered."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import fricp_oracle as fo
from tests.icp_cases import rot, rot_err

pytestmark = pytest.mark.gpu

PLACES = {"HDL-64": [0, 1, 2], "HAP": [4, 5], "mixed": [1, 2, 4]}
EXT = np.array([0.12, -0.05, 0.3, 0.002, -0.001, 0.01], np.float32)   # pose_ext (lidar-to-body) of the prior session


def _p4(xyz, rng):
    return np.column_stack([xyz, rng.integers(0, 256, len(xyz))]).astype(np.float32)


def _p6(R, t):
    return np.array([t[0], t[1], t[2], np.arctan2(R[2, 1], R[2, 2]), -np.arcsin(R[2, 0]), np.arctan2(R[1, 0], R[0, 0])], np.float32)


@pytest.fixture(scope="module")
def scene():
    """Body-frame key frames (3 HDL-64 and 2 HAP places, 80 000 HAP rays), two noise draws of each place (rep 0: the prior
    session, rep 1: the live scan) and the places' poses."""
    world = synth.city_world(half_extent=150.0, seed=6)
    rng = np.random.default_rng(3)
    kfs, poses = [], []
    for j, model in enumerate(["hdl64", "hdl64", "hdl64", "hdl64", "hap", "hap"]):
        st = synth.trajectory_state(4 * j)
        dirs = synth.lidar_dirs(model, np.random.default_rng(50 + j))
        if model == "hap":
            dirs = dirs[:80000]
        for rep in range(2):
            kfs.append(_p4(synth.scan_from_pose(world, st, dirs, np.random.default_rng(10 * j + rep), max_range=100.0, min_range=1.0), rng))
        R = synth.quat_to_mat(st[3:7]) @ synth.quat_to_mat(st[7:11])
        poses.append((R, st[0:3] + synth.quat_to_mat(st[3:7]) @ st[11:14]))
    return kfs, poses


@pytest.fixture(scope="module")
def store(scene):
    kfs, _ = scene
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, sum(len(k) for k in kfs) + 16, 64)
    for p in kfs:
        kf.append(capi.pack_pointtype(p[:, :3], p[:, 3]))
    yield kf
    kf.close()
    tree.close()


def _target(oracle, store, ids, poses6, ext=EXT):
    parts = []
    for j, k in enumerate(ids):
        c = store.download(k)[0]
        if ext is not None:
            c = oracle.transform_cloud_rpy(c, ext)
        parts.append(oracle.transform_cloud_rpy(c, poses6[j]))
    return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)


def _norm(g):
    return g["scale"], g["mu_source"], g["mu_target"]


def _first_pass_equal(store, oracle, src, ids, p6, init6=None, ext=EXT, what=""):
    for mode in (0, 4):
        g, gi, gr = store.fricp(src, ids, p6, tgt_pre_pose6=ext, src_pose6=init6, mode=mode, max_icp=0, correspondences=True)
        s = src if init6 is None else oracle.transform_cloud_rpy(src, init6)
        tgt = _target(oracle, store, ids, p6, ext)
        o, oi, orr, _ = fo.fricp(s, tgt, mode=mode, max_icp=0, norm=_norm(g))
        assert g["status"] == o["status"] == 0, what
        assert np.array_equal(gi, oi), (what, np.nonzero(gi != oi)[0][:5])
        assert np.array_equal(gr.view(np.uint64), orr.view(np.uint64)), what
        assert (g["nu_begin"], g["nu_end"]) == (o["nu_begin"], o["nu_end"]), what
        assert (g["n_source_finite"], g["n_target_finite"]) == (o["n_source_finite"], o["n_target_finite"])
    return g


def test_first_pass_and_scales_on_key_frames(scene, store, oracle):
    kfs, poses = scene
    for what, places in PLACES.items():
        ids = np.array([2 * k for k in places], np.int32)
        p6 = np.stack([_p6(*poses[k]) for k in places])
        a = places[len(places) // 2]
        init = _p6(*poses[a]) + np.array([0.4, -0.3, 0.05, 0.0, 0.0, 0.03], np.float32)
        for off in (np.zeros(6, np.float32), np.array([60.0, -90.0, 35.0, 0, 0, 0.3], np.float32)):   # the second: 20-150 m away
            g = _first_pass_equal(store, oracle, kfs[2 * a + 1], ids, p6, init + off, what=f"{what} off={off[:3]}")
            print(f"[fricp pass] {what}: {len(kfs[2 * a + 1])} -> {g['n_target']} points, nu {g['nu_begin']:.5f} -> {g['nu_end']:.6f}")


def test_first_pass_nan_duplicates_boundaries_and_tiny_targets(scene, oracle):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kfs, _ = scene
    base = kfs[0]
    tgt = np.concatenate([base[:30000], base[:5000]])   # duplicated target points: the lower index wins
    tgt[::101, 2] = np.nan
    src = base[3:40000].copy()
    src[::53, 0] = np.inf
    src[7::211, 1] = np.nan
    big = np.concatenate([kfs[2], kfs[3], kfs[6], kfs[8]])
    sizes = [sms * 256 - 1, sms * 256, sms * 256 + 1, 8 * sms * 256 - 1, 8 * sms * 256 + 1]
    assert len(big) >= max(sizes)
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(tgt) + sum(sizes) + 64, 32)
    kf.append(capi.pack_pointtype(tgt[:, :3], tgt[:, 3]))
    one = np.zeros((1, 6), np.float32)
    g = _first_pass_equal(kf, oracle, src, [0], one, ext=None, what="nan + duplicates")
    _, gi, _ = kf.fricp(src, [0], one, max_icp=0, correspondences=True)
    assert (gi[::53] == -1).all() and (gi >= 30000).sum() > 0
    for n in sizes:
        _first_pass_equal(kf, oracle, big[:n], [0], one, ext=None, what=f"n_source={n}")
        k = kf.append(capi.pack_pointtype(big[:n, :3], big[:n, 3]))
        _first_pass_equal(kf, oracle, src[:5000], [k], one, ext=None, what=f"n_target={n}")
    for n in range(1, 9):
        k = kf.append(capi.pack_pointtype(base[100:100 + n, :3] * 3.0, base[100:100 + n, 3]))
        if n == 1:
            g = kf.fricp(src[:100], [k], one)
            assert g["status_name"] == "FEW_TARGET" and np.array_equal(g["res_trans"], np.eye(4))
        else:
            _first_pass_equal(kf, oracle, src[:2000], [k], one, ext=None, what=f"{n} target points")
    kf.close()
    tree.close()


def _margins(log, stop):
    m = [np.inf]
    for _, e, prev, dT, _ in log:
        if np.isfinite(prev) and prev < 1e300:
            m.append(abs(e - prev) / max(abs(prev), 1e-300))
        m.append(abs(dT - stop) / stop)
    return min(m)


@pytest.mark.parametrize("mode", [0, 2, 3, 4])
def test_registration_follows_the_oracle(scene, store, oracle, mode):
    kfs, poses = scene
    places = [0, 1, 2]
    ids = np.array([2 * k for k in places], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in places])
    init = _p6(*poses[1]) + np.array([0.5, -0.4, 0.0, 0.0, 0.0, np.deg2rad(2.0)], np.float32)
    src = kfs[3]
    snap = [store.download(k) for k in range(len(kfs))]
    g, gi, gr, glog = store.fricp(src, ids, p6, tgt_pre_pose6=EXT, src_pose6=init, mode=mode, correspondences=True, log=True)
    g2 = store.fricp(src, ids, p6, tgt_pre_pose6=EXT, src_pose6=init, mode=mode)
    assert all(np.array_equal(np.asarray(g[k]), np.asarray(g2[k])) for k in g)   # two calls bit-identical
    for k, (p, c) in enumerate(snap):                                              # the store is unchanged
        q, d = store.download(k)
        assert np.array_equal(q.view(np.uint32), p.view(np.uint32)) and np.array_equal(d.view(np.uint32), c.view(np.uint32))
    s = oracle.transform_cloud_rpy(src, init)
    tgt = _target(oracle, store, ids, p6)
    o, oi, orr, olog = fo.fricp(s, tgt, mode=mode, norm=_norm(g))
    margin = _margins(olog, 1e-5)
    if margin > 1e-9:
        assert (g["stages"], g["iterations"], g["rejections"]) == (o["stages"], o["iterations"], o["rejections"])
        assert np.array_equal(glog[:, [0, 4]], olog[:, [0, 4]])
        assert np.abs(glog[:, 1] - olog[:, 1]).max() <= 1e-9 * np.abs(olog[:, 1]).max()
        assert abs(g["energy"] - o["energy"]) <= 1e-9 * abs(o["energy"])
    T, U = g["res_trans"], o["res_trans"]
    assert np.abs(T[:3, 3] - U[:3, 3]).max() <= 1e-6 and rot_err(T, U[:3, :3]) <= 1e-6, (T, U)
    print(f"[fricp] mode {mode}: {g['stages']} stages, {g['iterations']} iterations, {g['rejections']} rejections, "
          f"energy {g['energy']:.6g}, |dt| vs oracle {np.abs(T[:3, 3] - U[:3, 3]).max():.2e}, decision margin {margin:.3g}")


def test_recovery_of_a_displaced_scan_with_outliers(scene, store):
    kfs, poses = scene
    places = [0, 1, 2]
    ids = np.array([2 * k for k in places], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in places])
    world = np.concatenate([kfs[2 * k + 1][:, :3].astype(np.float64) @ poses[k][0].T + poses[k][1] for k in places])
    rng = np.random.default_rng(9)
    n_out = int(0.15 * len(world))
    lo, hi = world.min(0), world.max(0)
    outl = rng.uniform(lo, hi, size=(n_out, 3))   # stand-ins for dynamic objects
    R, t = rot((0.01, -0.01, np.deg2rad(8.0))), np.array([1.2, -0.9, 0.05])
    t = t / np.linalg.norm(t) * 1.5
    pts = np.concatenate([world, outl])
    src = ((pts - t) @ R).astype(np.float32)      # D^-1 x: the registration should return D = (R, t)
    errs = {}
    for mode in (4, 0):
        g = store.fricp(src, ids, p6, mode=mode)
        T = g["res_trans"]
        errs[mode] = (np.abs(T[:3, 3] - t).max(), rot_err(T, R))
        print(f"[fricp recovery] mode {mode}: {g['stages']} stages, {g['iterations']} iterations, "
              f"error {errs[mode][0] * 100:.2f} cm / {np.rad2deg(errs[mode][1]):.4f} deg")
    assert errs[4][0] < 0.02 and errs[4][1] < np.deg2rad(0.1)


def test_scratch_and_rejected_inputs(scene):
    kfs, poses = scene
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(kfs[0]) + 16, 4)
    kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
    one = np.zeros((1, 6), np.float32)
    assert kf.info()["map_scratch_bytes"] == 0
    g = kf.fricp(kfs[1], [0], one, max_icp=5)
    assert kf.info()["map_scratch_bytes"] >= 100 * len(kfs[0])
    kf.release_scratch()
    assert kf.info()["map_scratch_bytes"] == 0
    g2 = kf.fricp(kfs[1], [0], one, max_icp=5)
    assert all(np.array_equal(np.asarray(g[k]), np.asarray(g2[k])) for k in g)
    for mode in (1, 5, 6, 7, 8, -1):
        with pytest.raises(capi.FlbError, match=f"regMode {mode} is not supported"):
            kf.fricp(kfs[1], [0], one, mode=mode)
    for kw, msg in ((dict(max_icp=-1), "max_icp"), (dict(stop=np.nan), "stop"), (dict(anderson_m=0), "anderson_m"),
                    (dict(anderson_m=6), "anderson_m"), (dict(nu_end_k=0.0), "nu_begin_k and nu_end_k"),
                    (dict(nu_alpha=1.0), "nu_alpha"), (dict(src_pose6=[0, 0, np.inf, 0, 0, 0]), "finite")):
        with pytest.raises(capi.FlbError, match=msg):
            kf.fricp(kfs[1], [0], one, **kw)
    with pytest.raises(capi.FlbError, match="out of range"):
        kf.fricp(kfs[1], [3], one)
    g = kf.fricp(kfs[1][:0], [0], one)
    assert g["status_name"] == "NO_SOURCE" and g["iterations"] == 0
    kf.close()
    tree.close()
