"""GPU tests of the relocalisation Sparse ICP (flb_keyframes_sicp, regMode 7) against the sequential CPU oracle (orc_sicp in
tests/cpp/sicp_oracle.cpp), on the ray-cast HDL-64 and HAP street scenes of test_gpu_fricp.py.  Given the device's
normalisation, the first pass's matches are bit-equal to the oracle's and the first ADMM step lands within 1e-12; whole
registrations take the oracle's path (ICP iterations, ADMM iterations of each) wherever its logged stopping decisions have
margins above 1e-9 relative and land within 1e-6 m / 1e-6 rad of its res_trans; source sizes around the block and the
resident grid; repeat calls; one host synchronisation per ICP iteration; the rejected configs; a displaced, outlier-laden
scan is recovered."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi
from tests import sicp_oracle as so
from tests.icp_cases import rot, rot_err
from tests.test_gpu_fricp import EXT, PLACES, _norm, _p6, _target, scene, store  # noqa: F401  (the shared scene fixtures)

pytestmark = pytest.mark.gpu

STOP = 1e-5


def _sub(a, k):
    return np.ascontiguousarray(a[::k])


def _margin(log, stop=STOP, max_outer=100):
    m = [np.inf]
    for outer, primal, dual, st, _ in log:
        m.append(abs(st - stop) / stop)
        if outer < max_outer:   # the ADMM loop left on its own test
            m.append(max(abs(primal - stop), abs(dual - stop)) / stop if primal < stop or dual < stop else np.inf)
    return min(m)


def _compare(g, o, what, exact_path=True, tol=1e-6):
    assert g["status"] == o["status"] == 0, what
    assert (g["n_source_finite"], g["n_target_finite"]) == (o["n_source_finite"], o["n_target_finite"]), what
    T, U = g["res_trans"], o["res_trans"]
    assert np.abs(T[:3, 3] - U[:3, 3]).max() <= tol and rot_err(T, U[:3, :3]) <= tol, (what, T, U)


def _case(store, oracle, src, ids, p6, init6=None, ext=EXT, what="", **kw):
    g, gi, gr, glog = store.sicp(src, ids, p6, tgt_pre_pose6=ext, src_pose6=init6, correspondences=True, log=True, **kw)
    s = src if init6 is None else oracle.transform_cloud_rpy(src, init6)
    tgt = _target(oracle, store, ids, p6, ext)
    o, oi, orr, olog = so.sicp(s, tgt, norm=_norm(g), **kw)
    return g, gi, gr, glog, o, oi, orr, olog


def test_first_pass_and_first_admm_step(scene, store, oracle):
    kfs, poses = scene
    for what, places in PLACES.items():
        ids = np.array([2 * k for k in places], np.int32)
        p6 = np.stack([_p6(*poses[k]) for k in places])
        a = places[len(places) // 2]
        init = _p6(*poses[a]) + np.array([0.4, -0.3, 0.05, 0.0, 0.0, 0.03], np.float32)
        for off in (np.zeros(6, np.float32), np.array([60.0, -90.0, 35.0, 0, 0, 0.3], np.float32)):   # the second: 20-150 m away
            w = f"{what} off={off[:3]}"
            g, gi, gr, _, o, oi, orr, _ = _case(store, oracle, kfs[2 * a + 1], ids, p6, init + off, what=w, max_icp=1, max_outer=0)
            assert np.array_equal(gi, oi), (w, np.nonzero(gi != oi)[0][:5])
            assert np.array_equal(gr.view(np.uint64), orr.view(np.uint64)), w
            assert g["iterations"] == 1 and g["admm_iterations"] == 0 and np.array_equal(g["res_trans"], o["res_trans"]), w
            g, _, _, glog, o, _, _, olog = _case(store, oracle, _sub(kfs[2 * a + 1], 4), ids, p6, init + off, max_icp=1, max_outer=1)
            _compare(g, o, w, tol=1e-12)
            assert glog[0, 0] == olog[0, 0] == 1 and glog[0, 4] == olog[0, 4] == 12.0, w
            print(f"[sicp first step] {w}: {g['n_source']} -> {g['n_target']} points, "
                  f"|dt| {np.abs(g['res_trans'] - o['res_trans']).max():.2e}")


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
    src = _sub(kfs[2 * a + 1], 8)
    g, _, _, glog, o, _, _, olog = _case(store, oracle, src, ids, p6, init, max_icp=8)
    margin = _margin(olog)
    if margin > 1e-9:
        assert g["iterations"] == o["iterations"] and np.array_equal(glog[:, 0], olog[:, 0])
        assert g["admm_iterations"] == o["admm_iterations"]
        assert np.array_equal(glog[:, 4], olog[:, 4])
    _compare(g, o, what)
    print(f"[sicp] {what} far={far}: {g['iterations']} ICP / {g['admm_iterations']} ADMM iterations, stop {g['stop']:.3g}, "
          f"|dt| vs oracle {np.abs(g['res_trans'][:3, 3] - o['res_trans'][:3, 3]).max():.2e}, margin {margin:.3g}")


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
    g, gi, gr, _, o, oi, orr, _ = _case(kf, oracle, src, [0], one, shift, ext=None, max_icp=1, max_outer=0)
    assert np.array_equal(gi, oi) and np.array_equal(gr.view(np.uint64), orr.view(np.uint64))
    assert (gi[::53] == -1).all() and (gi[7::211] == -1).all()
    g, _, _, glog, o, _, _, olog = _case(kf, oracle, src, [0], one, shift, ext=None, max_icp=6)
    if _margin(olog) > 1e-9:
        assert np.array_equal(glog[:, 0], olog[:, 0])
    _compare(g, o, "nan + duplicates")
    for n in range(1, 9):
        k = kf.append(capi.pack_pointtype(base[100:100 + n, :3] * 3.0, base[100:100 + n, 3]))
        g, gi, _, glog, o, oi, _, olog = _case(kf, oracle, src[:2000], [k], one, ext=None, max_icp=5)
        assert np.array_equal(gi, oi)
        if _margin(olog) > 1e-9:
            assert np.array_equal(glog[:, 0], olog[:, 0])
        _compare(g, o, f"{n} target points")
    k = kf.append(capi.pack_pointtype(np.full((3, 3), np.nan, np.float32)))
    g = kf.sicp(src[:100], [k], one)
    assert g["status_name"] == "FEW_TARGET" and np.array_equal(g["res_trans"], np.eye(4))
    kf.close()
    tree.close()


def test_source_sizes_at_the_block_and_grid_boundaries(scene, oracle):
    kfs, _ = scene
    big = np.concatenate([kfs[2], kfs[3], kfs[6], kfs[8], kfs[9]])
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(kfs[0]) + 64, 4)
    kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
    one = np.zeros((1, 6), np.float32)
    shift = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.02], np.float32)
    resident = kf.sicp(big, [0], one, max_icp=1, max_outer=0)["admm_blocks"] * 256
    sizes = [1, 2, 255, 257, resident - 1, resident + 1, 2 * resident]
    assert len(big) >= max(sizes), (len(big), resident)
    for n in sizes:
        g, _, _, glog, o, _, _, olog = _case(kf, oracle, big[:n], [0], one, shift, ext=None, max_icp=2, max_outer=3)
        assert g["admm_blocks"] == min(resident // 256, (n + 255) // 256)
        assert np.array_equal(glog[:, 0], olog[:, 0]) or _margin(olog, max_outer=3) <= 1e-9
        _compare(g, o, f"n_source={n}", tol=1e-10)
    kf.close()
    tree.close()


def test_repeat_calls_syncs_scratch_and_rejected_configs(scene):
    kfs, _ = scene
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, len(kfs[0]) + 16, 4)
    kf.append(capi.pack_pointtype(kfs[0][:, :3], kfs[0][:, 3]))
    one = np.zeros((1, 6), np.float32)
    shift = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.02], np.float32)
    assert kf.info()["map_scratch_bytes"] == 0
    g = kf.sicp(kfs[1], [0], one, src_pose6=shift, max_icp=6, correspondences=True, log=True)
    r = g[0]
    assert r["syncs"] <= r["iterations"] + 6 and r["admm_iterations"] >= 10 * r["iterations"], r
    assert kf.info()["map_scratch_bytes"] >= 4 * 32 * len(kfs[1])
    g2 = kf.sicp(kfs[1], [0], one, src_pose6=shift, max_icp=6, correspondences=True, log=True)
    kf.release_scratch()
    assert kf.info()["map_scratch_bytes"] == 0
    g3 = kf.sicp(kfs[1], [0], one, src_pose6=shift, max_icp=6, correspondences=True, log=True)
    for other in (g2, g3):
        assert all(np.array_equal(np.asarray(r[k]), np.asarray(other[0][k])) for k in r)
        for a, b in zip(g[1:], other[1:]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    for kw, msg in ((dict(p=0.0), "p must be"), (dict(p=1.5), "p must be"), (dict(p=np.nan), "p must be"),
                    (dict(mu=0.0), "mu must be"), (dict(mu=np.inf), "mu must be"), (dict(max_mu=-1.0), "max_mu must be"),
                    (dict(max_mu=np.nan), "max_mu must be"), (dict(alpha=0.9), "alpha must be"), (dict(alpha=np.inf), "alpha must be"),
                    (dict(max_icp=-1), "max_icp"), (dict(max_outer=-1), "max_outer"), (dict(stop=np.nan), "stop"),
                    (dict(stop=-1e-6), "stop"), (dict(src_pose6=[0, 0, np.inf, 0, 0, 0]), "finite")):
        with pytest.raises(capi.FlbError, match=msg):
            kf.sicp(kfs[1], [0], one, **kw)
    with pytest.raises(capi.FlbError, match="regMode 7 is not supported"):
        kf.fricp(kfs[1], [0], one, mode=7)
    with pytest.raises(capi.FlbError, match="out of range"):
        kf.sicp(kfs[1], [3], one)
    g = kf.sicp(kfs[1][:0], [0], one)
    assert g["status_name"] == "NO_SOURCE" and g["iterations"] == 0
    kf.close()
    tree.close()


@pytest.mark.parametrize("shift_m,yaw_deg,required", [(0.5, 2.0, True), (1.5, 8.0, False)])
def test_recovery_of_a_displaced_scan_with_outliers(scene, store, shift_m, yaw_deg, required):
    kfs, poses = scene
    places = [0, 1, 2]
    ids = np.array([2 * k for k in places], np.int32)
    p6 = np.stack([_p6(*poses[k]) for k in places])
    world = np.concatenate([kfs[2 * k + 1][:, :3].astype(np.float64) @ poses[k][0].T + poses[k][1] for k in places])
    rng = np.random.default_rng(9)
    n_out = int(0.15 * len(world))
    lo, hi = world.min(0), world.max(0)
    outl = rng.uniform(lo, hi, size=(n_out, 3))   # stand-ins for dynamic objects
    R, t = rot((0.01, -0.01, np.deg2rad(yaw_deg))), np.array([1.2, -0.9, 0.05])
    t = t / np.linalg.norm(t) * shift_m
    pts = np.concatenate([world, outl])
    src = ((pts - t) @ R).astype(np.float32)      # D^-1 x: the registration should return D = (R, t)
    g = store.sicp(src, ids, p6)
    T = g["res_trans"]
    err = (np.abs(T[:3, 3] - t).max(), rot_err(T, R))
    print(f"[sicp recovery] {shift_m} m / {yaw_deg} deg: {g['iterations']} ICP / {g['admm_iterations']} ADMM iterations, "
          f"{g['syncs']} syncs, error {err[0] * 100:.2f} cm / {np.rad2deg(err[1]):.4f} deg")
    if required:
        assert err[0] < 0.02 and err[1] < np.deg2rad(0.1)
