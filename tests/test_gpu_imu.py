"""GPU tests of flb_imu_process: the forward propagation of UndistortPcl on the device against the IMU oracle
(tests/cpp/imu_oracle.cpp) and the front-end oracle's undistortion, the §3 quirks, sample counts, initialisation, a
closed loop through flb_scan_step, and the ImuProcessGpu facade.

Tolerances: prior state within 1e-12, P within 1e-12 max|P|, IMUpose within 1e-12 relative (device sincos may differ
from glibc in the last double ulp); undistorted points within 2 float ulp with >= 99.9 % bit-equal (the front-end bar);
closed loop 1e-4 m / 1e-4 rad per frame."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import imu_oracle as io
from tests.helpers import small_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_facade_smoke(out_dir):
    """g++ build of tests/cpp/imu_facade_smoke.cpp against the library (the header needs neither ROS nor Eigen)."""
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    libdir = os.path.dirname(capi.LIB_PATH)
    exe = os.path.join(out_dir, "imu_facade_smoke")
    cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "imu_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200", f"-Wl,-rpath,{libdir}",
           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def rel_close(a, b, rel=1e-12):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return a.shape == b.shape and (a.size == 0 or np.abs(a - b).max() <= rel * max(1.0, float(np.abs(b).max())))


def _ulp_close(a, b, ulps=2):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    tol = ulps * np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))
    return np.abs(a - b) <= tol


def state0():
    s = synth.trajectory_state(0)
    s[25] = -9.809
    return s


@pytest.fixture()
def rig():
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
    ses = capi.Session(tree, max_scan_points=1 << 17, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 17)
    yield tree, ses, fe
    fe.close()
    ses.close()
    tree.close()


def init_both(imu, o, rng, t0=-0.1):
    """One initialising scan (20 samples: init_iter_num 21 > MAX_INI_COUNT) on the device and on the oracle."""
    x, P = state0(), synth.default_cov()
    s = synth.imu_samples(t0, t0 + 0.1, 200.0, rng)
    xg, Pg, r = imu.process(s, t0, t0 + 0.1, x, P)
    so, xo, Po, _ = o.process(s, t0, t0 + 0.1, x, P)
    assert r.status == so == capi.IMU_INIT
    assert np.array_equal(xg, xo) and np.array_equal(Pg, Po)          # the init phase is bit-equal
    return xg, Pg


def compare_propagation(imu, o, samples, beg, end, x, P, leaf=0.0):
    xg, Pg, r = imu.process(samples, beg, end, x, P, leaf)
    so, xo, Po, po = o.process(samples, beg, end, x, P)
    assert r.status == so
    if so == capi.IMU_PROPAGATED:
        assert np.abs(xg - xo).max() <= 1e-12, np.abs(xg - xo).max()
        assert np.abs(Pg - Po).max() <= 1e-12 * np.abs(Po).max(), np.abs(Pg - Po).max()
        pg = imu.poses()
        assert r.n_poses == len(po) == len(pg) and r.n_predicts == r.n_poses
        assert rel_close(pg, po)
        gi, oi = imu.info(), o.info()
        assert rel_close(gi["angvel_last"], oi["angvel_last"]) and rel_close(gi["acc_s_last"], oi["acc_s_last"])
        assert gi["last_lidar_end_time"] == oi["last_lidar_end_time"] and np.array_equal(gi["last_imu"], oi["last_imu"])
    return xg, Pg, r, xo, Po, po


def test_one_scan_same_inputs_and_equivalence(rig, oracle):
    """Prior, P and IMUpose vs the oracle; the undistorted scan vs the front-end oracle fed with the oracle's IMUpose; and
    flb_imu_process == the oracle's IMUpose through the existing flb_frontend_undistort + flb_frontend_voxel_filter."""
    tree, ses, fe = rig
    sc = small_scene(seed=11, map_half=40.0, half_extent=100.0)
    rng = np.random.default_rng(5)
    xyz, inten, cur = synth.raw_scan_with_times(sc["body"], rng)
    pts48 = capi.pack_pointtype(xyz, inten, cur)
    imu = capi.Imu(fe)
    o = io.OracleImu()
    x, P = init_both(imu, o, rng)
    samples = synth.imu_samples(0.0, 0.1, 200.0, rng)
    fe.upload(pts48)
    xg, Pg, r, xo, Po, po = compare_propagation(imu, o, samples, 0.0, 0.1, x, P, leaf=0.5)
    assert r.n_poses == len(samples) + 1 and r.gpu_ms > 0
    g_und, g_cur, g_perm = fe.download_undistorted()
    o_xyz, o_perm = oracle.undistort(xyz, cur, po, xo)
    n = len(xyz)
    g_by_in = np.empty((n, 3), np.float32)
    o_by_in = np.empty((n, 3), np.float32)
    g_by_in[g_perm] = g_und[:, :3]
    o_by_in[o_perm] = o_xyz
    ok = _ulp_close(g_by_in, o_by_in)
    assert ok.all(), (~ok).sum()
    assert (g_by_in == o_by_in).mean() >= 0.999
    down, down_c = fe.download_down()
    assert len(down) == r.n_down == ses.n
    # equivalence: the same scan through the existing host-fed entry points with the oracle's IMUpose / end state
    fe.upload(pts48)
    fe.undistort(imu.poses(), xg)
    n3 = fe.voxel_filter(0.5)
    a_und, _, a_perm = fe.download_undistorted()
    a_down, a_c = fe.download_down()
    assert np.array_equal(a_perm, g_perm) and np.array_equal(a_und, g_und)
    assert n3 == r.n_down and np.array_equal(a_down, down) and np.array_equal(a_c, down_c)
    imu.close()


@pytest.mark.parametrize("n_imu", [1, 2, 21, 101, 255])
def test_sample_counts(rig, n_imu):
    tree, ses, fe = rig
    rng = np.random.default_rng(n_imu)
    imu = capi.Imu(fe)
    o = io.OracleImu()
    x, P = init_both(imu, o, rng)
    rate = max(n_imu / 0.1, 10.0)
    s = synth.imu_samples(0.0, 0.1, rate, rng)[:n_imu]
    assert len(s) == n_imu
    fe.upload(capi.pack_pointtype(rng.uniform(-20, 20, (3000, 3)).astype(np.float32), None,
                                  rng.uniform(0, 100, 3000).astype(np.float32)))
    compare_propagation(imu, o, s, 0.0, 0.1, x, P)
    imu.close()


def test_256_samples_rejected_state_untouched(rig):
    tree, ses, fe = rig
    rng = np.random.default_rng(2)
    imu = capi.Imu(fe)
    o = io.OracleImu()
    x, P = init_both(imu, o, rng)
    before = imu.info()
    s = synth.imu_samples(0.0, 0.1, 2560.0, rng)[:256]
    with pytest.raises(capi.FlbError, match="n_imu"):
        imu.process(s, 0.0, 0.1, x, P)
    bad = synth.imu_samples(0.0, 0.1, 200.0, rng)
    bad[3, 2] = np.nan
    with pytest.raises(capi.FlbError, match="non-finite"):
        imu.process(bad, 0.0, 0.1, x, P)
    with pytest.raises(capi.FlbError, match="lidar time"):
        imu.process(bad[:2] * 0 + 1, 0.0, np.inf, x, P)
    after = imu.info()
    for k, v in before.items():
        assert np.array_equal(np.asarray(v), np.asarray(after[k])), k
    # still usable, and still in step with the oracle
    compare_propagation(imu, o, synth.imu_samples(0.0, 0.1, 200.0, rng), 0.0, 0.1, x, P)
    imu.close()


def test_quirks_on_device(rig):
    """Skipped segments, dt from last_lidar_end_time_, the zero `in` of an all-skipped span, the forward final predict
    when the IMU ends after the scan, Q = process_noise_cov() until a segment ran, IMUpose[0] with the previous
    acc_s_last / angvel_last, last_lidar_end_time_ / acc_s_last starting at 0, accelerations in g, and Reset."""
    tree, ses, fe = rig
    rng = np.random.default_rng(7)
    cfg = dict(cov_gyr_scale=(0.2,) * 3, cov_acc_scale=(0.3,) * 3, cov_bias_gyr=(2e-4,) * 3, cov_bias_acc=(3e-4,) * 3)
    imu = capi.Imu(fe, **cfg)
    o = io.OracleImu(io.config_vector(gyr=(0.2,) * 3, acc=(0.3,) * 3, bias_gyr=(2e-4,) * 3, bias_acc=(3e-4,) * 3))
    info0 = imu.info()
    assert info0["last_lidar_end_time"] == 0 and np.array_equal(info0["acc_s_last"], np.zeros(3))
    x, P = init_both(imu, o, rng)
    assert np.array_equal(imu.info()["cov_acc"], [0.3] * 3) and np.array_equal(imu.info()["cov_gyr"], [0.2] * 3)
    # every sample older than last_lidar_end_time_ (0): all skipped, in = 0, Q = process_noise_cov()
    old = synth.imu_samples(-0.05, -0.01, 200.0, rng)
    x, P, r, *_ = compare_propagation(imu, o, old, 0.0, 0.1, x, P)
    assert r.n_poses == 1
    pose0 = imu.poses()[0]
    assert pose0[0] == 0.0 and np.array_equal(pose0[1:7], np.zeros(6))
    # head before last_lidar_end_time_ (0.1): dt = tail - 0.1; the IMU ends after the scan end 0.2
    late = synth.imu_samples(0.06, 0.23, 200.0, rng)
    x, P, r, *_ = compare_propagation(imu, o, late, 0.1, 0.2, x, P)
    assert 1 < r.n_poses < len(late) + 1
    # accelerations in g units after a Reset (re-initialisation without the first-frame branch)
    imu.reset()
    o.reset()
    assert imu.info()["b_first_frame"] == 0 and imu.info()["imu_need_init"] == 1 and imu.info()["n_poses"] == 0
    t = 0.3
    for k in range(2):
        s = synth.imu_samples(t, t + 0.1, 200.0, rng, g_units=True)
        x, P, r, xo, Po, _ = compare_propagation(imu, o, s, t, t + 0.1, x, P)
        if r.status == capi.IMU_INIT:
            assert np.array_equal(x, xo) and np.array_equal(P, Po)
        t += 0.1
    assert r.status == capi.IMU_PROPAGATED
    assert np.abs(x[14:17]).max() < 50
    imu.close()


def test_init_phase_bit_equal(rig):
    tree, ses, fe = rig
    rng = np.random.default_rng(12)
    imu = capi.Imu(fe, Lidar_T_wrt_IMU=(0.1, 0.0, -0.05),
                   Lidar_R_wrt_IMU=synth.quat_to_mat(synth.quat_from_rotvec([0.0, 0.1, 3.0])).ravel())
    o = io.OracleImu(io.config_vector(T=(0.1, 0.0, -0.05), R=synth.quat_to_mat(synth.quat_from_rotvec([0.0, 0.1, 3.0]))))
    x, P = state0(), synth.default_cov()
    t = 0.0
    for m in (4, 5, 1, 3):   # init_iter_num 5, 10 (still initialising), 11 (done), then a propagation
        s = synth.imu_samples(t, t + m * 0.005, 200.0, rng)
        t += m * 0.005
        xg, Pg, r = imu.process(s, t - 0.1, t, x, P)
        so, xo, Po, _ = o.process(s, t - 0.1, t, x, P)
        assert r.status == so
        gi, oi = imu.info(), o.info()
        assert gi["init_iter_num"] == oi["init_iter_num"] and gi["imu_need_init"] == oi["imu_need_init"]
        if so == capi.IMU_INIT:
            assert np.array_equal(xg, xo) and np.array_equal(Pg, Po)
            for k in ("mean_acc", "mean_gyr", "cov_acc", "cov_gyr"):
                assert np.array_equal(gi[k], oi[k]), k
        else:
            assert np.abs(xg - xo).max() <= 1e-12
        x, P = xg, Pg
    assert [imu.info()["init_iter_num"]] == [11]
    imu.close()


def test_closed_loop_driver_records(oracle):
    """100 scans: driver records + IMU -> flb_frontend_preprocess -> flb_imu_process -> flb_scan_step with the device
    posterior fed back, against the oracle chain (IMU oracle -> ESIKF update -> map_incremental on its own map) replaying
    every step from that same posterior, its map grown with it, so each frame is a comparison on identical inputs
    (DESIGN.md §6a: two free-running replays part at the first discrete event of the update — a converge test or a k-NN
    tie — whatever their priors).  The propagated priors must agree to 1e-12 on every frame.  The
    oracle update measures the device's feats_down_body: the undistortion and voxel filter have their own parity bar
    (test_one_scan_same_inputs_and_equivalence; a float summed in another order inside a leaf moves a closed loop by
    more than the pose bar), and the front-end oracle's undistortion of the same raw scan must filter to the same
    point count within 2."""
    seed = 4
    rng = np.random.default_rng(seed)
    world = synth.city_world(half_extent=150, seed=seed)
    ds, leaf = 0.2, 0.5
    tree = capi.KDTree(voxel_size=ds, max_points=1 << 21, max_blocks=1 << 18)
    ses = capi.Session(tree, max_scan_points=1 << 16, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 16)
    imu = capi.Imu(fe)
    try:
        _closed_loop(oracle, rng, world, ds, leaf, tree, ses, fe, imu)
    finally:   # the processor before its front end, the front end before its session
        imu.close()
        fe.close()
        ses.close()
        tree.close()


def _closed_loop(oracle, rng, world, ds, leaf, tree, ses, fe, imu):
    o = io.OracleImu()
    ref = oracle.make_map(ds=ds)
    cfg = capi.preprocess_config(capi.VELO16, n_scans=16, time_unit=capi.SEC, blind=2.0)
    speed = 2.0   # slow: every sweep is cast from one pose, so the undistortion's motion model is off by <= 0.2 m
    pos0, R0, _, _ = synth.imu_trajectory(0.0, speed=speed)
    st_true0 = synth.make_state(pos=pos0, rot=synth.trajectory_state(0)[3:7], offT=(0, 0, 0), vel=(speed, 0.3, 0))
    body0 = synth.voxel_downsample(synth.scan_from_pose(world, st_true0, synth.lidar_dirs("vlp16"), rng, max_range=60.0), ds)
    w0 = synth.body_to_world_np(st_true0, body0)
    tree.Build(w0)
    ref.Build(w0)
    x_g = x_c = st_true0.copy()
    P_g = P_c = synth.default_cov()
    irng = np.random.default_rng(99)
    log = []
    for k in range(102):
        beg, end = 0.1 * k, 0.1 * k + 0.1
        # a well-observed drive: no biases, small noise (the filter then stays close to the truth, where the
        # registration is well conditioned and two replays do not drift apart)
        samples = synth.imu_samples(beg, end, 200.0, irng, gyro_bias=(0, 0, 0), acc_bias=(0, 0, 0), gyro_noise=1e-4, acc_noise=1e-3,
                                    speed=speed)
        pos, R, _, _ = synth.imu_trajectory(end, speed=speed)   # the pose the undistortion compensates to
        st_true = synth.make_state(pos=pos, rot=synth.quat_from_rotvec([0, 0, np.arctan2(R[1, 0], R[0, 0])]), offT=(0, 0, 0))
        rec = synth.driver_records("vlp16", world, st_true, rng, max_range=60.0)
        fe.preprocess(rec, cfg)
        raw4, raw_c, _ = fe.download_undistorted()          # the raw scan in upload order (not undistorted yet)
        xg, Pg, r = imu.process(samples, beg, end, x_g, P_g, leaf)
        so, xo, Po, po = o.process(samples, beg, end, x_c, P_c)
        assert r.status == so
        if r.status != capi.IMU_PROPAGATED:
            x_g, P_g, x_c, P_c = xg, Pg, xo, Po
            continue
        dprior = float(np.abs(xg - xo).max())
        s_g, P_g, res = ses.scan_step(None, None, xg, Pg)
        o_xyz, o_perm = oracle.undistort(raw4[:, :3], raw_c, po, xo)
        o_ds, _, _ = oracle.voxel_grid(np.column_stack([o_xyz, raw4[o_perm, 3]]), leaf, order="stable")
        down, _ = fe.download_down()
        s_c, P_c, scr, _, _ = oracle.esikf_update(xo, Po, down[:, :3], ref, max_iter=3)
        oracle.map_incremental(s_g, down[:, :3], scr, ref, True, ds)   # both maps grow from the same posterior
        log.append((k, dprior, float(np.abs(s_g[:3] - s_c[:3]).max()), float(np.abs(s_g[3:7] - s_c[3:7]).max()),
                    len(o_ds) - r.n_down, res.update.effct_feat_num, float(np.abs(s_g[:3] - st_true[:3]).max())))
        x_g, x_c, P_c = s_g, s_g.copy(), P_g.copy()
    print("imu closed loop (k, |d prior|, |d pos|, |d quat|, d n_down, M, |pos - truth|):")
    for row in log:
        print(row)
    assert len(log) >= 100
    assert all(abs(row[4]) <= 2 for row in log)
    assert max(row[1] for row in log) <= 1e-12                     # the propagated priors
    assert max(row[2] for row in log) <= 1e-4 and 2 * max(row[3] for row in log) <= 1e-4


@pytest.mark.gpu
def test_facade_runs_on_gpu():
    with tempfile.TemporaryDirectory() as d:
        exe = build_facade_smoke(d)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
        assert "IMU_FACADE_OK" in out.stdout


pytestmark = pytest.mark.gpu
