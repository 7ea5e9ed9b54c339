"""CPU tests of the IMU propagation oracle (tests/cpp/imu_oracle.cpp) against an independent float64 numpy transcription
of ImuProcess (IMU_Processing.hpp:90-434) and esekf::predict (esekfom.hpp:280-384), the quirks the device kernel keeps,
the C ABI's argument checks without a GPU, and the compile of the ImuProcessGpu facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from better_fastlio2_b200 import synth
from tests import imu_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = 9.81
LEN = 98090.0 / 10000.0


# ------------------------------------------------------------------------------------------------ numpy transcription
def hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def qexp(v, scale):
    x2 = scale * scale * float(v @ v)
    if x2 >= 1.220703125e-4:
        x = np.sqrt(x2)
        c, s = np.cos(x), np.sin(x) / x
    else:   # Taylor branch of cos_sinc_sqrt
        c = 1 - x2 / 2 + x2 * x2 / 24 - x2 ** 3 / 720
        s = 1 - x2 / 6 + x2 * x2 / 120 - x2 ** 3 / 5040
    return np.r_[s * scale * v, c]


def qmul(a, b):
    return synth.quat_mul(a, b)


def A_matrix(v):
    n = np.linalg.norm(v)
    if n < 1e-11:
        return np.eye(3)
    H = hat(v)
    return np.eye(3) + (1 - np.cos(n)) / n ** 2 * H + (1 - np.sin(n) / n) / n ** 2 * H @ H


def Bx(v):
    L = LEN
    return np.array([[-v[1], -v[2]], [L - v[1] ** 2 / (L + v[0]), -v[2] * v[1] / (L + v[0])],
                     [-v[2] * v[1] / (L + v[0]), L - v[2] ** 2 / (L + v[0])]]) / L


def np_predict(x, P, qd, acc, gyr, dt):
    x = x.copy()
    R = synth.quat_to_mat(x[3:7])
    om = gyr - x[17:20]
    a_ = acc - x[20:23]
    fvel = R @ a_ + x[23:26]
    A = A_matrix(-om * dt)
    g = x[23:26]
    Mx = -hat(g) @ Bx(g)
    Nx = Bx(g).T @ hat(g) / LEN ** 2
    F = np.eye(23)
    F[0:3, 12:15] = np.eye(3) * dt
    F[3:6, 15:18] = -A * dt
    F[12:15, 3:6] = -R @ hat(a_) * dt
    F[12:15, 18:21] = -R * dt
    F[12:15, 21:23] = Mx * dt
    F[21:23, 21:23] = Nx @ Mx
    Gm = np.zeros((23, 12))
    Gm[3:6, 0:3] = -A
    Gm[12:15, 3:6] = -R
    Gm[15:18, 6:9] = np.eye(3)
    Gm[18:21, 9:12] = np.eye(3)
    P = F @ P @ F.T + (dt * Gm) @ np.diag(qd) @ (dt * Gm).T
    x[0:3] += dt * x[14:17]
    x[3:7] = qmul(x[3:7], qexp(om, dt / 2))
    x[14:17] += dt * fvel
    return x, P


class NpImu:
    """ImuProcess's members and Process restated in numpy."""

    def __init__(self, T=np.zeros(3), R=np.eye(3), gyr=(0.1,) * 3, acc=(0.1,) * 3, bg=(1e-4,) * 3, ba=(1e-4,) * 3):
        self.T, self.R = np.asarray(T, float), np.asarray(R, float)
        self.gyr_s, self.acc_s, self.bg, self.ba = [np.asarray(v, float) for v in (gyr, acc, bg, ba)]
        self.cov_acc, self.cov_gyr = np.full(3, 0.1), np.full(3, 0.1)
        self.Qd = np.r_[[1e-4] * 6, [1e-5] * 6]
        self.first = True
        self.acc_s_last = np.zeros(3)
        self.last_end = 0.0
        self.reset()

    def reset(self):
        self.mean_acc, self.mean_gyr, self.angvel_last = np.array([0, 0, -1.0]), np.zeros(3), np.zeros(3)
        self.need_init, self.N, self.last_imu = True, 1, np.zeros(7)

    def process(self, imu, beg, end, x, P):
        x, P = x.copy(), P.copy()
        if len(imu) == 0:
            return 0, x, P, None
        if self.need_init:
            if self.first:
                self.reset()
                self.N, self.first = 1, False
                self.mean_acc, self.mean_gyr = imu[0, 1:4].copy(), imu[0, 4:7].copy()
            for r in imu:
                N = self.N
                self.mean_acc = self.mean_acc + (r[1:4] - self.mean_acc) / N
                self.mean_gyr = self.mean_gyr + (r[4:7] - self.mean_gyr) / N
                self.cov_acc = self.cov_acc * (N - 1) / N + (r[1:4] - self.mean_acc) ** 2 * (N - 1) / N ** 2
                self.cov_gyr = self.cov_gyr * (N - 1) / N + (r[4:7] - self.mean_gyr) ** 2 * (N - 1) / N ** 2
                self.N += 1
            g = -self.mean_acc / np.linalg.norm(self.mean_acc) * G
            x[23:26] = g / np.linalg.norm(g) * LEN
            x[17:20], x[11:14] = self.mean_gyr, self.T
            from scipy.spatial.transform import Rotation
            q = Rotation.from_matrix(self.R).as_quat()
            x[7:11] = q if q[3] >= 0 else -q
            P = np.diag([1.0] * 6 + [1e-5] * 6 + [1.0] * 3 + [1e-4] * 3 + [1e-3] * 3 + [1e-5] * 2)
            self.last_imu = imu[-1].copy()
            if self.N > 10:
                self.need_init = False
                self.cov_acc, self.cov_gyr = self.acc_s.copy(), self.gyr_s.copy()
            return 1, x, P, None
        v = np.vstack([self.last_imu, imu])
        poses = [np.r_[0.0, self.acc_s_last, self.angvel_last, x[14:17], x[0:3], synth.quat_to_mat(x[3:7]).ravel()]]
        ia, ig = np.zeros(3), np.zeros(3)
        L = self.last_end
        for h, t in zip(v[:-1], v[1:]):
            if t[0] < L:
                continue
            ig = 0.5 * (h[4:7] + t[4:7])
            ia = 0.5 * (h[1:4] + t[1:4]) * G / np.linalg.norm(self.mean_acc)
            dt = t[0] - L if h[0] < L else t[0] - h[0]
            self.Qd = np.r_[self.cov_gyr, self.cov_acc, self.bg, self.ba]
            x, P = np_predict(x, P, self.Qd, ia, ig, dt)
            self.angvel_last = ig - x[17:20]
            self.acc_s_last = synth.quat_to_mat(x[3:7]) @ (ia - x[20:23]) + x[23:26]
            poses.append(np.r_[t[0] - beg, self.acc_s_last, self.angvel_last, x[14:17], x[0:3], synth.quat_to_mat(x[3:7]).ravel()])
        imu_end = v[-1, 0]
        dt = (1.0 if end > imu_end else -1.0) * (end - imu_end)
        x, P = np_predict(x, P, self.Qd, ia, ig, dt)
        self.last_imu, self.last_end = imu[-1].copy(), end
        return 2, x, P, np.array(poses)


# ------------------------------------------------------------------------------------------------ helpers
def close(a, b, rel=1e-12):
    a, b = np.asarray(a, float), np.asarray(b, float)
    scale = max(1.0, float(np.abs(b).max()) if b.size else 1.0)
    return np.abs(a - b).max() <= rel * scale if a.size else True


def state0():
    s = synth.make_state(pos=(1.0, 2.0, 0.5), rot=synth.quat_from_rotvec([0.01, -0.02, 0.3]), offT=(0, 0, 0), vel=(0.5, 0.1, 0))
    s[17:26] = 0.0
    s[25] = -LEN
    return s


def stream(n_scans, rate=200.0, seed=0, g_units=False, t0=0.0):
    rng = np.random.default_rng(seed)
    return [(synth.imu_samples(t0 + 0.1 * k, t0 + 0.1 * k + 0.1, rate, rng, g_units=g_units), t0 + 0.1 * k, t0 + 0.1 * k + 0.1)
            for k in range(n_scans)]


def run_both(scans, cfg_np=None, cfg_orc=None, x=None, P=None):
    o, n = io.OracleImu(cfg_orc), NpImu(**(cfg_np or {}))
    xo = xn = state0() if x is None else x
    Po = Pn = synth.default_cov() if P is None else P
    out = []
    for imu, beg, end in scans:
        so, xo, Po, po = o.process(imu, beg, end, xo, Po)
        sn, xn, Pn, pn = n.process(imu, beg, end, xn, Pn)
        assert so == sn
        assert close(xo, xn), np.abs(xo - xn).max()
        assert close(Po, Pn), np.abs(Po - Pn).max()
        if so == 2:
            assert len(po) == len(pn) and close(po, pn)
        out.append((so, xo, Po, po))
    return o, n, out


# ------------------------------------------------------------------------------------------------ tests
def test_predict_matches_numpy():
    rng = np.random.default_rng(1)
    for _ in range(20):
        x = state0()
        x[17:23] = rng.normal(0, 0.01, 6)
        g = rng.normal(0, 1, 3)
        x[23:26] = g / np.linalg.norm(g) * LEN
        A = rng.normal(0, 0.1, (23, 23))
        P = A @ A.T + np.eye(23) * 0.01
        qd = rng.uniform(1e-5, 0.2, 12)
        acc, gyr, dt = rng.normal(0, 3, 3), rng.normal(0, 0.5, 3), rng.uniform(0.0005, 0.02)
        xo, Po = io.predict(x, P, qd, acc, gyr, dt)
        xn, Pn = np_predict(x, P, qd, acc, gyr, dt)
        assert close(xo, xn) and close(Po, Pn), (np.abs(xo - xn).max(), np.abs(Po - Pn).max())
        assert np.abs(Po - Po.T).max() <= 1e-15 * np.abs(Po).max() * 23   # symmetric to rounding
        assert np.array_equal(xo[23:26], x[23:26]) and np.array_equal(xo[7:11], x[7:11])   # grav / offR: identity oplus


def test_predict_quirk_scalar_half_is_zero():
    """F's SO3 blocks are the identity (exp with scale 1/2 == 0) and the S2 block is Nx * I * Mx: the result does not
    depend on the rotation angle of seg_SO3 through F_x1 — checked by reconstructing F from P = F P F^T with Q = 0."""
    x = state0()
    P = np.diag(np.arange(1.0, 24.0))
    acc, gyr, dt = np.array([0.3, -0.2, 9.7]), np.array([0.5, -0.4, 1.2]), 0.05
    xo, Po = io.predict(x, P, np.zeros(12), acc, gyr, dt)
    # the rotation rows of F are e_r - dt A(seg) on 15-17 (no exp(seg) block on 3-5), so with a diagonal P the block is
    # P[3:6, 3:6] + dt^2 A P[15:18, 15:18] A^T; a rotation block would mix the distinct diagonal entries 4, 5, 6
    A = A_matrix(-(gyr - x[17:20]) * dt)
    assert close(Po[3:6, 3:6], P[3:6, 3:6] + dt * dt * A @ P[15:18, 15:18] @ A.T)
    g = x[23:26]
    NM = (Bx(g).T @ hat(g) / LEN ** 2) @ (-hat(g) @ Bx(g))
    assert close(Po[21:23, 21:23], NM @ P[21:23, 21:23] @ NM.T)


@pytest.mark.parametrize("rate,g_units", [(200.0, False), (1000.0, False), (200.0, True)])
def test_process_stream_matches_numpy(rate, g_units):
    scans = stream(16, rate=rate, seed=3, g_units=g_units)
    o, n, out = run_both(scans)
    st = [s for s, *_ in out]
    assert st[0] == 1 and 2 in st
    x, P = out[-1][1], out[-1][2]
    assert np.abs(P - P.T).max() <= 1e-14 * np.abs(P).max()
    # the gravity estimate points down with the S2 length 9.809, not 9.81
    assert abs(np.linalg.norm(x[23:26]) - LEN) < 1e-12 and x[25] < -9.7
    if g_units:   # accelerations in g: acc_avr * G_m_s2 / |mean_acc| rescales them to m/s^2
        assert abs(np.linalg.norm(o.info()["mean_acc"]) - 1.0) < 0.01


def test_init_boundary_and_dead_cov_scale():
    """init_iter_num crosses MAX_INI_COUNT = 10: still initialising at 10, done at 11; after init cov_acc / cov_gyr are
    the configured scales (the *= pow(...) line before them is dead)."""
    rng = np.random.default_rng(5)
    o = io.OracleImu(io.config_vector(gyr=(0.3, 0.2, 0.1), acc=(0.5, 0.6, 0.7)))
    n = NpImu(gyr=(0.3, 0.2, 0.1), acc=(0.5, 0.6, 0.7))
    x, P = state0(), synth.default_cov()
    sizes = [4, 5, 1, 3]   # samples per scan: N = 5, 10, 11 -> done
    t = 0.0
    seen = []
    for k, m in enumerate(sizes):
        imu = synth.imu_samples(t, t + m * 0.005, 200.0, rng)
        t += m * 0.005
        so, xo, Po, _ = o.process(imu, t - 0.1, t, x, P)
        sn, xn, Pn, _ = n.process(imu, t - 0.1, t, x, P)
        assert so == sn and close(xo, xn) and close(Po, Pn)
        info = o.info()
        seen.append((so, info["init_iter_num"], info["imu_need_init"]))
        assert np.array_equal(info["mean_acc"], n.mean_acc) or close(info["mean_acc"], n.mean_acc)
    assert seen[0] == (1, 5, 1) and seen[1] == (1, 10, 1) and seen[2] == (1, 11, 0)
    assert seen[3][0] == 2
    assert np.array_equal(o.info()["cov_acc"], [0.5, 0.6, 0.7]) and np.array_equal(o.info()["cov_gyr"], [0.3, 0.2, 0.1])


def test_init_state_and_gravity_length():
    rng = np.random.default_rng(2)
    R = synth.quat_to_mat(synth.quat_from_rotvec([0.1, -0.2, 2.9]))   # trace < 0 branch of the matrix -> quaternion
    cfg = dict(T=(0.1, -0.2, 0.3), R=R)
    o = io.OracleImu(io.config_vector(**cfg))
    imu = synth.imu_samples(0.0, 0.1, 200.0, rng)
    st, x, P, _ = o.process(imu, 0.0, 0.1, state0(), synth.default_cov())
    assert st == 1
    assert np.array_equal(x[11:14], [0.1, -0.2, 0.3])
    assert np.abs(synth.quat_to_mat(x[7:11]) - R).max() < 1e-14
    assert abs(np.linalg.norm(x[23:26]) - 9.809) < 1e-12
    assert np.array_equal(x[17:20], o.info()["mean_gyr"])
    assert np.array_equal(np.diag(P), [1.0] * 6 + [1e-5] * 6 + [1.0] * 3 + [1e-4] * 3 + [1e-3] * 3 + [1e-5] * 2)
    assert np.count_nonzero(P - np.diag(np.diag(P))) == 0


def _past_init(o, n=None, seed=9):
    rng = np.random.default_rng(seed)
    x, P = state0(), synth.default_cov()
    imu = synth.imu_samples(-0.1, 0.0, 200.0, rng)
    for obj in (o, n):
        if obj is not None:
            st, x1, P1, _ = obj.process(imu, -0.1, 0.0, x, P)
            assert st == 1
    return x1, P1


def test_skipped_segments_and_zero_input_final_predict():
    """Segments with tail < last_lidar_end_time_ are skipped; the final predict reuses the last `in`, the default (zero)
    input_ikfom when every segment was skipped, with dt = |pcl_end - imu_end| (forward even if the IMU ends later)."""
    o, n = io.OracleImu(), NpImu()
    x, P = _past_init(o, n)
    rng = np.random.default_rng(4)
    # first propagation: last_lidar_end_time_ = 0 (deviation: uninitialised in the reference) — no skip
    imu = synth.imu_samples(0.0, 0.1, 200.0, rng)
    so, xo, Po, po = o.process(imu, 0.0, 0.1, x, P)
    sn, xn, Pn, pn = n.process(imu, 0.0, 0.1, x, P)
    assert so == sn == 2 and close(xo, xn) and close(Po, Pn) and close(po, pn)
    # IMUpose[0] carries the previous acc_s_last / angvel_last at offset 0
    assert po[0, 0] == 0.0 and np.array_equal(po[0, 1:7], np.zeros(6))
    # every sample of the next span is older than the last scan end: all segments skipped, in = 0
    old = synth.imu_samples(0.02, 0.06, 200.0, rng)
    so, x2, P2, p2 = o.process(old, 0.1, 0.2, xo, Po)
    sn, y2, Q2, q2 = n.process(old, 0.1, 0.2, xn, Pn)
    assert so == 2 and len(p2) == 1 and close(x2, y2) and close(P2, Q2)
    xz, Pz = io.predict(xo, Po, o.info()["Qd"], np.zeros(3), np.zeros(3), 0.2 - old[-1, 0])
    assert close(x2, xz) and close(P2, Pz)
    # the IMU ends after the scan: dt = -(pcl_end - imu_end) > 0, propagation still forward
    late = synth.imu_samples(0.2, 0.33, 200.0, rng)
    so, x3, P3, p3 = o.process(late, 0.2, 0.3, x2, P2)
    sn, y3, Q3, q3 = n.process(late, 0.2, 0.3, y2, Q2)
    assert so == 2 and close(x3, y3) and close(P3, Q3) and close(p3, q3)
    # head before last_lidar_end_time_: dt = tail - last_lidar_end_time_ (covered by the numpy restatement above)
    assert p3[1, 0] == late[0, 0] - 0.2


def test_q_starts_from_process_noise_cov():
    """Q is process_noise_cov() until a segment overwrites its diagonal blocks with cov_gyr / cov_acc / cov_bias_*."""
    o = io.OracleImu(io.config_vector(gyr=(0.2,) * 3, acc=(0.3,) * 3, bias_gyr=(2e-4,) * 3, bias_acc=(3e-4,) * 3))
    x, P = _past_init(o)
    assert np.array_equal(o.info()["Qd"], [1e-4] * 6 + [1e-5] * 6)
    # a span whose samples are all older than last_lidar_end_time_ (0 here: negative stamps): Q untouched
    rng = np.random.default_rng(1)
    old = synth.imu_samples(-0.05, -0.01, 200.0, rng)
    st, x1, P1, p1 = o.process(old, 0.0, 0.1, x, P)
    assert st == 2 and len(p1) == 1
    xz, Pz = io.predict(x, P, [1e-4] * 6 + [1e-5] * 6, np.zeros(3), np.zeros(3), 0.1 - old[-1, 0])
    assert close(x1, xz) and close(P1, Pz)
    imu = synth.imu_samples(0.1, 0.2, 200.0, rng)
    o.process(imu, 0.1, 0.2, x1, P1)
    assert np.array_equal(o.info()["Qd"], [0.2] * 3 + [0.3] * 3 + [2e-4] * 3 + [3e-4] * 3)


def test_reset_keeps_first_frame_flag():
    o, n = io.OracleImu(), NpImu()
    x, P = _past_init(o, n)
    rng = np.random.default_rng(8)
    imu = synth.imu_samples(0.0, 0.1, 200.0, rng)
    o.process(imu, 0.0, 0.1, x, P)
    n.process(imu, 0.0, 0.1, x, P)
    o.reset()
    n.reset()
    info = o.info()
    assert info["imu_need_init"] == 1 and info["init_iter_num"] == 1 and info["b_first_frame"] == 0
    assert np.array_equal(info["mean_acc"], [0, 0, -1]) and info["n_poses"] == 0
    # re-initialisation without the first-frame branch: mean starts from (0, 0, -1), N from 1
    imu2 = synth.imu_samples(0.1, 0.2, 200.0, rng)
    so, xo, Po, _ = o.process(imu2, 0.1, 0.2, x, P)
    sn, xn, Pn, _ = n.process(imu2, 0.1, 0.2, x, P)
    assert so == sn == 1 and close(xo, xn) and close(o.info()["mean_acc"], n.mean_acc)


def test_empty_span_does_nothing():
    o = io.OracleImu()
    s0 = o.s.copy()
    st, x, P, _ = o.process(np.zeros((0, 7)), 0.0, 0.1, state0(), synth.default_cov())
    assert st == 0 and np.array_equal(o.s, s0) and np.array_equal(x, state0())


# ------------------------------------------------------------------------------------------------ C ABI without a GPU
@pytest.fixture(scope="module")
def lib():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def test_abi_argument_errors(lib):
    from better_fastlio2_b200 import capi
    c = capi.imu_config()
    assert list(c.cov_gyr_scale) == [0.1] * 3 and list(c.cov_bias_acc) == [1e-4] * 3 and list(c.Lidar_R_wrt_IMU)[::4] == [1.0] * 3
    h = ctypes.c_void_p()
    assert lib.flb_imu_create(None, ctypes.byref(c), ctypes.byref(h)) != 0 and not h.value
    assert b"null argument" in lib.flb_last_error()
    for field, idx, val, msg in [("cov_acc_scale", 1, float("nan"), b"cov_acc_scale[1] is not finite"),
                                 ("cov_bias_gyr", 0, -1.0, b"cov_bias_gyr[0] is negative"),
                                 ("Lidar_T_wrt_IMU", 2, float("inf"), b"Lidar_T_wrt_IMU[2] is not finite"),
                                 ("Lidar_R_wrt_IMU", 0, 2.0, b"Lidar_R_wrt_IMU is not a rotation")]:
        bad = capi.imu_config()
        getattr(bad, field)[idx] = val
        fake_fe = ctypes.c_void_p(1)   # never dereferenced: the configuration is checked first
        assert lib.flb_imu_create(fake_fe, ctypes.byref(bad), ctypes.byref(h)) != 0
        assert msg in lib.flb_last_error(), lib.flb_last_error()
    x = np.zeros(26)
    P = np.zeros((23, 23))
    r = capi.ImuResult()
    assert lib.flb_imu_process(None, None, 0, 0.0, 0.1, x.ctypes.data, P.ctypes.data, 0.0, ctypes.byref(r)) != 0
    assert b"null IMU processor" in lib.flb_last_error()
    assert lib.flb_imu_reset(None) != 0 and lib.flb_imu_info(None, None) != 0
    lib.flb_imu_destroy(None)


def test_facade_compiles():
    from tests.test_gpu_imu import build_facade_smoke
    with tempfile.TemporaryDirectory() as d:
        exe = build_facade_smoke(d)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, (out.stdout, out.stderr)
        assert "NO_GPU compile-only ok" in out.stdout or "IMU_FACADE_OK" in out.stdout
