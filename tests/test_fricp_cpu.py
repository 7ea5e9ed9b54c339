"""CPU tests of the relocalisation registration oracle (tests/cpp/fricp_oracle.cpp): its closed-form SE(3) log / exp against
scipy's matrix functions, its Anderson acceleration against a numpy transcription of AndersonAcceleration.h with a
least-squares min-norm solve, igl::median semantics, and whole small registrations in modes 0, 2, 3 and 4 against a
numpy / scipy (cKDTree) transcription of FRICP<3>::point_to_point.  Also compiles the facade smoke."""
import os
import subprocess

import numpy as np
import pytest
from scipy.linalg import expm, logm
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from tests import fricp_oracle as fo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _se3(rotvec, t):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rotvec).as_matrix()
    T[:3, 3] = t
    return T


@pytest.mark.parametrize("theta", [0.0, 1e-9, 1e-6, 3e-5, 0.3, 2.0, np.pi - 1e-3, np.pi - 1e-6, np.pi - 1e-9])
def test_log_exp_match_scipy(theta):
    rng = np.random.default_rng(int(theta * 1e6) % 1000 + 1)
    for _ in range(5):
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        T = _se3(theta * ax, rng.normal(size=3))
        L = fo.se3_log(T)
        assert np.allclose(L[3], 0) and np.allclose(L[:3, :3], -L[:3, :3].T, atol=0)
        assert np.abs(fo.se3_exp(L) - T).max() < 1e-9
        assert np.abs(expm(L) - T).max() < 1e-9
        if theta < np.pi - 1e-4:   # the principal log is unique away from pi
            assert np.abs(np.real(logm(T)) - L).max() < 1e-7
        else:                      # at pi the axis' sign is a choice: exp must still give T
            assert abs(np.linalg.norm([L[2, 1], L[0, 2], L[1, 0]]) - theta) < 1e-6
    L = np.zeros((4, 4))
    L[:3, :3] = [[0, -0.2, 0.1], [0.2, 0, -0.3], [-0.1, 0.3, 0]]
    L[:3, 3] = [0.5, -1.0, 2.0]
    assert np.abs(fo.se3_exp(L) - expm(L)).max() < 1e-12


class NpAnderson:
    """AndersonAcceleration.h in numpy, the normal equations solved by lstsq (min-norm)."""

    def __init__(self, m, u0):
        self.m, self.u, self.iter, self.col = m, np.array(u0, float), 0, 0
        self.dF = np.zeros((16, m))
        self.dG = np.zeros((16, m))
        self.M = np.zeros((m, m))
        self.scale = np.zeros(m)

    def compute(self, g):
        F = g - self.u
        if self.iter == 0:
            self.dF[:, 0], self.dG[:, 0], self.u = -F, -g, g.copy()
        else:
            c = self.col
            self.dF[:, c] += F
            self.dG[:, c] += g
            self.scale[c] = max(1e-14, np.linalg.norm(self.dF[:, c]))
            self.dF[:, c] /= self.scale[c]
            mk = min(self.m, self.iter)
            if mk == 1:
                n = np.linalg.norm(self.dF[:, c])
                self.M[0, 0] = n * n
                theta = np.array([(self.dF[:, c] / n) @ (F / n) if n > 1e-14 else 0.0])
            else:
                ip = self.dF[:, c] @ self.dF[:, :mk]
                self.M[c, :mk] = ip
                self.M[:mk, c] = ip
                theta = np.linalg.lstsq(self.M[:mk, :mk], self.dF[:, :mk].T @ F, rcond=mk * np.finfo(float).eps)[0]
            self.u = g - self.dG[:, :mk] @ (theta / self.scale[:mk])
            self.col = (c + 1) % self.m
            self.dF[:, self.col], self.dG[:, self.col] = -F, -g
        self.iter += 1


@pytest.mark.parametrize("m", [1, 2, 5])
def test_anderson_matches_numpy(m):
    rng = np.random.default_rng(m)
    u0 = rng.normal(size=16)
    ops = [0] * 9 + [1] + [0] * 4 + [2] + [0] * 8
    g = rng.normal(size=(len(ops), 16))
    g[5] = g[4]                                  # a repeated iterate: a rank-deficient history
    got = fo.anderson(m, u0, ops, g)
    ref = NpAnderson(m, u0)
    for k, op in enumerate(ops):
        if op == 0:
            ref.compute(g[k])
        elif op == 1:
            ref.u = g[k].copy()
        else:
            ref.u, ref.iter, ref.col = g[k].copy(), 0, 0
        assert np.abs(got[k] - ref.u).max() <= 1e-8 * max(1.0, np.abs(ref.u).max()), (k, op)


@pytest.mark.parametrize("n", [1, 2, 3, 6, 7, 100, 101])
def test_median_semantics(n):
    v = np.random.default_rng(n).normal(size=n)
    assert fo.median(v) == np.median(v)
    assert fo.median(np.repeat(v[:1], n)) == v[0]


# ------------------------------------------------------------------------------------------------ numpy FR-ICP
def np_fricp(src, tgt, mode, max_icp=100, stop=1e-5, m=5, nu_begin_k=3.0, nu_end_k=1 / (3 * np.sqrt(3)), nu_alpha=0.5):
    welsch, use_aa = mode in (3, 4), mode in (2, 4)
    X = src[np.isfinite(src[:, :3]).all(1), :3].astype(np.float64)
    Y = tgt[np.isfinite(tgt[:, :3]).all(1), :3].astype(np.float64)
    scale = max(np.linalg.norm(X.max(0) - X.min(0)), np.linalg.norm(Y.max(0) - Y.min(0)))
    X, Y = X / scale, Y / scale
    ms, mt = X.mean(0), Y.mean(0)
    X, Y = X - ms, Y - mt
    tree = cKDTree(Y)

    def closest(T):
        d, j = tree.query(X @ T[:3, :3].T + T[:3, 3])
        return Y[j], d

    def energy(r, nu):
        return np.sum(1 - np.exp(-r * r / (2 * nu * nu))) if welsch else np.sum(r * r)

    def step(Q, r, nu):
        w = np.exp(-r * r / (2 * nu * nu)) if welsch else np.ones(len(r))
        w = w / w.sum()
        xm, qm = w @ X, w @ Q
        U, _, Vt = np.linalg.svd(((X - xm) * w[:, None]).T @ (Q - qm))
        S = np.diag([1, 1, -1 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1])
        T = np.eye(4)
        T[:3, :3] = Vt.T @ S @ U.T
        T[:3, 3] = qm - T[:3, :3] @ xm
        return T

    T = np.eye(4)
    Q, r = closest(T)
    nu1 = nu2 = 1.0
    if welsch:
        d, _ = tree.query(Y, k=min(7, len(Y)))
        nu2 = nu_end_k * np.sqrt(np.median(np.median(d[:, 1:] ** 2, axis=1)))
        nu1 = max(nu_begin_k * np.median(r), nu2)
    aa = NpAnderson(m, np.real(logm(T)).T.reshape(16))
    svd_T, To2, last, path = T.copy(), T.copy(), np.inf, []
    while True:
        stage = []
        for _ in range(max_icp):
            e = energy(r, nu1)
            acc = 1
            if use_aa:
                if e < last:
                    last = e
                else:
                    acc = 0
                    aa.u = np.real(logm(svd_T)).T.reshape(16)
                    Q, r = closest(svd_T)
                    last = energy(r, nu1)
            T = step(Q, r, nu1)
            svd_T = T.copy()
            if use_aa:
                aa.compute(np.real(logm(T)).T.reshape(16))
                T = expm(aa.u.reshape(4, 4).T)
            Q, r = closest(T)
            stage.append(acc)
            s2 = np.linalg.norm(T - To2)
            To2 = T.copy()
            if s2 < stop:
                break
        path.append(stage)
        if not welsch:
            break
        done = abs(nu1 - nu2) < 1e-6
        nu1 = max(nu1 * nu_alpha, nu2)
        if use_aa:
            aa.u, aa.iter, aa.col = np.real(logm(T)).T.reshape(16), 0, 0
            last = np.inf
        if done:
            break
    res = T.copy()
    res[:3, 3] = (T[:3, 3] - T[:3, :3] @ ms + mt) * scale
    return res, path, energy(r, nu1)


def _scene(seed, n_t=3000, n_s=1500):
    """Three rough planes of a corner and a ridge (a well-constrained shape), a displaced noisy subset as the source."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-5, 5, size=(n_t, 2))
    k = rng.integers(0, 3, n_t)
    P = np.where(k[:, None] == 0, np.c_[a, 0.2 * np.sin(a[:, 0])],
                 np.where(k[:, None] == 1, np.c_[a[:, 0], np.full(n_t, -5.0), a[:, 1] + 5], np.c_[np.full(n_t, -5.0), a + [0, 5]]))
    tgt = P.astype(np.float32)
    R = Rotation.from_euler("xyz", [0.02, -0.03, 0.08]).as_matrix()
    sel = rng.choice(n_t, n_s, replace=False)
    src = ((P[sel] - [0.3, -0.2, 0.1]) @ R + rng.normal(scale=0.01, size=(n_s, 3))).astype(np.float32)
    return src, tgt


@pytest.mark.parametrize("mode", [0, 2, 3, 4])
def test_registration_matches_numpy_transcription(mode):
    src, tgt = _scene(mode + 11)
    o, corr, resid, log = fo.fricp(src, tgt, mode=mode)
    ref, path, e = np_fricp(src, tgt, mode)
    assert o["status"] == 0 and o["stages"] == len(path) and o["iterations"] == sum(len(s) for s in path)
    got_path = [[int(a) for st, _, _, _, a in log if st == k] for k in range(o["stages"])]
    assert got_path == path
    assert np.abs(o["res_trans"][:3, 3] - ref[:3, 3]).max() < 1e-6
    assert np.abs(o["res_trans"][:3, :3] - ref[:3, :3]).max() < 1e-7
    assert abs(o["energy"] - e) <= 1e-9 * max(abs(e), 1e-300)
    assert (corr >= 0).all() and np.isfinite(resid).all()


def test_non_finite_points_and_tiny_targets():
    src, tgt = _scene(5, n_t=400, n_s=200)
    bad_s, bad_t = src.copy(), tgt.copy()
    bad_s[::17, 1] = np.nan
    bad_t[::13, 2] = np.inf
    o, corr, _, _ = fo.fricp(bad_s, bad_t)
    assert o["n_source_finite"] == len(src) - len(src[::17]) and o["n_target_finite"] == len(tgt) - len(tgt[::13])
    assert (corr[::17] == -1).all() and np.isfinite(bad_t[corr[corr >= 0], :3]).all()
    for n in (0, 1):
        o, corr, _, _ = fo.fricp(src, tgt[:n])
        assert o["status"] == 1 and np.array_equal(o["res_trans"], np.eye(4)) and (corr == -1).all()
    o, _, _, _ = fo.fricp(src[:0], tgt)
    assert o["status"] == 2
    for n in (2, 3, 5, 7, 8):   # fewer than 7 targets: the median of the k - 1 > 0 neighbours there are
        o, _, _, _ = fo.fricp(src[:50], tgt[:n], mode=4)
        Y = (tgt[:n].astype(np.float64) / o["scale"]) - o["mu_target"]
        d2 = ((Y[:, None] - Y[None]) ** 2).sum(-1)
        d2.sort(1)
        k = min(7, n)
        assert o["nu_end"] == pytest.approx(1 / (3 * np.sqrt(3)) * np.sqrt(np.median(np.median(d2[:, 1:k], axis=1))), rel=1e-12)


def test_facade_smoke_compiles():
    src = os.path.join(ROOT, "tests", "cpp", "fricp_facade_smoke.cpp")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
                    src], check=True)
