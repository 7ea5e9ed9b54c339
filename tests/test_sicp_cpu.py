"""CPU tests of the Sparse ICP oracle (orc_sicp in tests/cpp/sicp_oracle.cpp): whole small registrations against a numpy /
scipy (cKDTree) transcription of SICP::point_to_point (ICP.h:275-380), the shrink operator and its thresholds against a
direct transcription of ICP.h:238-256 at its edges and along the μ schedule, the oracle's handling of non-finite points
and tiny targets, and the facade smoke's syntax."""
import math
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from tests import sicp_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def np_sicp(src, tgt, p=0.4, mu=10.0, alpha=1.2, max_mu=1e5, max_icp=100, max_outer=100, stop=1e-5):
    """SICP::point_to_point with Registeration's normalisation, in numpy.  Returns (res_trans, ADMM iterations per ICP
    iteration)."""
    X = src[np.isfinite(src[:, :3]).all(1), :3].astype(np.float64)
    Y = tgt[np.isfinite(tgt[:, :3]).all(1), :3].astype(np.float64)
    scale = max(np.linalg.norm(X.max(0) - X.min(0)), np.linalg.norm(Y.max(0) - Y.min(0)))
    X, Y = X / scale, Y / scale
    ms, mt = X.mean(0), Y.mean(0)
    X, Y = X - ms, Y - mt
    tree = cKDTree(Y)
    n = len(X)
    w = 1.0 / n
    C = np.zeros_like(X)
    Xo2 = X.copy()
    T = np.eye(4)
    path = []
    for _ in range(max_icp):
        Q = Y[tree.query(X)[1]]
        m = mu
        outers = 0
        for _ in range(max_outer):
            Z = X - Q + C / m
            Ba = ((2.0 / m) * (1.0 - p)) ** (1.0 / (2.0 - p))
            ha = Ba + (p / m) * Ba ** (p - 1.0)
            nz = np.linalg.norm(Z, axis=1)
            with np.errstate(divide="ignore", invalid="ignore"):
                s = (Ba / nz + 1.0) / 2.0
                for _ in range(3):
                    s = 1.0 - (p / m) * nz ** (p - 2.0) * s ** (p - 1.0)
            Z = Z * np.where(nz > ha, s, 0.0)[:, None]
            U = Q + Z - C / m
            xm, um = (X * w).sum(0), (U * w).sum(0)
            Us, _, Vt = np.linalg.svd(((X - xm) * w).T @ (U - um))
            S = np.diag([1, 1, -1 if np.linalg.det(Us) * np.linalg.det(Vt) < 0 else 1])
            cur = np.eye(4)
            cur[:3, :3] = Vt.T @ S @ Us.T
            cur[:3, 3] = um - cur[:3, :3] @ xm
            Xn = X @ cur[:3, :3].T + cur[:3, 3]
            dual = ((Xn - X) ** 2).sum() / n
            X = Xn
            T = cur @ T
            P = X - Q - Z
            C = C + m * P
            if m < max_mu:
                m *= alpha
            outers += 1
            if np.linalg.norm(P, axis=1).max() < stop and dual < stop:
                break
        path.append(outers)
        s_v = np.linalg.norm(X - Xo2, axis=1).max()
        Xo2 = X.copy()
        if s_v < stop:
            break
    res = T.copy()
    res[:3, 3] = (T[:3, 3] - T[:3, :3] @ ms + mt) * scale
    return res, path


def _scene(seed, n_t=1500, n_s=600, outliers=0.0):
    """A corner of three rough planes and a ridge, a displaced noisy subset as the source, optionally with outliers."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-5, 5, size=(n_t, 2))
    k = rng.integers(0, 3, n_t)
    P = np.where(k[:, None] == 0, np.c_[a, 0.2 * np.sin(a[:, 0])],
                 np.where(k[:, None] == 1, np.c_[a[:, 0], np.full(n_t, -5.0), a[:, 1] + 5], np.c_[np.full(n_t, -5.0), a + [0, 5]]))
    R = Rotation.from_euler("xyz", [0.02, -0.03, 0.06]).as_matrix()
    sel = rng.choice(n_t, n_s, replace=False)
    src = (P[sel] - [0.25, -0.2, 0.1]) @ R + rng.normal(scale=0.005, size=(n_s, 3))
    n_o = int(outliers * n_s)
    src[:n_o] = rng.uniform(-5, 5, size=(n_o, 3))
    return src.astype(np.float32), P.astype(np.float32)


@pytest.mark.parametrize("seed,outliers,max_icp", [(1, 0.0, 100), (2, 0.1, 100), (3, 0.0, 4)])
def test_registration_matches_numpy_transcription(seed, outliers, max_icp):
    src, tgt = _scene(seed, outliers=outliers)
    o, corr, resid, log = so.sicp(src, tgt, max_icp=max_icp)
    ref, path = np_sicp(src, tgt, max_icp=max_icp)
    assert o["status"] == 0 and o["iterations"] == len(path) and [int(r[0]) for r in log] == path
    assert o["admm_iterations"] == sum(path)
    assert np.abs(o["res_trans"][:3, 3] - ref[:3, 3]).max() < 1e-7
    assert np.abs(o["res_trans"][:3, :3] - ref[:3, :3]).max() < 1e-8
    assert (corr >= 0).all() and np.isfinite(resid).all()
    print(f"[sicp oracle] seed {seed}: {o['iterations']} ICP iterations, {o['admm_iterations']} ADMM iterations")


def test_first_admm_step_is_one_kabsch_onto_the_shrunk_targets():
    src, tgt = _scene(4, n_t=600, n_s=300)
    o, _, _, log = so.sicp(src, tgt, max_icp=1, max_outer=1)
    ref, path = np_sicp(src, tgt, max_icp=1, max_outer=1)
    assert path == [1] and log[0, 0] == 1 and log[0, 4] == 12.0   # μ after one update: 10 * 1.2
    assert np.abs(o["res_trans"] - ref).max() < 1e-12


def _shrink_py(n, mu, p, Ba, ha):
    if not n > ha:
        return 0.0
    s = (Ba / n + 1.0) / 2.0
    for _ in range(3):
        s = 1.0 - ((p / mu) * math.pow(n, p - 2.0)) * math.pow(s, p - 1.0)
    return s


def _schedule(mu=10.0, alpha=1.2, max_mu=1e5, max_outer=100):
    out = []
    for _ in range(max_outer):
        out.append(mu)
        if mu < max_mu:
            mu *= alpha
    return out


@pytest.mark.parametrize("p", [0.4, 0.1, 1.0])
def test_shrink_operator_matches_its_transcription(p):
    for mu in _schedule():
        Ba, ha = so.sicp_thresholds(mu, p)
        Ba_py = math.pow((2.0 / mu) * (1.0 - p), 1.0 / (2.0 - p))
        assert (Ba, ha) == (Ba_py, Ba_py + (p / mu) * math.pow(Ba_py, p - 1.0))
        for n in (0.0, ha, np.nextafter(ha, 0.0), np.nextafter(ha, np.inf), 1e-300, 1e300, 0.5 * ha, 2.0 * ha, 1.0):
            got, want = so.sicp_shrink(n, mu, p, Ba, ha), _shrink_py(n, mu, p, Ba, ha)
            assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (mu, n)
        assert so.sicp_shrink(ha, mu, p, Ba, ha) == 0.0
        if p < 1:   # the ℓp jump (p = 1 is the soft threshold, continuous at ha)
            assert so.sicp_shrink(np.nextafter(ha, np.inf), mu, p, Ba, ha) > 0.1
        assert so.sicp_shrink(1e300, mu, p, Ba, ha) == 1.0   # far outside: Z kept as it is


def test_non_finite_points_and_tiny_targets():
    src, tgt = _scene(5, n_t=400, n_s=200)
    bad_s, bad_t = src.copy(), tgt.copy()
    bad_s[::17, 1] = np.nan
    bad_t[::13, 2] = np.inf
    o, corr, _, _ = so.sicp(bad_s, bad_t, max_icp=5)
    assert o["n_source_finite"] == len(src) - len(src[::17]) and o["n_target_finite"] == len(tgt) - len(tgt[::13])
    assert (corr[::17] == -1).all() and np.isfinite(bad_t[corr[corr >= 0], :3]).all()
    o, corr, _, _ = so.sicp(src, tgt[:0])
    assert o["status"] == 1 and np.array_equal(o["res_trans"], np.eye(4)) and (corr == -1).all()
    o, _, _, _ = so.sicp(src[:0], tgt)
    assert o["status"] == 2
    o, _, _, _ = so.sicp(src[:1], tgt, max_icp=3)   # one source point: a pure translation onto its match
    assert np.array_equal(o["res_trans"][:3, :3], np.eye(3))
    for n in range(1, 9):   # one target point is enough for Sparse ICP
        o, corr, _, _ = so.sicp(src[:50], tgt[:n], max_icp=10)
        assert o["status"] == 0 and (corr < n).all() and np.isfinite(o["res_trans"]).all()


def test_facade_smoke_compiles():
    src = os.path.join(ROOT, "tests", "cpp", "sicp_facade_smoke.cpp")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
                    src], check=True)
