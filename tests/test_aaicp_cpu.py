"""CPU tests of the AA-ICP oracle (orc_aaicp in tests/cpp/aaicp_oracle.cpp): whole small registrations against a numpy /
scipy (cKDTree) transcription of AAICP::point_to_point_aaicp (ICP.h:841-1033); eulerAngles(0, 1, 2) round trips, its
range and both branches; the column-pivoting QR solve against scipy's pivoted QR (LAPACK geqp3, the same pivot rule) and
lstsq; the first heuristic at 0/0 and x/0; non-finite points and tiny targets; the facade smoke's syntax."""
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from tests import aaicp_oracle as ao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def np_euler(R):
    """Eigen 3.3.7 eulerAngles(0, 1, 2)."""
    a = np.arctan2(R[1, 2], R[2, 2])
    c2 = np.hypot(R[0, 0], R[0, 1])
    if a > 0:
        a -= np.pi
        b = np.arctan2(-R[0, 2], -c2)
    else:
        b = np.arctan2(-R[0, 2], c2)
    c = np.arctan2(np.sin(a) * R[2, 0] - np.cos(a) * R[1, 0], np.cos(a) * R[1, 1] - np.sin(a) * R[2, 1])
    return -np.array([a, b, c])


def np_mat4(v):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_euler("XYZ", v[:3]).as_matrix()   # intrinsic X, Y, Z: AngleAxis X * AngleAxis Y * AngleAxis Z
    T[:3, 3] = v[3:]
    return T


def np_vec6(T):
    return np.r_[np_euler(T[:3, :3]), T[:3, 3]]


def np_qr_solve(A, b):
    """The basic solution of a column-pivoted Householder QR (rank from the pivots, free variables 0)."""
    Q, R, P = scipy.linalg.qr(A, pivoting=True, mode="economic")
    d = np.abs(np.diag(R))
    rank = int((d > d.max() * np.finfo(float).eps * np.sqrt(6)).sum()) if d.size and d.max() > 0 else 0
    x = np.zeros(A.shape[1])
    if rank:
        x[P[:rank]] = scipy.linalg.solve_triangular(R[:rank, :rank], (Q.T @ b)[:rank])
    return x


def np_next_u(u, g, f):
    sol, na = g[-1].copy(), 1
    for i in range(2, len(f) + 1):
        F = np.array(f[-i:]).T
        A = F[:, -1:] - F[:, :-1]
        al = np_qr_solve(A, F[:, -1])
        al = np.r_[al, 1 - al.sum()]
        if not (-10 < al.min() and al.max() < 10 and al[-1] > 0):
            break
        sol, na = np.array(g[-i:]).T @ al, i
    return sol, na


def np_aaicp(src, tgt, max_icp=100, stop=1e-5, thr=0.05):
    """point_to_point_aaicp with Registeration's normalisation, par.f = NONE, in numpy.  Returns (res_trans, log of
    (outcome, α count) per iteration, iterations, per-iteration energies, convergence energy, history columns)."""
    X0 = src[np.isfinite(src[:, :3]).all(1), :3].astype(np.float64)
    Y = tgt[np.isfinite(tgt[:, :3]).all(1), :3].astype(np.float64)
    scale = max(np.linalg.norm(X0.max(0) - X0.min(0)), np.linalg.norm(Y.max(0) - Y.min(0)))
    X0, Y = X0 / scale, Y / scale
    ms, mt = X0.mean(0), Y.mean(0)
    X0, Y = X0 - ms, Y - mt
    tree = cKDTree(Y)
    X = X0.copy()
    T, To2, tr, fin = np.eye(4), np.eye(4), np.eye(4), np.eye(4)
    u, g, f = [], [], []
    prev = np.finfo(float).max
    path, energies = [], []
    Q = np.zeros_like(X0)
    icp = 0
    while icp < max_icp:
        Q = Y[tree.query(X)[1]]
        xm, qm = X.mean(0), Q.mean(0)
        U_, _, Vt = np.linalg.svd((X - xm).T @ (Q - qm) / len(X))
        S = np.diag([1, 1, -1 if np.linalg.det(U_) * np.linalg.det(Vt) < 0 else 1])
        step = np.eye(4)
        step[:3, :3] = Vt.T @ S @ U_.T
        step[:3, 3] = qm - step[:3, :3] @ xm
        T = step @ T
        fin = T.copy()
        energy = (np.linalg.norm(X - Q, axis=1) ** 2).sum()
        energies.append(energy)
        gk = np_vec6(tr @ fin)
        if icp:
            with np.errstate(divide="ignore", invalid="ignore"):
                up = (energy - prev) / prev > thr
            if up:
                u_next = u_k = g[-1]
                prev = np.finfo(float).max
                u, g, f = u[-2:], g[-1:], f[-1:]
                path.append((0, 1))
            else:
                prev = energy
                g.append(gk)
                f.append(gk - u_k)
                u_next, na = np_next_u(u, g, f)
                u.append(u_next)
                u_k = u_next
                path.append((1, na))
        else:
            prev = energy
            u = [np_vec6(np.eye(4)), gk]
            g, f = [gk], [gk - u[0]]
            u_next = u_k = gk
            path.append((-1, 1))
        tr = np_mat4(u_next) @ np.linalg.inv(fin)
        fin = np_mat4(u_next)
        X = X0 @ fin[:3, :3].T + fin[:3, 3]
        stop2 = np.linalg.norm(fin - To2)
        To2 = fin
        if stop2 < stop and icp:
            break
        icp += 1
    conv = (np.linalg.norm(X - Q, axis=1) ** 2).sum()   # the last matches against the re-seated X
    res = fin.copy()
    res[:3, 3] = (fin[:3, 3] - fin[:3, :3] @ ms + mt) * scale
    return res, path, icp, np.array(energies), conv, len(u)


def _scene(seed, n_t=1500, n_s=600, outliers=0.0, rpy=(0.02, -0.03, 0.06), shift=(0.25, -0.2, 0.1)):
    """A corner of three rough planes and a ridge, a displaced noisy subset as the source, optionally with outliers."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-5, 5, size=(n_t, 2))
    k = rng.integers(0, 3, n_t)
    P = np.where(k[:, None] == 0, np.c_[a, 0.2 * np.sin(a[:, 0])],
                 np.where(k[:, None] == 1, np.c_[a[:, 0], np.full(n_t, -5.0), a[:, 1] + 5], np.c_[np.full(n_t, -5.0), a + [0, 5]]))
    R = Rotation.from_euler("xyz", rpy).as_matrix()
    sel = rng.choice(n_t, n_s, replace=False)
    src = (P[sel] - shift) @ R + rng.normal(scale=0.005, size=(n_s, 3))
    n_o = int(outliers * n_s)
    src[:n_o] = rng.uniform(-5, 5, size=(n_o, 3))
    return src.astype(np.float32), P.astype(np.float32)


def _margin(log, thr=0.05):
    """The smallest relative margin of the logged decisions: the stop test, the first heuristic and alphas_cond."""
    m = [np.inf]
    for k, (e, p, out, _, s2, am) in enumerate(log):
        m.append(abs(s2 - 1e-5) / 1e-5)
        if k:
            with np.errstate(divide="ignore", invalid="ignore"):
                r = (e - p) / p
            m.append(abs(r - thr) / thr if np.isfinite(r) else np.inf)
            m.append(am)
    return min(m)


@pytest.mark.parametrize("seed,outliers,max_icp,rpy", [(1, 0.0, 100, (0.02, -0.03, 0.06)), (2, 0.1, 100, (0.02, -0.03, 0.06)),
                                                      (3, 0.0, 4, (0.02, -0.03, 0.06)), (4, 0.0, 100, (-0.03, 0.02, -0.05))])
def test_registration_matches_numpy_transcription(seed, outliers, max_icp, rpy):
    src, tgt = _scene(seed, outliers=outliers, rpy=rpy)
    o, corr, resid, log = ao.aaicp(src, tgt, max_icp=max_icp)
    ref, path, iters, energies, conv, hist = np_aaicp(src, tgt, max_icp=max_icp)
    assert o["status"] == 0
    if _margin(log) > 1e-6:
        assert o["iterations"] == iters and [(int(r[2]), int(r[3])) for r in log] == path
        assert o["accepted"] == sum(p[0] == 1 for p in path) and o["resets"] == sum(p[0] == 0 for p in path)
        assert o["history"] == hist
        assert np.abs(log[:, 0] - energies).max() <= 1e-9 * energies.max()
    assert abs(o["energy"] - conv) <= 1e-6 * conv, (o["energy"], conv)   # the convergence energy
    assert np.abs(o["res_trans"][:3, 3] - ref[:3, 3]).max() < 1e-7
    assert np.abs(o["res_trans"][:3, :3] - ref[:3, :3]).max() < 1e-8
    assert (corr >= 0).all() and np.isfinite(resid).all()
    assert o["history"] == 2 + o["accepted"] if o["resets"] == 0 else o["history"] >= 2
    print(f"[aaicp oracle] seed {seed}: {o['iterations']} iterations, {o['accepted']} accepted, {o['resets']} resets, "
          f"history {o['history']}, margin {_margin(log):.3g}")


def test_first_step_is_one_kabsch():
    src, tgt = _scene(5, n_t=600, n_s=300)
    o, _, _, log = ao.aaicp(src, tgt, max_icp=1)
    ref, path, iters, energies, conv, _ = np_aaicp(src, tgt, max_icp=1)
    assert path == [(-1, 1)] and o["iterations"] == iters == 1 and log[0, 2] == -1
    assert np.abs(o["res_trans"] - ref).max() < 1e-12
    assert abs(log[0, 0] - energies[0]) <= 1e-12 * energies[0] and abs(o["energy"] - conv) <= 1e-9 * conv


def test_max_icp_zero_energy_is_the_source_norm():
    src, tgt = _scene(6, n_t=400, n_s=200)
    o, corr, _, log = ao.aaicp(src, tgt, max_icp=0)
    X = src.astype(np.float64) / o["scale"] - o["mu_source"]
    assert o["iterations"] == 0 and len(log) == 0 and np.array_equal(o["res_trans"][:3, :3], np.eye(3))
    assert abs(o["energy"] - (np.linalg.norm(X, axis=1) ** 2).sum()) < 1e-12 * o["energy"]
    assert (corr == -1).all()


def test_euler_round_trip_range_and_branches():
    rng = np.random.default_rng(7)
    Rs = list(Rotation.random(200, random_state=3).as_matrix())
    for roll in (-1e-3, -0.3, 1e-3, 0.3, 0.0):   # a small negative roll comes back near π, the others reflected
        Rs.append(Rotation.from_euler("XYZ", [roll, 0.2, -0.1]).as_matrix())
    for pitch in (np.pi / 2, -np.pi / 2, np.pi / 2 - 1e-9, -np.pi / 2 + 1e-9):
        Rs.append(Rotation.from_euler("XYZ", [0.3, pitch, 0.2]).as_matrix())
        Rs.append(Rotation.from_euler("XYZ", [-0.3, pitch, 0.2]).as_matrix())
    for R in Rs:
        e = ao.euler(R)
        assert 0.0 <= e[0] <= np.pi, e
        assert np.abs(e - np_euler(R)).max() < 1e-12
        v = np.r_[e, rng.normal(size=3)]
        assert np.abs(ao.mat4(v)[:3, :3] - R).max() < 1e-9
        assert np.abs(ao.mat4(v) - np_mat4(v)).max() < 1e-14
    e = ao.euler(Rotation.from_euler("XYZ", [-1e-3, 0.2, -0.1]).as_matrix())
    assert abs(e[0] - (np.pi - 1e-3)) < 1e-9 and abs(e[1] - (np.pi - 0.2)) < 1e-9 and abs(e[2] - (np.pi - 0.1)) < 1e-9   # (roll + π, π - pitch, yaw + π)
    e = ao.euler(Rotation.from_euler("XYZ", [1e-3, 0.2, -0.1]).as_matrix())
    assert np.abs(e - [1e-3, 0.2, -0.1]).max() < 1e-12
    assert np.array_equal(ao.mat4(np.r_[ao.euler(np.eye(3)), 0, 0, 0]), np.eye(4))


def test_inverse_of_rigid_transforms():
    for k in range(20):
        T = np.eye(4)
        T[:3, :3] = Rotation.random(random_state=k).as_matrix()
        T[:3, 3] = np.random.default_rng(k).normal(size=3)
        assert np.abs(ao.inv4(T) - np.linalg.inv(T)).max() < 1e-14


def test_qr_solve_matches_lapack_pivoting():
    rng = np.random.default_rng(11)
    for n in range(1, 7):   # full column rank: the least-squares solution
        for _ in range(20):
            A, b = rng.normal(size=(6, n)), rng.normal(size=6)
            x, r = ao.qr_solve(A, b)
            assert r == n and np.abs(x - np.linalg.lstsq(A, b, rcond=None)[0]).max() < 1e-10
    checked = 0
    for n in range(7, 12):  # wide: the basic solution on the first 6 pivots, free variables 0
        for _ in range(20):
            A, b = rng.normal(size=(6, n)) * rng.uniform(0.1, 10, size=n), rng.normal(size=6)
            _, R, P = scipy.linalg.qr(A, pivoting=True)
            norms = np.sort(np.linalg.norm(A, axis=0))[::-1]
            if norms[0] - norms[1] < 1e-3 * norms[0]:
                continue   # no margin on the first pivot choice
            x, r = ao.qr_solve(A, b)
            assert r == 6 and (x != 0).sum() == 6 and np.abs(A @ x - b).max() < 1e-9
            assert np.abs(x - np_qr_solve(A, b)).max() < 1e-8, (n, P)
            checked += 1
    assert checked > 50
    A = rng.normal(size=(6, 3))   # rank deficient: a repeated column
    A = np.c_[A, A[:, 1]]
    x, r = ao.qr_solve(A, A @ [1.0, 2.0, 3.0, 0.0])
    assert r == 3 and np.abs(A @ x - A @ [1.0, 2.0, 3.0, 0.0]).max() < 1e-12 and (x == 0).sum() == 1
    # a zero matrix: the pivot threshold is 0 itself, so every pivot counts and the solve divides by zero (get_next_u's
    # alphas_cond then fails on the non-finite α)
    with np.errstate(all="ignore"):
        x, r = ao.qr_solve(np.zeros((6, 2)), np.ones(6))
    assert r == 2 and not np.isfinite(x).all()


def test_first_heuristic_at_zero_previous_energy():
    # 0/0: one source point on a target point never moves (a zero cross-covariance gives R = I, the step t = 0), every
    # energy is 0 and NaN > threshold is false, so the step is accepted
    tgt = np.array([[-1, 0, 0, 0], [1, 0, 0, 0], [0, 0, 0, 0]], np.float32)
    o, _, _, log = ao.aaicp(np.zeros((1, 4), np.float32), tgt)
    assert np.array_equal(log[:, 0], [0.0, 0.0]) and log[1, 1] == 0.0 and log[1, 2] == 1 and o["iterations"] == 1
    assert np.array_equal(o["res_trans"], np.eye(4))
    # x/0: the same cloud as source and target starts at energy 0; a step with rounding moves it off by a little, and
    # x / 0 = inf resets.  Whichever the rounding gives, the decision follows IEEE division.
    src, tgt = _scene(8, n_t=300, n_s=300)
    o, _, _, log = ao.aaicp(tgt, tgt, max_icp=10)
    assert log[0, 0] == 0.0
    seen = set()
    for e, p, out, _, _, _ in log[1:]:
        with np.errstate(divide="ignore", invalid="ignore"):
            assert out == (0 if (e - p) / p > 0.05 else 1)
        if p == 0.0:
            seen.add("0/0" if e == 0.0 else "x/0")
    print(f"[aaicp heuristic] same cloud: {seen}, log {log[:, :3].tolist()}")
    assert np.abs(o["res_trans"] - np.eye(4)).max() < 1e-9


def test_non_finite_points_and_tiny_targets():
    src, tgt = _scene(9, n_t=400, n_s=200)
    bad_s, bad_t = src.copy(), tgt.copy()
    bad_s[::17, 1] = np.nan
    bad_t[::13, 2] = np.inf
    o, corr, _, _ = ao.aaicp(bad_s, bad_t, max_icp=5)
    assert o["n_source_finite"] == len(src) - len(src[::17]) and o["n_target_finite"] == len(tgt) - len(tgt[::13])
    assert (corr[::17] == -1).all() and np.isfinite(bad_t[corr[corr >= 0], :3]).all()
    o, corr, _, _ = ao.aaicp(src, tgt[:0])
    assert o["status"] == 1 and np.array_equal(o["res_trans"], np.eye(4)) and (corr == -1).all()
    o, _, _, _ = ao.aaicp(src[:0], tgt)
    assert o["status"] == 2
    o, _, _, _ = ao.aaicp(src[:1], tgt, max_icp=3)   # one source point: a pure translation onto its match
    assert np.abs(o["res_trans"][:3, :3] - np.eye(3)).max() < 1e-12
    for n in range(1, 9):   # one target point is enough
        o, corr, _, _ = ao.aaicp(src[:50], tgt[:n], max_icp=10)
        assert o["status"] == 0 and (corr < n).all() and np.isfinite(o["res_trans"]).all()


def test_facade_smoke_compiles():
    src = os.path.join(ROOT, "tests", "cpp", "aaicp_facade_smoke.cpp")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
                    src], check=True)
