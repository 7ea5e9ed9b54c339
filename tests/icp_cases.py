"""An independent float64 numpy / scipy restatement of the loop-closure ICP contract (DESIGN.md §9), and the clouds the
ICP tests share.  Points and transforms are float32 as in the contract (the same operation order, no FMA); the
algebra (means, cross-covariance, SVD, convergence test) is float64 numpy; the 1-NN is scipy's cKDTree."""
import numpy as np
from scipy.spatial import cKDTree

DBL_MAX = np.finfo(np.float64).max
F = np.float32


def apply(T, x):
    """transformPointCloud with a float 4x4: ((m0 x + m1 y) + m2 z) + m3 per row, float32."""
    T = np.asarray(T, np.float32)
    out = x.copy()
    for r in range(3):
        out[:, r] = ((T[r, 0] * x[:, 0] + T[r, 1] * x[:, 1]) + T[r, 2] * x[:, 2]) + T[r, 3]
    return out


def mul4(A, B):
    C = np.zeros((4, 4), np.float32)
    for r in range(4):
        for c in range(4):
            C[r, c] = ((F(A[r, 0] * B[0, c]) + F(A[r, 1] * B[1, c])) + F(A[r, 2] * B[2, c])) + F(A[r, 3] * B[3, c])
    return C


def d2_of(x, t, idx):
    """float32 (dx*dx + dy*dy) + dz*dz between x[i] and t[idx[i]]."""
    d = t[idx, :3] - x[:, :3]
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


class NN:
    def __init__(self, tgt):
        self.t = np.ascontiguousarray(tgt[:, :3], np.float32)
        self.fin = np.nonzero(np.isfinite(self.t).all(1))[0]
        self.tree = cKDTree(self.t[self.fin].astype(np.float64)) if len(self.fin) else None

    def __call__(self, x):
        """Nearest finite target of every finite query: (index or -1, float32 d² or inf)."""
        idx = np.full(len(x), -1, np.int64)
        d2 = np.full(len(x), np.inf, np.float32)
        f = np.isfinite(x[:, :3]).all(1)
        if f.any():
            _, j = self.tree.query(x[f, :3].astype(np.float64), k=1)
            idx[f] = self.fin[j]
            d2[f] = d2_of(x[f], self.t, idx[f])
        return idx, d2


def np_icp(src, tgt, max_correspondence_distance=200.0, max_iterations=100, transformation_epsilon=1e-6,
           euclidean_fitness_epsilon=1e-6, reflections=None):
    """Returns (result dict as the oracle's, idx, d2 of the last iteration).  reflections: a list that receives, per
    iteration, whether det U det V < 0."""
    x = np.ascontiguousarray(src[:, :3], np.float32).copy()
    nn = NN(tgt)
    t = nn.t
    final = np.eye(4, dtype=np.float32)
    res = {"converged": False, "iterations": 0, "state": 0, "n_correspondences": 0, "fitness_score": DBL_MAX}
    idx = np.full(len(x), -1, np.int64)
    d2 = np.full(len(x), np.inf, np.float32)
    if len(x) == 0 or nn.tree is None:
        res["final_transformation"] = final
        return res, idx, d2
    max_d2 = float(max_correspondence_distance) ** 2
    prev = DBL_MAX
    while True:
        idx, d2 = nn(x)
        keep = (idx >= 0) & (d2.astype(np.float64) <= max_d2)
        n = int(keep.sum())
        res["n_correspondences"] = n
        if n < 3:
            res["state"] = 5
            break
        ps = x[keep].astype(np.float64)
        pt = t[idx[keep]].astype(np.float64)
        ms, mt = ps.mean(0), pt.mean(0)
        H = (pt - mt).T @ (ps - ms)
        U, _, Vt = np.linalg.svd(H)
        flip = np.linalg.det(U) * np.linalg.det(Vt) < 0
        if reflections is not None:
            reflections.append(bool(flip))
        R = U @ np.diag([1.0, 1.0, -1.0 if flip else 1.0]) @ Vt
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = R.astype(np.float32)
        T[:3, 3] = (mt - R @ ms).astype(np.float32)
        x = apply(T, x)
        final = mul4(T, final)
        res["iterations"] += 1
        Td = T.astype(np.float64)
        cosa = 0.5 * (Td[0, 0] + Td[1, 1] + Td[2, 2] - 1.0)
        tr2 = Td[0, 3] ** 2 + Td[1, 3] ** 2 + Td[2, 3] ** 2
        mse = float(d2[keep].astype(np.float64).sum()) / n
        if res["iterations"] >= max_iterations:
            res["state"] = 1
        elif cosa >= 1.0 - transformation_epsilon and tr2 <= transformation_epsilon:
            res["state"] = 2
        elif abs(mse - prev) < 1e-12:
            res["state"] = 3
        elif abs(mse - prev) / prev < euclidean_fitness_epsilon:
            res["state"] = 4
        else:
            prev = mse
        if res["state"]:
            res["converged"] = True
            break
    res["final_transformation"] = final
    y = apply(final, np.ascontiguousarray(src[:, :3], np.float32))
    _, fd = nn(y)
    ok = np.isfinite(y).all(1)
    if ok.any():
        res["fitness_score"] = float(fd[ok].astype(np.float64).sum()) / int(ok.sum())
    return res, idx, d2


def rot(rpy):
    r, p, y = rpy
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
    Ry = np.array([[np.cos(p), 0, np.sin(p)], [0, 1, 0], [-np.sin(p), 0, np.cos(p)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(r), -np.sin(r)], [0, np.sin(r), np.cos(r)]])
    return Rz @ Ry @ Rx


def surface_cloud(n, seed, extent=30.0):
    """Points on a few planes and a cylinder (a ground, walls, a pole), float32 (n, 4) with intensity."""
    rng = np.random.default_rng(seed)
    k = n // 4
    g = np.column_stack([rng.uniform(-extent, extent, k), rng.uniform(-extent, extent, k), rng.normal(0, 0.02, k)])
    w1 = np.column_stack([rng.uniform(-extent, extent, k), np.full(k, 0.6 * extent) + rng.normal(0, 0.02, k), rng.uniform(0, 8, k)])
    w2 = np.column_stack([np.full(k, -0.5 * extent) + rng.normal(0, 0.02, k), rng.uniform(-extent, extent, k), rng.uniform(0, 8, k)])
    m = n - 3 * k
    a = rng.uniform(0, 2 * np.pi, m)
    c = np.column_stack([5 + 1.5 * np.cos(a), -4 + 1.5 * np.sin(a), rng.uniform(0, 10, m)])
    p = np.concatenate([g, w1, w2, c])
    return np.column_stack([p, rng.integers(0, 256, n)]).astype(np.float32)


def moved(cloud, rpy, t):
    """cloud moved by the rigid motion (R(rpy), t) in float64, rounded to float32."""
    out = cloud.copy()
    out[:, :3] = (cloud[:, :3].astype(np.float64) @ rot(rpy).T + np.asarray(t)).astype(np.float32)
    return out


def rot_err(T, R_true):
    """Angle (rad) between the rotation part of T and R_true."""
    M = np.asarray(T, np.float64)[:3, :3].T @ R_true
    w = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return float(np.arctan2(np.linalg.norm(w), 0.5 * (np.trace(M) - 1.0)))   # well conditioned near 0
