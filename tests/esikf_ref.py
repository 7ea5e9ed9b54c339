"""An independent float64 numpy restatement of the iterated update, update_iterated_dyn_share_modified
(esekfom.hpp:1620-1938), used to check the oracle (oracle/lio_oracle.cpp) and, through it, both update engines.

It shares no code with the oracle or the engines: the SO3 / S2 manifold operations are written from their formulas
(Rodrigues; S2.hpp Bx, boxplus, boxminus, Nx_yy, Mx), and the linear algebra goes through LAPACK (np.linalg.solve).
The measurement is a callback, so the same loop runs with the oracle's h_share_model or with any other row source.

`device_gain` is a numpy model of the device engine's gain form (esikf_device.cuh: the 12- or 6-dimensional measured
subspace, Q (T11 + H^T H)^-1 with Gauss-Jordan inverses without pivoting).  Running `update` with it next to the
reference gain, with the normal equations summed in several orders (normal_equations), predicts on the CPU how far
each engine may sit from the oracle on a given covariance.
"""
import numpy as np

NS = 23
TOL = 1e-11                   # MTK::tolerance<double>()
S2_LEN = 98090.0 / 10000.0    # |grav| of MTK::S2<double, 98090, 10000, 1>


# ------------------------------------------------------------------------------------------------ SO3
def hat(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def rodrigues(v):
    """exp([v]x) as a rotation matrix."""
    th = np.linalg.norm(v)
    K = hat(v)
    if th < 1e-8:
        return np.eye(3) + K + 0.5 * K @ K
    return np.eye(3) + np.sin(th) / th * K + (1.0 - np.cos(th)) / th ** 2 * K @ K


def quat_exp(v):
    """Unit quaternion (x, y, z, w) of the rotation vector v."""
    th = np.linalg.norm(v)
    s = 0.5 - th * th / 48.0 if th < 1e-6 else np.sin(th / 2) / th
    return np.array([s * v[0], s * v[1], s * v[2], np.cos(th / 2)])


def quat_mul(a, b):
    av, aw, bv, bw = a[:3], a[3], b[:3], b[3]
    return np.r_[aw * bv + bw * av + np.cross(av, bv), aw * bw - av @ bv]


def quat_conj(q):
    return np.r_[-q[:3], q[3]]


def quat_log(q):
    """Rotation vector of q with the toolkit's sign convention: 2 atan(|v| / w) v / |v|, so q and -q give the same
    vector (SOn.hpp:293-297)."""
    nv = max(np.linalg.norm(q[:3]), TOL)
    return 2.0 * np.arctan(nv / q[3]) / nv * q[:3]


def A_matrix(v):
    """I + (1 - cos t) / t^2 [v]x + (1 - sin t / t) / t^2 [v]x^2 (mtkmath.hpp:235-247)."""
    t2 = v @ v
    t = np.sqrt(t2)
    if t < TOL:
        return np.eye(3)
    K = hat(v)
    return np.eye(3) + (1.0 - np.cos(t)) / t2 * K + (1.0 - np.sin(t) / t) / t2 * K @ K


# ------------------------------------------------------------------------------------------------ S2 (S2_typ == 1)
def s2_Bx(g):
    """Orthonormal basis (3x2) of the tangent plane at g (S2.hpp:215-231)."""
    L = S2_LEN
    if g[0] + L > TOL:
        c = L + g[0]
        return np.array([[-g[1], -g[2]],
                         [L - g[1] * g[1] / c, -g[2] * g[1] / c],
                         [-g[2] * g[1] / c, L - g[2] * g[2] / c]]) / L
    return np.array([[0.0, 0.0], [0.0, -1.0], [1.0, 0.0]])


def s2_boxplus(g, d):
    return rodrigues(s2_Bx(g) @ d) @ g


def s2_boxminus(g, o):
    """g [-] o (S2.hpp:144-167)."""
    v_sin = np.linalg.norm(np.cross(g, o))
    theta = np.arctan2(v_sin, g @ o)
    if v_sin < TOL:
        return np.array([3.1415926 if abs(theta) > TOL else 0.0, 0.0])
    return theta / v_sin * s2_Bx(o).T @ np.cross(o, g)


def s2_Nx_yy(g):
    return s2_Bx(g).T @ hat(g) / S2_LEN ** 2


def s2_Mx(g, d):
    """S2.hpp:266-280.  exp(Bu, scalar(1/2)) there is an integer 1/2 == 0, an identity rotation: only A(Bu)^T stays."""
    B = s2_Bx(g)
    if np.hypot(d[0], d[1]) < TOL:
        return -hat(g) @ B
    return -hat(g) @ A_matrix(B @ d).T @ B


# ------------------------------------------------------------------------------------------------ state26
def boxplus(s, d):
    """state26 [+] d23 (build_manifold.hpp:188-190; layout of include/fastlio_b200.h)."""
    o = np.array(s, np.float64).copy()
    o[0:3] += d[0:3]
    o[3:7] = quat_mul(s[3:7], quat_exp(d[3:6]))
    o[7:11] = quat_mul(s[7:11], quat_exp(d[6:9]))
    o[11:14] += d[9:12]
    o[14:17] += d[12:15]
    o[17:20] += d[15:18]
    o[20:23] += d[18:21]
    o[23:26] = s2_boxplus(s[23:26], d[21:23])
    return o


def boxminus(a, b):
    """a [-] b as a 23-vector."""
    r = np.zeros(NS)
    r[0:3] = a[0:3] - b[0:3]
    r[3:6] = quat_log(quat_mul(quat_conj(b[3:7]), a[3:7]))
    r[6:9] = quat_log(quat_mul(quat_conj(b[7:11]), a[7:11]))
    r[9:21] = a[11:23] - b[11:23]
    r[21:23] = s2_boxminus(a[23:26], b[23:26])
    return r


def projection(d, g, gp):
    """The block-diagonal Jacobian of esekfom.hpp:1665-1703 / :1841-1918: A(d_rot)^T, A(d_offR)^T and
    Nx_yy(g) Mx(gp, d_grav) on the diagonal, identity elsewhere."""
    J = np.eye(NS)
    J[3:6, 3:6] = A_matrix(d[3:6]).T
    J[6:9, 6:9] = A_matrix(d[6:9]).T
    J[21:23, 21:23] = s2_Nx_yy(g) @ s2_Mx(gp, d[21:23])
    return J


# ------------------------------------------------------------------------------------------------ gains
ORDERS = (None, "blocked", "reversed", "shuffled")


def normal_equations(hx, h, order=None):
    """(H^T H, H^T h) over the 12 measured columns, summed in one of several orders: None (one BLAS product),
    "blocked" (132 partials of consecutive rows added in turn, the shape of the GPU's reduction on 132 SMs),
    "reversed" and "shuffled" (row by row, backwards or in a seeded random order).  The spread of the update over these
    orders is the rounding a different summation order of the same rows can cause."""
    if order is None:
        return hx.T @ hx, hx.T @ h
    if order == "blocked":
        parts = np.array_split(np.arange(len(h)), 132)
    else:
        rows = np.arange(len(h))[::-1] if order == "reversed" else np.random.default_rng(len(h)).permutation(len(h))
        parts = np.array_split(rows, max(1, len(h) // 8))
    HTH, HTh = np.zeros((12, 12)), np.zeros(12)
    for r in parts:
        HTH += hx[r].T @ hx[r]
        HTh += hx[r].T @ h[r]
    return HTH, HTh


def reference_gain(P, R, hx, h, order=None):
    """(K_x, K_h) of esekfom.hpp: explicit rows for M < 23 (:1720-1750), information form otherwise (:1788-1815),
    solved with LAPACK.  `order`: the summation order of the normal equations (normal_equations)."""
    M = len(h)
    if M < NS:
        H = np.zeros((M, NS))
        H[:, :12] = hx
        S = H @ P @ H.T / R + np.eye(M)
        K = np.linalg.solve(S, H @ P).T / R
        return K @ H, K @ h
    HTH, HTh = normal_equations(hx, h, order)
    A = np.linalg.solve(P / R, np.eye(NS))
    A[:12, :12] += HTH
    Kx = np.zeros((NS, NS))
    Kx[:, :12] = np.linalg.solve(A, np.vstack([HTH, np.zeros((NS - 12, 12))]))
    return Kx, np.linalg.solve(A, np.r_[HTh, np.zeros(NS - 12)])


def gauss_jordan_nopivot(A):
    """The device's b_inverse_spd: N sweeps of Gauss-Jordan without pivoting."""
    A = np.array(A, np.float64)
    n = len(A)
    for k in range(n):
        inv = 1.0 / A[k, k]
        B = A - np.outer(A[:, k], A[k, :] * inv)
        B[k, :] = A[k, :] * inv
        B[:, k] = -A[:, k] * inv
        B[k, k] = inv
        A = B
    return A


def device_gain(P, R, hx, h, md, order=None):
    """(K_x, K_h) in the device's form: T11 = (P11 / R)^-1, Q = P[:, :md] T11 / R, V = (T11 + H^T H)^-1 and
    [K_x | K_h] = Q V [H^T H | H^T h] on the measured md columns (md = 12 with extrinsic estimation, else 6).
    The M < 23 branch runs on the host in the product, so it keeps the reference form here."""
    if len(h) < NS:
        return reference_gain(P, R, hx, h)
    HTH, HTh = normal_equations(hx, h, order)
    HTH, HTh = HTH[:md, :md], HTh[:md]
    T11 = gauss_jordan_nopivot(P[:md, :md] / R)
    Q = P[:, :md] @ T11 / R
    V = gauss_jordan_nopivot(T11 + HTH)
    Kx = np.zeros((NS, NS))
    Kx[:, :md] = Q @ (V @ HTH)
    return Kx, Q @ (V @ HTh)


# ------------------------------------------------------------------------------------------------ the iterated update
def update(state26, P, measure, R=0.001, max_iter=4, limit=None, gain=reference_gain):
    """update_iterated_dyn_share_modified.  measure(state26, search) -> (M, hx[M, 12], h[M]) is one h_share_model pass
    at the iterate (search = dyn_share.converge).  Returns (state26, P, stats) with stats = [passes, search passes,
    last M, converged count] in the oracle's order."""
    lim = np.full(NS, 0.001) if limit is None else np.asarray(limit, np.float64)
    xp = np.array(state26, np.float64)
    Pp = np.array(P, np.float64).reshape(NS, NS)
    x, Pc = xp.copy(), Pp.copy()
    converge, t = True, 0
    passes = searches = lastM = 0
    for it in range(-1, max_iter):
        M, hx, h = measure(x, converge)
        passes += 1
        searches += int(converge)
        if M < 1:
            continue
        lastM = M
        dx = boxminus(x, xp)
        J = projection(dx, x[23:26], xp[23:26])
        dx_new = J @ dx
        Pc = J @ Pp @ J.T
        Kx, Kh = gain(Pc, R, hx, h)
        dx_ = Kh + (Kx - np.eye(NS)) @ dx_new
        x = boxplus(x, dx_)
        converge = not (np.abs(dx_) > lim).any()
        t += int(converge)
        if not t and it == max_iter - 2:
            converge = True
        if t > 1 or it == max_iter - 1:
            J = projection(dx_, x[23:26], xp[23:26])
            Pc = J @ Pc @ J.T - (J @ Kx)[:, :12] @ (Pc @ J.T)[:12, :]
            return x, Pc, np.array([passes, searches, lastM, t])
    return x, (Pc if lastM else Pp), np.array([passes, searches, lastM, t])


class OracleMeasurement:
    """measure() for `update`: the oracle's h_share_model (orc_residual_pass) with a map search on search passes.  Like
    laserMapping.cpp, point_selected_surf and the neighbours persist over the passes of one scan."""

    def __init__(self, oracle, body, map_obj, extrinsic_est_en=False):
        self.oracle, self.body, self.map, self.ext = oracle, np.ascontiguousarray(body, np.float32), map_obj, extrinsic_est_en
        self.sel = np.ones(len(body), np.uint8)
        self.nbr = self.d2 = self.cnt = None

    def __call__(self, state26, search):
        world = self.oracle.transform(state26, self.body)
        if search:
            self.nbr, self.d2, self.cnt = self.map.Nearest_Search(world, 5)
        M, hx, h, _, _ = self.oracle.residual_pass(state26, self.body, world, self.nbr, self.d2, self.cnt, search, self.sel,
                                                   self.ext)
        return M, hx, h
