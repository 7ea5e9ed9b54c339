"""Seeded inputs for the dense-covariance tests of the iterated update: scenes with non-trivial states, and three
families of dense prior covariances.

synth.default_cov() is diagonal, and with a diagonal prior the gain rows of velocity, biases and gravity are exactly
zero, so those rows never move.  After IMU propagation the prior the node hands to the update is dense; these families
reproduce that:
  * propagated   - default_cov() carried through one scan interval of P <- F P F^T + F_w Q F_w^T with the blocks of
                   df_dx / df_dw (use-ikfom.hpp:70-97) and the reference's default IMU noise (laserMapping.cpp:51);
  * correlated   - D^1/2 C D^1/2 with a random correlation C and the diagonal scales of default_cov(), cond(P) from
                   about 1e3 to 1e8;
  * posterior    - the posterior of a previous dense update plus process noise (what the closed loop feeds).
"""
import numpy as np

from better_fastlio2_b200 import synth
from tests import esikf_ref as ref
from tests.helpers import small_scene

GYR_COV, ACC_COV, B_GYR_COV, B_ACC_COV = 0.1, 0.1, 0.0001, 0.0001   # laserMapping.cpp:51 defaults


def propagate_cov(state26, P, n_steps=20, dt=0.005, acc=(0.35, -0.2, 9.9), gyr=(0.02, -0.03, 0.25)):
    """n_steps IMU steps (200 Hz) of the covariance propagation: F = I + df_dx dt with the rotation block
    Exp(-omega dt), F_w = df_dw dt, Q = diag(gyr, acc, bias_gyr, bias_acc)."""
    P = np.array(P, np.float64).reshape(23, 23).copy()
    q = np.array(state26[3:7], np.float64)
    bg, ba, g = state26[17:20], state26[20:23], state26[23:26]
    w = np.asarray(gyr) - bg
    a = np.asarray(acc) - ba
    Qn = np.diag([GYR_COV] * 3 + [ACC_COV] * 3 + [B_GYR_COV] * 3 + [B_ACC_COV] * 3)
    grav_block = -ref.hat(g) @ ref.s2_Bx(g)                    # S2_Mx at a zero increment (use-ikfom.hpp:82-84)
    for _ in range(n_steps):
        Rm = synth.quat_to_mat(q)
        F = np.eye(23)
        F[0:3, 12:15] = np.eye(3) * dt
        F[3:6, 3:6] = ref.rodrigues(-w * dt)
        F[3:6, 15:18] = -np.eye(3) * dt
        F[12:15, 3:6] = -Rm @ ref.hat(a) * dt
        F[12:15, 18:21] = -Rm * dt
        F[12:15, 21:23] = grav_block * dt
        Fw = np.zeros((23, 12))
        Fw[3:6, 0:3] = -np.eye(3) * dt
        Fw[12:15, 3:6] = -Rm * dt
        Fw[15:18, 6:9] = np.eye(3) * dt
        Fw[18:21, 9:12] = np.eye(3) * dt
        P = F @ P @ F.T + Fw @ Qn @ Fw.T
        q = ref.quat_mul(q, ref.quat_exp(w * dt))
    return 0.5 * (P + P.T)


def correlated_cov(rng, log10_spread):
    """D^1/2 C D^1/2: C a random correlation matrix whose eigenvalues span 10^log10_spread before normalisation."""
    Qm, _ = np.linalg.qr(rng.normal(size=(23, 23)))
    S = Qm @ np.diag(np.logspace(0, -log10_spread, 23)) @ Qm.T
    d = 1.0 / np.sqrt(np.diag(S))
    C = S * d[:, None] * d[None, :]
    D = np.sqrt(np.diag(synth.default_cov()))
    P = C * D[:, None] * D[None, :]
    return 0.5 * (P + P.T)


def tilt(g_dir):
    g = np.asarray(g_dir, np.float64)
    return g / np.linalg.norm(g) * synth.G_LEN


# gravity directions: along -z, tilted, just off -x (the ordinary branch of Bx) and exactly -x (its other branch)
GRAVITY = {"down": (0, 0, -1), "tilted": (0.3, -0.2, -1), "near_-x": (-1, 1e-3, 2e-3), "-x": (-1, 0, 0)}


def true_state(offR_deg=(0, 0, 0), vel=(1.5, -0.4, 0.1), bg=(0.004, -0.003, 0.002), ba=(0.05, -0.03, 0.02), grav="down"):
    s = synth.trajectory_state(0)
    s[7:11] = synth.quat_from_rotvec(np.deg2rad(offR_deg))
    s[14:17], s[17:20], s[20:23] = vel, bg, ba
    s[23:26] = tilt(GRAVITY[grav])
    return s


def prior_from(st_true, rng, pos_m, rot_deg):
    """A prior pos_m metres and rot_deg degrees off the truth (fixed magnitudes, random directions), velocity and
    biases perturbed as well."""
    s = st_true.copy()
    u = rng.normal(size=3)
    s[0:3] += pos_m * u / np.linalg.norm(u)
    v = rng.normal(size=3)
    s[3:7] = ref.quat_mul(s[3:7], ref.quat_exp(np.deg2rad(rot_deg) * v / np.linalg.norm(v)))
    s[14:17] += rng.normal(0, 0.2, 3)
    s[17:20] += rng.normal(0, 0.002, 3)
    s[20:23] += rng.normal(0, 0.02, 3)
    return s


def scene(seed=5, offR_deg=(0, 0, 0), grav="down", every=4):
    """A small city scene scanned from a true state with non-zero velocity / biases (and an optional extrinsic
    rotation: the scan is taken through it), plus a map around it.  Body cloud thinned to every `every`-th point."""
    rng = np.random.default_rng(seed)
    sc = small_scene(seed=seed, map_half=25.0, half_extent=80.0)
    st = true_state(offR_deg=offR_deg, grav=grav)
    body = synth.scan_from_pose(sc["world"], st, synth.lidar_dirs("vlp16"), rng)[::every]
    return dict(st_true=st, body=np.ascontiguousarray(body), map=sc["map"], rng=rng)


def nonuniform_limit():
    lim = np.full(23, 0.001)
    lim[0:3] = 0.002
    lim[3:6] = 0.0005
    lim[12:15] = 0.01
    lim[21:23] = 0.003
    return lim


def family_cov(family, prior, rng, oracle=None, body=None, map_obj=None):
    """The prior covariance of one family at `prior`."""
    if family == "propagated":
        return propagate_cov(prior, synth.default_cov())
    if family.startswith("correlated"):
        return correlated_cov(rng, float(family.split("_")[1]))
    if family == "posterior":
        # posterior of a dense update on the same scene, then one more interval of propagation with process noise
        P0 = propagate_cov(prior, synth.default_cov())
        _, P1, _, _, _ = oracle.esikf_update(prior, P0, body, map_obj, max_iter=4)
        return propagate_cov(prior, 0.5 * (P1 + P1.T))
    raise ValueError(family)


FAMILIES = ["propagated", "correlated_1", "correlated_3", "correlated_6", "posterior"]


def cond_tol(P, scale):
    """Agreement bound for two float64 implementations of the update on prior P: `scale` for a well-conditioned P,
    growing linearly with cond(P / R) = cond(P) above 1e6."""
    ev = np.linalg.eigvalsh(P)
    return scale * (1.0 + ev.max() / ev.min() / 1e6)


def engine_bounds(prior, P, R, max_iter, limit, md, make_measure):
    """Predicted largest |state| and |P| difference from the oracle of each engine on this input, as
    {"device": (bx, bP), "host": (bx, bP)}, derived on the CPU.  Both engines take H^T H and H^T h summed on the GPU in
    an order of their own; the device engine then forms the gain in the measured subspace with Gauss-Jordan inverses
    (esikf_ref.device_gain), the host engine solves the reference's information form (esikf_ref.reference_gain).  The
    spread of each engine's numpy model over the summation orders of esikf_ref.ORDERS, against the reference gain on
    one BLAS product, times 10, floored at 1e-12 (state) and 1e-12 max|P| (covariance)."""
    s_r, P_r, _ = ref.update(prior, P, make_measure(), R=R, max_iter=max_iter, limit=limit)
    gains = {"device": lambda order: (lambda Pc, R_, hx, h: ref.device_gain(Pc, R_, hx, h, md, order)),
             "host": lambda order: (lambda Pc, R_, hx, h: ref.reference_gain(Pc, R_, hx, h, order))}
    out = {}
    for engine, gain in gains.items():
        dx = dP = 0.0
        for order in ref.ORDERS:
            s_m, P_m, _ = ref.update(prior, P, make_measure(), R=R, max_iter=max_iter, limit=limit, gain=gain(order))
            dx, dP = max(dx, np.abs(s_m - s_r).max()), max(dP, np.abs(P_m - P_r).max())
        out[engine] = (max(1e-12, 10 * dx), max(1e-12 * np.abs(P_r).max(), 10 * dP))
    return out


# seeded update cases shared by the CPU host-engine test and the GPU engine test:
# (family, max_iterations, extrinsic estimation, scene, R, limit, prior rotation error in degrees)
ENGINE_CASES = [
    ("propagated", 0, False, "plain", 1e-3, None, 1.0),
    ("correlated_1", 1, True, "offR", 1e-3, None, 1.0),
    ("correlated_3", 2, False, "offR", 1e-2, "nonuniform", 3.0),
    ("correlated_6", 3, True, "plain", 1e-3, None, 0.5),
    ("posterior", 4, False, "plain", 1e-4, None, 2.0),
    ("propagated", 5, True, "offR", 1e-3, "nonuniform", 3.0),
    ("posterior", 6, True, "plain", 1e-3, None, 1.0),
    ("correlated_6", 7, False, "offR", 1e-2, None, 1.0),
    ("correlated_3", 4, True, "plain", 1e-3, None, 1.0),
    ("propagated", 3, False, "plain", 1e-3, None, 1.0),
]
ENGINE_CASE_IDS = [f"{c[0]}-it{c[1]}-{'md12' if c[2] else 'md6'}" for c in ENGINE_CASES]


def engine_case(case, scenes, oracle):
    """(prior, P, R, max_iter, limit, ext, scene) of one ENGINE_CASES entry."""
    fam, max_iter, ext, key, R, lim_kind, rot_deg = case
    sc = scenes[key]
    rng = np.random.default_rng(21 + max_iter)
    prior = prior_from(sc["st_true"], rng, 0.2, rot_deg)
    P = family_cov(fam, prior, rng, oracle, sc["body"], sc["mp"])
    lim = nonuniform_limit() if lim_kind else np.full(23, 0.001)
    return prior, P, R, max_iter, lim, ext, sc
