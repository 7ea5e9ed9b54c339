"""CPU: the iterated update under DENSE prior covariances, every max_iterations setting, non-default R / limit, large
prior errors and states with velocity, biases, an extrinsic rotation and tilted gravity.

Three implementations meet here: the oracle's restatement (oracle/lio_oracle.cpp), the product's host engine
(csrc/esikf_host.hpp through tests/cpp/esikf_host_shim.cpp) and the independent float64 numpy restatement
tests/esikf_ref.py.  With a diagonal prior the rows of velocity, biases and gravity never move, so nothing else in the
suite checks them; every case here moves them."""
import numpy as np
import pytest

from better_fastlio2_b200 import synth
from tests import dense_cases as dc
from tests import esikf_ref as ref
from tests.test_esikf_host_cpu import iu  # noqa: F401  (the compiled host-engine shim, a module fixture)


# ------------------------------------------------------------------------------------------------ manifold operations
def _rand_state(rng, grav=None, neg_w=False):
    q = ref.quat_exp(rng.normal(0, 1.0, 3))
    if neg_w and q[3] > 0:
        q = -q
    g = dc.tilt(grav if grav is not None else rng.normal(0, 1, 3) + [0, 0, -2])
    return synth.make_state(pos=rng.normal(0, 5, 3), rot=q, offR=ref.quat_exp(rng.normal(0, 0.1, 3)), offT=rng.normal(0, 0.1, 3),
                            vel=rng.normal(0, 2, 3), bg=rng.normal(0, 0.01, 3), ba=rng.normal(0, 0.05, 3), grav=g)


@pytest.mark.parametrize("rot_scale", [1e-4, 0.01, 0.05, 0.3])     # the half-angle series of cos_sinc_sqrt below ~1.27 deg, sincos above
def test_boxplus_boxminus_match_oracle(oracle, rot_scale):
    L = oracle.lio()
    rng = np.random.default_rng(11)
    for k in range(200):
        grav = [None, (-1, 1e-3, 2e-3), (-1, 0, 0), (0.3, -0.2, -1)][k % 4]
        s = _rand_state(rng, grav=grav, neg_w=k % 2 == 1)
        d = rng.normal(0, 0.05, 23)
        d[3:9] = rng.normal(0, rot_scale, 6)
        d[21:23] = rng.normal(0, rot_scale, 2)
        a = s.copy()
        L.orc_boxplus(a, d)
        b = ref.boxplus(s, d)
        assert np.abs(a - b).max() < 1e-13, (k, np.abs(a - b).max())
        r_o = np.zeros(23)
        L.orc_boxminus(a, s, r_o)
        r_n = ref.boxminus(a, s)
        assert np.abs(r_o - r_n).max() < 1e-12 * max(1.0, np.abs(r_n).max() / 1e-3), (k, np.abs(r_o - r_n).max())
        assert np.abs(r_n - d).max() < 1e-9                      # and it inverts boxplus


def test_A_matrix_matches_oracle_at_the_branch_edge(oracle):
    L = oracle.lio()
    rng = np.random.default_rng(12)
    for norm in (0.5e-11, 0.99e-11, 1.01e-11, 2e-11, 1e-6, 1e-3, 0.3, 2.5):
        for _ in range(5):
            u = rng.normal(size=3)
            v = u / np.linalg.norm(u) * norm
            A = np.zeros(9)
            L.orc_A_matrix(v, A)
            assert np.abs(A.reshape(3, 3) - ref.A_matrix(v)).max() < 1e-12 * max(1.0, 1e-6 / norm), norm


def test_s2_matrices_match_oracle_at_the_branch_edges(oracle):
    """Bx, Nx_yy and Mx at random gravities, at exactly -x (the second branch of Bx), just off -x (g[0] + len a few
    tolerances above zero) and with |delta| on both sides of 1e-11 (the two branches of Mx)."""
    L = oracle.lio()
    rng = np.random.default_rng(13)
    gs = [dc.tilt(rng.normal(0, 1, 3)) for _ in range(20)]
    gs += [dc.tilt((-1, 0, 0)), dc.tilt((-1, 1e-3, 0)), dc.tilt((-1, 0, 1e-2)), dc.tilt((0, 0, -1)), dc.tilt((0.3, -0.2, -1))]
    deltas = [np.zeros(2), np.array([0.7e-11, 0.0]), np.array([0.0, 1.3e-11]), rng.normal(0, 1e-3, 2), rng.normal(0, 0.05, 2),
              rng.normal(0, 0.5, 2)]
    for g in gs:
        for d in deltas:
            Bx, Nx, Mx = np.zeros(6), np.zeros(6), np.zeros(6)
            L.orc_s2_mats(g, d, Bx, Nx, Mx)
            assert np.abs(Bx.reshape(3, 2) - ref.s2_Bx(g)).max() < 1e-13
            assert np.abs(Nx.reshape(2, 3) - ref.s2_Nx_yy(g)).max() < 1e-13
            assert np.abs(Mx.reshape(3, 2) - ref.s2_Mx(g, d)).max() < 1e-12, (g, d)
    # the -x branch really is taken there, and gives an orthonormal tangent basis
    B = ref.s2_Bx(dc.tilt((-1, 0, 0)))
    assert np.array_equal(B, [[0, 0], [0, -1], [1, 0]])


def test_s2_boxminus_near_parallel_and_antipodal(oracle):
    """v_sin = |g x o| on both sides of 1e-11, and g = -o (theta = pi, v_sin = 0)."""
    L = oracle.lio()
    rng = np.random.default_rng(14)
    base = _rand_state(rng)
    g = base[23:26]
    axis = np.cross(g, rng.normal(size=3))
    axis /= np.linalg.norm(axis)
    for v_sin in (0.3e-11, 0.5e-11, 3e-11, 1e-9, 1e-6):
        eps = v_sin / synth.G_LEN ** 2
        o = ref.rodrigues(axis * eps) @ g
        a, b = base.copy(), base.copy()
        b[23:26] = o
        r_o = np.zeros(23)
        L.orc_boxminus(a, b, r_o)
        r_n = ref.boxminus(a, b)
        assert np.abs(r_o[21:23] - r_n[21:23]).max() < 1e-15 + 1e-6 * np.abs(r_n[21:23]).max(), (v_sin, r_o[21:23], r_n[21:23])
    b = base.copy()
    b[23:26] = -g
    r_o = np.zeros(23)
    L.orc_boxminus(base, b, r_o)
    assert np.array_equal(r_o[21:23], ref.boxminus(base, b)[21:23]) and r_o[21] == 3.1415926


# ------------------------------------------------------------------------------------------------ the iterated update
@pytest.fixture(scope="module")
def scenes(oracle):
    """Scenes by extrinsic rotation, each with its map (the reference ikd-Tree when present)."""
    out = {}
    for key, offR in (("plain", (0, 0, 0)), ("offR", (1.5, -2.0, 3.0))):
        sc = dc.scene(seed=5, offR_deg=offR)
        mp = oracle.make_map(ds=0.2)
        mp.Build(sc["map"])
        sc["mp"] = mp
        out[key] = sc
    return out


def _case(oracle, scenes, family, *, max_iter=4, R=0.001, limit=None, pos_m=0.2, rot_deg=1.0, offR=False, ext=False,
          grav="down", neg_q=False, seed=1):
    sc = scenes["offR" if offR else "plain"]
    rng = np.random.default_rng(seed)
    st = sc["st_true"].copy()
    st[23:26] = dc.tilt(dc.GRAVITY[grav])
    prior = dc.prior_from(st, rng, pos_m, rot_deg)
    if neg_q:
        prior[3:7] = -prior[3:7]
    P = dc.family_cov(family, prior, rng, oracle, sc["body"], sc["mp"])
    return dict(prior=prior, P=P, body=sc["body"], mp=sc["mp"], max_iter=max_iter, R=R, limit=limit, ext=ext)


def _tols(c):
    """State and covariance bounds between two float64 implementations: rounding of values of order one (state) and of
    the prior's entries (the posterior covariance is the prior's minus a gain term), growing with cond(P / R).
    With extrinsic estimation the 12 measured columns are nearly dependent (position and extrinsic translation enter the
    rows almost alike), which costs one more digit."""
    scale = 1e-11 if c["ext"] else 1e-12
    return dc.cond_tol(c["P"], scale), dc.cond_tol(c["P"], scale) * np.abs(c["P"]).max()


def _oracle_vs_ref(oracle, c):
    s_o, P_o, _, st_o, _ = oracle.esikf_update(c["prior"], c["P"], c["body"], c["mp"], max_iter=c["max_iter"], R=c["R"],
                                               extrinsic_est_en=c["ext"], limit=c["limit"])
    s_r, P_r, st_r = ref.update(c["prior"], c["P"], ref.OracleMeasurement(oracle, c["body"], c["mp"], c["ext"]), R=c["R"],
                                max_iter=c["max_iter"], limit=c["limit"])
    assert list(st_o) == list(st_r), (st_o, st_r)            # passes, search passes, last M, converged count
    tx, tP = _tols(c)
    assert np.abs(s_o - s_r).max() <= tx, (np.abs(s_o - s_r).max(), tx)
    assert np.abs(P_o - P_r).max() <= tP, (np.abs(P_o - P_r).max(), tP)
    return s_o, P_o, st_o


def test_covariance_families_are_dense_and_span_the_conditioning(oracle, scenes):
    conds = []
    for fam in dc.FAMILIES:
        P = _case(oracle, scenes, fam)["P"]
        ev = np.linalg.eigvalsh(P)
        assert ev.min() > 0 and np.allclose(P, P.T, rtol=0, atol=1e-18)
        assert np.abs(P[12:23, 0:12]).max() > 1e-3 * np.sqrt(np.diag(P)[12:23].max() * np.diag(P)[0:12].max()), fam
        conds.append(ev.max() / ev.min())
    assert min(conds) < 2e3 and max(conds) > 1e8, conds


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("max_iter", range(8))
def test_oracle_matches_numpy_reference_every_iteration_count(oracle, scenes, family, max_iter):
    c = _case(oracle, scenes, family, max_iter=max_iter)
    s, P, st = _oracle_vs_ref(oracle, c)
    assert st[0] >= 1 and st[2] > 23


@pytest.mark.parametrize("R", [1e-4, 1e-3, 1e-2])
@pytest.mark.parametrize("limit", ["uniform", "nonuniform"])
@pytest.mark.parametrize("prior", [(0.05, 0.3), (0.3, 3.0)])
def test_oracle_matches_numpy_reference_settings(oracle, scenes, R, limit, prior):
    lim = dc.nonuniform_limit() if limit == "nonuniform" else None
    c = _case(oracle, scenes, "propagated", max_iter=5, R=R, limit=lim, pos_m=prior[0], rot_deg=prior[1])
    _oracle_vs_ref(oracle, c)


STATES = {
    "vel_bias": dict(),
    "offR": dict(offR=True),
    "offR_est": dict(offR=True, ext=True),
    "est": dict(ext=True),
    "grav_tilted": dict(grav="tilted"),
    "grav_near_-x": dict(grav="near_-x"),
    "grav_-x": dict(grav="-x"),
}


@pytest.mark.parametrize("state", sorted(STATES))
@pytest.mark.parametrize("family", ["propagated", "correlated_3", "posterior"])
def test_oracle_matches_numpy_reference_states(oracle, scenes, state, family):
    c = _case(oracle, scenes, family, max_iter=4, **STATES[state])
    _oracle_vs_ref(oracle, c)


def test_q_and_minus_q_give_the_same_posterior(oracle, scenes):
    a = _case(oracle, scenes, "propagated", rot_deg=2.0)
    b = _case(oracle, scenes, "propagated", rot_deg=2.0, neg_q=True)
    assert np.array_equal(a["prior"][3:7], -b["prior"][3:7])
    sa, Pa, _ = _oracle_vs_ref(oracle, a)
    b["P"] = a["P"]
    sb, Pb, _ = _oracle_vs_ref(oracle, b)
    sb[3:7] = -sb[3:7]
    assert np.abs(sa - sb).max() < 1e-12 and np.abs(Pa - Pb).max() < 1e-15


@pytest.mark.parametrize("family", dc.FAMILIES)
def test_dense_prior_moves_velocity_biases_and_gravity(oracle, scenes, family):
    """Under a dense prior the update moves every block and couples them in the posterior; under the diagonal
    default_cov() the same scan leaves velocity, biases and gravity exactly where they were."""
    c = _case(oracle, scenes, family)
    s, P, _ = _oracle_vs_ref(oracle, c)
    moved = np.abs(ref.boxminus(s, c["prior"]))
    assert moved[12:15].max() > 1e-3 and moved[15:21].max() > 1e-6 and moved[21:23].max() > 1e-7, moved
    assert np.abs(P[12:23, 0:12]).max() > 1e-9
    s0, P0, _, _, _ = oracle.esikf_update(c["prior"], synth.default_cov(), c["body"], c["mp"], max_iter=4)
    assert np.array_equal(s0[14:26], c["prior"][14:26]) and not P0[12:23, 0:12].any()


# ------------------------------------------------------------------------------------------------ the product's host engine
def _host_engine(L, oracle, c):
    """flb's host-driven engine with the oracle standing in for the GPU measurement kernels."""
    lim = np.full(23, 0.001) if c["limit"] is None else np.asarray(c["limit"], np.float64)
    h = L.iu_create(np.ascontiguousarray(c["prior"]), np.ascontiguousarray(c["P"]).reshape(-1), c["R"], c["max_iter"], lim)
    meas = ref.OracleMeasurement(oracle, c["body"], c["mp"], c["ext"])
    passes = searches = lastM = 0
    st = np.zeros(26)
    while L.iu_more(h):
        L.iu_current_state(h, st)
        search = bool(L.iu_need_search(h))
        M, hx, hv = meas(st, search)
        passes += 1
        searches += int(search)
        if M < 1:
            L.iu_skip(h)
            continue
        lastM = M
        if M < 23:
            L.iu_step_rows(h, np.ascontiguousarray(hx).reshape(-1), np.ascontiguousarray(hv), M)
        else:
            L.iu_step(h, np.ascontiguousarray(hx.T @ hx).reshape(-1), np.ascontiguousarray(hx.T @ hv))
    out_s, out_P = np.zeros(26), np.zeros(23 * 23)
    L.iu_result(h, out_s, out_P)
    t = L.iu_converged_count(h)
    L.iu_destroy(h)
    return out_s, out_P.reshape(23, 23), [passes, searches, lastM, t]


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("max_iter", [0, 1, 2, 5, 7])
@pytest.mark.parametrize("state", ["vel_bias", "offR_est", "grav_-x"])
def test_host_engine_matches_oracle_dense(iu, oracle, scenes, family, max_iter, state):  # noqa: F811
    c = _case(oracle, scenes, family, max_iter=max_iter, R=1e-2 if max_iter == 5 else 1e-3,
              limit=dc.nonuniform_limit() if max_iter == 7 else None, rot_deg=3.0 if max_iter == 2 else 1.0, **STATES[state])
    s_o, P_o, _, st_o, _ = oracle.esikf_update(c["prior"], c["P"], c["body"], c["mp"], max_iter=c["max_iter"], R=c["R"],
                                               extrinsic_est_en=c["ext"], limit=c["limit"])
    s, P, st = _host_engine(iu, oracle, c)
    assert st == list(st_o), (st, st_o)
    tx, tP = _tols(c)
    assert np.abs(s - s_o).max() <= tx and np.abs(P - P_o).max() <= tP


@pytest.mark.parametrize("family", ["propagated", "correlated_6", "posterior"])
def test_host_engine_underdetermined_dense(iu, oracle, scenes, family):  # noqa: F811
    """M < 23 (explicit-row gain) under a dense prior: a dozen well-supported points."""
    c = _case(oracle, scenes, family, max_iter=3)
    world = oracle.transform(c["prior"], c["body"])
    _, d2, cnt = c["mp"].Nearest_Search(world, 5)
    c["body"] = np.ascontiguousarray(c["body"][np.where((cnt == 5) & (d2[:, 4] < 0.2))[0][:14]])
    s_o, P_o, st_o = _oracle_vs_ref(oracle, c)
    assert 0 < st_o[2] < 23
    s, P, st = _host_engine(iu, oracle, c)
    assert st == list(st_o)
    tx, tP = _tols(c)
    assert np.abs(s - s_o).max() <= tx and np.abs(P - P_o).max() <= tP


def test_engine_gain_models_predict_small_differences(oracle, scenes):
    """The numpy models of both engines' gains, over several summation orders of the normal equations, agree with the
    reference on every family: the bounds the GPU tests derive from them stay far below the 1e-4 m / rad bar."""
    for fam in dc.FAMILIES:
        for ext in (False, True):
            c = _case(oracle, scenes, fam, ext=ext)
            bounds = dc.engine_bounds(c["prior"], c["P"], c["R"], c["max_iter"], c["limit"], 12 if ext else 6,
                                      lambda: ref.OracleMeasurement(oracle, c["body"], c["mp"], c["ext"]))
            for engine, (bx, bP) in bounds.items():
                assert bx < 1e-9 and bP < 1e-9 * np.abs(c["P"]).max(), (fam, ext, engine, bx, bP)


@pytest.mark.parametrize("case", dc.ENGINE_CASES, ids=dc.ENGINE_CASE_IDS)
def test_host_engine_matches_oracle_engine_cases(iu, oracle, scenes, case):  # noqa: F811
    """The cases the GPU runs both engines on.  With extrinsic estimation the information form's P_temp is
    ill-conditioned: the host engine solves for the gain from its LU factors; forming P_temp^-1 and multiplying by
    H^T H put it 6.6e-10 from the oracle on propagated-it5-md12."""
    prior, P, R, max_iter, lim, ext, sc = dc.engine_case(case, scenes, oracle)
    c = dict(prior=prior, P=P, body=sc["body"], mp=sc["mp"], max_iter=max_iter, R=R, limit=lim, ext=ext)
    s_o, P_o, st_o = _oracle_vs_ref(oracle, c)
    s, Pm, st = _host_engine(iu, oracle, c)
    assert st == list(st_o), (st, st_o)
    tx, tP = _tols(c)
    assert np.abs(s - s_o).max() <= tx and np.abs(Pm - P_o).max() <= tP, (np.abs(s - s_o).max(), tx)
