"""CPU checks that every constructed measurement case (tests/meas_edge_cases.py) is what it claims to be: the exact
float properties hold, the oracle's decisions match each family's intent, and away from the 0.1 threshold those
decisions and the fitted normals agree with an independent float64 least-squares fit."""
import numpy as np
import pytest

from tests import meas_edge_cases as mc

F32 = np.float32
EPS32 = float(np.finfo(np.float32).eps)
FLT_MIN = float(np.finfo(np.float32).tiny)


@pytest.fixture(scope="module")
def cases(oracle):
    return {c["name"]: c for c in mc.neighbourhood_cases(oracle.esti_plane)}


def _seq_sq_norm(col):
    s = F32(0)
    for v in np.asarray(col, F32):
        s = F32(s + F32(v * v))
    return s


def test_exact_properties(cases):
    # zero columns are exactly zero
    assert (cases["wall_x0"]["pts"][:, 0] == 0).all() and (cases["ground_z0"]["pts"][:, 2] == 0).all()
    # skip at the first pivot: the biggest column has exact zeros below its first row
    p = cases["skip_k0_plane"]["pts"]
    norms = [_seq_sq_norm(p[:, j]) for j in range(3)]
    assert int(np.argmax(norms)) == 0 and p[0, 0] == 16 and (p[1:, 0] == 0).all()
    # subnormal tails: every column's squared norm is a small multiple of FLT_MIN, so the Householder tails sit at it
    for s in ("2e-20", "6e-20"):
        q = cases[f"subnormal_tail_{s}"]["pts"].astype(np.float64)
        assert ((q ** 2).sum(0) < 64 * FLT_MIN).all()
    # exact multiples: the origin line's y and z columns are x/2 and x/4 in float32
    q = cases["collinear_origin_line"]["pts"]
    assert np.array_equal(q[:, 1] * 2, q[:, 0]) and np.array_equal(q[:, 2] * 4, q[:, 0])
    assert (cases["duplicates_345"]["pts"] == [3, 4, 5]).all() and (cases["origin_x5"]["pts"] == 0).all()
    # pivot ties: bit-equal sequential float32 sums, and they are the biggest column
    for name in [n for n in cases if n.startswith("pivot_tie")]:
        p = cases[name]["pts"]
        nx, ny, nz = (_seq_sq_norm(p[:, j]) for j in range(3))
        assert nx.view(np.uint32) == ny.view(np.uint32) and nx > nz, name
    # norm downdate: after the first reflection (the biggest column projected out, in float64) another column keeps
    # under 1 % of its norm, far below the sqrt(sqrt(eps)) ~ 1.9 % where the downdate switches to a recompute
    for name in [n for n in cases if n.startswith("downdate")]:
        A = cases[name]["pts"].astype(np.float64)
        k = int(np.argmax(np.linalg.norm(A, axis=0)))
        u = A[:, k] / np.linalg.norm(A[:, k])
        rest = [np.linalg.norm(A[:, j] - u * (u @ A[:, j])) / np.linalg.norm(A[:, j]) for j in range(3) if j != k]
        assert min(rest) < 0.01, (name, rest)


@pytest.mark.parametrize("pose", ["A", "B"])
def test_d2_gate_exact(oracle, pose):
    state = {"A": mc.POSE_A, "B": mc.POSE_B}[pose]
    cs = mc.d2_gate_cases(state, oracle.transform)
    assert len(cs) == 4
    for c in cs:
        w = oracle.transform(state, c["body"][None])[0]
        assert np.array_equal(w, c["query"])
        d = mc.sorted_d2(c["pts"], w)
        if "d2_eq5" in c["branches"]:
            assert d[4] == F32(5.0) and d[3] < 5, c["name"]
        else:
            assert d[4] == np.nextafter(F32(5.0), F32(9)) or (d[4] > 5 and d[4] < 5.0001), (c["name"], d[4])
        assert oracle.esti_plane(c["pts"])[0]
        sel = np.ones(1, np.uint8)
        oracle.residual_pass(state, c["body"][None], w[None], c["pts"][None], d[None], np.array([5], np.int32), True, sel)
        assert sel[0] == (1 if "d2_eq5" in c["branches"] else 0), c["name"]


def test_intents(oracle, cases):
    for name, c in cases.items():
        ok, pabcd = oracle.esti_plane(c["pts"])
        if c["expect"] == "accept":
            assert ok, name
        elif c["expect"] == "reject":
            assert not ok, name
        elif c["expect"] == "nan":
            # accepted (NaN > 0.1 is false) with a NaN plane, then dropped by the s gate (NaN > 0.9 is false)
            assert ok and np.isnan(pabcd).all(), name
            for st in (mc.POSE_A, mc.POSE_B):
                body = mc.world_to_body(st, c["query"])
                w = oracle.transform(st, body)
                sel = np.ones(1, np.uint8)
                M = oracle.residual_pass(st, body, w, c["pts"][None], mc.sorted_d2(c["pts"], w[0])[None],
                                         np.array([5], np.int32), True, sel)[0]
                assert sel[0] == 0 and M == 0
    # the rank-1 duplicates fit the plane z = 5 (to a float step)
    ok, p = oracle.esti_plane(cases["duplicates_345"]["pts"])
    assert ok and p[0] == 0 and p[1] == 0 and p[2] == -1 and abs(p[3] - 5) < 1e-5
    # the exact ground z = 1.8 is accepted at 1 km and rejected at 5 and 20 km (float conditioning)
    assert oracle.esti_plane(cases["ground_x1000"]["pts"])[0]
    for name in ("ground_x5000", "ground_diag5000", "ground_x20000", "ground_diag20000"):
        assert not oracle.esti_plane(cases[name]["pts"])[0], name


def test_threshold_pairs_straddle(oracle, cases):
    pairs = sorted({n.rsplit("_", 1)[0] for n in cases if n.startswith("thr")})
    assert len(pairs) == 4
    for p in pairs:
        cin, cout = cases[p + "_in"], cases[p + "_out"]
        assert np.nextafter(F32(cin["offset"]), F32(1)) == F32(cout["offset"]), p
        ok_in, pin = oracle.esti_plane(cin["pts"])
        ok_out, pout = oracle.esti_plane(cout["pts"])
        assert ok_in and not ok_out
        r_in, r_out = mc.on_plane(cin["pts"], pin).max(), mc.on_plane(cout["pts"], pout).max()
        assert r_in <= mc.THR < r_out, (p, r_in, r_out)
        # within a few ulps of 0.1f, or of the coordinates' own float step where that is coarser
        tol = 4 * np.spacing(mc.THR) + 2 * np.spacing(np.abs(cin["pts"]).max())
        assert mc.THR - r_in <= tol and r_out - mc.THR <= tol, (p, r_in, r_out, tol)
    for n in ("thr0_pos_in", "thr0_pos_out", "thr0_neg_in", "thr0_neg_out"):   # next to the origin: 1.5e-7 at most
        c = cases[n]
        assert abs(mc.on_plane(c["pts"], oracle.esti_plane(c["pts"])[1]).max() - mc.THR) <= 32 * np.spacing(mc.THR), n


def test_float64_agreement(oracle, cases):
    """Away from the threshold by more than the float32 error bound, the oracle decides as a float64 fit does and its
    normal agrees within the bound of test_oracle_math. Far cases test parity only."""
    checked = 0
    for name, c in cases.items():
        if c["far"] or c["expect"] == "nan":
            continue
        A = c["pts"].astype(np.float64)
        cond = np.linalg.cond(A)
        if not np.isfinite(cond) or cond > 1e6:
            continue
        x = np.linalg.lstsq(A, -np.ones(5), rcond=None)[0]
        nn = np.linalg.norm(x)
        ref = np.r_[x / nn, 1 / nn]
        res = np.abs(A @ ref[:3] + ref[3]).max()
        scale = max(1.0, np.abs(A).max())
        ok, pabcd = oracle.esti_plane(c["pts"])
        if abs(res - 0.1) > 40 * EPS32 * cond * scale:
            assert ok == (res <= 0.1), (name, res)
        if ok:
            tol = max(2e-4, 40 * 1.2e-7 * cond)
            assert np.allclose(pabcd[:3], ref[:3], atol=tol), (name, pabcd, ref)
            assert abs(pabcd[3] - ref[3]) < tol * scale * 2, (name, pabcd, ref)
        checked += 1
    assert checked >= 20


@pytest.mark.parametrize("pose", ["A", "B"])
def test_s_gate_cases(oracle, pose):
    state = {"A": mc.POSE_A, "B": mc.POSE_B}[pose]
    cs = mc.s_gate_cases(state, oracle.transform, oracle.esti_plane, lambda *a: oracle.residual_pass(*a))
    names = {c["name"] for c in cs}
    assert {"bn0_pd2_nonzero", "s_in0", "s_out0", "s_in1", "s_out1"} <= names
    assert ("bn0_pd2_zero" in names) == (pose == "B")
    for c in cs:
        body = c["body"][None]
        w = oracle.transform(state, body)
        assert np.array_equal(w[0], c["query"])
        ok, pabcd = oracle.esti_plane(c["pts"])
        assert ok or "tiny_bn" in c["branches"], c["name"]
        sel = np.ones(1, np.uint8)
        oracle.residual_pass(state, body, w, c["pts"][None], mc.sorted_d2(c["pts"], w[0])[None], np.array([5], np.int32),
                             True, sel)
        pd2 = mc.on_plane(w, pabcd)[0]
        if "bn0" in c["branches"]:
            assert (c["body"] == 0).all() and sel[0] == 0
            assert (pd2 == 0) == (c["name"] == "bn0_pd2_zero"), c["name"]
        if "s_in" in c["branches"] or "s_out" in c["branches"]:
            assert sel[0] == (1 if "s_in" in c["branches"] else 0), c["name"]
    for k in (0, 1):
        b_in = [c for c in cs if c["name"] == f"s_in{k}"][0]["body"]
        b_out = [c for c in cs if c["name"] == f"s_out{k}"][0]["body"]
        assert np.nextafter(b_in[2], b_out[2]) == b_out[2] and np.array_equal(b_in[:2], b_out[:2])


def test_pass_sequence_scene(oracle):
    """At pose B the queries above their plane fail the s gate and the others pass."""
    cs, sa, sb = mc.pass_sequence_scene(np.random.default_rng(21))
    body = np.array([mc.world_to_body(sa, c["query"])[0] for c in cs], np.float32)
    nbr = np.array([c["pts"] for c in cs], np.float32)
    w_a = oracle.transform(sa, body)
    d2 = np.array([mc.sorted_d2(c["pts"], w) for c, w in zip(cs, w_a)], np.float32)
    cnt = np.full(len(cs), 5, np.int32)
    sel = np.ones(len(cs), np.uint8)
    assert oracle.residual_pass(sa, body, w_a, nbr, d2, cnt, True, sel)[0] == len(cs)
    M = oracle.residual_pass(sb, body, oracle.transform(sb, body), nbr, d2, cnt, False, sel)[0]
    assert 0 < M < len(cs)


@pytest.mark.parametrize("fs", [0.5, 0.25, 0.2])
def test_classifier_cases(oracle, fs):
    """Each classifier case is decided as named, and its equality is exact in the float arithmetic the classifier uses."""
    want = {"nonneed": 2, "strict_lt": 1, "nearer": 0, "strict_gt": 1}
    for name, pts, q, branch in mc.classifier_cases(fs):
        d = mc.sorted_d2(pts, q)
        order = np.argsort(((pts - q) ** 2).sum(1), kind="stable")
        nbr = pts[order][None]
        world, cls = oracle.map_incremental_classify(mc.POSE_A, q[None], nbr, np.array([5], np.int32), True, fs)
        assert np.array_equal(world[0], q)
        mid = (np.floor(q.astype(np.float64) / fs) * fs + 0.5 * fs).astype(F32)
        n0 = nbr[0, 0]
        if branch == "strict_gt" and fs != 0.2:   # 0.5 * 0.2 is no float: the tie exists on exact faces only
            eq = np.abs(n0 - mid).astype(np.float64) == 0.5 * fs
            assert int(eq.sum()) == int(name.split("_")[1][0]), name
        if branch == "strict_lt" and fs != 0.2:
            dq = ((q[0] - mid[0]) * (q[0] - mid[0]) + (q[1] - mid[1]) * (q[1] - mid[1])) + (q[2] - mid[2]) * (q[2] - mid[2])
            dn = [((p[0] - mid[0]) * (p[0] - mid[0]) + (p[1] - mid[1]) * (p[1] - mid[1])) + (p[2] - mid[2]) * (p[2] - mid[2])
                  for p in nbr[0]]
            assert min(dn) == dq, name
        if branch in want and (fs != 0.2 or branch in ("nonneed", "nearer")):   # the ties hold on exact faces only
            assert cls[0] == want[branch], (name, cls[0])
        assert d[4] < 5
