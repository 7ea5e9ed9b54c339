"""GPU: Nearest_Search on the constructed k-NN edge cases of tests/knn_edge_cases.py (voxel, block and coarse faces, the
completeness test of every search phase, exact ties, overflow chains, sparse and far maps, the max_dist bound) for every
k from 1 to 20, against the float32 brute force with a comparator stricter than helpers.knn_equal; the scan path's
5-NN on the same queries, with the phase that finished each family; and the reference ikd-Tree on the same cases."""
import ctypes as C

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import knn_edge_cases as kc

pytestmark = pytest.mark.gpu

F32 = np.float32
KS = range(1, 21)


def _tree(ds, max_points=1 << 14):
    return capi.KDTree(voxel_size=ds, max_points=max_points, max_blocks=1 << 12)


def _built(c):
    t = _tree(c["ds"])
    if len(c["map"]):
        t.Build(c["map"])
    return t


@pytest.fixture(scope="module")
def cases():
    return kc.search_cases()


def _exact_rows(c):
    """Queries the exact kernel finishes (the stencil left them unresolved): their tie groups are in (x, y, z) order."""
    return np.array([kc.expected_phase(c["map"], q, c["ds"], kc.K_SCAN, c["max_dist"])[0] > 0 for q in c["queries"]])


def test_every_k_on_every_case(cases):
    bad = {}
    for c in cases:
        t = _built(c)
        md = 0.0 if c["max_dist"] is None else float(c["max_dist"])
        lex = _exact_rows(c)
        for k in KS:
            xyz, d2, cnt = t.Nearest_Search(c["queries"], k, max_dist=md)
            b = kc.check_knn(c["map"], c["queries"], k, xyz, d2, cnt, c["max_dist"], lex=lex if k == kc.K_SCAN else None)
            if c.get("lex_exact") and k == kc.K_SCAN:
                bx, _, _ = kc.brute(c["map"], c["queries"], k, c["max_dist"])
                if not np.array_equal(bx.view(np.uint32), xyz.view(np.uint32)):
                    b.append(f"tie rule: {xyz.tolist()} != {bx.tolist()}")
            if b:
                bad[(c["name"], k)] = b[:2]
        t.close()
    assert not bad, dict(list(bad.items())[:12])


def test_max_dist_against_reference(oracle):
    """Neighbours at d2 = fl(md * md), at the largest float not above the double square and a step either side: the
    counts are the reference's (called with the same float widened to double)."""
    for c in kc.max_dist_cases():
        t = _built(c)
        xyz, d2, cnt = t.Nearest_Search(c["queries"], 20, max_dist=float(c["max_dist"]))
        t.close()
        assert not kc.check_knn(c["map"], c["queries"], 20, xyz, d2, cnt, c["max_dist"]), c["name"]
        if oracle.have_ref():
            r = oracle.RefIkdTree(ds=c["ds"])
            r.Build(c["map"])
            rx, rd2, rc = r.Nearest_Search_md(c["queries"], 20, float(c["max_dist"]))
            r.close()
            assert np.array_equal(rc, cnt) and np.array_equal(rd2, d2), c["name"]


def test_out_of_range_queries_get_no_neighbours():
    """Queries at or beyond 4e6 ds per axis, infinite or NaN: no neighbours (DESIGN.md section 5)."""
    for ds in kc.DS_LIST:
        t = _tree(ds)
        t.Build(np.array([[0, 0, 0], [ds, ds, ds]], F32))
        q = kc.out_of_range_queries(ds)
        xyz, d2, cnt = t.Nearest_Search(q, 5)
        assert (cnt == 0).all() and np.isinf(d2).all() and np.isnan(xyz).all(), ds
        t.close()


def _replay(ops, max_points=1 << 14):
    t = _tree(0.2, max_points)
    for op, a in ops:
        if op == "build":
            t.Build_xyzi(a)
        elif op == "delete":
            t.Delete_Points(a)
        else:
            t.Add_Points_xyzi(a, False)
    return t


def _check_xyzi(t, content, q, oracle=None, ops=None):
    for k in KS:
        out, d2, cnt = t.Nearest_Search_xyzi(q, k)
        bad = kc.check_knn(content[:, :3], q, k, out[..., :3], d2, cnt, extra=out[..., 3:], mp_extra=content[:, 3:])
        assert not bad, (k, bad[:3])
        xyz, d2b, cntb = t.Nearest_Search(q, k)
        assert np.array_equal(d2b, d2) and np.array_equal(cntb, cnt)
    if oracle is not None and oracle.have_ref():
        r = oracle.RefIkdTree(ds=0.2)
        for op, a in ops:
            r.Build_xyzi(a) if op == "build" else (r.Delete_Points(a) if op == "delete" else r.Add_Points_xyzi(a, False))
        for k in (5, 20):
            ro, rd, rc = r.Nearest_Search_xyzi(q, k)
            go, gd, gc = t.Nearest_Search_xyzi(q, k)
            assert np.array_equal(rc, gc) and np.array_equal(rd, gd)
            for i in range(len(q)):
                # the reference's order of equal records depends on its traversal: multisets per query, without the
                # tie group at position k when it is cut there (which of its members are kept is traversal order too)
                n = int(rc[i])
                if n == k:
                    n = int(np.nonzero(rd[i, :n] == rd[i, n - 1])[0][0])
                assert sorted(kc._rows(ro[i, :n])) == sorted(kc._rows(go[i, :n])), (k, i)
        r.close()


def test_overflow_chains(oracle):
    """Chains from a verbatim Build with heads, middles and tails deleted, then a verbatim insert into the freed nodes."""
    ops, final, qs = kc.chain_ops()
    t = _replay(ops)
    assert sorted(kc._rows(t.flatten_xyzi())) == sorted(kc._rows(final))
    _check_xyzi(t, final, qs, oracle, ops)
    t.close()


def test_duplicate_intensities(oracle):
    """Duplicated coordinates with distinct intensities: every duplicate returned carries its own record's intensity."""
    pts4, qs = kc.duplicate_points()
    t = _replay([("build", pts4)])
    _check_xyzi(t, pts4, qs, oracle, [("build", pts4)])
    t.close()


def test_chains_to_the_end_of_the_pool():
    """max_points = 2048: a Build whose chains take all 1024 overflow nodes, the last of them included."""
    pts, qs = kc.pool_end_points()
    t = _tree(0.2, 2048)
    t.Build(pts)
    assert t.validnum() == len(pts)
    for k in KS:
        xyz, d2, cnt = t.Nearest_Search(qs, k)
        bad = kc.check_knn(pts, qs, k, xyz, d2, cnt)
        assert not bad, (k, bad[:3])
    t.close()


def _stencil_unresolved(tree, q):
    f = capi.lib().flb_debug_knn_bench
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int),
                  C.c_void_p, C.c_void_p]
    q = np.ascontiguousarray(q, F32)
    ms, unres = C.c_float(0), C.c_int(0)
    assert f(tree.h, q.ctypes.data, len(q), 12, 0, 1, C.byref(ms), C.byref(unres), None, None) == 0
    return unres.value


def test_scan_path_phases(cases):
    """The scan path's 5-NN (h_share_model at the identity pose, the queries as the body points) equals the brute
    force; every completeness and tie family finishes in the phase it targets (knn_phase), and the stencil leaves
    exactly the queries it cannot prove complete."""
    state = synth.make_state(offT=(0.0, 0.0, 0.0))
    groups = {}
    for c in cases:
        if c["name"].startswith(("complete_", "tie_", "faces_", "sparse", "far")) and len(c["map"]) and c["max_dist"] is None:
            groups.setdefault(c["name"], c)
    for name, c in groups.items():
        t = _built(c)
        q = c["queries"][np.isfinite(c["queries"]).all(1)]
        want = np.array([kc.expected_phase(c["map"], p, c["ds"], kc.K_SCAN)[0] for p in q])
        assert _stencil_unresolved(t, q) == int((want > 0).sum()), name
        t.profile_enable(True)
        t.profile_read(reset=True)
        ses = capi.Session(t, max_scan_points=max(len(q), 16), max_iterations=1, filter_size_map_min=c["ds"])
        ses.scan_upload(q)
        ses.h_share_model(state, True)
        nb = ses.neighbors()
        assert np.array_equal(nb["world"], q), name
        bad = kc.check_knn(c["map"], q, kc.K_SCAN, nb["nbr"], nb["d2"], nb["cnt"], lex=want > 0)
        assert not bad, (name, bad[:3])
        ph = t.profile_read(reset=True)["knn_phase"]
        assert ph == [int((want == j).sum()) for j in range(4)], (name, ph)
        ses.close()
        t.close()
