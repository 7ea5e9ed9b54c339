"""The k-NN edge cases of tests/knn_edge_cases.py are what they claim to be (float properties, keys, which search
region each point falls in, which phase finishes each query) and their float32 brute force agrees with the reference
ikd-Tree on every case: distances bit-equal and points equal as multisets within each tie group."""
import numpy as np
import pytest

from tests import knn_edge_cases as kc

F32 = np.float32


@pytest.fixture(scope="module")
def cases():
    return kc.search_cases()


def _by_prefix(cases, prefix):
    out = [c for c in cases if c["name"].startswith(prefix)]
    assert out, prefix
    return out


def test_outside_keyed_faces():
    """Points keyed across a face from where their coordinate lies exist for the non-binary voxel sizes only, and
    each one is what it claims."""
    for ds in kc.DS_LIST:
        found = kc.outside_keyed_faces(ds, 300)
        for k, x, side in found:
            f = kc.face(k, ds)
            if side > 0:
                assert x < f and kc.key(x, ds) == k
            else:
                assert x >= f and kc.key(x, ds) == k - 1
        if ds in (0.25, 0.5, 1.0):
            assert not found, ds
        else:
            assert len(found) > 10, ds
    # about one face in ten at 0.2 holds a point a few float steps below fl(k ds) keyed to voxel k
    n = sum(1 for _, _, s in kc.outside_keyed_faces(0.2, 300) if s > 0)
    assert 0.05 * 300 < n < 0.25 * 300, n


def test_face_cases_sit_on_faces(cases):
    for c in _by_prefix(cases, "faces_"):
        ds = c["ds"]
        for a in (c["map"], c["queries"]):
            v = a[np.isfinite(a)].ravel()
            k = np.round(v.astype(np.float64) / ds)
            near = np.abs(v - (k * ds).astype(F32)) <= 4 * np.spacing(np.abs((k * ds).astype(F32)) + F32(1e-30))
            assert (near | (np.abs(v) < 1e-37)).all(), c["name"]
        assert (c["map"] == 0).any() and np.signbit(c["map"][c["map"] == 0]).any(), c["name"]


def test_completeness_cases(cases):
    """The K-th neighbour is keyed inside the region within [c - mg, c + ulps] of its face, the competitor keyed
    outside it one float step nearer or farther; the region's stop test fails and the intended next phase finishes."""
    for c in _by_prefix(cases, "complete_"):
        ds, q, comp, kth = c["ds"], c["queries"][0], c["comp"], c["kth"]
        k = c["face_k"]
        f = kc.face(k, ds)
        assert comp[0] <= f and kc.key(comp[0], ds) == k, c["name"]           # keyed outside, not beyond the face
        assert kc.key(kth[0], ds) < k, c["name"]
        dcomp, dk = kc.sqdist(q, comp), kc.sqdist(q, kth)
        assert (dcomp < dk) == (c["variant"] == "near"), c["name"]
        assert abs(int(dk.view(np.int32)) - int(dcomp.view(np.int32))) <= 3, c["name"]
        cdist = F32(f - q[0])
        mg = kc.margin(q, ds)
        assert F32(cdist - mg) ** 2 <= dk <= np.nextafter(cdist * cdist, F32(np.inf), dtype=F32) * F32(1 + 1e-6), c["name"]
        ph, r = kc.expected_phase(c["map"], q, ds, kc.K_SCAN)
        assert ph == kc.NEXT_PHASE[c["region"]], (c["name"], ph, r)
        if c["region"].startswith("ring") and c["region"] != "ring8":
            assert r == int(c["region"][4:]) + 1, (c["name"], r)
        # the +x face is the region's nearest; without the margin its stop test would pass, and lose the nearer competitor
        own = {"stencil": (0, 0), "coarse": (2, 0)}.get(c["region"]) or (1, int(c["region"][4:]))
        if c["variant"] == "near" and ds not in (0.25, 0.5, 1.0):
            assert kc.expected_phase(c["map"], q, ds, kc.K_SCAN, margin_scale=0.0) == own, c["name"]
        # the K-th neighbour overall is the nearer of the two
        _, d2, _ = kc.brute(c["map"], c["queries"], kc.K_SCAN)
        assert d2[0, -1] == min(dcomp, dk)


def test_tie_cases(cases):
    for c in _by_prefix(cases, "tie_"):
        q = c["queries"][0].astype(np.float64)
        d, p, _ = kc.candidates(c["map"], c["queries"][0])
        d64 = ((p.astype(np.float64) - q) ** 2).sum(1)
        # the tie is exact in float64 geometry too (coordinates on a 1/64 grid)
        vals, counts = np.unique(d, return_counts=True)
        assert counts.max() >= 2, c["name"]
        for v in vals[counts >= 2]:
            assert np.ptp(d64[d == v]) == 0, c["name"]
        pos = np.nonzero(d == d[kc.K_SCAN - 1])[0]
        assert pos.min() < kc.K_SCAN - 1 + 1 <= pos.max() + 1 and len(d) > kc.K_SCAN, c["name"]   # straddles position K
        ph, r = kc.expected_phase(c["map"], c["queries"][0], c["ds"], kc.K_SCAN)
        if c["lex_exact"]:
            qb = kc.key(c["queries"][0], c["ds"]) >> 2
            assert np.abs((kc.key(c["ring1"], c["ds"]) >> 2) - qb).max() == 1, c["name"]
            assert np.abs((kc.key(c["ring2"], c["ds"]) >> 2) - qb).max() == 2, c["name"]
            assert (ph, r) == (1, 2), c["name"]
        else:
            assert ph == 0, c["name"]


def test_max_dist_cases():
    """The float square rounds up for 0.1, so a point at d2 = fl(md * md) lies beyond the reference's bound.  It rounds
    down for 0.3, 0.7 and 1.3; a rounded-down nearest float is already the largest float not above the double square,
    so there the two bounds agree."""
    for c in kc.max_dist_cases():
        m = c["max_dist"]
        fsq, dsq = c["fsq"], c["dsq"]
        exact = float(m) * float(m)
        assert float(dsq) <= exact < float(np.nextafter(dsq, F32(np.inf), dtype=F32))
        if float(m) in (float(F32(0.1)),):
            assert float(fsq) > exact
        if float(m) in (float(F32(0.3)), float(F32(0.7)), float(F32(1.3))):
            assert float(fsq) < exact and dsq == fsq
        d = kc.sqdist(c["queries"][0], c["map"])
        for t in (fsq, dsq, kc.step(dsq, 1)):
            assert (d == t).any(), (c["name"], t)
        _, _, cnt = kc.brute(c["map"], c["queries"], 20, m)
        assert cnt[0] == int((d <= dsq).sum())


def _ref_search(oracle, c, k):
    t = oracle.make_map(ds=c["ds"])
    if len(c["map"]):
        t.Build(c["map"])
    qs = c["queries"][np.isfinite(c["queries"]).all(1)]
    if c["max_dist"] is not None:
        assert isinstance(t, oracle.RefIkdTree)
        r = t.Nearest_Search_md(qs, k, float(c["max_dist"]))
    else:
        r = t.Nearest_Search(qs, k)
    t.close()
    return qs, r


@pytest.mark.parametrize("k", [1, 5, 20])
def test_brute_matches_reference(oracle, cases, k):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    bad = {}
    for c in cases:
        if len(c["map"]) == 0:
            continue
        qs, (xyz, d2, cnt) = _ref_search(oracle, c, k)
        b = kc.check_knn(c["map"], qs, k, xyz, d2, cnt, c["max_dist"])
        if b:
            bad[c["name"]] = b[:3]
    assert not bad, bad


def test_reference_max_dist_is_double(oracle):
    """The reference keeps d2 <= max_dist^2 in double: a float-square bound disagrees with it on these cases."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    differs = []
    for c in kc.max_dist_cases():
        _, (xyz, d2, cnt) = _ref_search(oracle, c, 20)
        d = kc.sqdist(c["queries"][0], c["map"])
        assert cnt[0] == int((d <= c["dsq"]).sum()), c["name"]
        if cnt[0] != int((d <= c["fsq"]).sum()):
            differs.append(c["name"])
    assert differs == ["max_dist_0.1"]


def _ref_replay(oracle, ops, ds=0.2):
    t = oracle.RefIkdTree(ds=ds)
    for op, a in ops:
        if op == "build":
            t.Build_xyzi(a)
        elif op == "delete":
            t.Delete_Points(a)
        else:
            t.Add_Points_xyzi(a, False)
    return t


def test_chains_and_duplicates_reference(oracle):
    """The chain and duplicate scenes: the reference's content after the same operations is the constructed content,
    and its k-NN with intensities agrees with the brute force (records compared as multisets per tie group)."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    ops, final, qs = kc.chain_ops()
    pts4, dq = kc.duplicate_points()
    for ops_, content, q in ((ops, final, qs), ([("build", pts4)], pts4, dq)):
        t = _ref_replay(oracle, ops_)
        got = t.flatten_xyzi()
        assert sorted(kc._rows(got)) == sorted(kc._rows(content))
        for k in (1, 5, 20):
            out, d2, cnt = t.Nearest_Search_xyzi(q, k)
            bad = kc.check_knn(content[:, :3], q, k, out[..., :3], d2, cnt, extra=out[..., 3:], mp_extra=content[:, 3:])
            assert not bad, bad[:3]
        t.close()


def test_reference_searches_out_of_range_queries(oracle):
    """Finite queries beyond the map's coordinate bound get neighbours from the reference (the GPU map returns none:
    DESIGN.md section 5)."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    q = kc.out_of_range_queries(0.2)
    q = q[np.isfinite(q).all(1)]
    t = oracle.make_map(ds=0.2)
    t.Build(np.array([[0, 0, 0], [1, 1, 1]], F32))
    _, _, cnt = t.Nearest_Search(q, 1)
    assert (cnt == 1).all()
    t.close()
