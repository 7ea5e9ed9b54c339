"""GPU: the k-NN work-list hand-over between the stencil kernel and the exact kernel, which runs beside it and takes the
unresolved queries as they are published.  Results must not depend on how many queries go through the list or on what
an earlier search left in it: exact 5-NN against a brute-force float32 restatement (scipy cKDTree candidates) with
many, none and all queries unresolved, and bounded by max_dist; back-to-back device-driven steps, two in flight, whose
unresolved counts alternate between large and small, each bit-equal to the same scan stepped alone in a fresh session;
the largest max_iterations, against the host-driven engine; and the stencil-only debug harness, which must leave the list
empty for the next search."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

from better_fastlio2_b200 import capi, synth
from tests.helpers import knn_equal, sort_rows

pytestmark = pytest.mark.gpu

DS = 0.2


def ref_knn(mp, q, k=5, max_dist=None):
    """Exact k-NN as the kernels define it: float32 squared distances ((dx*dx + dy*dy) + dz*dz), ascending, equal
    distances ordered by (x, y, z), only points with d2 <= max_dist^2 (float32) when bounded.  The candidates come from
    a float64 cKDTree query of 12 neighbours, which holds the float32 top k."""
    mp = np.ascontiguousarray(mp, np.float32)
    q = np.ascontiguousarray(q, np.float32)
    ub = np.inf if max_dist is None else max_dist * 1.001 + 1e-3
    _, idx = cKDTree(mp.astype(np.float64)).query(q.astype(np.float64), k=12, distance_upper_bound=ub)
    ok = idx < len(mp)
    p = mp[np.where(ok, idx, 0)]
    d = q[:, None, :] - p
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    if max_dist is not None:
        ok &= d2 <= np.float32(max_dist) * np.float32(max_dist)
    d2 = np.where(ok, d2, np.float32(np.inf)).astype(np.float32)
    x, y, z = (np.where(ok, p[..., j], np.float32(np.inf)) for j in range(3))
    order = np.lexsort((z, y, x, d2), axis=-1)[:, :k]
    d2 = np.take_along_axis(d2, order, 1)
    xyz = np.take_along_axis(p, order[..., None], 1)
    fin = np.isfinite(d2)
    xyz = np.where(fin[..., None], xyz, np.float32(np.nan)).astype(np.float32)
    return xyz, d2, fin.sum(1).astype(np.int32)


def check_knn(tree, mp, q, max_dist=None):
    xyz, d2, cnt = tree.Nearest_Search(q, 5, max_dist=max_dist or 0.0)
    rx, rd2, rcnt = ref_knn(mp, q, 5, max_dist)
    d2 = np.where(np.arange(5)[None, :] < cnt[:, None], d2, np.float32(np.inf)).astype(np.float32)
    knn_equal(d2, xyz, cnt, rd2, rx, rcnt)
    return cnt


def stencil_unresolved(tree, q, variant=0, iters=1):
    """flb_debug_knn_bench: the stencil kernel (0) or its bulk-copy variant (1) alone; the number of queries it leaves
    to the exact kernel."""
    f = capi.lib().flb_debug_knn_bench
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int),
                  C.c_void_p, C.c_void_p]
    q = np.ascontiguousarray(q, np.float32)
    ms, unres = C.c_float(0), C.c_int(0)
    rc = f(tree.h, q.ctypes.data, len(q), 12, variant, iters, C.byref(ms), C.byref(unres), None, None)
    assert rc == 0, capi.lib().flb_last_error()
    return unres.value


def _tree(points, max_points=1 << 20):
    t = capi.KDTree(voxel_size=DS, max_points=max_points, max_blocks=1 << 17)
    t.Build(np.ascontiguousarray(points, np.float32))
    return t


@pytest.fixture(scope="module")
def world():
    return synth.city_world(half_extent=100.0, seed=21)


@pytest.fixture(scope="module")
def frontier(world):
    """The map is one scan (world frame); the queries are the next scan, taken 5 m further on."""
    rng = np.random.default_rng(5)
    dirs = synth.lidar_dirs("vlp16", rng)
    st0 = synth.trajectory_state(0)
    st1 = st0.copy()
    st1[0] += 5.0
    mp = synth.body_to_world_np(st0, synth.scan_from_pose(world, st0, dirs, rng))
    q = synth.body_to_world_np(st1, synth.scan_from_pose(world, st1, dirs, rng))
    return mp, q


def test_map_frontier(frontier):
    """Tens of thousands of unresolved queries stream through the list while the stencil kernel runs."""
    mp, q = frontier
    t = _tree(mp)
    assert stencil_unresolved(t, q) > 10000
    cnt = check_knn(t, mp, q)
    assert (cnt == 5).all()
    t.close()


def test_nothing_unresolved(world):
    """Queries on a dense map whose 5th neighbour lies well inside the 5x5x5 voxel stencil: the list stays empty and
    the exact kernel ends on the closed list alone."""
    rng = np.random.default_rng(6)
    mp = synth.sample_surface_map(world, (0, 0, 0), 20.0, DS, rng)
    q = (mp[rng.choice(len(mp), 20000, replace=False)] + rng.normal(0, 0.01, (20000, 3))).astype(np.float32)
    d, _ = cKDTree(mp.astype(np.float64)).query(q.astype(np.float64), k=5)
    v = np.floor(q.astype(np.float64) / DS)
    cover = np.minimum(q - (v - 2) * DS, (v + 3) * DS - q).min(1)   # distance to the stencil's faces
    q = np.ascontiguousarray(q[d[:, 4] < 0.8 * cover - 0.01])
    assert len(q) > 1000
    t = _tree(mp)
    assert stencil_unresolved(t, q) == 0
    check_knn(t, mp, q)
    t.close()


def test_everything_unresolved(world):
    """Queries 40-60 m above the map: the stencil finds nothing, every query goes to the exact kernel and on to the
    coarse levels; unbounded and bounded by max_dist (some queries then have fewer than 5 or no neighbours)."""
    rng = np.random.default_rng(7)
    mp = synth.sample_surface_map(world, (0, 0, 0), 15.0, DS, rng)
    q = mp[rng.choice(len(mp), 3000, replace=False)].copy()
    q[:, 2] += rng.uniform(40.0, 60.0, len(q)).astype(np.float32)
    q = np.ascontiguousarray(q, np.float32)
    t = _tree(mp)
    assert stencil_unresolved(t, q) == len(q)
    assert (check_knn(t, mp, q) == 5).all()
    cnt = check_knn(t, mp, q, max_dist=50.0)
    assert (cnt == 0).any() and (cnt == 5).any()
    t.close()


def _scene_scans(world):
    """Two scans of one street: the whole scan (the map covers only |x|, |y| <= 12 m of it, so most of its points are
    unresolved) and the same scan cut to the mapped area (nearly all resolved by the stencil)."""
    rng = np.random.default_rng(8)
    mp = synth.sample_surface_map(world, (0, 0, 0), (12.0, 12.0, 25.0), DS, rng)
    st_true = synth.trajectory_state(0)
    body = synth.scan_from_pose(world, st_true, synth.lidar_dirs("vlp16", rng), rng)
    w = synth.body_to_world_np(st_true, body)
    inside = (np.abs(w[:, 0]) < 10.0) & (np.abs(w[:, 1]) < 10.0)
    scans = []
    for b in (body, body[inside]):
        scans.append(dict(body=np.ascontiguousarray(b), prior=synth.perturb_state(st_true, rng), P=synth.default_cov()))
    return mp, scans


def test_stale_entries_two_in_flight(world):
    """Device-driven steps back to back, two in flight, with large and small unresolved counts alternating: each
    posterior is bit-equal to the same scan stepped alone in a fresh session on a twin map with the same history, and
    agrees with the host-driven engine on that map (update_iterated_dyn_share_modified, as in test_update_engines_agree)."""
    import torch
    mp, (big, small) = _scene_scans(world)
    order = [big, small, big, small, big]
    probe = _tree(mp)
    n_big = stencil_unresolved(probe, synth.body_to_world_np(big["prior"], big["body"]))
    n_small = stencil_unresolved(probe, synth.body_to_world_np(small["prior"], small["body"]))
    probe.close()
    assert n_big > 5000 and n_small * 10 < n_big, (n_big, n_small)
    cap = max(len(sc["body"]) for sc in order)
    t = _tree(mp)
    ses = capi.Session(t, max_scan_points=cap, max_iterations=3)
    devs = []
    for sc in order:
        b4 = np.zeros((len(sc["body"]), 4), np.float32)
        b4[:, :3] = sc["body"]
        devs.append(torch.from_numpy(b4).cuda())
    torch.cuda.synchronize()
    sts = [sc["prior"].copy() for sc in order]
    Ps = [sc["P"].copy() for sc in order]
    ses.scan_set_device(devs[0].data_ptr(), len(order[0]["body"]))
    ses.scan_step_begin(None, sts[0], Ps[0], True)
    for i in range(len(order)):
        if i + 1 < len(order):
            ses.scan_set_device(devs[i + 1].data_ptr(), len(order[i + 1]["body"]))
            ses.scan_step_begin(None, sts[i + 1], Ps[i + 1], True)
        ses.scan_step_finish(None, sts[i], Ps[i])
    ses.close()
    twin = _tree(mp)
    for i, sc in enumerate(order):
        host = capi.Session(twin, max_scan_points=cap, max_iterations=3)
        host.set_update_engine(False)
        host.scan_upload(sc["body"])
        s_h, P_h, _ = host.update_iterated_dyn_share_modified(sc["prior"], sc["P"])
        host.close()
        alone = capi.Session(twin, max_scan_points=cap, max_iterations=3)
        s_a, P_a, _ = alone.scan_step(None, sc["body"], sc["prior"], sc["P"], True)
        alone.close()
        assert np.array_equal(sts[i], s_a) and np.array_equal(Ps[i], P_a), i
        assert np.abs(s_a - s_h).max() < 1e-11, i
        assert np.allclose(P_a, P_h, rtol=1e-7, atol=1e-14), i
    assert np.array_equal(sort_rows(t.flatten()), sort_rows(twin.flatten()))
    t.close()
    twin.close()


def test_max_iterations_7(world):
    """max_iterations = 7, the largest a session accepts: the device-driven sequence holds eight passes, each with its
    own work-list counters zeroed by k_esikf_begin (a ninth pass would use the memset counters of launch_knn, which the
    host-driven engine and Nearest_Search use on every search); it agrees with the host-driven engine."""
    mp, (big, _) = _scene_scans(world)
    prior = big["prior"].copy()
    prior[0:2] += 0.4
    out = {}
    t = _tree(mp)
    for dev in (True, False):
        ses = capi.Session(t, max_scan_points=len(big["body"]), max_iterations=7)
        ses.set_update_engine(dev)
        ses.scan_upload(big["body"])
        out[dev] = ses.update_iterated_dyn_share_modified(prior, big["P"])
        ses.close()
    (s1, P1, st1), (s0, P0, st0) = out[True], out[False]
    for k in ("passes", "search_passes", "effct_feat_num", "converged_count"):
        assert st1[k] == st0[k], k
    assert np.abs(s1 - s0).max() < 1e-11
    assert np.allclose(P1, P0, rtol=1e-7, atol=1e-14)
    with pytest.raises(capi.FlbError):
        capi.Session(t, max_scan_points=16, max_iterations=8)
    t.close()


def test_debug_harness_leaves_the_list_empty(frontier, world):
    """flb_debug_knn_bench fills the list without a consumer (both variants, several launches): the next search and
    the next scan step give what they give on a map that never ran it."""
    mp, q = frontier
    mp2, (big, _) = _scene_scans(world)
    res = []
    for harness in (True, False):
        t = _tree(mp2)
        if harness:
            assert stencil_unresolved(t, q, 0, 3) > 10000
            assert stencil_unresolved(t, q, 1, 2) > 10000
        x, d2, cnt = t.Nearest_Search(q, 5)
        ses = capi.Session(t, max_scan_points=len(big["body"]), max_iterations=3)
        s, P, r = ses.scan_step(None, big["body"], big["prior"], big["P"], True)
        ses.close()
        res.append((x, d2, cnt, s, P, r.map_valid))
        t.close()
    (x1, d1, c1, s1, P1, v1), (x0, d0, c0, s0, P0, v0) = res
    assert np.array_equal(c1, c0) and np.array_equal(d1, d0) and np.array_equal(np.nan_to_num(x1), np.nan_to_num(x0))
    assert np.array_equal(s1, s0) and np.array_equal(P1, P0) and v1 == v0
