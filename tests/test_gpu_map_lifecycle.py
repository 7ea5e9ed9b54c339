"""The device map driven for a long run as a node drives it — a sliding window that inserts ahead and deletes behind, scan
after scan — against the reference ikd-Tree fed the same operations through the map API (no closed loop: nothing can
diverge between the two).  This is the regime that exercises the block and overflow free stacks, tombstones and rehashes,
and the coarse level (cells created and emptied, rebuilt from the live blocks) that far searches walk.  The file runs in
about 40 s on one H100.

Generated points keep 0.01 * ds from every voxel face and tie rows are compared with knn_equal (DESIGN.md §5, the two
documented deviations), so every comparison with the reference is exact."""
import time

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import map_lifecycle_cases as mc
from tests.helpers import knn_equal, sort_rows

pytestmark = pytest.mark.gpu

CHECK_EVERY = 25


def _compare(t, ref, queries):
    assert np.array_equal(sort_rows(t.flatten()), sort_rows(ref.flatten()))
    for q in queries:
        if len(q):
            xg, dg, cg = t.Nearest_Search(q, 5)
            xr, dr, cr = ref.Nearest_Search(q, 5)
            knn_equal(dg, xg, cg, dr, xr, cr)


def _ref_validnum(ref, timeout=10.0):
    """validnum of the reference tree, which answers -1 while its background rebuild holds the tree (ikd_Tree.cpp:129-145)."""
    deadline = time.monotonic() + timeout
    while True:
        v = ref.validnum()
        if v >= 0:
            return v
        assert time.monotonic() < deadline, f"the reference tree's rebuild held it for more than {timeout} s"
        time.sleep(0.001)


def test_sparse_corridor(oracle):
    """64 points per step, each alone in its own coarse cell, window of 8 columns: every delete empties whole coarse cells.
    The coarse level must stay bounded by the live cells (a table sized for the live map used to fill up after ~32 steps
    and fail every later call with "coarse hash full", long before any rehash)."""
    steps = 400
    t = capi.KDTree(voxel_size=mc.DS, max_points=1 << 16, max_blocks=1 << 14)
    ref = oracle.make_map(ds=mc.DS)
    cor = mc.Corridor()
    rng = np.random.default_rng(1)
    for s in range(steps):
        p = cor.points(s)
        if s == 0:   # (the reference tree's Add_Points needs a root)
            t.Build(p)
            ref.Build(p)
        else:
            t.Add_Points(p, True)
            ref.Add_Points(p, True)
        box = cor.delete_box(s)
        if box is not None:
            assert t.Delete_Point_Boxes(box[None]) == ref.Delete_Point_Boxes(box[None]) == mc.Corridor.PER_STEP, s
        assert t.validnum() == _ref_validnum(ref) == cor.live_cells(s), s
        st = t.stats()
        assert st["blocks_in_use"] == cor.live_cells(s), (s, st)
        assert st["coarse_cells"] <= cor.live_cells(s), (s, st)   # one block per cell: no more cells than live blocks
        if s % CHECK_EVERY == 0 or s == steps - 1:
            _compare(t, ref, cor.queries(s, rng))
    assert steps * mc.Corridor.PER_STEP > 10 * 2048
    t.close()


def test_build_more_coarse_cells_than_an_eighth_of_the_blocks(oracle):
    """A Build whose points all sit in different coarse cells, more of them than max_blocks / 8 (the coarse table's size
    before it was sized by max_blocks), with max_blocks well above the point count: it succeeds and searches exactly."""
    max_blocks = 1 << 16
    n = max_blocks // 8 + 1
    pts = mc.distinct_cells(n)
    t = capi.KDTree(voxel_size=mc.DS, max_points=1 << 17, max_blocks=max_blocks)
    ref = oracle.make_map(ds=mc.DS)
    t.Build(pts)
    ref.Build(pts)
    assert t.validnum() == _ref_validnum(ref) == n
    st = t.stats()
    assert st["coarse_cells"] == st["blocks_in_use"] == n
    rng = np.random.default_rng(2)
    lo, hi = pts.min(0), pts.max(0)
    near = mc.face_filter(rng.uniform(lo, hi, (2000, 3)).astype(np.float32))
    far = mc.face_filter((rng.uniform(lo, hi, (64, 3)) + np.array([0, 0, 1.5 * (hi[2] - lo[2])])).astype(np.float32))
    _compare(t, ref, (near, far))
    mc.assert_knn_exact(pts, far, *t.Nearest_Search(far, 5))
    t.close()


ROUTE_STEPS = 360
ROUTE_MAX_BLOCKS = 1 << 14   # the live window peaks at ~14k blocks; ~53k distinct blocks are allocated over the route


@pytest.fixture(scope="module")
def route():
    r = mc.Route(ROUTE_STEPS)
    r.steps = [r.step(k) for k in range(ROUTE_STEPS)]
    return r


def test_driven_route(oracle, route):
    """Delete boxes of lasermap_fov_segment (cube 120 m, detection range 30 m), then the downsampled scan and a verbatim
    batch inserted, every step, and 40 points deleted by Delete_Points every 10th step.  max_blocks holds the live window
    with margin but not everything the route allocates, so the run succeeds only if freed blocks are reused, and it goes
    through at least three rehashes.

    Delete_Points is checked on the device map's own content: the reference tree's result for it varied by a point
    between identical runs (its background rebuild thread), so after each such delete the reference is rebuilt from the
    device map's (checked) content and the comparison goes on from there."""
    t = capi.KDTree(voxel_size=mc.DS, max_points=1 << 18, max_blocks=ROUTE_MAX_BLOCKS)
    ref = oracle.make_map(ds=mc.DS)
    fov = oracle.FovSegment(120.0, 30.0)
    rng = np.random.default_rng(4)
    peak = 0
    seen = set()
    for k in range(ROUTE_STEPS):
        _, down, verb = route.steps[k]
        boxes = fov.step(route.pos_lid(route.truth(k)))
        if len(boxes):
            assert t.Delete_Point_Boxes(boxes) == ref.Delete_Point_Boxes(boxes), k
        if k == 0:
            t.Build(down)
            ref.Build(down)
        else:
            t.Add_Points(down, True)
            ref.Add_Points(down, True)
        t.Add_Points(verb, False)
        ref.Add_Points(verb, False)
        if k % 10 == 5:
            before = t.flatten()
            gone = before[rng.choice(len(before), 40, replace=False)]
            keep = ~(np.abs(before[:, None, :] - gone[None, :, :]) < 1e-6).all(2).any(1)   # same_point: every copy goes
            assert t.Delete_Points(gone) == int((~keep).sum()), k
            after = t.flatten()
            assert np.array_equal(sort_rows(after), sort_rows(before[keep])), k
            ref.close()   # a fresh tree: Build on a tree whose background rebuild is running is not safe
            ref = oracle.make_map(ds=mc.DS)
            ref.Build(after)
        assert t.validnum() == _ref_validnum(ref), k
        st = t.stats()
        # max_blocks is a power of two: the coarse level holds no more cells than there are live blocks
        assert st["coarse_cells"] <= st["blocks_in_use"], (k, st)
        if k % 5 == 0 or len(boxes) or k == ROUTE_STEPS - 1:
            content = t.flatten()
            blocks = {tuple(b) for b in np.unique(mc.coarse_keys(content)[1], axis=0)}
            assert st["blocks_in_use"] == len(blocks), (k, st)   # empty blocks go back to the free stack
            seen |= blocks
            peak = max(peak, len(blocks))
        if k % CHECK_EVERY == 0 or k == ROUTE_STEPS - 1:
            q = mc.face_filter(down[rng.choice(len(down), min(256, len(down)), replace=False)]
                               + rng.normal(0, 0.3, (min(256, len(down)), 3)).astype(np.float32))
            far = route.far_queries(k, rng)
            _compare(t, ref, (q, far))
            content = t.flatten()
            for qq in (q, far):
                mc.assert_knn_exact(content, qq, *t.Nearest_Search(qq, 5))
    st = t.stats()
    print(f"[route] peak live blocks {peak}, distinct blocks over the route {len(seen)}, stats {st}")
    assert peak < ROUTE_MAX_BLOCKS < len(seen)
    assert st["rehash_count"] >= 3, st
    t.close()


SCAN_MAX_BLOCKS = 1 << 15


def test_scan_path_route(route):
    """The same route through Session.scan_step with lasermap_fov_segment on the device: the scan path's own inserts
    (classified and fused into the scan's kernels), its box deletes and the map checks at the end of each step, 359 steps.
    Priors are the truth plus 2 cm / 0.2 deg noise.  Every step succeeds, and the map stays consistent: the block count is
    the number of blocks its content occupies, the coarse level holds no more cells than there are blocks, freed blocks
    are reused (the route allocates more blocks than max_blocks), and 5-NN over the final map, near and far, equals brute
    force.

    The posterior is not held to the truth: the map is built from the posteriors, and on this route the estimate drifts
    upwards by a few millimetres per scan (the CPU restatement of the reference's update and map_incremental drifts the
    same way: 3 cm after 20 scans, 7 cm after 40, 25 cm after 100); only a gross failure is caught."""
    t = capi.KDTree(voxel_size=mc.DS, max_points=1 << 19, max_blocks=SCAN_MAX_BLOCKS)
    rng = np.random.default_rng(5)
    bodies = [synth.voxel_downsample(b, 0.5) for b, _, _ in route.steps]
    t.Build(synth.sample_surface_map(route.world, route.truth(0)[:3], 20.0, mc.DS, rng))   # the map a node has by then
    ses = capi.Session(t, max_scan_points=max(len(b) for b in bodies), max_iterations=4)
    fov = capi.make_fov(120.0, 30.0)
    P = synth.default_cov()
    peak, seen, worst = 0, set(), 0.0
    for k in range(1, ROUTE_STEPS):
        truth = route.truth(k)
        prior = synth.perturb_state(truth, rng, sig_pos=0.02, sig_rot_deg=0.2)
        st, _, r = ses.scan_step(fov, bodies[k], prior, P, True)   # fov keeps the previous posterior's LiDAR position
        worst = max(worst, float(np.abs(st[:3] - truth[:3]).max()))
        assert np.abs(st[:3] - truth[:3]).max() < 2.0, (k, st[:3], truth[:3])
        stats = t.stats()
        assert r.map_valid == stats["valid_points"], k
        assert stats["coarse_cells"] <= stats["blocks_in_use"], (k, stats)
        if k % 5 == 0 or k == ROUTE_STEPS - 1:
            content = t.flatten()
            blocks = {tuple(b) for b in np.unique(mc.coarse_keys(content)[1], axis=0)}
            assert stats["blocks_in_use"] == len(blocks), (k, stats)
            seen |= blocks
            peak = max(peak, len(blocks))
    stats = t.stats()
    print(f"[scan path] worst position error {worst:.3f} m, peak live blocks {peak}, distinct blocks {len(seen)}, stats {stats}")
    assert peak < SCAN_MAX_BLOCKS < len(seen)
    assert stats["rehash_count"] >= 1, stats
    content = t.flatten()
    q = content[rng.choice(len(content), 256, replace=False)] + rng.normal(0, 0.3, (256, 3)).astype(np.float32)
    for qq in (q.astype(np.float32), route.far_queries(ROUTE_STEPS - 1, rng)):
        mc.assert_knn_exact(content, qq, *t.Nearest_Search(qq, 5))
    ses.close()
    t.close()
