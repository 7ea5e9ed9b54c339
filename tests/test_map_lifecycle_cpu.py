"""The lifecycle scenarios' generators (tests/map_lifecycle_cases.py) do what the GPU lifecycle tests rely on: no point
near a voxel face, the corridor really creates far more coarse cells than a coarse table sized for the live map, and a
shortened run of each scenario leaves the same map in our CPU port of the ikd-Tree as in the reference tree."""
import numpy as np
import pytest

from tests import map_lifecycle_cases as mc
from tests.helpers import sort_rows

CORRIDOR_STEPS = 400
PARENT_COARSE_CAP = 2048   # next_pow2(max(1024, max_blocks / 8)) at max_blocks = 1 << 14, the sizing before the coarse rebuild


def test_face_margin_holds():
    cor = mc.Corridor()
    pts = np.concatenate([cor.points(s) for s in range(40)] + [mc.distinct_cells(3000)])
    route = mc.Route(6)
    for k in range(0, 6, 2):
        _, down, verb = route.step(k)
        pts = np.concatenate([pts, down, verb, route.far_queries(k, np.random.default_rng(k))])
    near, far = cor.queries(20, np.random.default_rng(0))
    pts = np.concatenate([pts, near, far])
    f = pts.astype(np.float64) / np.float64(np.float32(mc.DS))
    r = f - np.floor(f)
    assert r.min() >= mc.FACE_MARGIN and r.max() <= 1 - mc.FACE_MARGIN
    # and the float32 division the map keys with agrees with the float64 one on every point
    assert np.array_equal(np.floor(pts / np.float32(mc.DS)).astype(np.int64), np.floor(f).astype(np.int64))


def test_corridor_creates_ten_coarse_tables_of_cells():
    cor = mc.Corridor()
    cells = []
    for s in range(CORRIDOR_STEPS):
        p = cor.points(s)
        assert len(p) == mc.Corridor.PER_STEP
        c, b = mc.coarse_keys(p)
        assert mc.n_unique_rows(c) == len(p)                    # one point, so one block, per coarse cell
        assert np.array_equal(c[:, 0], np.full(len(p), s))      # all in the step's column
        cells.append(c)
    cells = np.concatenate(cells)
    assert mc.n_unique_rows(cells) == len(cells) > 10 * PARENT_COARSE_CAP
    # the delete box of a step removes exactly the columns that left the window
    box = cor.delete_box(30)
    p = np.concatenate([cor.points(s) for s in range(31)])
    inside = ((p >= box[:3]) & (p < box[3:])).all(1)
    assert inside.sum() == (31 - cor.window) * mc.Corridor.PER_STEP
    assert mc.n_unique_rows(mc.coarse_keys(p[~inside])[0]) == cor.live_cells(30)


def test_distinct_cells():
    p = mc.distinct_cells(2049)
    c, _ = mc.coarse_keys(p)
    assert mc.n_unique_rows(c) == 2049


def _run_corridor(m, steps):
    cor = mc.Corridor()
    for s in range(steps):
        if s == 0:
            m.Build(cor.points(s))   # (the reference tree's Add_Points needs a root)
        else:
            m.Add_Points(cor.points(s), True)
        box = cor.delete_box(s)
        if box is not None:
            m.Delete_Point_Boxes(box[None])
    return m.validnum(), sort_rows(m.flatten())


def _run_route(m, steps, oracle):
    route = mc.Route(steps)
    fov = oracle.FovSegment(120.0, 30.0)
    for k in range(steps):
        _, down, verb = route.step(k)
        boxes = fov.step(route.pos_lid(route.truth(k)))
        if len(boxes):
            m.Delete_Point_Boxes(boxes)
        if k == 0:
            m.Build(down)
        else:
            m.Add_Points(down, True)
        m.Add_Points(verb, False)
    return m.validnum(), sort_rows(m.flatten())


@pytest.mark.parametrize("scenario", ["corridor", "route"])
def test_port_matches_reference_tree(oracle, scenario):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    run = (lambda m: _run_corridor(m, 40)) if scenario == "corridor" else (lambda m: _run_route(m, 40, oracle))
    vp, fp = run(oracle.PortMap(ds=mc.DS))
    vr, fr = run(oracle.RefIkdTree(ds=mc.DS))
    assert vp == vr == len(fr) and vr > 0
    assert np.array_equal(fp, fr)
