"""CPU checks of the constructed grid-search cases (tests/icp_grid_cases.py): every case exercises what it claims, on the
float32 restatement of the registrations' grid, and the brute-force reference agrees bit for bit with the k-d tree 1-NN of
tests/cpp/icp_oracle.cpp, which the GPU ICP tests rely on at ties."""
import numpy as np
import pytest

from tests import icp_grid_cases as gc
from tests import icp_oracle as io

F = np.float32
CASES = gc.cases()


def _ids():
    return [c.name for c in CASES]


@pytest.mark.parametrize("case", CASES, ids=_ids())
def test_brute_force_equals_the_kd_tree_oracle(case):
    bi, bd = gc.brute_nn(case.qry, case.tgt)
    oi, od = io.nearest(case.qry, case.tgt)
    assert np.array_equal(bi, oi), (case.name, np.nonzero(bi != oi)[0][:5])
    assert np.array_equal(bd.view(np.uint32), od.view(np.uint32)), case.name


def _cheb(a, b):
    return np.abs(a - b).max(1)


@pytest.mark.parametrize("case", CASES, ids=_ids())
def test_each_case_exercises_what_it_claims(case):
    c, g = case.claims, gc.grid_of(case.tgt)
    fin = np.isfinite(case.tgt).all(1)
    t = case.tgt[fin]
    bi, bd, cnt, second = gc.brute_nn(case.qry, case.tgt, ties=True)
    qc = gc.cells(g, case.qry)
    wc = gc.cells(g, case.tgt[np.maximum(bi, 0)])
    ring = _cheb(qc, wc)

    def tied_cells(j):
        """The cells of every target at query j's best d²."""
        d = case.tgt[:, :3] - case.qry[j]
        with np.errstate(over="ignore", invalid="ignore"):
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        return gc.cells(g, case.tgt[d2 == bd[j]])

    if "binned_across" in c:   # float binning puts a point one cell away from where its coordinate lies
        assert (gc.raw_cells(g, t) != gc.exact_cells(g, t)).any(1).sum() >= c["binned_across"]
    if "binned_across_coarse" in c:
        raw, ex = gc.raw_cells(g, t), gc.exact_cells(g, t)
        assert ((raw // gc.ICP_C) != (ex // gc.ICP_C)).any(1).sum() >= c["binned_across_coarse"]
    if "tie_across_cells" in c:
        n = sum(1 for j in np.flatnonzero(cnt >= 2) if len(np.unique(tied_cells(j), axis=0)) > 1)
        assert n >= c["tie_across_cells"], n
    if "one_step_apart" in c:   # the pair one coordinate step apart: the runner-up within 1e-4 relative, not tied
        with np.errstate(invalid="ignore"):
            assert ((second > bd) & (second - bd <= 1e-4 * bd)).sum() >= c["one_step_apart"]
    if "ring2" in c:   # the handoff: the nearest target at the last fine ring and at the first coarse-walk ring
        assert (ring == 2).sum() >= c["ring2"] and (ring == 3).sum() >= c["ring3"], np.bincount(ring)
        assert (ring == 3).sum() > 0 and max(ring) >= 3
    if "ties" in c:
        for k in c["ties"]:
            assert (cnt == k).sum() > 100, (k, np.bincount(cnt))
        assert set(np.unique(cnt)) == set(c["ties"])
    if "far_ties" in c:   # one tied target inside the fine rings, the other reachable only by the far path
        n = 0
        for j in np.flatnonzero(cnt == 2):
            r = sorted(_cheb(tied_cells(j), qc[j][None]))
            n += r[0] <= gc.ICP_RINGS < r[1] and not gc.ring_done(g, case.qry[j], qc[j], gc.ICP_RINGS + 1, bd[j])
        assert n >= c["far_ties"], n
    if "min_coarse_ring" in c:
        assert _cheb(qc // gc.ICP_C, wc // gc.ICP_C).min() >= c["min_coarse_ring"]
    if "outside" in c:
        q = case.qry[:c["outside"]]
        lo, hi = t.min(0), t.max(0)
        assert ((q < lo) | (q > hi)).any(1).all()
        raw = gc.raw_cells(g, q)
        assert ((raw < 0) | (raw >= np.array(g.dims))).any(1).sum() > len(q) // 2   # the border clamp
        assert (np.abs(q - (lo + hi) / 2).max(1) > 900).sum() >= 100                   # 1 km out
        ov = slice(c["outside"], c["outside"] + c["overflow"])
        assert np.isinf(bd[ov]).all() and (bi[ov] == np.flatnonzero(fin)[0]).all() and np.flatnonzero(fin)[0] > 0
    if "n_fin" in c:
        assert fin.sum() == c["n_fin"] and g.dims == (8, 8, 8)
    if "zero_extent" in c:
        assert (t.max(0) == t.min(0)).sum() == c["zero_extent"]
        if c["zero_extent"] == 3:
            assert (cnt[np.isfinite(case.qry).all(1)] == len(t)).all() and (bi == 0).all()   # every target tied: index 0
    if "gz" in c:
        assert g.dims[2] == c["gz"]
    if "tiny" in c:
        ext = t.max(0).astype(np.float64) - t.min(0)
        assert 0 < ext.max() <= c["tiny"]
    if "mult8" in c:   # floor(ext / e) + 1 on (8) or one past (9) a multiple of 8, within an ulp of the integer
        k = c["mult8"]
        assert all(abs(r - 8.0) < 1e-12 and int(np.floor(r)) + 1 == k for r in g.ext_over_e)
        assert g.dims == ((8, 8, 8) if k == 8 else (16, 16, 16))
        # the far corner bins to cell 8 either way: the last cell of the 16-cell axis, or clamped into cell 7 of the 8-cell one
        assert (gc.raw_cells(g, t) == 8).any()
    if "slack_from_coordinates" in c:
        assert F(4e-6) * F(np.abs(t).max()) > F(1e-3) * g.e
    if "open_after_fine_rings" in c:
        assert g.slack > 50 * g.e
        assert not any(gc.ring_done(g, case.qry[j], qc[j], r, bd[j]) for j in range(0, len(case.qry), 7)
                       for r in range(1, gc.ICP_RINGS + 2))
    if "gate" in c:
        md, n_lo, n_at, n_hi = c["gate"]
        M = md * md
        top = F(M) if float(F(M)) <= M else np.nextafter(F(M), F(0))
        assert (bd == np.nextafter(top, F(0))).sum() == n_lo and (bd == top).sum() == n_at
        assert (bd == np.nextafter(top, F(np.inf))).sum() == n_hi and float(np.nextafter(top, F(np.inf))) > M
        assert (bi == np.arange(len(bi))).all()
    if "slack_traps" in c:   # the nearest target lies in a cell only the slack keeps: slack 0 gives a wrong answer
        m0, n, least = c["slack_traps"]
        assert n >= least and m0 + n == len(case.qry)
        index = gc.cell_index(g, case.tgt)
        for j in range(m0, m0 + n):
            closed, i0, d0 = gc.fine_search(g, case.tgt, case.qry[j], index, slack=0.0)
            assert closed and (i0, d0) != (bi[j], bd[j]), j
            assert gc.raw_cells(g, case.tgt[bi[j]][None])[0].tolist() != gc.exact_cells(g, case.tgt[bi[j]][None])[0].tolist()
            closed, i1, d1 = gc.fine_search(g, case.tgt, case.qry[j], index)
            assert not closed or (i1, d1.view(np.uint32)) == (bi[j], bd[j].view(np.uint32)), j
    if "knn7_outside" in c:
        assert gc.knn7_outside_fraction(case) >= c["knn7_outside"]


def test_both_multiple_of_8_boxes_are_present():
    assert sorted(c.claims["mult8"] for c in CASES if "mult8" in c.claims) == [8, 9]


def test_lattice_takes_one_cap_step_and_its_analytic_answer_is_exact():
    """Family h: the 256³ lattice at 0.125 m first sizes to 520³ > 2^27 cells and takes one 1.25 step to 416³; the analytic
    nearest lattice point equals the brute force and the k-d tree on a sub-lattice of the queries."""
    n = gc.LATTICE_N
    top = (n - 1) * gc.LATTICE_PITCH
    g = gc.grid((0, 0, 0), (top, top, top), n ** 3)
    assert g.cap_steps == 1 and g.dims == (416, 416, 416), (g.cap_steps, g.dims)
    assert 520 ** 3 > gc.MAX_CELLS >= 416 ** 3 and abs(float(g.e) - 0.0778) < 1e-3
    lat = np.concatenate([gc.lattice_keyframe(k) for k in range(16)])
    assert np.array_equal(lat[12345 * 67], np.array([(12345 * 67) % n, (12345 * 67 // n) % n, 12345 * 67 // n ** 2], F) * F(0.125))
    q = gc.lattice_queries()
    ai, ad = gc.lattice_nn(q)
    assert ((q % F(0.125)) == F(0.0625)).any(1).mean() > 0.3   # many queries on a lattice mid-plane: ties
    # the brute force on a 12³ block of the lattice, for the queries whose answer lies inside it
    blk = lat.reshape(n, n, n, 3)[40:52, 100:112, 7:19].reshape(-1, 3)
    idx_blk = (np.arange(40, 52)[:, None, None] * n + np.arange(100, 112)[None, :, None]) * n + np.arange(7, 19)[None, None, :]
    lo, hi = blk.min(0) + 0.2, blk.max(0) - 0.2
    sel = np.flatnonzero(((q >= lo) & (q <= hi)).all(1))[:3000]
    bi, bd = gc.brute_nn(q[sel], blk)
    assert np.array_equal(idx_blk.reshape(-1)[bi], ai[sel]) and np.array_equal(bd.view(np.uint32), ad[sel].view(np.uint32))
    # the k-d tree over the whole lattice on a subsample of the queries
    sub = q[::512]
    oi, od = io.nearest(sub, lat)
    assert np.array_equal(oi, ai[::512]) and np.array_equal(od.view(np.uint32), ad[::512].view(np.uint32))
