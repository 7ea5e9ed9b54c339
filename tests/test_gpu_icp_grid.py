"""GPU tests of the registrations' grid nearest-neighbour search on the constructed cases of tests/icp_grid_cases.py
(cell and coarse faces, exact ties, the fine-to-coarse handoff, empty regions, queries outside the box, degenerate boxes,
far-from-origin scenes, the cell cap and the correspondence gate).  The loop ICP's 1-NN equals the brute force (or, on
the 2^24-point lattice, the analytic answer) in index and d² bits; every pair of a batched call equals flb_keyframes_icp
bit for bit, also when the batch needs a second round; fricp's double first pass, its Welsch scales (the 7-NN
self-query) and the first passes of sicp and aaicp equal the sequential oracles given the device's normalisation."""
import time

import numpy as np
import pytest

from better_fastlio2_b200 import capi
from tests import aaicp_oracle as ao
from tests import fricp_oracle as fo
from tests import icp_grid_cases as gc
from tests import sicp_oracle as so

pytestmark = pytest.mark.gpu

EYE = np.eye(3, 4, dtype=np.float32).reshape(1, 12)
ZERO = [0.0] * 6
Z6 = np.zeros((1, 6), np.float32)
CASES = gc.cases()


def _pack(xyz):
    return capi.pack_pointtype(np.asarray(xyz, np.float32), np.zeros(len(xyz), np.float32))


@pytest.fixture(scope="module")
def grid_store():
    """Every case's target and queries as two key frames, an all-NaN and a one-point key frame, the 2^24-point lattice
    as 16 key frames and its 2^20 queries."""
    total = sum(len(c.tgt) + len(c.qry) for c in CASES) + (17 << 20) + 64
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, total, 2 * len(CASES) + 32)
    ids = []
    for c in CASES:
        ids.append((kf.append(_pack(c.tgt)), kf.append(_pack(c.qry))))
    nan_k = kf.append(_pack(np.full((50, 3), np.nan, np.float32)))
    one_k = kf.append(_pack(np.array([[0.25, 0.5, -0.75]], np.float32)))
    lat = [kf.append(_pack(gc.lattice_keyframe(k))) for k in range(16)]
    lq = gc.lattice_queries()
    lq_k = kf.append(_pack(lq))
    yield kf, ids, nan_k, one_k, lat, lq_k, lq
    kf.close()
    tree.close()


def _loop(kf, s, t, md=200.0):
    return kf.icp([s], list(t) if np.ndim(t) else [t], src_affines=EYE, tgt_affines=np.repeat(EYE, np.size(t), 0), max_iterations=1,
                  max_correspondence_distance=md, correspondences=True)


@pytest.mark.parametrize("j", range(len(CASES)), ids=[c.name for c in CASES])
def test_loop_icp_nearest_equals_the_brute_force(grid_store, j):
    kf, ids, *_ = grid_store
    c = CASES[j]
    tk, qk = ids[j]
    src, _ = kf.assemble([qk], affines=EYE)
    tgt, _ = kf.assemble([tk], affines=EYE)
    assert np.array_equal(src[:, :3], c.qry, equal_nan=True) and np.array_equal(tgt[:, :3], c.tgt, equal_nan=True)
    t0 = time.perf_counter()
    g, gi, gd = _loop(kf, qk, tk, c.max_dist)
    ms = (time.perf_counter() - t0) * 1e3
    bi, bd = gc.brute_nn(c.qry, c.tgt)
    assert np.array_equal(gi, bi), (c.name, np.nonzero(gi != bi)[0][:5], gi[gi != bi][:5], bi[gi != bi][:5])
    assert np.array_equal(gd.view(np.uint32), bd.view(np.uint32)), (c.name, np.nonzero(gd.view(np.uint32) != bd.view(np.uint32))[0][:5])
    want = int(((bi >= 0) & (bd.astype(np.float64) <= c.max_dist * c.max_dist)).sum())
    assert g["n_correspondences"] == want, (g["n_correspondences"], want)
    if "gate" in c.claims:
        assert want == c.claims["gate"][1] + c.claims["gate"][2]
    print(f"[icp grid] {c.name}: {len(c.qry)} -> {len(c.tgt)} points, call {ms:.1f} ms")


def test_loop_icp_on_the_capped_lattice(grid_store):
    kf, _, _, _, lat, lq_k, lq = grid_store
    t0 = time.perf_counter()
    g, gi, gd = _loop(kf, lq_k, lat)
    ms = (time.perf_counter() - t0) * 1e3
    ai, ad = gc.lattice_nn(lq)
    assert g["n_target"] == 1 << 24 and g["n_source"] == len(lq)
    assert np.array_equal(gi, ai), np.nonzero(gi != ai)[0][:5]
    assert np.array_equal(gd.view(np.uint32), ad.view(np.uint32))
    print(f"[icp grid] lattice 2^24 targets, {len(lq)} queries (416³ cells after one cap step): {ms:.0f} ms per call")


def _bits(r):
    return (r["state"], r["converged"], r["iterations"], r["n_source"], r["n_target"], r["n_correspondences"],
            r["final_transformation"].tobytes(), np.float64(r["fitness_score"]).tobytes())


CFG = dict(max_correspondence_distance=200.0, max_iterations=1)


def _single(kf, pair):
    si, sp, ti, tp = pair
    return kf.icp(np.asarray(si, np.int32), np.asarray(ti, np.int32), src_poses6=np.asarray(sp, np.float32).reshape(-1, 6),
                  tgt_poses6=np.asarray(tp, np.float32).reshape(-1, 6), **CFG)


def test_batched_icp_equals_the_loop_icp_pair_by_pair(grid_store):
    kf, ids, nan_k, one_k, lat, lq_k, _ = grid_store
    pairs = []
    for j, (tk, qk) in enumerate(ids):
        pairs.append(([qk], [ZERO], [tk], [ZERO]))
        fill = (([], [], [tk], [ZERO]), ([qk], [ZERO], [nan_k], [ZERO]), ([qk], [ZERO], [one_k], [ZERO]))[j % 3]
        pairs.append(fill)   # empty, all-NaN and one-point selections shift the packed offsets
    singles = [_single(kf, p) for p in pairs]
    got, st = kf.icp_batch(pairs, leaf=0.0, **CFG)
    for p, (g, r) in enumerate(zip(got, singles)):
        assert _bits(g) == _bits(r), (p, g, r)
    assert st["rounds"] == 1, st
    # two copies of the lattice pair: their two 416³ grids exceed one round's cells, so the second opens a new round
    h = ([lq_k], [ZERO], lat, [ZERO] * len(lat))
    h_single = _single(kf, h)
    mixed = pairs[:7] + [h] + pairs[7:20] + [h] + pairs[20:]
    got, st = kf.icp_batch(mixed, leaf=0.0, **CFG)
    assert st["rounds"] >= 2, st
    want = singles[:7] + [h_single] + singles[7:20] + [h_single] + singles[20:]
    for p, (g, r) in enumerate(zip(got, want)):
        assert _bits(g) == _bits(r), (p, g, r)
    print(f"[icp grid batch] {len(pairs)} pairs in one round; with two lattice pairs: {st}")


def _norm(g):
    return g["scale"], g["mu_source"], g["mu_target"]


DOUBLE = [j for j, c in enumerate(CASES) if c.double_path]


@pytest.mark.parametrize("j", DOUBLE, ids=[CASES[j].name for j in DOUBLE])
def test_fricp_first_pass_and_scales_equal_the_oracle(grid_store, j):
    kf, ids, *_ = grid_store
    c = CASES[j]
    tk, _ = ids[j]
    tgt, _ = kf.assemble([tk], poses6=Z6)
    for mode in (0, 4):
        t0 = time.perf_counter()
        g, gi, gr = kf.fricp(c.qry, [tk], Z6, mode=mode, max_icp=0, correspondences=True)
        ms = (time.perf_counter() - t0) * 1e3
        o, oi, orr, _ = fo.fricp(c.qry, tgt, mode=mode, max_icp=0, norm=_norm(g))
        assert g["status"] == o["status"] == 0, (c.name, g["status_name"])
        assert np.array_equal(gi, oi), (c.name, mode, np.nonzero(gi != oi)[0][:5])
        assert np.array_equal(gr.view(np.uint64), orr.view(np.uint64)), (c.name, mode)
        assert (g["nu_begin"], g["nu_end"]) == (o["nu_begin"], o["nu_end"]), (c.name, mode)
        assert (g["n_source_finite"], g["n_target_finite"]) == (o["n_source_finite"], o["n_target_finite"])
    print(f"[fricp grid] {c.name}: nu {g['nu_begin']:.6g} -> {g['nu_end']:.6g}, call {ms:.1f} ms")


@pytest.mark.parametrize("name", ["7-NN: isolated clusters of 2-6 points", "c: ties between the fine rings and the far path"])
def test_sicp_and_aaicp_first_passes_read_the_same_search(grid_store, name):
    kf, ids, *_ = grid_store
    j = [c.name for c in CASES].index(name)
    c = CASES[j]
    tk, _ = ids[j]
    tgt, _ = kf.assemble([tk], poses6=Z6)
    g, fi, fr = kf.fricp(c.qry, [tk], Z6, mode=0, max_icp=0, correspondences=True)
    gs, si, sr = kf.sicp(c.qry, [tk], Z6, max_icp=1, max_outer=0, correspondences=True)
    o, oi, orr, _ = so.sicp(c.qry, tgt, max_icp=1, max_outer=0, norm=_norm(gs))
    assert np.array_equal(si, oi) and np.array_equal(sr.view(np.uint64), orr.view(np.uint64)), name
    ga, ai, ar = kf.aaicp(c.qry, [tk], Z6, max_icp=1, correspondences=True)
    o, oi, orr, _ = ao.aaicp(c.qry, tgt, max_icp=1, norm=_norm(ga))
    assert np.array_equal(ai, oi) and np.array_equal(ar.view(np.uint64), orr.view(np.uint64)), name
    # one normalisation and one search: before any step, fricp and sicp match the same targets
    assert _norm(g)[0] == _norm(gs)[0] == _norm(ga)[0]
    assert np.array_equal(fi, si) and np.array_equal(fr.view(np.uint64), sr.view(np.uint64)), name
