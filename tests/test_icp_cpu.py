"""CPU tests of the loop-closure ICP (flb_keyframes_icp): the sequential oracle (tests/cpp/icp_oracle.cpp) against an
independent float64 numpy / scipy restatement on seeded clouds, directed cases that reach every branch of the contract
(each convergence state, the distance boundary, fewer than 3 pairs, empty and all-NaN clouds, the reflection branch,
duplicated target points), the C structs' layout, argument checking before any device work and the C++ facade
compiled as src/laserMapping.cpp would use it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import icp_oracle as io
from tests.icp_cases import DBL_MAX, NN, moved, np_icp, rot, surface_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same_run(o, n, what=""):
    assert (o["state"], o["converged"], o["iterations"]) == (n["state"], n["converged"], n["iterations"]), (what, o, n)
    assert o["n_correspondences"] == n["n_correspondences"], what
    T, U = o["final_transformation"].astype(np.float64), n["final_transformation"].astype(np.float64)
    assert np.abs(T[:3, 3] - U[:3, 3]).max() <= 1e-6, (what, T, U)
    M = T[:3, :3].T @ U[:3, :3]
    assert np.arccos(np.clip(0.5 * (np.trace(M) - 1), -1, 1)) <= 1e-6 or np.abs(T[:3, :3] - U[:3, :3]).max() <= 1e-6, what
    if n["fitness_score"] == DBL_MAX:
        assert o["fitness_score"] == DBL_MAX
    else:
        assert abs(o["fitness_score"] - n["fitness_score"]) <= 1e-9 * abs(n["fitness_score"]) + 1e-300, (what, o, n)


def _same_pairs(oi, od, ni, nd):
    """The last iteration's correspondences equal, except where two candidates' float distances lie within 2 ulp."""
    diff = np.nonzero(oi != ni)[0]
    for i in diff:
        a, b = od[i], nd[i]
        assert oi[i] >= 0 and ni[i] >= 0
        assert abs(int(np.float32(a).view(np.int32)) - int(np.float32(b).view(np.int32))) <= 2, (i, a, b)
    assert np.array_equal(od[oi == ni], nd[oi == ni])
    return len(diff)


@pytest.mark.parametrize("n,seed", [(1000, 1), (8000, 2), (50000, 3)])
def test_oracle_equals_numpy_on_seeded_clouds(n, seed):
    tgt = surface_cloud(n, seed)
    src = moved(surface_cloud(n, seed + 100), (0.01, -0.02, 0.05), (0.8, -0.5, 0.1))
    o, oi, od, log = io.icp(src, tgt)
    r, ni, nd = np_icp(src, tgt)
    _same_run(o, r, f"n={n}")
    assert o["converged"] and o["iterations"] >= 3
    ndiff = _same_pairs(oi, od, ni.astype(np.int32), nd)
    print(f"[icp oracle] n={n}: {o['iterations']} iterations, {o['state_name']}, fitness {o['fitness_score']:.6g}, "
          f"{ndiff} near-tie pairs differ")


def test_nearest_equals_numpy_with_nan_and_duplicates():
    rng = np.random.default_rng(4)
    tgt = surface_cloud(5000, 5)
    tgt[::97, 1] = np.nan
    tgt = np.concatenate([tgt, tgt[:300]])          # duplicates: indices i and 5000 + i hold the same point
    q = surface_cloud(4000, 6)
    q[:50, :3] = tgt[1:51, :3]                       # exact hits on duplicated points (d² 0 at both copies)
    q[60:70, 0] = np.inf
    q[70:80, 2] = np.nan
    q[80:200, :3] += rng.uniform(40, 150, (120, 3)).astype(np.float32)   # far from every target point
    oi, od = io.nearest(q, tgt)
    ni, nd = NN(tgt)(q)
    assert (oi[60:80] == -1).all() and np.isinf(od[60:80]).all()
    good = np.arange(len(q))
    same = oi == ni
    for i in good[~same]:   # only exact ties may differ, and then the oracle holds the lower index
        assert od[i] == nd[i] and oi[i] < ni[i], (i, oi[i], ni[i], od[i], nd[i])
    assert (oi[:50] == np.arange(1, 51)).all() and (od[:50] == 0).all()


def test_states_and_branches():
    base = surface_cloud(3000, 7)
    moved_src = moved(surface_cloud(3000, 8), (0.0, 0.01, -0.03), (0.5, 0.2, 0.0))
    cases = {
        "ITERATIONS": (moved_src, base, dict(max_iterations=2)),
        "ITERATIONS_at_0": (moved_src, base, dict(max_iterations=0)),   # nr_iterations >= 0 after the first iteration
        "TRANSFORM": (base, base, {}),
        "ABS_MSE": (base, base, dict(transformation_epsilon=-1.0)),
        "REL_MSE": (moved_src, base, dict(transformation_epsilon=-1.0, euclidean_fitness_epsilon=0.999)),
        "NO_CORRESPONDENCES": (moved(base, (0, 0, 0), (0, 0, 50)), base, dict(max_correspondence_distance=1.0)),
    }
    want = {"ITERATIONS": (1, 2), "ITERATIONS_at_0": (1, 1), "TRANSFORM": (2, 1), "ABS_MSE": (3, 2), "REL_MSE": (4, 2),
            "NO_CORRESPONDENCES": (5, 0)}
    for name, (s, t, kw) in cases.items():
        o, _, _, _ = io.icp(s, t, **kw)
        r, _, _ = np_icp(s, t, **kw)
        _same_run(o, r, name)
        assert (o["state"], o["iterations"]) == want[name], (name, o)
        assert o["converged"] == (name != "NO_CORRESPONDENCES")
    o, _, _, _ = io.icp(*cases["NO_CORRESPONDENCES"][:2], **cases["NO_CORRESPONDENCES"][2])
    assert np.array_equal(o["final_transformation"], np.eye(4, dtype=np.float32)) and o["fitness_score"] < DBL_MAX


def test_distance_boundary_and_fewer_than_three_pairs():
    tgt = np.array([[0, 0, 0, 0], [100, 0, 0, 0], [0, 100, 0, 0], [0, 0, 100, 0]], np.float32)
    src = tgt.copy()
    src[:, 0] += 2.0                                  # d² exactly 4
    src[3, 0] = np.float32(np.nextafter(np.float32(2.0), np.float32(3.0)))   # just beyond 2 m
    o, oi, od, _ = io.icp(src, tgt, max_correspondence_distance=2.0, max_iterations=1)
    assert od[0] == 4.0 and o["n_correspondences"] == 3 and o["state"] == 1   # d² == max² is kept
    r, _, _ = np_icp(src, tgt, max_correspondence_distance=2.0, max_iterations=1)
    _same_run(o, r, "boundary")
    o, _, _, _ = io.icp(src, tgt, max_correspondence_distance=float(np.nextafter(2.0, 0.0)), max_iterations=5)
    assert o["state"] == 5 and not o["converged"] and o["iterations"] == 0 and o["n_correspondences"] == 0
    # exactly two pairs within reach: not converged, identity kept
    src2 = tgt.copy()
    src2[2:, 2] += 10.0
    o, _, _, _ = io.icp(src2, tgt, max_correspondence_distance=1.0)
    assert o["state"] == 5 and o["n_correspondences"] == 2 and not o["converged"]
    assert np.array_equal(o["final_transformation"], np.eye(4, dtype=np.float32))


def test_empty_and_all_nan_clouds():
    c = surface_cloud(500, 9)
    nan = np.full((40, 4), np.nan, np.float32)
    for s, t in ((c[:0], c), (c, c[:0]), (c, nan), (c[:0], c[:0])):
        for res in (io.icp(s, t)[0], np_icp(s, t)[0]):
            assert not res["converged"] and res["iterations"] == 0 and res["state"] == 0
            assert res["fitness_score"] == DBL_MAX
            assert np.array_equal(res["final_transformation"], np.eye(4, dtype=np.float32))
    # an all-NaN source: no pairs at all
    o, oi, od, _ = io.icp(nan, c)
    assert o["state"] == 5 and (oi == -1).all() and o["fitness_score"] == DBL_MAX


def test_reflection_branch():
    rng = np.random.default_rng(10)
    tgt = np.column_stack([rng.uniform(1, 4, 12), rng.uniform(-60, 60, 12), rng.uniform(-60, 60, 12), np.zeros(12)]).astype(np.float32)
    src = tgt.copy()
    src[:, 0] = -src[:, 0]                             # the mirror image: each point's nearest target is its original
    flips = []
    r, ni, _ = np_icp(src, tgt, max_iterations=1, reflections=flips)
    assert flips == [True] and (ni == np.arange(12)).all()
    o, _, _, _ = io.icp(src, tgt, max_iterations=1)
    _same_run(o, r, "reflection")
    assert np.linalg.det(o["final_transformation"][:3, :3].astype(np.float64)) > 0.999   # a rotation, not the mirror


def test_oracle_recovers_a_known_motion():
    tgt = surface_cloud(20000, 11)
    R = rot((0.0, 0.0, np.deg2rad(3.0)))
    t = np.array([0.9, -0.4, 0.05])
    src = tgt.copy()                                  # src = motion^-1 (tgt): final should be the motion
    src[:, :3] = ((tgt[:, :3].astype(np.float64) - t) @ R).astype(np.float32)
    o, _, _, _ = io.icp(src, tgt, transformation_epsilon=1e-10, euclidean_fitness_epsilon=1e-10)
    T = o["final_transformation"].astype(np.float64)
    assert np.abs(T[:3, 3] - t).max() < 0.02 and np.abs(T[:3, :3] - R).max() < np.deg2rad(0.1)


# ------------------------------------------------------------------------------------------------ C ABI without a GPU
@pytest.fixture(scope="module")
def L():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def test_struct_layout_matches_the_c_compiler():
    from better_fastlio2_b200 import capi
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "fastlio_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(flb_icp_config), offsetof(flb_icp_config, max_iterations),
         offsetof(flb_icp_config, transformation_epsilon), offsetof(flb_icp_config, euclidean_fitness_epsilon), sizeof(flb_icp_result),
         offsetof(flb_icp_result, converged), offsetof(flb_icp_result, state), offsetof(flb_icp_result, n_correspondences),
         offsetof(flb_icp_result, fitness_score));
  return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "layout.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "layout")
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    ic, ir = capi.IcpConfig, capi.IcpResult
    want = [C.sizeof(ic), ic.max_iterations.offset, ic.transformation_epsilon.offset, ic.euclidean_fitness_epsilon.offset,
            C.sizeof(ir), ir.converged.offset, ir.state.offset, ir.n_correspondences.offset, ir.fitness_score.offset]
    assert got == want


def test_invalid_arguments_are_rejected_with_a_message(L):
    from better_fastlio2_b200 import capi
    p = capi._p
    ids = np.array([0, 1], np.int32)
    tr = np.zeros(24, np.float32)
    good = capi.IcpConfig(200.0, 100, 1e-6, 1e-6)
    out = capi.IcpResult()
    out.iterations = 77

    def cfg(**kw):
        c = capi.IcpConfig(200.0, 100, 1e-6, 1e-6)
        for k, v in kw.items():
            setattr(c, k, v)
        return C.byref(c)

    f = L.flb_keyframes_icp
    g, o = C.byref(good), C.byref(out)
    cases = [
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), g, None, None, None), "null result"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), None, o, None, None), "null config"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), cfg(max_iterations=-1), o, None, None), "max_iterations >= 0"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), cfg(max_correspondence_distance=-1.0), o, None, None),
         "max_correspondence_distance >= 0"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), cfg(max_correspondence_distance=float("nan")), o, None, None),
         "finite"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), cfg(transformation_epsilon=float("inf")), o, None, None),
         "finite"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), cfg(euclidean_fitness_epsilon=float("nan")), o, None, None),
         "finite"),
        (lambda: f(None, p(ids), -1, 1, p(tr), None, p(ids), 2, 1, p(tr), g, o, None, None), "negative n_src or n_tgt"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), -2, 1, p(tr), g, o, None, None), "negative n_src or n_tgt"),
        (lambda: f(None, None, 2, 1, p(tr), None, p(ids), 2, 1, p(tr), g, o, None, None), "null ids or transforms"),
        (lambda: f(None, p(ids), 2, 1, None, None, p(ids), 2, 1, p(tr), g, o, None, None), "null ids or transforms"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, None, 2, 1, p(tr), g, o, None, None), "null ids or transforms"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, None, g, o, None, None), "null ids or transforms"),
        (lambda: f(None, p(ids), 2, 2, p(tr), None, p(ids), 2, 1, p(tr), g, o, None, None), "transform kinds"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, -1, p(tr), g, o, None, None), "transform kinds"),
        (lambda: f(None, p(ids), 2, 1, p(tr), None, p(ids), 2, 1, p(tr), g, o, None, None), "null key-frame store"),
        (lambda: f(None, None, 0, 0, None, None, None, 0, 0, None, g, o, None, None), "null key-frame store"),
    ]
    for call, msg in cases:
        assert call() != 0
        assert msg in L.flb_last_error().decode(), (msg, L.flb_last_error().decode())
    assert out.iterations == 77          # nothing written on failure


def test_python_layer_checks_transform_shapes():
    from better_fastlio2_b200 import capi

    class _FakeStore(capi.KeyFrameStore):
        def __init__(self):
            self.h = None

    s = _FakeStore()
    with pytest.raises(ValueError):
        s.icp([0, 1], [0], src_poses6=[[0] * 6], tgt_poses6=[[0] * 6])
    with pytest.raises(ValueError):
        s.icp([0], [0], src_poses6=[[0] * 6], src_affines=[[0] * 12], tgt_poses6=[[0] * 6])
    with pytest.raises(ValueError):
        s.icp([0], [0], src_affines=[[0] * 12], tgt_affines=[[0] * 6])


def test_header_documents_icp():
    src = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for name in ("flb_keyframes_icp", "flb_icp_config", "flb_icp_result", "FLB_ICP_NO_CORRESPONDENCES 5", "FLB_ICP_REL_MSE 4"):
        assert name in src


def test_icp_facade_compiles_and_fails_loudly_without_a_gpu(L):
    from better_fastlio2_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "icp_facade_smoke")
        cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", "icp_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
               f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    if capi.device_count() > 0:
        assert out.returncode == 0 and "ICP_FACADE_OK" in out.stdout, (out.returncode, out.stdout, out.stderr)
    else:   # no device: the store cannot be attached, and the facade says so on stderr
        assert out.returncode == 2 and "NO_GPU" in out.stdout and "KeyFrameStore::attach" in out.stderr, (out.stdout, out.stderr)
