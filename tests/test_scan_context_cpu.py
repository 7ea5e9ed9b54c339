"""CPU tests of the Scan Context readers of the key-frame store: the oracle (tests/cpp/scan_context_oracle.cpp) against an
independent numpy restatement of makeScancontext on directed edge cases, argument checking of both C entry points
before any device work, no store without a device, and the C++ facade methods compiled as src/laserMapping.cpp would use
them."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import scan_context_oracle as sco
from tests.scan_context_cases import edge_points, np_scan_context

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("h", [1.5, 0.0, -2.25])
def test_oracle_equals_numpy_on_directed_cases(h):
    pts = edge_points(h)
    o, sens, mask = sco.scan_context(pts, h)
    assert np.array_equal(o, np_scan_context(pts, h))
    # 90, 180 and 270 degrees (x = +0 with y != 0, the -x axis) lie on sector boundaries; 0 degrees, -90 degrees
    # (x = -0, y > 0) and NaN angles do not
    x, y = pts[:, 0], pts[:, 1]
    kept = (np.hypot(x, y) <= 80) & (pts[:, 2] + h > -1000)
    on_boundary = kept & (((x == 0) & ~np.signbit(x) & (y != 0)) | ((x < 0) & (y == 0)))
    assert on_boundary.sum() >= 8 and sens[on_boundary].all()
    assert not sens[kept & (x == 0) & np.signbit(x) & (y > 0)].any() and not sens[kept & (x > 0) & (y == 0)].any()
    # each point alone: the same bin and value in both
    for p in pts:
        assert np.array_equal(sco.scan_context(p[None], h)[0], np_scan_context(p[None], h))


def test_documented_consequences():
    h = 1.5
    one = lambda x, y, z: sco.scan_context(np.array([[x, y, z, 0]], np.float32), h)[0]
    d = one(-0.0, 7.0, 1.0)                # x = -0, y > 0: -90 degrees, sector 1 (ring 2)
    assert d[1, 0] == 2.5 and np.count_nonzero(d) == 1
    d = one(0.0, 7.0, 1.0)                 # x = +0, y > 0: 90 degrees, sector 15
    assert d[1, 14] == 2.5 and np.count_nonzero(d) == 1
    for x, y in ((0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0)):   # NaN angle, range 0: ring 1, sector 1
        d = one(x, y, 1.0)
        assert d[0, 0] == 2.5 and np.count_nonzero(d) == 1
    d = one(np.nan, 3.0, 1.0)              # NaN range is not skipped: int(NaN) clamps to ring 1 / sector 1
    assert d[0, 0] == 2.5 and np.count_nonzero(d) == 1
    assert not one(3.0, 4.0, np.nan).any()                          # NaN height: no bin changes
    assert not one(np.float32(np.nextafter(np.float32(80), np.float32(100))), 0.0, 1.0).any()   # one ulp beyond 80 m
    d = one(80.0, 0.0, 1.0)
    assert d[19, 0] == 2.5                 # exactly 80 m: ring 20; angle 0 -> sector ceil(0) = 0 -> 1
    assert not one(10.0, 10.0, -1001.5).any()                       # pt.z == -1000 does not beat the initial -1000
    d = one(10.0, 10.0, np.nextafter(np.float32(-1001.5), np.float32(0)))
    assert d[3, 7] == np.float32(np.nextafter(np.float32(-1001.5), np.float32(0)) + np.float32(1.5))
    assert not sco.scan_context(np.zeros((0, 4), np.float32), h)[0].any()   # empty cloud: all zeros


def test_oracle_equals_numpy_on_random_clouds():
    rng = np.random.default_rng(1)
    p = np.empty((50000, 4), np.float32)
    p[:, 0] = rng.uniform(-90, 90, len(p))
    p[:, 1] = rng.uniform(-90, 90, len(p))
    p[:, 2] = rng.uniform(-3, 8, len(p))
    p[:, 3] = 0
    o, sens, mask = sco.scan_context(p, 1.5)
    n = np_scan_context(p, 1.5)
    assert np.array_equal(o[~mask], n[~mask])        # numpy's arctan may differ from glibc's on sensitive points only
    assert sens.sum() < 20 and (o != 0).sum() > 1000


@pytest.fixture(scope="module")
def L():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def _err(L):
    return L.flb_last_error().decode()


def test_invalid_arguments_are_rejected_with_a_message(L):
    from better_fastlio2_b200 import capi
    ids = np.array([0, 1], np.int32)
    tr = np.zeros(24, np.float32)
    out = np.full(2 * 1200, 7.0)
    p = capi._p
    one = L.flb_keyframes_scan_context
    cases = [
        (lambda: one(None, p(ids), -1, 1, p(tr), C.c_double(1.5), p(out)), "negative n_ids"),
        (lambda: one(None, p(ids), 2, 1, p(tr), C.c_double(1.5), None), "null out_desc"),
        (lambda: one(None, None, 2, 1, p(tr), C.c_double(1.5), p(out)), "null ids or transforms"),
        (lambda: one(None, p(ids), 2, 1, None, C.c_double(1.5), p(out)), "null ids or transforms"),
        (lambda: one(None, p(ids), 2, 2, p(tr), C.c_double(1.5), p(out)), "transform_kind"),
        (lambda: one(None, p(ids), 2, -1, p(tr), C.c_double(1.5), p(out)), "transform_kind"),
        (lambda: one(None, p(ids), 2, 0, p(tr), C.c_double(float("nan")), p(out)), "lidar_height must be finite"),
        (lambda: one(None, p(ids), 2, 0, p(tr), C.c_double(float("inf")), p(out)), "lidar_height must be finite"),
        (lambda: one(None, p(ids), 2, 0, p(tr), C.c_double(1.5), p(out)), "null key-frame store"),
        (lambda: one(None, None, 0, 0, None, C.c_double(1.5), p(out)), "null key-frame store"),
    ]
    many = L.flb_keyframes_scan_contexts
    cases += [
        (lambda: many(None, p(ids), -3, C.c_double(1.5), p(out)), "negative n_ids"),
        (lambda: many(None, None, 2, C.c_double(1.5), p(out)), "null ids or out_descs"),
        (lambda: many(None, p(ids), 2, C.c_double(1.5), None), "null ids or out_descs"),
        (lambda: many(None, p(ids), 2, C.c_double(-float("inf")), p(out)), "lidar_height must be finite"),
        (lambda: many(None, p(ids), 2, C.c_double(1.5), p(out)), "null key-frame store"),
    ]
    for call, msg in cases:
        assert call() != 0
        assert msg in _err(L), (msg, _err(L))
    assert (out == 7.0).all()          # nothing written on failure


def test_no_store_without_a_device():
    from better_fastlio2_b200 import capi
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(capi.FlbError, match="no CUDA device"):
        capi.KDTree(voxel_size=0.2)


def test_python_layer_checks_transform_shapes():
    from better_fastlio2_b200 import capi

    class _FakeStore(capi.KeyFrameStore):
        def __init__(self):
            self.h = None

    s = _FakeStore()
    with pytest.raises(ValueError):
        s.scan_context([0, 1], poses6=[[0] * 6])
    with pytest.raises(ValueError):
        s.scan_context([0], poses6=[[0] * 6], affines=[[0] * 12])
    with pytest.raises(ValueError):
        s.scan_context([0], affines=[[0] * 6])


def test_header_documents_scan_context():
    src = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for name in ("flb_keyframes_scan_context", "flb_keyframes_scan_contexts", "FLB_SC_RINGS 20", "FLB_SC_SECTORS 60"):
        assert name in src


def test_scan_context_facade_compiles(L):
    from better_fastlio2_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "scan_context_facade_smoke")
        cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", "scan_context_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
               f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "NO_GPU compile-only ok" in out.stdout or "SCAN_CONTEXT_FACADE_OK" in out.stdout
