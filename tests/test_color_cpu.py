"""CPU tests of the camera-coloured and IMU-frame publishers (publish_frame_world_color, laserMapping.cpp:310-392;
publish_frame_body, :1543-1558): the oracle (tests/cpp/color_oracle.cpp) against a float64 numpy restatement that sums
in index order, directed cases of the projection contract (DESIGN.md §9) with exact extrinsics, the ctypes signatures,
argument rejection before any device work and the C++ facade compiled as src/laserMapping.cpp would use it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from better_fastlio2_b200 import synth
from tests import color_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = co.W_MAX, co.H_MAX


def _qrot(q, v):
    """Eigen's q * v on (n, 3) float64 rows, in the order of _transformVector."""
    qx, qy, qz, qw = (float(c) for c in q)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    ux, uy, uz = qy * z - qz * y, qz * x - qx * z, qx * y - qy * x
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    cx, cy, cz = qy * uz - qz * uy, qz * ux - qx * uz, qx * uy - qy * ux
    return np.stack([(x + qw * ux) + cx, (y + qw * uy) + cy, (z + qw * uz) + cz], 1)


def np_colorize(cam_ex, cam_in, img, pts, st, width=W, height=H):
    ex = np.asarray(cam_ex, np.float64).reshape(4, 4)
    ki = np.asarray(cam_in, np.float64).reshape(3, 4)
    M = np.empty((3, 4))
    for r in range(3):
        for c in range(4):
            s = ki[r, 0] * ex[0, c]
            for k in range(1, 4):
                s = s + ki[r, k] * ex[k, c]
            M[r, c] = s
    p = np.asarray(pts, np.float32)
    x, y, z = (p[:, k].astype(np.float64) for k in range(3))
    with np.errstate(divide="ignore", invalid="ignore"):   # 0 * inf and x / 0 are part of the contract
        cam = [((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] * 1.0 for r in range(3)]
        u, v = cam[0] / cam[2], cam[1] / cam[2]
    ok = np.isfinite(u) & np.isfinite(v) & (u > -2147483649.0) & (u < 2147483648.0) & (v > -2147483649.0) & (v < 2147483648.0)
    ui = np.zeros(len(p), np.int64)
    vi = np.zeros(len(p), np.int64)
    ui[ok], vi[ok] = np.trunc(u[ok]).astype(np.int64), np.trunc(v[ok]).astype(np.int64)
    keep = ok & (ui >= 0) & (ui < width) & (vi >= 0) & (vi < height) & (p[:, 0] > 0)
    idx = np.nonzero(keep)[0].astype(np.int32)
    im = np.zeros((height, width, 3), np.uint8) if img is None else img
    px = im[vi[idx], ui[idx]].astype(np.uint32)
    bgra = px[:, 0] | (px[:, 1] << 8) | (px[:, 2] << 16) | np.uint32(255 << 24)
    a = _qrot(st[7:11], np.stack([x[idx], y[idx], z[idx]], 1)) + st[11:14]
    g = _qrot(st[3:7], a) + st[0:3]
    xyzi = np.column_stack([g.astype(np.float32), p[idx, 3]]).astype(np.float32)
    return xyzi, bgra.astype(np.uint32), idx


def hap_cloud(seed, n=None):
    rng = np.random.default_rng(seed)
    d = synth.lidar_dirs("hap", rng)
    if n is not None:
        d = d[:n]
    r = rng.uniform(0.5, 90.0, len(d))
    xyz = d * r[:, None] + rng.normal(0, 0.01, (len(d), 3))
    return np.column_stack([xyz, rng.uniform(0, 255, len(d))]).astype(np.float32)


def state(seed):
    rng = np.random.default_rng(seed)
    st = synth.make_state(pos=rng.uniform(-50, 50, 3), rot=synth.quat_from_rotvec(rng.normal(0, 0.5, 3)),
                          offR=synth.quat_from_rotvec(rng.normal(0, 0.05, 3)))
    return st


def image(seed, height=H, width=W):
    return np.random.default_rng(seed).integers(0, 256, (height, width, 3), dtype=np.uint8)


@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_equals_numpy_on_hap_clouds(seed):
    pts = hap_cloud(seed)
    ex, ki = co.forward_camera(fx=900.0 + seed, fy=899.5, t=(0.05, -0.02, 0.1))
    st, img = state(seed), image(seed)
    o = co.colorize(ex, ki, img, pts, st)
    n = np_colorize(ex, ki, img, pts, st)
    assert 20000 < len(o[2]) < len(pts)
    for a, b in zip(o, n):
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    want = (_qrot(st[7:11], pts[:, :3].astype(np.float64)) + st[11:14]).astype(np.float32)
    got = co.to_imu(pts, st)
    assert np.array_equal(got[:, :3].view(np.uint32), want.view(np.uint32)) and np.array_equal(got[:, 3], pts[:, 3])


def _one(x, y, z, cam=None, img=None, st=None):
    ex, ki = cam if cam is not None else co.forward_camera()
    st = synth.make_state(offT=(0, 0, 0)) if st is None else st
    pts = np.array([[x, y, z, 5.0]], np.float32)
    o = co.colorize(ex, ki, img, pts, st)
    n = np_colorize(ex, ki, img, pts, st)
    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(o, n))
    return len(o[2]) == 1


def _pixel_cam():
    """Extrinsic identity, intrinsic [[1,0,0,0],[0,1,0,0],[0,0,1,0]]: u = x / z, v = y / z exactly."""
    return np.eye(4).reshape(-1), np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float64)


def test_directed_projection_edges():
    cam = _pixel_cam()
    # u at -0.5 (truncates to pixel 0: kept), 0, W - eps, W; v at H
    assert _one(1.0, 0.0, 2.0, cam) and _one(2.0, 0.0, 1.0, cam)      # u = 0.5, 2
    assert _one(0.5, 1.0, -1.0, cam) is False                          # u = -0.5, v = -1
    assert _one(1.0, 0.0, -2.0, cam)                                   # u = -0.5, v = -0: pixel (0, 0), kept
    assert _one(1.0, 3.0, 1.0, cam)                                    # z == 1: u = 1, v = 3
    w_eps = np.float32(np.nextafter(np.float32(W), np.float32(0)))
    assert _one(w_eps, 10.0, 1.0, cam)                                 # u = W - eps
    assert not _one(float(W), 10.0, 1.0, cam)                          # u = W
    assert _one(5.0, float(np.nextafter(np.float32(H), np.float32(0))), 1.0, cam)
    assert not _one(5.0, float(H), 1.0, cam)                           # v = H
    assert not _one(1.0, 0.0, -1.0, cam)                               # u = -1 (trunc -1)
    # c2 < 0 in bounds is kept (u = 1/-2 -> pixel 0, v = -6/-2 = 3); c2 = 0 is rejected (u = inf; v = 0/0)
    assert _one(1.0, -6.0, -2.0, cam) and not _one(4.0, 6.0, 0.0, cam) and not _one(4.0, 0.0, 0.0, cam)
    # c2 < 0 with a positive pixel: the camera looks along -z (u = -x/z)
    flip = (np.eye(4).reshape(-1), np.array([-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0], np.float64))
    assert _one(4.0, 6.0, -2.0, flip)
    # x = 0, -0.0 and < 0 are rejected whatever the pixel (the camera here ignores x for u)
    ex, ki = np.eye(4).reshape(-1), np.array([0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1], np.float64)   # u = y, v = z, c2 = 1
    assert _one(1.0, 3.0, 4.0, (ex, ki))
    for x in (0.0, -0.0, -1.0):
        assert not _one(x, 3.0, 4.0, (ex, ki))
    # non-finite points
    for bad in ((np.nan, 1, 1), (1, np.nan, 1), (1, 1, np.nan), (np.inf, 1, 1), (1, np.inf, 1), (1, 1, np.inf), (1, -np.inf, 1)):
        assert not _one(*bad, cam=(ex, ki)) and not _one(*bad, cam=cam)
    # beyond int32: rejected
    assert not _one(1.0, 3e9, 1.0, (ex, ki)) and not _one(1.0, -3e9, 1.0, (ex, ki))


def test_colour_and_fields():
    ex, ki = np.eye(4).reshape(-1), np.array([0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1], np.float64)
    img = image(4)
    pts = np.array([[1, 3.7, 4.2, 9], [2, 1279.9, 719.9, 8], [3, 0.0, 0.0, 7]], np.float32)
    xyzi, bgra, idx = co.colorize(ex, ki, img, pts, synth.make_state(), W, H)
    assert idx.tolist() == [0, 1, 2]
    for k, (u, v) in enumerate(((3, 4), (1279, 719), (0, 0))):
        b, g, r = img[v, u]
        assert bgra[k] == (int(b) | int(g) << 8 | int(r) << 16 | 255 << 24)
    assert xyzi[:, 3].tolist() == [9, 8, 7]
    # all-zero image: colour word is alpha only
    _, bgra0, _ = co.colorize(ex, ki, None, pts, synth.make_state())
    assert (bgra0 == np.uint32(255 << 24)).all()


def test_empty_cloud():
    ex, ki = co.forward_camera()
    xyzi, bgra, idx = co.colorize(ex, ki, None, np.zeros((0, 4), np.float32), synth.make_state())
    assert len(xyzi) == len(bgra) == len(idx) == 0
    assert len(co.to_imu(np.zeros((0, 4), np.float32), synth.make_state())) == 0


def test_projection_is_in_index_order():
    ex, ki = co.forward_camera(fx=913.25, fy=907.5, t=(0.1, 0.2, 0.3))
    M = co.projection(ex, ki)
    e, k = ex.reshape(4, 4), ki.reshape(3, 4)
    for r in range(3):
        for c in range(4):
            assert M[r, c] == ((k[r, 0] * e[0, c] + k[r, 1] * e[1, c]) + k[r, 2] * e[2, c]) + k[r, 3] * e[3, c]


# ------------------------------------------------------------------------------------------------ C ABI, no device
@pytest.fixture(scope="module")
def L():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def test_ctypes_signatures(L):
    vp, ip = C.c_void_p, C.POINTER(C.c_int)
    assert L.flb_frontend_camera_config.argtypes == [vp, vp, vp, C.c_int, C.c_int]
    assert L.flb_frontend_camera_image.argtypes == [vp, vp, C.c_int, C.c_int, C.c_int]
    assert L.flb_frontend_points_colorize.argtypes == [vp, C.c_int, vp, vp, vp, C.c_int, ip]
    assert L.flb_frontend_points_to_imu.argtypes == [vp, vp, vp, C.c_int, ip]
    for f in ("flb_frontend_camera_config", "flb_frontend_camera_image", "flb_frontend_points_colorize", "flb_frontend_points_to_imu"):
        assert getattr(L, f).restype is C.c_int


def test_arguments_are_rejected_before_device_work(L):
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    err = lambda: L.flb_last_error().decode()    # noqa: E731
    ex, ki = co.forward_camera()
    ex, ki = np.ascontiguousarray(ex), np.ascontiguousarray(ki)
    n = C.c_int(-7)
    assert L.flb_frontend_camera_config(None, None, p(ki), W, H) != 0 and "null argument" in err()
    assert L.flb_frontend_camera_config(None, p(ex), None, W, H) != 0 and "null argument" in err()
    for w, h in ((0, H), (W, 0), (-1, H)):
        assert L.flb_frontend_camera_config(None, p(ex), p(ki), w, h) != 0 and "must be positive" in err()
    for k, bad in ((3, np.nan), (15, np.inf)):
        e2 = ex.copy()
        e2[k] = bad
        assert L.flb_frontend_camera_config(None, p(e2), p(ki), W, H) != 0 and f"cam_ex[{k}] is not finite" in err()
    k2 = ki.copy()
    k2[11] = -np.inf
    assert L.flb_frontend_camera_config(None, p(ex), p(k2), W, H) != 0 and "cam_in[11] is not finite" in err()
    assert L.flb_frontend_camera_config(None, p(ex), p(ki), W, H) != 0 and "null front end" in err()
    img = image(1, 4, 4)
    assert L.flb_frontend_camera_image(None, None, 4, 4, 12) != 0 and "null image" in err()
    assert L.flb_frontend_camera_image(None, p(img), 0, 4, 12) != 0 and "must be positive" in err()
    assert L.flb_frontend_camera_image(None, p(img), 4, 4, 11) != 0 and "row step 11" in err()
    assert L.flb_frontend_camera_image(None, p(img), 4, 4, 12) != 0 and "null front end" in err()
    st = synth.make_state()
    out = np.empty((4, 4), np.float32)
    col = np.empty(4, np.uint32)
    for which in (-1, 2):
        assert L.flb_frontend_points_colorize(None, which, p(st), p(out), p(col), 4, C.byref(n)) != 0 and "which must be" in err()
    assert L.flb_frontend_points_colorize(None, 0, None, p(out), p(col), 4, C.byref(n)) != 0 and "null argument" in err()
    assert L.flb_frontend_points_colorize(None, 0, p(st), p(out), p(col), 4, None) != 0 and "null argument" in err()
    assert L.flb_frontend_points_colorize(None, 0, p(st), None, p(col), 4, C.byref(n)) != 0 and "null output" in err()
    assert L.flb_frontend_points_colorize(None, 0, p(st), p(out), None, 4, C.byref(n)) != 0 and "null output" in err()
    assert L.flb_frontend_points_colorize(None, 0, p(st), p(out), p(col), -1, C.byref(n)) != 0 and "negative" in err()
    assert L.flb_frontend_points_colorize(None, 1, p(st), None, None, 0, C.byref(n)) != 0 and "null front end" in err()
    assert L.flb_frontend_points_to_imu(None, None, p(out), 4, C.byref(n)) != 0 and "null state" in err()
    assert L.flb_frontend_points_to_imu(None, p(st), p(out), 4, C.byref(n)) != 0 and "null front end" in err()


def test_python_layer_checks_shapes():
    from better_fastlio2_b200 import capi

    class _Fake(capi.FrontEnd):
        def __init__(self):
            self.h = None

    f = _Fake()
    with pytest.raises(ValueError):
        f.set_camera(np.zeros(15), np.zeros(12))
    with pytest.raises(ValueError):
        f.upload_image(np.zeros((4, 4), np.uint8))
    with pytest.raises(ValueError):
        f.upload_image(np.zeros((4, 4, 3), np.float32))


def test_header_documents_the_publishers():
    src = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for cite in ("laserMapping.cpp:310-392", ":279-289", ":250-276", "laserMapping.cpp:1543-1558", ":1113-1122", ":2045-2046"):
        assert cite in src, cite


def test_color_facade_compiles_and_fails_loudly_without_a_gpu(L):
    from better_fastlio2_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "color_facade_smoke")
        cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", "color_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
               f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    if capi.device_count() > 0:
        assert out.returncode == 0 and "COLOR_FACADE_OK" in out.stdout, (out.returncode, out.stdout, out.stderr)
    else:   # no device: the front end cannot be attached, and the facade says so on stderr
        assert out.returncode == 0 and "NO_GPU" in out.stdout and "set_camera" in out.stderr, (out.stdout, out.stderr)
