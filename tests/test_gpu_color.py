"""GPU tests of the camera-coloured and IMU-frame publishers (flb_frontend_camera_config / _camera_image /
_points_colorize / _points_to_imu) against the CPU oracle (tests/cpp/color_oracle.cpp): bit-exact count, order, world
x, y, z, intensity and colour on a Livox HAP scan through flb_frontend_process, the image handling, the projection's
directed cases, cloud sizes on the kernels' launch boundaries, and no effect on the scan step that follows."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import color_oracle as co
from tests.helpers import small_scene

pytestmark = pytest.mark.gpu

W, H = co.W_MAX, co.H_MAX
ALPHA = np.uint32(255 << 24)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


@pytest.fixture(scope="module")
def hap():
    sc = small_scene(seed=21, model="hap", map_half=40.0, half_extent=100.0)
    rng = np.random.default_rng(8)
    xyz, inten, cur = synth.raw_scan_with_times(sc["body"], rng)
    poses, end = synth.imu_pose_sequence(sc["st_true"], rng)
    return dict(scene=sc, pts48=np.ascontiguousarray(capi.pack_pointtype(xyz, inten, cur)),
                poses=np.ascontiguousarray(poses, np.float64), end=np.ascontiguousarray(end, np.float64))


def _rig(cap=1 << 18, scan_cap=1 << 18):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
    ses = capi.Session(tree, max_scan_points=scan_cap, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=cap)
    return tree, ses, fe


@pytest.fixture()
def rig():
    tree, ses, fe = _rig()
    yield tree, ses, fe
    fe.close()
    ses.close()
    tree.close()


def _process(fe, hap, leaf=0.5):
    b = hap["pts48"]
    return fe.process_ptr(b.ctypes.data, len(b), hap["poses"], hap["end"], leaf)


def _camera(seed=0):
    return co.forward_camera(fx=900.0 + 0.25 * seed, fy=899.75, t=(0.04, -0.03, 0.12))


def _state(hap):
    st = hap["scene"]["st_true"].copy()
    st[7:11] = synth.quat_from_rotvec((0.01, -0.02, 0.015))
    return st


def _image(seed, rows=H, cols=W):
    return np.random.default_rng(seed).integers(0, 256, (rows, cols, 3), dtype=np.uint8)


@pytest.mark.parametrize("which", [0, 1])
def test_hap_scan_bit_exact_against_oracle(hap, rig, which):
    tree, ses, fe = rig
    n_down = _process(fe, hap)
    und, _, _ = fe.download_undistorted()
    down, _ = fe.download_down()
    cloud = down if which == 0 else und
    assert len(down) == n_down and len(und) == len(hap["pts48"]) > 50000
    ex, ki = _camera(which)
    img = _image(31 + which)
    fe.set_camera(ex, ki)
    fe.upload_image(img)
    st = _state(hap)
    xyzi, bgra, n = fe.colorize(which, st)
    o_xyzi, o_bgra, o_idx = co.colorize(ex, ki, img, cloud, st)
    assert n == len(o_idx) == len(xyzi) and 0 < n < len(cloud)
    assert _same(xyzi, o_xyzi) and _same(bgra, o_bgra)
    # world coordinates are flb_frontend_points_to_world's at the kept indices
    w = fe.points_to_world(which, st)
    assert _same(xyzi, w[o_idx])
    assert (bgra >> 24 == 255).all() and len(np.unique(bgra)) > 100


def test_to_imu_bit_exact(hap, rig):
    tree, ses, fe = rig
    _process(fe, hap)
    und, _, _ = fe.download_undistorted()
    st = _state(hap)
    got = fe.to_imu(st)
    assert _same(got, co.to_imu(und, st))
    # identity extrinsic rotation still goes through the quaternion (no shortcut): the oracle agrees bit for bit
    st2 = st.copy()
    st2[7:11] = (0, 0, 0, 1)
    assert _same(fe.to_imu(st2), co.to_imu(und, st2))


def test_image_handling(hap, rig):
    tree, ses, fe = rig
    _process(fe, hap)
    und, _, _ = fe.download_undistorted()
    st = _state(hap)
    ex, ki = _camera()
    with pytest.raises(capi.FlbError, match="camera not configured"):
        fe.colorize(1, st)
    with pytest.raises(capi.FlbError, match="camera not configured"):
        fe.upload_image(_image(1))
    fe.set_camera(ex, ki)
    # before any image: every colour is zero
    xyzi, bgra, n = fe.colorize(1, st)
    o = co.colorize(ex, ki, None, und, st)
    assert n == len(o[2]) > 0 and (bgra == ALPHA).all() and _same(xyzi, o[0])
    # a second upload replaces the first
    a, b = _image(2), _image(3)
    fe.upload_image(a)
    fe.upload_image(b)
    _, bgra, _ = fe.colorize(1, st)
    assert _same(bgra, co.colorize(ex, ki, b, und, st)[1])
    # padded rows: a (H, W) window of a wider buffer (row step 3 * (W + 13) bytes)
    wide = _image(4, H, W + 13)
    view = wide[:, :W]
    assert view.strides[0] == 3 * (W + 13)
    fe.upload_image(view)
    _, bgra, _ = fe.colorize(1, st)
    assert _same(bgra, co.colorize(ex, ki, wide[:, :W], und, st)[1])
    # a larger image: its top-left H x W window
    big = _image(5, H + 9, W + 21)
    fe.upload_image(big)
    _, bgra, _ = fe.colorize(1, st)
    assert _same(bgra, co.colorize(ex, ki, big, und, st)[1])
    # a smaller image is rejected and leaves the last one in place
    for small in (_image(6, H - 1, W), _image(6, H, W - 1)):
        with pytest.raises(capi.FlbError, match="smaller than the configured"):
            fe.upload_image(small)
    _, bgra2, _ = fe.colorize(1, st)
    assert _same(bgra, bgra2)
    # configuring the camera again zero-fills the image; another size bounds the pixels
    fe.set_camera(ex, ki, 640, 480)
    xyzi, bgra, n = fe.colorize(1, st)
    o = co.colorize(ex, ki, None, und, st, 640, 480)
    assert n == len(o[2]) and (bgra == ALPHA).all() and _same(xyzi, o[0])
    fe.upload_image(big)
    _, bgra, _ = fe.colorize(1, st)
    assert _same(bgra, co.colorize(ex, ki, big[:480, :640], und, st, 640, 480)[1])
    with pytest.raises(capi.FlbError, match="not finite"):
        fe.set_camera(np.where(np.arange(16) == 5, np.nan, ex), ki)


def _directed_points():
    """Lidar-frame points for the pixel camera u = x / z, v = y / z and the camera u = y, v = z (c2 = 1)."""
    w_eps, h_eps = np.nextafter(np.float32(W), np.float32(0)), np.nextafter(np.float32(H), np.float32(0))
    pix = [(1, 0, 2), (2, 0, 1), (0.5, 1, -1), (1, 0, -2), (1, 3, 1), (w_eps, 10, 1), (W, 10, 1), (5, h_eps, 1), (5, H, 1),
           (1, 0, -1), (1, -6, -2), (4, 6, 0), (4, 0, 0), (1, 3e9, 1), (np.nan, 1, 1), (1, np.inf, 1), (np.inf, 1, 1)]
    yz = [(1, 3, 4), (0.0, 3, 4), (-0.0, 3, 4), (-1, 3, 4), (1, -0.5, 4), (1, -1, 4), (1, w_eps, h_eps), (1, W, 3), (1, 3, H),
          (1, np.nan, 1), (1, 1, -np.inf), (1, -3e9, 1), (2.5, 0, 0)]
    return np.array(pix, np.float32), np.array(yz, np.float32)


def test_directed_cases_on_device(rig):
    tree, ses, fe = rig
    pix, yz = _directed_points()
    cams = [(np.eye(4).reshape(-1), np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float64)),
            (np.eye(4).reshape(-1), np.array([-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0], np.float64)),
            (np.eye(4).reshape(-1), np.array([0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1], np.float64))]
    img = _image(9)
    st = synth.make_state(pos=(1.5, -2.0, 0.25), rot=synth.quat_from_rotvec((0.1, 0.2, -0.3)))
    for pts in (pix, yz):
        inten = np.arange(len(pts), dtype=np.float32) + 0.5
        fe.upload(capi.pack_pointtype(pts, inten, np.zeros(len(pts), np.float32)))
        p4 = np.column_stack([pts, inten]).astype(np.float32)
        for ex, ki in cams:
            fe.set_camera(ex, ki)
            fe.upload_image(img)
            xyzi, bgra, n = fe.colorize(1, st)
            o = co.colorize(ex, ki, img, p4, st)
            assert n == len(o[2]) and _same(xyzi, o[0]) and _same(bgra, o[1]), (o[2], n)
    # the cases the contract singles out did what it says (pixel camera, then u = y, v = z)
    ex, ki = cams[0]
    kept = set(co.colorize(ex, ki, img, np.column_stack([pix, np.zeros(len(pix))]), st)[2].tolist())
    assert {0, 1, 3, 4, 5, 7, 10} <= kept and not kept & {2, 6, 8, 9, 11, 12, 13, 14, 15, 16}
    ex, ki = cams[2]
    kept = set(co.colorize(ex, ki, img, np.column_stack([yz, np.zeros(len(yz))]), st)[2].tolist())
    assert kept == {0, 4, 6, 12}


SIZES = [0, 1, 255, 256, 257, 132 * 8 * 256 - 1, 132 * 8 * 256, 132 * 8 * 256 + 1, 400000]


def test_sizes_and_capacity():
    tree, ses, fe = _rig(cap=1 << 19, scan_cap=1 << 12)
    try:
        rng = np.random.default_rng(12)
        ex, ki = _camera(3)
        fe.set_camera(ex, ki)
        img = _image(13)
        fe.upload_image(img)
        st = synth.make_state(pos=(3.0, 1.0, -0.5), rot=synth.quat_from_rotvec((0.0, 0.1, 0.4)))
        allp = np.column_stack([rng.uniform(-5, 60, 400000), rng.uniform(-40, 40, 400000), rng.uniform(-20, 20, 400000),
                                rng.uniform(0, 200, 400000)]).astype(np.float32)
        for n in SIZES:
            p4 = allp[:n]
            fe.upload(capi.pack_pointtype(p4[:, :3], p4[:, 3], np.zeros(n, np.float32)))
            xyzi, bgra, k = fe.colorize(1, st)
            o = co.colorize(ex, ki, img, p4, st)
            assert k == len(o[2]) and _same(xyzi, o[0]) and _same(bgra, o[1]), n
            assert _same(fe.to_imu(st), co.to_imu(p4, st)), n
            if k > 2:   # cap below the count: the first cap records, the full count
                for cap in (0, 1, k // 2, k - 1):
                    x2, b2, k2 = fe.colorize(1, st, cap=cap)
                    assert k2 == k and _same(x2, o[0][:cap]) and _same(b2, o[1][:cap]), (n, cap)
        # feats_down_body of an empty filtered scan
        fe.upload(capi.pack_pointtype(np.zeros((0, 3), np.float32)))
        assert fe.voxel_filter(0.5) == 0
        assert fe.colorize(0, st)[2] == 0
    finally:
        fe.close()
        ses.close()
        tree.close()


def test_no_side_effects(hap):
    sc = hap["scene"]
    outs = []
    for colour in (False, True):
        tree, ses, fe = _rig()
        try:
            tree.Build(sc["map"])
            _process(fe, hap)
            first = None
            if colour:
                ex, ki = _camera()
                fe.set_camera(ex, ki)
                fe.upload_image(_image(17))
                st = _state(hap)
                first = [fe.colorize(w, st) for w in (0, 1)] + [fe.to_imu(st)]
                again = [fe.colorize(w, st) for w in (0, 1)] + [fe.to_imu(st)]
                for a, b in zip(first[:2], again[:2]):
                    assert _same(a[0], b[0]) and _same(a[1], b[1]) and a[2] == b[2]
                assert _same(first[2], again[2])
            down, dc = fe.download_down()
            und, uc, perm = fe.download_undistorted()
            s, P, r = ses.scan_step(None, None, sc["prior"], sc["P"])
            outs.append((down, dc, und, uc, perm, s, P, r.update.effct_feat_num, r.n_to_add, tree.validnum()))
        finally:
            fe.close()
            ses.close()
            tree.close()
    a, b = outs
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert _same(x, y)
        else:
            assert x == y
