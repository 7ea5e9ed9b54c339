"""GPU parity tests of flb_frontend_preprocess (Preprocess::process on the device) against the CPU oracle
(tests/cpp/preprocess_oracle.cpp), and of the chain driver records -> preprocess -> UndistortPcl -> VoxelGrid -> update.

Exactness: output count and order, x, y, z and intensity are bit-exact, and so is every curvature not derived from
atan2.  For Velodyne clouds without per-point time the synthesised times go through the device's double atan2
(within 2 ulp; glibc's is close to correctly rounded): identical drop / keep / wrap decisions, curvature within 1 float
ulp and at least 99.99 % of curvatures bit-equal."""
import subprocess
import tempfile

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import preprocess_cases as pc
from tests import preprocess_oracle as po
from tests.helpers import small_scene

pytestmark = pytest.mark.gpu

CASES = pc.cases()


@pytest.fixture(scope="module")
def rig():
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
    ses = capi.Session(tree, max_scan_points=1 << 18, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 18)
    yield tree, ses, fe
    fe.close()
    ses.close()
    tree.close()


def _synthesised(rec, cfg):
    if cfg["lidar_type"] != capi.VELO16 or len(rec) == 0:
        return False
    return "time" not in rec.dtype.names or not (rec["time"][-1] > 0)


def _ulp_close(a, b, ulps=1):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    tol = ulps * np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))
    return (np.abs(a - b) <= tol) | (np.isnan(a) & np.isnan(b))


def _bits_equal(a, b):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _check(fe, rec, cfg):
    n, last = fe.preprocess(rec, cfg)
    g_xyzi, g_cur, perm = fe.download_undistorted()      # no undistortion yet: upload (= message) order
    o_xyzi, o_cur, o_last = po.preprocess(rec, cfg)
    assert n == len(o_xyzi) == len(g_xyzi)
    assert np.array_equal(perm, np.arange(n))
    assert _bits_equal(g_xyzi, o_xyzi).all()
    if _synthesised(rec, cfg):
        assert _ulp_close(g_cur, o_cur).all(), np.abs(g_cur - o_cur).max()
        assert _bits_equal(g_cur, o_cur).mean() >= 0.9999 if n else True
        assert _ulp_close(last, o_last).all()
    else:
        assert _bits_equal(g_cur, o_cur).all()
        assert _bits_equal(last, o_last)
    return g_xyzi, g_cur


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_match_oracle(rig, name):
    _check(rig[2], *CASES[name])


@pytest.mark.parametrize("model,with_time", [("hdl64", True), ("hdl64", False), ("vlp16", False), ("os64", True), ("hap", True)])
def test_full_sweeps_match_oracle(rig, model, with_time):
    rec, cfg = pc.synthetic(model, with_time=with_time)
    xyzi, cur = _check(rig[2], rec, cfg)
    assert len(xyzi) > 5000
    if cfg["lidar_type"] == capi.VELO16 and not with_time:
        assert cur.max() > 90.0      # the synthesised times span the sweep


def test_decimation_and_layout_variants(rig):
    """point_filter_num on full sweeps and a field-order variant (time before ring, 32-byte aligned records)."""
    rec, cfg = pc.synthetic("hdl64", with_time=False)
    for pfn in (3, 4):
        _check(rig[2], rec, dict(cfg, point_filter_num=pfn))
    dt = np.dtype({"names": ["x", "y", "z", "intensity", "time", "ring"], "formats": ["<f4"] * 5 + ["<u2"],
                   "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
    rec2 = np.zeros(len(rec), dt)
    for k in ("x", "y", "z", "intensity", "ring"):
        rec2[k] = rec[k]
    _check(rig[2], rec2, cfg)


def test_ring_out_of_range_and_capacity(rig):
    tree, ses, fe = rig
    rec, cfg = CASES["velo_notime_wrap"]
    with pytest.raises(capi.FlbError, match="ring 3 >= n_scans=3"):
        fe.preprocess(rec, dict(cfg, n_scans=3))
    assert fe.download_undistorted()[0].shape[0] == 0       # the failed call leaves an empty scan
    _check(fe, rec, cfg)                                     # and the front end stays usable
    small = capi.FrontEnd(ses, max_raw_points=100)
    with pytest.raises(capi.FlbError, match="max_raw_points"):
        small.preprocess(rec[:101], cfg)
    n, _ = small.preprocess(rec[:100], cfg)
    assert n == 96
    small.close()


def test_preprocess_then_undistort_and_filter(rig, oracle):
    tree, ses, fe = rig
    rng = np.random.default_rng(5)
    rec, cfg = pc.synthetic("vlp16", with_time=False)
    poses, end = synth.imu_pose_sequence(synth.trajectory_state(0), rng)
    fe.preprocess(rec, cfg)
    fe.undistort(poses, end)
    und, ucur, perm = fe.download_undistorted()
    o_xyzi, o_cur, _ = po.preprocess(rec, cfg)
    assert _ulp_close(ucur, o_cur[perm]).all()
    o_xyz, o_perm = oracle.undistort(o_xyzi[:, :3], o_cur, poses, end)
    g_by_in = np.empty((len(und), 3), np.float32)
    o_by_in = np.empty((len(und), 3), np.float32)
    g_by_in[perm] = und[:, :3]
    o_by_in[o_perm] = o_xyz
    assert _ulp_close(g_by_in, o_by_in, ulps=2).all()
    assert (g_by_in == o_by_in).mean() > 0.999
    n_out = fe.voxel_filter(0.5)
    g, gc = fe.download_down()
    o, oc, _ = oracle.voxel_grid(und, 0.5, curvature=ucur, order="stable")
    assert n_out == len(o) and np.array_equal(g, o) and np.array_equal(gc, oc)


@pytest.mark.parametrize("with_time", [True, False])
def test_driver_records_to_posterior(rig, oracle, with_time):
    """driver records -> preprocess -> UndistortPcl -> VoxelGrid -> update on the GPU vs the same chain on the oracle."""
    tree, ses, fe = rig
    sc = small_scene(seed=11, map_half=40.0, half_extent=100.0)
    rng = np.random.default_rng(17)
    rec = synth.driver_records("vlp16", sc["world"], sc["st_true"], rng, with_time=with_time)
    cfg = dict(lidar_type=capi.VELO16, n_scans=16, scan_rate=10, point_filter_num=1, time_unit=capi.SEC, blind=2.0)
    poses, end = synth.imu_pose_sequence(sc["st_true"], rng)
    tree.Build(sc["map"])
    n, last = fe.preprocess(rec, cfg)
    fe.undistort(poses, end)
    n_out = fe.voxel_filter(0.5)
    assert n_out > 1000
    s_gpu, P_gpu, r = ses.scan_step(None, None, sc["prior"], sc["P"])
    o_xyzi, o_cur, o_last = po.preprocess(rec, cfg)
    assert n == len(o_xyzi) and _ulp_close(last, o_last).all()
    o_xyz, o_perm = oracle.undistort(o_xyzi[:, :3], o_cur, poses, end)
    o_ds, _, _ = oracle.voxel_grid(np.column_stack([o_xyz, o_xyzi[o_perm, 3]]), 0.5, order="pcl")
    assert abs(len(o_ds) - n_out) <= 2                      # a 1-ulp time may move a point across a leaf face
    ref = oracle.make_map(ds=0.2)
    ref.Build(sc["map"])
    s_cpu, P_cpu, *_ = oracle.esikf_update(sc["prior"], sc["P"], o_ds[:, :3], ref, max_iter=3)
    assert np.abs(s_gpu[:3] - s_cpu[:3]).max() <= 1e-4
    assert np.abs(s_gpu[3:7] - s_cpu[3:7]).max() <= 1e-4
    assert r.update.effct_feat_num > 500


def test_preprocess_facade_on_device():
    from tests.test_oracle_preprocess import build_facade_smoke
    with tempfile.TemporaryDirectory() as d:
        exe = build_facade_smoke(d)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "PREPROCESS_FACADE_OK" in out.stdout
