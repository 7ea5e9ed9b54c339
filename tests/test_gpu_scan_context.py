"""GPU tests of the Scan Context readers of the key-frame store (flb_keyframes_scan_context / _scan_contexts) against the
CPU oracle (tests/cpp/scan_context_oracle.cpp, a literal restatement of makeScancontext).  The only tolerated difference
is the device's double atan (within 2 ulp of glibc's): bins an atan-sensitive point could reach are left out of the
comparison, and the number of such points is asserted small and reported.  Everything else is bit-exact."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import scan_context_oracle as sco
from tests.scan_context_cases import edge_points, sc_distance

pytestmark = pytest.mark.gpu

H = 1.5
EYE = np.eye(3, 4, dtype=np.float32).reshape(12)


def _scan(world, model, pos=(3.0, 2.0, 1.8), yaw=0.0, seed=0, n_rays=None):
    """One ray-cast scan in the LiDAR frame, the sensor yawed by `yaw` in the world.  The ray azimuths are turned by a
    non-grid angle, so that a spinning LiDAR's columns do not sit on 6-degree sector boundaries."""
    rng = np.random.default_rng(seed)
    dirs = synth.lidar_dirs(model, np.random.default_rng(100 + seed))
    if n_rays:
        dirs = dirs[:n_rays]
    c, s = np.cos(0.0123), np.sin(0.0123)
    dirs = dirs @ np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]).T
    st = synth.make_state(pos=pos, rot=synth.quat_from_rotvec([0.0, 0.0, yaw]))
    return synth.scan_from_pose(world, st, dirs, rng, max_range=100.0, min_range=1.0)


def _p4(xyz, seed=0):
    rng = np.random.default_rng(seed)
    return np.column_stack([xyz, rng.integers(0, 256, len(xyz))]).astype(np.float32)


@pytest.fixture(scope="module")
def clouds():
    world = synth.city_world(half_extent=150.0, seed=4)
    c = [_p4(_scan(world, "hdl64", seed=0), 0),
         _p4(_scan(world, "hap", pos=(8.0, -1.0, 1.8), seed=1, n_rays=80000), 1),
         edge_points(H),
         np.zeros((0, 4), np.float32),
         _p4(_scan(world, "hdl64", pos=(-6.0, 4.0, 1.8), yaw=0.7, seed=2), 2)]
    return world, c


@pytest.fixture()
def store(clouds):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, 1 << 20, 16)
    for p in clouds[1]:
        kf.append(capi.pack_pointtype(p[:, :3], p[:, 3], np.linspace(0, 1, len(p), dtype=np.float32)))
    yield kf
    kf.close()
    tree.close()


def _agree(gpu, pts, h=H, what=""):
    """gpu equals the oracle's descriptor of pts on every bin no atan-sensitive point reaches; returns the number of
    sensitive points."""
    o, sens, mask = sco.scan_context(pts, h)
    assert gpu.shape == (20, 60) and gpu.dtype == np.float64
    bad = (gpu != o) & ~mask
    assert not bad.any(), (what, np.argwhere(bad)[:5], gpu[bad][:5], o[bad][:5])
    assert (np.isnan(gpu) == np.isnan(o)).all()
    # the edge-case key frame puts 9 points on the 90 / 180 / 270 degree boundaries on purpose; ray-cast scans have
    # a few per million
    assert sens.sum() <= max(16, len(pts) // 2000), (what, int(sens.sum()))
    if len(pts):
        print(f"[scan_context] {what}: {len(pts)} points, {int(sens.sum())} atan-sensitive, {int(mask.sum())} bins left out, "
              f"{int(((gpu != o) & mask).sum())} of them differ")
    return int(sens.sum())


def _snapshot(kf, n):
    return [kf.download(k) for k in range(n)]


def _same_store(kf, snap):
    for k, (p, c) in enumerate(snap):
        q, d = kf.download(k)
        assert np.array_equal(q.view(np.uint32), p.view(np.uint32)) and np.array_equal(d.view(np.uint32), c.view(np.uint32))


def test_saver_equals_oracle(clouds, store):
    _, cs = clouds
    snap = _snapshot(store, len(cs))
    ids = np.arange(len(cs), dtype=np.int32)
    for h in (H, 0.0, -0.75):
        descs = store.scan_contexts(ids, lidar_height=h)
        assert descs.shape == (len(cs), 20, 60)
        for j, p in enumerate(cs):
            _agree(descs[j], p, h, f"key frame {j}, lidar_height {h}")
        assert not descs[3].any() and (descs[0] != 0).sum() > 300 and (descs[1] != 0).sum() > 100
    # permuted and repeated ids: each descriptor is its key frame's
    perm = np.array([4, 2, 0, 2, 3], np.int32)
    dp = store.scan_contexts(perm)
    d = store.scan_contexts(ids)
    assert np.array_equal(dp, d[perm])
    assert store.scan_contexts([]).shape == (0, 20, 60)
    _same_store(store, snap)


def test_saver_equals_single_selection_bit_for_bit(clouds, store):
    ids = np.array([0, 1, 2, 3, 4], np.int32)
    descs = store.scan_contexts(ids)
    for j, k in enumerate(ids):
        one = store.scan_context([k], affines=EYE[None])
        assert np.array_equal(one.view(np.uint64), descs[j].view(np.uint64))


def _poses(n):
    return np.array([[1.5 * j, -0.5 * j, 0.1 * j, 0.01 * j, -0.02 * j, 0.3 * j] for j in range(n)], np.float32)


def test_loop_submap_equals_oracle_of_assembly(clouds, store, oracle):
    _, cs = clouds
    snap = _snapshot(store, len(cs))
    poses = _poses(len(cs))
    for ids in ([0, 1, 2, 3, 4], [4, 3, 0, 2], [1, 1, 0], [3], [2]):   # in order, permuted with the empty one, repeated
        ids = np.array(ids, np.int32)
        g = store.scan_context(ids, poses6=poses[ids], lidar_height=H)
        dense, _ = store.assemble(ids, poses6=poses[ids])
        _agree(g, dense, H, f"pose6 {ids.tolist()}")
        # the fused kernel and the oracle's own transformPointCloud cannot drift apart unnoticed
        sub = np.concatenate([oracle.transform_cloud_rpy(cs[i], poses[i]) for i in ids])
        # (bit for bit except NaN payloads: the edge-case key frame's Inf * 0 makes the device's and x86's default NaNs)
        nan = np.isnan(dense)
        assert np.array_equal(nan, np.isnan(sub)) and np.array_equal(dense.view(np.uint32)[~nan], sub.view(np.uint32)[~nan])
        _agree(g, sub, H, f"pose6 via oracle transform {ids.tolist()}")
    # affines, with the identity entry (stored records copied) as loopFindNearKeyframes passes them
    rng = np.random.default_rng(2)
    A = oracle.rpy_matrix(np.array([1.0, -2.0, 0.5, 0.1, 0.2, -0.3], np.float32)).reshape(12)
    B = rng.normal(size=12).astype(np.float32)
    for ids, aff in (([0, 4, 1], [EYE, A, B]), ([4, 0, 2, 4], [A, EYE, EYE, EYE]), ([3, 1], [A, EYE])):
        ids = np.array(ids, np.int32)
        aff = np.stack(aff)
        g = store.scan_context(ids, affines=aff, lidar_height=-0.25)
        dense, _ = store.assemble(ids, affines=aff)
        _agree(g, dense, -0.25, f"affines {ids.tolist()}")
    # an empty selection and a selection of empty key frames: all zeros
    assert not store.scan_context([], poses6=np.zeros((0, 6), np.float32)).any()
    assert not store.scan_context([3, 3], affines=np.stack([A, EYE])).any()
    _same_store(store, snap)


def test_invalid_arguments_on_a_store(store):
    snap = _snapshot(store, 5)
    with pytest.raises(capi.FlbError, match="out of range"):
        store.scan_context([0, 5], poses6=_poses(2))
    with pytest.raises(capi.FlbError, match="out of range"):
        store.scan_context([-1], affines=EYE[None])
    with pytest.raises(capi.FlbError, match="out of range"):
        store.scan_contexts([1, 9])
    with pytest.raises(capi.FlbError, match="finite"):
        store.scan_contexts([1], lidar_height=float("nan"))
    with pytest.raises(capi.FlbError, match="finite"):
        store.scan_context([1], affines=EYE[None], lidar_height=float("inf"))
    _same_store(store, snap)


def test_yaw_shift_is_found_by_the_reference_distance(clouds):
    world, _ = clouds
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, 1 << 21, 16)
    kf.append(capi.pack_pointtype(_scan(world, "hdl64", seed=5)))
    ms = (3, 17, 41)
    for m in ms:
        kf.append(capi.pack_pointtype(_scan(world, "hdl64", yaw=np.deg2rad(6.0 * m), seed=5)))
    d = kf.scan_contexts(np.arange(1 + len(ms)))
    for j, m in enumerate(ms):
        dist, shift = sc_distance(d[0], d[1 + j])
        print(f"[scan_context] yaw {6 * m} deg: distance {dist:.4f}, shift {shift}")
        assert dist < 0.3 and min((shift - m) % 60, (m - shift) % 60) <= 1, (m, dist, shift)
    kf.close()
    tree.close()


def test_scratch_is_reported_and_released(clouds, store):
    ids = np.arange(5, dtype=np.int32)
    store.release_scratch()
    assert store.info()["map_scratch_bytes"] == 0
    a = store.scan_contexts(ids)
    s1 = store.info()["map_scratch_bytes"]
    assert s1 >= 5 * 1200 * 4
    b = store.scan_context(ids, poses6=_poses(5))
    assert store.info()["map_scratch_bytes"] >= s1
    store.release_scratch()
    assert store.info()["map_scratch_bytes"] == 0
    assert np.array_equal(store.scan_contexts(ids), a) and np.array_equal(store.scan_context(ids, poses6=_poses(5)), b)
    store.release_scratch()
    assert store.info()["map_scratch_bytes"] == 0
