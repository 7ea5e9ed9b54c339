"""GPU tests of the device key-frame store (flb_keyframes) and its readers: append from the host and from the front end,
the sub-map rebuild from stored clouds, and the map assembly (pose6 / explicit affines, dense / VoxelGrid), against the
host-cloud entry point and the CPU oracle (oracle.transform_cloud_rpy + oracle.voxel_grid, stable order).  Everything
here is bit-exact: the assembly is the same float arithmetic as transformPointCloud (no FMA), the filter the same sums."""
import ctypes as C

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests.helpers import small_scene, sort_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def raw():
    sc = small_scene(seed=11, map_half=40.0, half_extent=100.0)
    rng = np.random.default_rng(5)
    xyz, inten, cur = synth.raw_scan_with_times(sc["body"], rng)
    poses, end = synth.imu_pose_sequence(sc["st_true"], rng)
    return dict(xyz=xyz, inten=inten, cur=cur, poses=poses, end=end, scene=sc, pts48=capi.pack_pointtype(xyz, inten, cur))


def _clouds(raw, seed=9, k=5, m=6000, empty_at=2):
    """k body-frame key frames of m points (x,y,z,intensity + curvature) and their poses; one empty key frame inserted."""
    rng = np.random.default_rng(seed)
    p4s, curs, poses = [], [], []
    for j in range(k):
        idx = rng.choice(len(raw["xyz"]), m, replace=False)
        p4s.append(np.column_stack([raw["xyz"][idx], raw["inten"][idx]]).astype(np.float32))
        curs.append(raw["cur"][idx].astype(np.float32))
        poses.append([3.0 * j, 0.2 * j, 0.1, 0.01 * j, -0.02, 0.3 * j])
    if empty_at is not None:
        p4s.insert(empty_at, np.zeros((0, 4), np.float32))
        curs.insert(empty_at, np.zeros(0, np.float32))
        poses.insert(empty_at, [0, 0, 0, 0, 0, 0])
    return p4s, curs, np.array(poses, np.float32)


def _pack(p4, cur):
    return capi.pack_pointtype(p4[:, :3], p4[:, 3], cur)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _store(tree, p4s, curs, max_points=1 << 20, max_kf=64):
    kf = capi.KeyFrameStore(tree, max_points, max_kf)
    for j, (p, c) in enumerate(zip(p4s, curs)):
        assert kf.append(_pack(p, c)) == j
    return kf


def _affine_np(t12, p4):
    """transformPointCloud with an explicit affine, float32, left to right, one rounding per operation."""
    t = np.asarray(t12, np.float32).reshape(12)
    x, y, z = p4[:, 0], p4[:, 1], p4[:, 2]
    out = np.empty_like(p4)
    for r in range(3):
        out[:, r] = ((t[4 * r] * x + t[4 * r + 1] * y) + t[4 * r + 2] * z) + t[4 * r + 3]
    out[:, 3] = p4[:, 3]
    return out


def test_host_append_download_bit_equal(raw):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    p4s, curs, _ = _clouds(raw)
    p4s[0][:3, 0] = [-0.0, np.nan, np.inf]          # stored as they are
    curs[0][:2] = [-0.0, np.nan]
    kf = _store(tree, p4s, curs)
    info = kf.info()
    assert info["n_keyframes"] == len(p4s) and info["n_points"] == sum(len(p) for p in p4s)
    assert info["device_bytes"] >= 20 * (1 << 20)
    for j, (p, c) in enumerate(zip(p4s, curs)):
        g, gc = kf.download(j)
        assert kf.size(j) == len(p) == len(g)
        assert np.array_equal(_bits(g), _bits(p)) and np.array_equal(_bits(gc), _bits(c))
    kf.close()
    tree.close()


@pytest.fixture()
def rig():
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
    ses = capi.Session(tree, max_scan_points=1 << 17, max_iterations=3)
    fe = capi.FrontEnd(ses, max_raw_points=1 << 17)
    yield tree, ses, fe
    fe.close()
    ses.close()
    tree.close()


def test_frontend_append_equals_feats_undistort(raw, rig):
    tree, ses, fe = rig
    kf = capi.KeyFrameStore(tree, 1 << 20, 8)
    fe.upload(raw["pts48"])                                   # no undistortion: upload order
    a = kf.append_frontend(fe)
    ref0 = fe.download_undistorted()
    fe.undistort(raw["poses"], raw["end"])                    # feats_undistort: time order, compensated
    b = kf.append_frontend(fe)
    ref1 = fe.download_undistorted()
    buf = np.ascontiguousarray(raw["pts48"])
    fe.process_ptr(buf.ctypes.data, len(buf), np.ascontiguousarray(raw["poses"], np.float64),
                   np.ascontiguousarray(raw["end"], np.float64), 0.5)
    c = kf.append_frontend(fe)
    ref2 = fe.download_undistorted()
    fe.upload(np.zeros((0, 12), np.float32))                 # an empty scan is an empty key frame
    d = kf.append_frontend(fe)
    assert (a, b, c, d) == (0, 1, 2, 3)
    for k, ref in zip((a, b, c), (ref0, ref1, ref2)):
        g, gc = kf.download(k)
        assert np.array_equal(_bits(g), _bits(ref[0])) and np.array_equal(_bits(gc), _bits(ref[1]))
    assert not np.array_equal(kf.download(a)[0], kf.download(b)[0])
    assert kf.size(d) == 0 and kf.info()["n_points"] == 3 * len(buf)
    kf.close()


def _host_rebuild(tree, p4s, poses, leaf):
    return capi.reconstruct_keyframes(tree, [capi.pack_pointtype(p[:, :3], p[:, 3]) for p in p4s], poses, leaf)


def test_reconstruct_from_store_equals_host_clouds(raw, oracle):
    p4s, curs, poses = _clouds(raw)
    leaf = 0.4
    ta = capi.KDTree(voxel_size=0.2, max_points=1 << 20, max_blocks=1 << 17)
    tb = capi.KDTree(voxel_size=0.2, max_points=1 << 20, max_blocks=1 << 17)
    tb.Build(raw["scene"]["map"][:5000])                      # previous content must disappear
    kf = _store(tb, p4s, curs)
    for ids in ([0, 1, 2, 3, 4, 5], [4, 0, 2, 5, 3, 1], [3, 3, 1]):   # in order, permuted (with the empty one), repeated
        ids = np.array(ids, np.int32)
        fa = _host_rebuild(ta, [p4s[i] for i in ids], poses[ids], leaf)
        fb = kf.reconstruct(ids, poses[ids], leaf)
        sub = np.concatenate([oracle.transform_cloud_rpy(p4s[i], poses[i]) for i in ids])
        o, _, _ = oracle.voxel_grid(sub, leaf, order="stable")
        assert np.array_equal(fb, fa) and np.array_equal(fb, o)
        assert tb.validnum() == ta.validnum() == len(o) == tb.size()
        assert np.array_equal(sort_rows(tb.flatten()), sort_rows(ta.flatten()))
        assert np.array_equal(sort_rows(tb.flatten_xyzi()), sort_rows(o))
    assert len(kf.reconstruct([], np.zeros((0, 6), np.float32), leaf)) == 0 and tb.validnum() == 0   # empty selection
    assert len(kf.reconstruct([2], poses[2:3], leaf)) == 0 and tb.validnum() == 0                   # only an empty key frame
    kf.close()
    ta.close()
    tb.close()


def test_scan_step_after_store_rebuild_is_identical(raw):
    """The posterior of a scan step right after the rebuild does not depend on where the key-frame clouds came from."""
    sc = raw["scene"]
    mp = np.asarray(sc["map"], np.float32)
    rng = np.random.default_rng(4)
    parts = np.array_split(rng.permutation(len(mp)), 4)
    p4s, poses = [], []
    for j, idx in enumerate(parts):
        t = np.array([0.5 * j, -0.25 * j, 0.1], np.float32)
        p4s.append(np.column_stack([mp[idx] - t, np.full(len(idx), j, np.float32)]).astype(np.float32))
        poses.append([t[0], t[1], t[2], 0, 0, 0])
    poses = np.array(poses, np.float32)
    ids = np.arange(4, dtype=np.int32)
    out = []
    for use_store in (False, True):
        tree = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
        ses = capi.Session(tree, max_scan_points=len(sc["body"]), max_iterations=3)
        if use_store:
            kf = _store(tree, p4s, [np.zeros(len(p), np.float32) for p in p4s])
            kf.reconstruct(ids, poses, 0.2)
        else:
            _host_rebuild(tree, p4s, poses, 0.2)
        st, P, r = ses.scan_step(None, sc["body"], sc["prior"], sc["P"])
        out.append((st, P, r.update.effct_feat_num, tree.validnum()))
        if use_store:
            kf.close()
        ses.close()
        tree.close()
    (sa, Pa, ma, va), (sb, Pb, mb, vb) = out
    assert ma > 500 and ma == mb and va == vb
    assert np.array_equal(sa, sb) and np.array_equal(Pa, Pb)


def test_assemble_pose6(raw, oracle):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    p4s, curs, poses = _clouds(raw)
    kf = _store(tree, p4s, curs)
    ids = np.array([3, 0, 2, 5, 1], np.int32)
    dense, dc = kf.assemble(ids, poses6=poses[ids])
    sub = np.concatenate([oracle.transform_cloud_rpy(p4s[i], poses[i]) for i in ids])
    assert np.array_equal(_bits(dense), _bits(sub)) and (dc == 0).all() and not np.signbit(dc).any()
    for leaf in (0.7, 0.3):
        g, gc = kf.assemble(ids, poses6=poses[ids], leaf=leaf)
        o, oc, ovf = oracle.voxel_grid(sub, leaf, curvature=np.zeros(len(sub), np.float32), order="stable")
        assert not ovf and np.array_equal(g, o) and np.array_equal(gc, oc)
    kf.close()
    tree.close()


def test_assemble_affine_and_identity_copy(raw, oracle):
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    p4s, curs, poses = _clouds(raw, empty_at=None)
    p4s[1][:2, :3] = -0.0                                     # -0 survives a copy (a computed identity would give +0)
    curs[1][:2] = -0.0
    kf = _store(tree, p4s, curs)
    rng = np.random.default_rng(2)
    A = oracle.rpy_matrix(np.array([1.0, -2.0, 0.5, 0.1, 0.2, -0.3], np.float32)).reshape(12)
    B = rng.normal(size=12).astype(np.float32)
    eye = np.eye(3, 4, dtype=np.float32).reshape(12)
    ids = np.array([0, 1, 4, 1], np.int32)
    aff = np.stack([A, eye, B, eye])
    dense, dc = kf.assemble(ids, affines=aff)
    want = np.concatenate([_affine_np(A, p4s[0]), p4s[1], _affine_np(B, p4s[4]), p4s[1]])
    want_c = np.concatenate([np.zeros(len(p4s[0]), np.float32), curs[1], np.zeros(len(p4s[4]), np.float32), curs[1]])
    assert np.array_equal(_bits(dense), _bits(want)) and np.array_equal(_bits(dc), _bits(want_c))
    # a rotation-free affine is not the identity: arithmetic (curvature 0)
    shift = eye.copy()
    shift[3] = 0.5
    g, gc = kf.assemble([2], affines=shift[None])
    assert np.array_equal(g, _affine_np(shift, p4s[2])) and (gc == 0).all()
    # filtered with curvature carried: the identity keeps the stored curvature, so the centroids average it
    g, gc = kf.assemble([0, 3], affines=np.stack([eye, eye]), leaf=0.5)
    o, oc, _ = oracle.voxel_grid(np.concatenate([p4s[0], p4s[3]]), 0.5, curvature=np.concatenate([curs[0], curs[3]]), order="stable")
    assert np.array_equal(g, o) and np.array_equal(gc, oc) and (gc != 0).any()
    kf.close()
    tree.close()


def test_assemble_overflow_guard_returns_input():
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    kf = capi.KeyFrameStore(tree, 1 << 10, 4)
    far = np.array([[0, 0, 0, 1], [500, 500, 500, 2], [-100, 3, 9, 3]], np.float32)
    cur = np.array([5, 6, 7], np.float32)
    kf.append(_pack(far, cur))
    g, gc = kf.assemble([0], affines=np.eye(3, 4, dtype=np.float32)[None], leaf=0.001)
    assert np.array_equal(g, far) and np.array_equal(gc, cur)
    g, gc = kf.assemble([0], poses6=np.zeros((1, 6), np.float32), leaf=0.001)
    assert np.array_equal(g[:, :3], far[:, :3]) and (gc == 0).all()
    kf.close()
    tree.close()


def test_error_paths_leave_the_store_unchanged(raw, rig):
    tree, ses, fe = rig
    kf = capi.KeyFrameStore(tree, 10000, 3)
    p4s, curs, poses = _clouds(raw, k=3, m=4000, empty_at=None)
    kf.append(_pack(p4s[0], curs[0]))
    kf.append(_pack(p4s[1], curs[1]))
    before = kf.info()
    with pytest.raises(capi.FlbError, match="does not fit"):      # point capacity
        kf.append(_pack(p4s[2], curs[2]))
    fe.upload(raw["pts48"][:4000])
    with pytest.raises(capi.FlbError, match="does not fit"):
        kf.append_frontend(fe)
    assert kf.info() == before
    assert np.array_equal(kf.download(1)[0], p4s[1])
    kf.append(_pack(p4s[2][:10], curs[2][:10]))
    with pytest.raises(capi.FlbError, match="store full"):       # key-frame capacity
        kf.append(_pack(p4s[2][:10], curs[2][:10]))
    assert kf.info()["n_keyframes"] == 3
    # ids out of range: nothing runs, the map keeps its content
    tree.Build(raw["scene"]["map"][:3000])
    v = tree.validnum()
    with pytest.raises(capi.FlbError, match="out of range"):       # cap given: the library's own check is reached
        kf.reconstruct([0, 3], poses[:2], 0.4, cap=10)
    with pytest.raises(capi.FlbError, match="out of range"):
        kf.assemble([-1], poses6=poses[:1], cap=10)
    with pytest.raises(capi.FlbError, match="out of range"):
        kf.download(3)
    with pytest.raises(capi.FlbError):
        kf.size(7)
    assert tree.validnum() == v
    # a front end (and a map) of another map
    t2 = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    s2 = capi.Session(t2, max_scan_points=1 << 12)
    f2 = capi.FrontEnd(s2, max_raw_points=1 << 12)
    f2.upload(raw["pts48"][:100])
    with pytest.raises(capi.FlbError, match="another map"):
        kf.append_frontend(f2)
    n = C.c_int(0)
    ids = np.array([0], np.int32)
    assert capi.lib().flb_map_reconstruct_from_keyframes(t2.h, kf.h, capi._p(ids), 1, capi._p(poses[:1]), C.c_float(0.4), None, 0,
                                                         C.byref(n)) != 0
    assert b"another map" in capi.lib().flb_last_error()
    # cap smaller than the output: the first cap points, *n_out the full size
    full, fc = kf.assemble([1, 0], poses6=poses[[1, 0]])
    part, pc, n_full = kf.assemble([1, 0], poses6=poses[[1, 0]], cap=10, return_size=True)
    assert n_full == len(full) == 8000 and np.array_equal(part, full[:10]) and np.array_equal(pc, fc[:10])
    _, _, n_ds = kf.assemble([1, 0], poses6=poses[[1, 0]], leaf=0.5, cap=0, return_size=True)
    assert 0 < n_ds < 8000
    with pytest.raises(capi.FlbError):
        kf.assemble([0], poses6=poses[:1], leaf=-1.0)
    assert kf.info()["n_points"] == 8010
    f2.close()
    s2.close()
    t2.close()
    kf.close()


def test_cfg3_size_rebuild_agrees(oracle):
    """40 key frames of 240k points (the cfg3 sub-map) through both entry points."""
    rng = np.random.default_rng(3)
    base = []
    for j in range(4):
        p = np.empty((240000, 4), np.float32)
        p[:, 0] = rng.uniform(2, 60, 240000)
        p[:, 1] = rng.uniform(-20, 20, 240000)
        p[:, 2] = rng.uniform(-2, 2, 240000)
        p[:, 3] = rng.integers(0, 256, 240000)
        base.append(p)
    p4s = [base[k % 4] for k in range(40)]
    poses = np.array([[0.25 * k, 0.05 * k, 0.0, 0.0, 0.0, 0.02 * k] for k in range(40)], np.float32)
    ta = capi.KDTree(voxel_size=0.1, max_points=1 << 23, max_blocks=1 << 20)
    tb = capi.KDTree(voxel_size=0.1, max_points=1 << 23, max_blocks=1 << 20)
    fa = _host_rebuild(ta, p4s, poses, 0.2)
    kf = capi.KeyFrameStore(tb, 40 * 240000, 40)
    for p in p4s:
        kf.append(capi.pack_pointtype(p[:, :3], p[:, 3]))
    fb = kf.reconstruct(np.arange(40), poses, 0.2)
    assert len(fb) > 100000 and np.array_equal(fa, fb)
    assert ta.validnum() == tb.validnum() == len(fb)
    # the CPU oracle on a slice of the same sub-map (the full one takes minutes on one core)
    sub = np.concatenate([oracle.transform_cloud_rpy(p4s[k], poses[k]) for k in range(3)])
    o, _, _ = oracle.voxel_grid(sub, 0.2, order="stable")
    assert np.array_equal(kf.reconstruct(np.arange(3), poses[:3], 0.2), o)
    kf.close()
    ta.close()
    tb.close()


def test_scratch_is_sized_per_path_reported_and_released(raw, oracle):
    """A dense assembly allocates no filter buffers; the map-side scratch is reported and can be given back, after which
    every reader still works (and gives the same answer)."""
    tree = capi.KDTree(voxel_size=0.2, max_points=1 << 20, max_blocks=1 << 17)
    p4s, curs, poses = _clouds(raw, empty_at=None)
    kf = _store(tree, p4s, curs)
    ids = np.arange(len(p4s), dtype=np.int32)
    n = sum(len(p) for p in p4s)
    assert kf.info()["map_scratch_bytes"] == 0
    dense, dc = kf.assemble(ids, poses6=poses)
    after_dense = kf.info()["map_scratch_bytes"]
    assert 20 * n <= after_dense < 2 * 20 * n                 # kf_in + its curvature (+ growth margin, segment table)
    g, gc = kf.assemble(ids, poses6=poses, leaf=0.5)
    after_filter = kf.info()["map_scratch_bytes"]
    assert after_filter > 2 * after_dense                     # + kf_out, its curvature, the voxel-grid workspace
    kf.release_scratch()
    assert kf.info()["map_scratch_bytes"] == 0
    g2, gc2 = kf.assemble(ids, poses6=poses, leaf=0.5)
    assert np.array_equal(g2, g) and np.array_equal(gc2, gc)
    feats = kf.reconstruct(ids, poses, 0.4)
    sub = np.concatenate([oracle.transform_cloud_rpy(p, q) for p, q in zip(p4s, poses)])
    assert np.array_equal(feats, oracle.voxel_grid(sub, 0.4, order="stable")[0])
    kf.release_scratch()
    assert tree.validnum() == len(feats)                       # the map's contents are not scratch
    assert np.array_equal(_host_rebuild(tree, p4s, poses, 0.4), feats)
    kf.close()
    tree.close()
