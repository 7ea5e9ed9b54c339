"""GPU: the host layer's grow-only scratch and record uploads.  A buffer baked into a captured scan graph that is
regrown after the capture (the k-NN work list by a large Nearest_Search, the insert's scratch hash by a large
downsampled Add_Points) makes the next step re-capture: its result equals a fresh session's on a twin map.  Host
records keep their per-entry-point intensity / curvature meaning, and every scan upload path gives the same step.  An
under-determined scan that runs in step slot 1 hands over to the host engine like one in slot 0."""
import ctypes as C

import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import dense_cases as dc
from tests.helpers import small_scene, sort_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scans():
    return [small_scene(seed=s, map_half=25.0, half_extent=80.0) for s in (7, 8)]


def _tree(points):
    t = capi.KDTree(voxel_size=0.2, max_points=1 << 20, max_blocks=1 << 17)
    t.Build(points)
    return t


def _session(tree, scs):
    return capi.Session(tree, max_scan_points=max(len(sc["body"]) for sc in scs) + 64, max_iterations=3)


def _step(ses, sc):
    return ses.scan_step(None, sc["body"], sc["prior"], sc["P"], True)


def _same_step(a, b):
    (sa, Pa, ra), (sb, Pb, rb) = a, b
    assert np.array_equal(sa, sb) and np.array_equal(Pa, Pb)
    assert (ra.map_valid, ra.n_to_add, ra.n_no_downsample) == (rb.map_valid, rb.n_to_add, rb.n_no_downsample)


def _regrown_step_equals_fresh_session(scs, regrow):
    """Step 1 (captures the scan graph), regrow(tree, rng), step 2 on one session == the same on a twin map whose
    step 2 runs on a new session."""
    mp = scs[0]["map"]
    trees = [_tree(mp) for _ in range(2)]
    ses = _session(trees[0], scs)
    _step(ses, scs[0])
    regrow(trees[0], np.random.default_rng(4))
    again = _step(ses, scs[1])
    ses.close()
    first = _session(trees[1], scs)
    _step(first, scs[0])
    regrow(trees[1], np.random.default_rng(4))
    first.close()
    fresh = _session(trees[1], scs)
    captured = _step(fresh, scs[1])
    fresh.close()
    _same_step(again, captured)
    assert np.array_equal(sort_rows(trees[0].flatten_xyzi()), sort_rows(trees[1].flatten_xyzi()))
    for t in trees:
        t.close()


def test_worklist_regrown_after_capture(scans):
    """More queries than the work list's 131072-entry floor (and the session's capacity) regrow it."""
    cap = max(len(sc["body"]) for sc in scans) + 64
    nq = 140000
    assert cap < 131072 < nq

    def search(tree, rng):
        mp = scans[0]["map"]
        q = (mp[rng.integers(0, len(mp), nq)] + rng.normal(0, 0.05, (nq, 3))).astype(np.float32)
        before = tree.validnum()
        _, _, cnt = tree.Nearest_Search(q, 5)
        assert len(cnt) == nq and tree.validnum() == before
    _regrown_step_equals_fresh_session(scans, search)


def test_scratch_hash_regrown_after_capture(scans):
    """A downsampled insert of four times the session's capacity needs a larger scratch hash than the capture ensured."""
    cap = max(len(sc["body"]) for sc in scans) + 64

    def add(tree, rng):
        mp = scans[0]["map"]
        pts = (mp[rng.integers(0, len(mp), 4 * cap)] + rng.normal(0, 0.05, (4 * cap, 3))).astype(np.float32)
        assert tree.Add_Points(pts, True) > 0
    _regrown_step_equals_fresh_session(scans, add)


# ------------------------------------------------------------------------------------------------ host records
def _grid4(n=2000, seed=0):
    """n points on distinct 0.2 m voxels, 4th float a non-zero intensity."""
    rng = np.random.default_rng(seed)
    idx = rng.choice(40 * 40 * 40, n, replace=False)
    xyz = np.stack([idx % 40, (idx // 40) % 40, idx // 1600], axis=1).astype(np.float32) * 0.6 + 0.1
    return np.column_stack([xyz, rng.uniform(1, 255, n)]).astype(np.float32)


def test_build_of_xyzi_rows_carries_the_fourth_float():
    a4 = _grid4()
    t = capi.KDTree(voxel_size=0.2, max_points=1 << 16, max_blocks=1 << 12)
    t.Build(a4)                                       # flb_map_build, stride 16, no intensity offset
    assert np.array_equal(sort_rows(t.flatten_xyzi()), sort_rows(a4))
    t.close()


def test_scan_upload_of_xyzi_rows_carries_the_fourth_float(scans):
    """flb_scan_upload of (n, 4) rows == flb_scan_upload_pt with the intensity at byte 12: the same map, intensities
    included."""
    sc = scans[0]
    b4 = np.column_stack([sc["body"], 1.0 + np.arange(len(sc["body"])) % 199]).astype(np.float32)
    maps = []
    for xyzi in (False, True):
        t = _tree(sc["map"])
        ses = _session(t, scans)
        if xyzi:
            ses.scan_upload_xyzi(b4)
        else:
            ses.scan_upload(b4)
        s, P, _ = ses.update_iterated_dyn_share_modified(sc["prior"], sc["P"])
        ses.map_incremental(s)
        maps.append(sort_rows(t.flatten_xyzi()))
        ses.close()
        t.close()
    assert np.array_equal(maps[0], maps[1])
    added = maps[0][maps[0][:, 3] != 0]                 # (the map was built without intensities)
    assert len(added) > 0 and np.isin(added[:, 3], b4[:, 3]).all()


def test_frontend_upload_of_16_byte_records_without_offsets_gives_zero_intensity_and_curvature(scans):
    sc = scans[0]
    t = _tree(sc["map"])
    ses = _session(t, scans)
    fe = capi.FrontEnd(ses, max_raw_points=8192)
    a4 = _grid4(3000, seed=1)
    fe.upload_ptr(a4.ctypes.data, len(a4), stride=16, off_i=-1, off_c=-1)
    xyzi, cur, perm = fe.download_undistorted()
    assert np.array_equal(xyzi[:, :3], a4[:, :3]) and np.array_equal(perm, np.arange(len(a4)))
    assert not xyzi[:, 3].any() and not cur.any()
    fe.close()
    ses.close()
    t.close()


def test_every_scan_upload_path_gives_the_same_step(scans):
    """flb_scan_upload_pt with strides 12, 16 and 32 (intensity at byte 20), flb_scan_prefetch with strides 12 and 16
    and flb_scan_set_device: the same step, bit for bit; the map carries the intensity wherever the records do."""
    import torch
    sc = scans[0]
    body = sc["body"]
    n = len(body)
    inten = (1.0 + np.arange(n) % 199).astype(np.float32)
    r12 = np.ascontiguousarray(body, np.float32)
    r16 = np.column_stack([body, inten]).astype(np.float32)
    r32 = np.zeros((n, 8), np.float32)
    r32[:, :3] = body
    r32[:, 5] = inten
    r32[:, 3] = -7.0                                  # a field the upload must not read as the intensity
    dev = torch.from_numpy(r16).cuda()
    torch.cuda.synchronize()
    paths = {"pt12": ("pt", r12, 12, -1), "pt16": ("pt", r16, 16, -1), "pt32": ("pt", r32, 32, 20),
             "prefetch12": ("prefetch", r12, 12, None), "prefetch16": ("prefetch", r16, 16, None), "device": ("device", None, 0, None)}
    out = {}
    for name, (kind, rec, stride, off) in paths.items():
        t = _tree(sc["map"])
        ses = _session(t, scans)
        if kind == "pt":
            capi._chk(capi.lib().flb_scan_upload_pt(ses.h, C.c_void_p(rec.ctypes.data), n, stride, off))
            ses.n = n
        elif kind == "prefetch":
            ses.scan_prefetch_ptr(rec.ctypes.data, n, stride)
        else:
            ses.scan_set_device(dev.data_ptr(), n)
        st, P = sc["prior"].copy(), np.ascontiguousarray(sc["P"], np.float64).copy()
        r = ses.scan_step_ptr(None, None, 0, 0, st, P)
        out[name] = (st, P, r, sort_rows(t.flatten_xyzi()))
        ses.close()
        t.close()
    ref = out["pt16"]
    for name, (st, P, r, mp) in out.items():
        _same_step((st, P, r), ref[:3])
        assert np.array_equal(sort_rows(mp[:, :3]), sort_rows(ref[3][:, :3])), name
    for name in ("pt32", "prefetch16", "device"):          # the scan's intensities travelled into the map
        assert np.array_equal(out[name][3], ref[3]), name
    added = ref[3][ref[3][:, 3] != 0]
    assert len(added) > 0 and np.isin(added[:, 3], inten).all()
    for name in ("pt12", "prefetch12"):                   # no intensity in 12-byte records (the map was built without)
        assert not out[name][3][:, 3].any(), name


# ------------------------------------------------------------------------------------------------ step slots
def test_underdetermined_scan_in_slot_1_hands_over_to_the_host_engine():
    """Scan 1 runs in slot 0 (begin / finish), scan 2 — 14 points, fewer than 23 rows — in slot 1: the device engine
    stops and the host's explicit-row branch finishes it, with the host engine's result on the same map."""
    sc = dc.scene(seed=5)
    rng = np.random.default_rng(3)
    prior = dc.prior_from(sc["st_true"], rng, 0.1, 0.5)
    P = dc.propagate_cov(prior, synth.default_cov())
    probe = _tree(sc["map"])
    _, d2, cnt = probe.Nearest_Search(synth.body_to_world_np(prior, sc["body"]), 5)
    probe.close()
    few = np.ascontiguousarray(sc["body"][np.where((cnt == 5) & (d2[:, 4] < 0.2))[0][:14]])
    assert len(few) == 14
    results = []
    for device_second in (True, False):
        t = _tree(sc["map"])
        ses = capi.Session(t, max_scan_points=len(sc["body"]) + 64, max_iterations=3)
        st, Pm = prior.copy(), P.copy()
        ses.scan_upload(sc["body"])
        ses.scan_step_begin(None, st, Pm)
        ses.scan_step_finish(None, st, Pm)                # slot 0
        ses.set_update_engine(device_second)
        st2, P2 = prior.copy(), P.copy()
        ses.scan_upload(few)
        ses.scan_step_begin(None, st2, P2)                # slot 1
        r = ses.scan_step_finish(None, st2, P2)
        assert 0 < r.update.effct_feat_num < 23
        results.append((st2, P2, r, sort_rows(t.flatten())))
        ses.close()
        t.close()
    (s_d, P_d, r_d, m_d), (s_h, P_h, r_h, m_h) = results
    assert np.array_equal(s_d, s_h) and np.array_equal(P_d, P_h)
    assert (r_d.update.passes, r_d.update.effct_feat_num, r_d.map_valid, r_d.n_to_add) == \
        (r_h.update.passes, r_h.update.effct_feat_num, r_h.map_valid, r_h.n_to_add)
    assert np.array_equal(m_d, m_h)
