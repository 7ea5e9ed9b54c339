"""GPU: both update engines under dense prior covariances and every max_iterations setting, against the oracle with
bounds predicted on the CPU by the numpy model of the device's gain form (tests/esikf_ref.py); the measurement and
map_incremental kernels at their round boundaries; per-point state carried from one scan to the next; a closed loop
carrying a dense propagated covariance; the range check of max_iterations."""
import numpy as np
import pytest

from better_fastlio2_b200 import capi, synth
from tests import dense_cases as dc
from tests import esikf_ref as ref
from tests.helpers import small_scene, sort_rows

pytestmark = pytest.mark.gpu


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ dense update, both engines
@pytest.fixture(scope="module")
def dense_scenes(oracle):
    out = {}
    for key, offR in (("plain", (0, 0, 0)), ("offR", (1.5, -2.0, 3.0))):
        sc = dc.scene(seed=5, offR_deg=offR)
        mp = oracle.make_map(ds=0.2)
        mp.Build(sc["map"])
        sc["mp"] = mp
        out[key] = sc
    return out


def _tree(points):
    t = capi.KDTree(voxel_size=0.2, max_points=1 << 21, max_blocks=1 << 18)
    t.Build(points)
    return t


@pytest.mark.parametrize("case", dc.ENGINE_CASES, ids=dc.ENGINE_CASE_IDS)
def test_dense_update_both_engines_match_oracle(oracle, dense_scenes, case):
    prior, P, R, max_iter, lim, ext, sc = dc.engine_case(case, dense_scenes, oracle)
    md = 12 if ext else 6
    s_o, P_o, _, st_o, _ = oracle.esikf_update(prior, P, sc["body"], sc["mp"], max_iter=max_iter, R=R, extrinsic_est_en=ext,
                                                 limit=lim)
    bounds = dc.engine_bounds(prior, P, R, max_iter, lim, md, lambda: ref.OracleMeasurement(oracle, sc["body"], sc["mp"], ext))
    assert np.abs(ref.boxminus(s_o, prior)[12:23]).max() > 1e-7         # velocity / biases / gravity moved
    t = _tree(sc["map"])
    for device in (True, False):
        engine = "device" if device else "host"
        bx, bP = bounds[engine]
        ses = capi.Session(t, max_scan_points=len(sc["body"]) + 64, extrinsic_est_en=ext, max_iterations=max_iter,
                           laser_point_cov=R, limit=lim)
        ses.set_update_engine(device)
        ses.scan_upload(sc["body"])
        runs = [ses.update_iterated_dyn_share_modified(prior, P) for _ in range(2)]   # graph capture, then replay
        (s1, P1, st1), (s2, P2, _) = runs
        assert np.array_equal(s1, s2) and np.array_equal(P1, P2)
        got = [st1["passes"], st1["search_passes"], st1["effct_feat_num"], st1["converged_count"]]
        assert got == list(st_o), (engine, got, st_o)
        dx, dP = np.abs(s1 - s_o).max(), np.abs(P1 - P_o).max()
        print(f"DENSE case={case[0]}-it{max_iter}-md{md} engine={engine} dx={dx:.2e} bound_x={bx:.2e} dP={dP:.2e} bound_P={bP:.2e}")
        assert dx <= bx and dP <= bP, (engine, dx, bx, dP, bP)
        ses.close()
    t.close()
    # the whole step (update + map_incremental) through the scan graph twice in a row on one session: the first call
    # captures the graph, the second replays it on the map the first one grew.  The first is checked against the
    # oracle; the replay against a fresh session's captured step on a map grown by the same first step, bit for bit.
    bx, bP = bounds["device"]
    trees = [_tree(sc["map"]) for _ in range(2)]
    kw = dict(max_scan_points=len(sc["body"]) + 64, extrinsic_est_en=ext, max_iterations=max_iter, laser_point_cov=R, limit=lim)
    ses = capi.Session(trees[0], **kw)
    s3, P3, r = ses.scan_step(None, sc["body"], prior, P)
    assert r.update.passes == st_o[0] and r.update.effct_feat_num == st_o[2]
    assert np.abs(s3 - s_o).max() <= bx and np.abs(P3 - P_o).max() <= bP
    replay = ses.scan_step(None, sc["body"], prior, P)
    ses.close()
    first = capi.Session(trees[1], **kw)
    assert np.array_equal(first.scan_step(None, sc["body"], prior, P)[0], s3)
    first.close()
    fresh = capi.Session(trees[1], **kw)
    captured = fresh.scan_step(None, sc["body"], prior, P)
    fresh.close()
    assert np.array_equal(replay[0], captured[0]) and np.array_equal(replay[1], captured[1])
    assert replay[2].map_valid == captured[2].map_valid
    assert np.array_equal(sort_rows(trees[0].flatten()), sort_rows(trees[1].flatten()))
    for tr in trees:
        tr.close()


@pytest.mark.parametrize("family", ["propagated", "correlated_6", "posterior"])
def test_dense_underdetermined_device_hands_over_to_host(oracle, dense_scenes, family):
    """M < 23 under a dense prior: the device engine stops and the host's explicit-row branch finishes the scan."""
    sc = dense_scenes["plain"]
    rng = np.random.default_rng(3)
    prior = dc.prior_from(sc["st_true"], rng, 0.1, 0.5)
    P = dc.family_cov(family, prior, rng, oracle, sc["body"], sc["mp"])
    world = oracle.transform(prior, sc["body"])
    _, d2, cnt = sc["mp"].Nearest_Search(world, 5)
    few = np.ascontiguousarray(sc["body"][np.where((cnt == 5) & (d2[:, 4] < 0.2))[0][:14]])
    s_o, P_o, _, st_o, _ = oracle.esikf_update(prior, P, few, sc["mp"], max_iter=3)
    assert 0 < st_o[2] < 23
    t = _tree(sc["map"])
    for device in (True, False):
        ses = capi.Session(t, max_scan_points=64, max_iterations=3)
        ses.set_update_engine(device)
        ses.scan_upload(few)
        s, Pg, st = ses.update_iterated_dyn_share_modified(prior, P)
        assert st["effct_feat_num"] == st_o[2] and st["passes"] == st_o[0]
        assert np.abs(s - s_o).max() <= 1e-10 and np.abs(Pg - P_o).max() <= 1e-9 * np.abs(P).max()
        ses.close()
    t.close()


def test_max_iterations_range_is_checked():
    t = _tree(small_scene(seed=1, map_half=10.0, half_extent=40.0)["map"])
    for bad in (-1, -5, 8):
        with pytest.raises(capi.FlbError, match="max_iterations"):
            capi.Session(t, max_scan_points=1000, max_iterations=bad)
    for ok in (0, 7):
        capi.Session(t, max_scan_points=1000, max_iterations=ok).close()
    t.close()


# ------------------------------------------------------------------------------------------------ round boundaries
@pytest.fixture(scope="module")
def big():
    """A map and a scan of up to `cap` points (jittered copies of one VLP-16 scan), with S = SMs x threads of
    k_residual for both variants and the stride of k_classify."""
    sm = _sm_count()
    S1024, S896, classify = sm * 1024, sm * 896, sm * 8 * 256
    cap = max(2 * S1024 + 1, classify + 1) + 4096
    sc = small_scene(seed=1)
    rng = np.random.default_rng(8)
    reps = -(-cap // len(sc["body"]))
    body = np.concatenate([sc["body"] + rng.normal(0, 0.01, sc["body"].shape) for _ in range(reps)])[:cap]
    return dict(S1024=S1024, S896=S896, classify=classify, cap=cap, body=np.ascontiguousarray(body, np.float32),
                map=sc["map"], prior=sc["prior"], st_true=sc["st_true"])


def _sizes(big, S):
    return sorted({1, 22, 23, 24, 31, 32, 33, 127, 128, 129, S - 1, S, S + 1, 2 * S + 1, big["cap"]})


@pytest.mark.parametrize("ext", [False, True])
def test_pass_and_classify_at_round_boundaries(oracle, big, ext):
    S = big["S896"] if ext else big["S1024"]
    t = _tree(big["map"])
    ses = capi.Session(t, max_scan_points=big["cap"], extrinsic_est_en=ext, max_iterations=3)
    prior = big["prior"]
    sizes = _sizes(big, S)
    assert max(sizes) > big["classify"] and 2 * S + 1 in sizes
    for n in sizes:
        body = big["body"][:n]
        ses.scan_upload(body)
        r = ses.h_share_model(prior, converge=True)
        nb = ses.neighbors()
        world = oracle.transform(prior, body)
        assert np.array_equal(nb["world"], world), n
        sel = np.ones(n, np.uint8)
        M, hx, h, nv, tot = oracle.residual_pass(prior, body, world, nb["nbr"], nb["d2"], nb["cnt"], True, sel, ext)
        assert r["effct_feat_num"] == M, (n, r["effct_feat_num"], M)
        assert np.array_equal(nb["sel"], sel), n
        s = sel.astype(bool)
        assert np.array_equal(nb["normvec"][s], nv[s]), n
        if M:
            HTH, HTh = hx.T @ hx, hx.T @ h
            assert np.abs(r["HTH"] - HTH).max() <= 1e-9 * np.abs(HTH).max(), n
            assert np.abs(r["HTh"] - HTh).max() <= 1e-9 * max(np.abs(HTh).max(), 1e-300), n
        assert abs(r["total_residual"] - tot) <= 1e-9 * max(tot, 1e-300), n
        if n >= S - 1 or n == 129:
            _, cls = oracle.map_incremental_classify(prior, body, nb["nbr"], nb["cnt"], True, 0.2)
            a, b = ses.map_incremental(prior, True)
            assert (a, b) == (int((cls == 1).sum()), int((cls == 2).sum())), n
    # before the filter is initialised every point is a downsampled insert (class 1): the count is exactly n, so a point
    # classified twice or never shows, whatever class the map would give it.  Over k_classify's stride, last (it grows
    # the map by the whole scan).
    n = max(sizes)
    _, cls = oracle.map_incremental_classify(prior, big["body"][:n], nb["nbr"], nb["cnt"], False, 0.2)
    assert int((cls == 1).sum()) == n
    assert ses.map_incremental(prior, False) == (n, 0)
    ses.close()
    t.close()


@pytest.mark.parametrize("ext", [False, True])
def test_no_state_carries_over_between_scans(oracle, big, ext):
    """One session through large -> small -> just under a boundary -> tiny -> over two rounds: every update equals a fresh
    session's bit for bit (the scan graph is captured at capacity and replayed with each scan's n)."""
    S = big["S896"] if ext else big["S1024"]
    t = _tree(big["map"])
    rng = np.random.default_rng(4)
    P = dc.propagate_cov(big["prior"], synth.default_cov())
    ses = capi.Session(t, max_scan_points=big["cap"], extrinsic_est_en=ext, max_iterations=4)
    for n in (big["cap"], 5000, S - 1, 40, 2 * S + 1):
        body = big["body"][rng.permutation(big["cap"])[:n]] if n < big["cap"] else big["body"]
        ses.scan_upload(body)
        got = ses.update_iterated_dyn_share_modified(big["prior"], P)
        fresh = capi.Session(t, max_scan_points=big["cap"], extrinsic_est_en=ext, max_iterations=4)
        fresh.scan_upload(body)
        want = fresh.update_iterated_dyn_share_modified(big["prior"], P)
        fresh.close()
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), n
        for k in ("passes", "search_passes", "effct_feat_num", "converged_count"):
            assert got[2][k] == want[2][k], (n, k)
    ses.close()
    t.close()


# ------------------------------------------------------------------------------------------------ closed loop
def test_closed_loop_dense_covariance(oracle):
    """8 scans of test_closed_loop_sequence's scene, each prior carrying the previous posterior's covariance through
    one propagation interval (dense), on both sides: per-frame posterior within 1e-4 m / 1e-4 rad of the oracle's, and
    velocity, biases and gravity following it."""
    seed = 3
    rng = np.random.default_rng(seed)
    world = synth.city_world(half_extent=150, seed=seed)
    dirs = synth.lidar_dirs("vlp16")
    ds = 0.2
    t = capi.KDTree(voxel_size=ds, max_points=1 << 21, max_blocks=1 << 18)
    mp = oracle.make_map(ds=ds)
    fov_g = capi.make_fov(cube_len=120.0, det_range=30.0)
    fov_c = oracle.FovSegment(cube_len=120.0, det_range=30.0)
    pos_lid_c = np.zeros(3)
    ses = None
    moved = 0.0
    for k in range(9):
        st_true = synth.trajectory_state(k, speed=20.0)
        body = synth.voxel_downsample(synth.scan_from_pose(world, st_true, dirs, rng, max_range=60.0), ds)
        if k == 0:
            w0 = synth.body_to_world_np(st_true, body)
            t.Build(w0)
            mp.Build(w0)
            s_g, s_c = st_true.copy(), st_true.copy()
            P_g = P_c = synth.default_cov()
            ses = capi.Session(t, max_scan_points=60000, max_iterations=4)
            continue

        def propagate(s_prev, P_prev):
            noise = np.random.default_rng(100 + k)
            s = s_prev.copy()
            s[0:3] += synth.trajectory_state(k, speed=20.0)[0:3] - synth.trajectory_state(k - 1, speed=20.0)[0:3]
            s[3:7] = synth.trajectory_state(k, speed=20.0)[3:7]
            return synth.perturb_state(s, noise, 0.03, 0.3), dc.propagate_cov(s, P_prev)

        pri_g, Pp_g = propagate(s_g, P_g)
        pri_c, Pp_c = propagate(s_c, P_c)
        s_g, P_g, r = ses.scan_step(fov_g, body, pri_g, Pp_g, True)
        boxes = fov_c.step(pos_lid_c)
        if len(boxes):
            mp.Delete_Point_Boxes(boxes)
        s_c, P_c, sc, _, _ = oracle.esikf_update(pri_c, Pp_c, body, mp, max_iter=4)
        pos_lid_c = s_c[0:3] + synth.quat_to_mat(s_c[3:7]) @ s_c[11:14]
        oracle.map_incremental(s_c, body, sc, mp, True, ds)
        d = np.abs(ref.boxminus(s_g, s_c))
        assert d[0:3].max() <= 1e-4 and d[3:6].max() <= 1e-4, (k, d[0:6])
        assert d[12:23].max() <= 1e-4, (k, d[12:23])
        moved = max(moved, np.abs(ref.boxminus(s_c, pri_c)[12:23]).max())
    assert moved > 1e-4
    ses.close()
    t.close()
