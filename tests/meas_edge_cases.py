"""Constructed neighbourhoods for the point-to-plane measurement (esti_plane, the three gates of h_share_model) and the
map_incremental classifier, at the branches and boundaries natural scenes never reach.

Plain numpy. A case is one map cluster plus one query point. The builders that have to land on a float boundary take
the CPU oracle's functions as arguments and bisect on them, so every literal below is regenerated deterministically.

QR branches named below are those of esti_plane (column-pivoted Householder QR, include/common_lib.h:506-536 of the
reference, Eigen 3.3 ColPivHouseholderQR):
  skip       - the Householder tail is <= FLT_MIN: tau = 0 (hCoeffs[k] == 0), beta = c0, the tail zeroed
  rankdef    - the biggest remaining column norm falls under the threshold: nonzero_pivots < 3
  pivot_tie  - two columns with bit-equal norms: the first maximum wins
  downdate   - a column loses nearly all its norm in one reflection: its norm is recomputed, not downdated
  thr_in / thr_out - the largest residual |n.p + d| a few float steps below / above 0.1f
"""
import numpy as np

from better_fastlio2_b200 import synth

F32 = np.float32
THR = F32(0.1)
SEPARATION = 20.0  # metres between clusters of one map: the 5-NN of a query are exactly its own cluster

# poses: A is the identity (body == world bit for bit), B is rotated and translated so body-to-world rounding feeds the gates
POSE_A = synth.make_state(offT=(0.0, 0.0, 0.0))
POSE_B = synth.make_state(pos=(3.25, -2.5, 0.5), rot=synth.quat_from_rotvec([0.1, -0.2, 0.7]),
                          offR=synth.quat_from_rotvec([0.01, 0.02, -0.03]))


def by_distance(pts, q):
    """The cluster in the k-NN's order: ascending float32 squared distance from q (the fit's rounding depends on it)."""
    pts = np.asarray(pts, F32)
    d = pts - np.asarray(q, F32)
    return pts[np.argsort((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2], kind="stable")]


def case(name, family, pts, query=None, expect=None, branches=(), far=False, **kw):
    pts = np.asarray(pts, np.float64).astype(F32)
    q = pts.mean(0).astype(F32) if query is None else np.asarray(query, F32)
    return dict(name=name, family=family, pts=by_distance(pts, q), query=q, expect=expect, branches=tuple(branches),
                far=far, **kw)


SQUARE = np.array([[-1, -1], [1, -1], [-1, 1], [1, 1], [0.25, 0.125]])  # four corners and an inner point


def plane_points(centre, normal, rng, spread=0.3, noise=0.0, layout=None):
    """Five points of a plane through `centre`, in float64 (the caller rounds): random in a square of half-side
    `spread`, or `layout` (5 x 2, in units of `spread`)."""
    n = np.asarray(normal, np.float64)
    n = n / np.linalg.norm(n)
    u = np.cross(n, [0.3, 1.0, 0.2])
    u /= np.linalg.norm(u)
    v = np.cross(n, u)
    a = rng.uniform(-spread, spread, (5, 2)) if layout is None else np.asarray(layout, np.float64) * spread
    return np.asarray(centre, np.float64) + a[:, :1] * u + a[:, 1:] * v + rng.normal(0, noise, (5, 1)) * n


def on_plane(c, pabcd):
    """float32 residuals |a x + b y + c z + d| evaluated left to right, as common_lib.h:530 does."""
    p = np.asarray(c, F32)
    a, b, cc, d = (F32(v) for v in pabcd)
    return np.abs(((a * p[:, 0] + b * p[:, 1]) + cc * p[:, 2]) + d)


# ------------------------------------------------------------------------------------------------ neighbourhood families
def control(rng):
    """1. Well-conditioned planes in random orientations within 60 m of the origin."""
    out = []
    for k in range(6):
        n = rng.normal(0, 1, 3)
        c = np.array([-60.0 + 24 * k, 40.0 * (-1) ** k, 3.0])
        out.append(case(f"control{k}", "control", plane_points(c, n, rng, 0.4, 0.003), expect="accept"))
    return out


def exact_zeros():
    """2. Binary-fraction planes with exact zero components. The biggest column has one nonzero entry, so its tail is 0
    and the first Householder step is skipped (hCoeffs[0] == 0); the same with a tail of subnormal squares."""
    out = []
    # x column (16, 0, 0, 0, 0) dominates; the rest of the plane is x/8 + z = 3 in binary fractions
    # (the query sits next to the first point, so the k-NN puts that point first)
    p = np.array([[16, 1, 1], [0, 1.5, 3], [0, -1, 3], [0, 2, 3], [0, -0.5, 3]], np.float64)
    out.append(case("skip_k0_plane", "exact_zeros", p, query=[14, 1, 1.25], branches=("skip",)))
    # the wall y = 40 (exact zero normal components) through binary-fraction points
    p = np.array([[0.5, 40, 0.25], [0.25, 40, 0.75], [0.75, 40, 0.5], [0.5, 40, 1.0], [0.0, 40, 0.5]]) + [-90, 0, 0]
    out.append(case("wall_y40_binary", "exact_zeros", p, expect="accept"))
    # a plane 1e-19 from the origin: every column's tail is of the order of FLT_MIN, so which branch each step takes
    # decides the plane's last bits (the tail entries are the whole information, not rounding noise)
    g = np.array([[0, 0], [0.4, 0], [0, 0.4], [0.4, 0.4], [0.2, 0.1]])
    for s in (2.5e-20, 6e-20, 1.5e-19):
        out.append(case(f"subnormal_tail_{s:.0e}", "exact_zeros", np.c_[g * s * 2.5, np.full(5, 1e-19)],
                        query=[0, 0, 1e-19], expect="accept", branches=("skip",)))
    return out


def rank_deficient():
    """3. Rank deficiency: zero column, collinear points, duplicates, five points at the origin."""
    out = []
    wall = np.array([[0, 30, 1], [0, 30.5, 1.25], [0, 31, 1.5], [0, 30.25, 2], [0, 30.75, 1.75]], np.float64)
    out.append(case("wall_x0", "rank_deficient", wall, expect="reject", branches=("rankdef", "skip")))
    ground = np.array([[-30, 30, 0], [-30.5, 30.25, 0], [-29.5, 30.5, 0], [-30.25, 29.5, 0], [-29.75, 29.75, 0]])
    out.append(case("ground_z0", "rank_deficient", ground, expect="reject", branches=("rankdef", "skip")))
    # a line through the origin: the y and z columns are exact multiples of x, so after one reflection both are 0
    t = np.array([0.0, 0.25, 0.5, 0.75, 1.0])
    out.append(case("collinear_origin_line", "rank_deficient", np.c_[32 + t, 16 + t / 2, 8 + t / 4], expect=None,
                    branches=("rankdef", "skip")))
    # a line off the origin (rank 2 in exact arithmetic)
    out.append(case("collinear_offset_line", "rank_deficient", np.c_[60 + t, np.full(5, -60.0), 4 + t], expect=None,
                    branches=("rankdef",)))
    out.append(case("duplicates_345", "rank_deficient", np.tile([3.0, 4.0, 5.0], (5, 1)), query=[3, 4, 5.0625],
                    expect="accept", branches=("rankdef", "skip")))
    out.append(case("origin_x5", "rank_deficient", np.zeros((5, 3)), query=[0.125, 0, 0], expect="nan",
                    branches=("skip",)))
    return out


def pivot_ties():
    """4. x and y columns are permutations of each other with exactly representable squares: bit-equal norms at the
    first pivot, so the first maximum (x) must win."""
    base = np.array([[10, 11, 2.5], [11, 10, 2.5], [10.5, 10.5, 2.5], [10, 10, 3], [11, 11, 2]], np.float64)  # x+y+2z=26
    out = []
    for k, sh in enumerate(([0, 0, 0], [40, 40, 0], [-64, -64, 1], [24, 24, -3])):
        out.append(case(f"pivot_tie{k}", "pivot_tie", base + sh, expect="accept", branches=("pivot_tie",)))
    # a tilted tie: x + y + z/4 = const, the x/y columns tie and dominate
    b2 = np.array([[6, 7, 4], [7, 6, 4], [6.5, 6.5, 4], [6, 6, 8], [7, 7, 0]], np.float64)
    out.append(case("pivot_tie_tilted", "pivot_tie", b2 + [-40, -40, 0], expect="accept", branches=("pivot_tie",)))
    return out


def norm_downdate(rng):
    """5. Nearly parallel x and y columns (x ~ y on every point): after the first reflection the other column keeps
    well under 2 % of its norm, so temp2 <= sqrt(eps) and the norm is recomputed."""
    out = []
    for k in range(4):
        u = rng.uniform(0.0, 0.5, 5)
        c = 30.0 + 25 * k
        x = c + u
        y = c + u + rng.normal(0, 2e-3, 5)
        z = 2.0 + 0.2 * u + rng.normal(0, 2e-3, 5)
        out.append(case(f"downdate{k}", "downdate", np.c_[x, -y, z] if k % 2 else np.c_[x, y, z],
                        branches=("downdate",)))
    return out


def threshold_pairs(esti_plane, rng):
    """6. One point pushed along the normal so that the largest residual lands just below (accepted) and just above
    (rejected) 0.1f: the two pushes are adjacent float32 values, bisected with the oracle's esti_plane. Next to the
    origin the coordinates resolve the residual to a few ulps of 0.1f; 90 m out, to the coordinates' own float step."""
    out = []
    for k, (c, n, spread) in enumerate((([0.25, -0.125, 0.375], [0.1, 0.2, 1.0], 0.125),
                                        ([50.0, -70.0, 6.0], [1.0, 0.3, 0.2], 0.4))):
        p0 = plane_points(c, n, rng, spread, layout=SQUARE)
        nn = np.asarray(n) / np.linalg.norm(n)
        q = p0.mean(0).astype(F32)
        for sign in (1.0, -1.0):
            def pts_for(off):
                p = p0.copy()
                p[3] += sign * float(off) * nn
                return by_distance(p.astype(F32), q)

            lo, hi = _bisect_f32(lambda off: esti_plane(pts_for(off))[0], 0.0, 1.0)  # accepted at 0, rejected at 1 m
            s = "pos" if sign > 0 else "neg"
            for tag, off, exp in (("in", lo, "accept"), ("out", hi, "reject")):
                out.append(case(f"thr{k}_{s}_{tag}", "threshold", pts_for(off), query=q, expect=exp,
                                branches=(f"thr_{tag}",), offset=float(off)))
    return out


def far_from_origin(rng):
    """7. Control planes and the exact ground z = 1.8 at 1, 5 and 20 km along x and along the diagonal."""
    out = []
    g = np.array([[0, 0], [0.4, 0], [0, 0.4], [0.4, 0.4], [0.2, 0.1]])
    for dist in (1000.0, 5000.0, 20000.0):
        for axis, d in (("x", np.array([1.0, 0, 0])), ("diag", np.array([1.0, 1.0, 0]) / np.sqrt(2))):
            c = dist * d
            out.append(case(f"ground_{axis}{int(dist)}", "far", np.c_[c[0] + g[:, 0], c[1] + g[:, 1], np.full(5, 1.8)],
                            far=True))
            n = rng.normal(0, 1, 3)
            out.append(case(f"plane_{axis}{int(dist)}", "far", plane_points(c + [0, 0, 4], n, rng, 0.5, 0.003),
                            far=True))
    return out


def neighbourhood_cases(esti_plane, seed=7):
    rng = np.random.default_rng(seed)
    return (control(rng) + exact_zeros() + rank_deficient() + pivot_ties() + norm_downdate(rng)
            + threshold_pairs(esti_plane, rng) + far_from_origin(rng))


def batches(cases, sep=SEPARATION):
    """Group cases into maps whose clusters (and queries) are at least `sep` apart."""
    out = []
    for c in cases:
        pc = np.vstack([c["pts"], c["query"][None]]).astype(np.float64)
        for b in out:
            other = np.vstack([np.vstack([o["pts"], o["query"][None]]) for o in b]).astype(np.float64)
            if np.sqrt(((pc[:, None, :] - other[None]) ** 2).sum(-1)).min() >= sep:
                b.append(c)
                break
        else:
            out.append([c])
    return out


# ------------------------------------------------------------------------------------------------ body <-> world
def world_to_body(state, w):
    """float64 inverse of the body-to-world transform (laserMapping.cpp:1894-1898), rounded to float32."""
    R = synth.quat_to_mat(state[3:7])
    Rl = synth.quat_to_mat(state[7:11])
    w = np.atleast_2d(np.asarray(w, np.float64))
    a = (w - state[0:3]) @ R                 # R^T (w - pos)
    return ((a - state[11:14]) @ Rl).astype(F32)


def sorted_d2(pts, q):
    """Ascending float32 squared distances (dx*dx + dy*dy) + dz*dz of the 5 cluster points from q."""
    d = pts.astype(F32) - np.asarray(q, F32)
    return np.sort(((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32))


# ------------------------------------------------------------------------------------------------ gate cases
def _bisect_f32(pred, lo, hi):
    """Adjacent float32 values (a, b) between lo and hi with pred(a) true and pred(b) false (pred(lo) and not pred(hi)),
    by bisection on the ordering of float32 bit patterns (lo and hi of the same sign)."""
    lo, hi = F32(lo), F32(hi)
    assert pred(lo) and not pred(hi)
    li, hu = int(lo.view(np.int32)), int(hi.view(np.int32))
    while abs(hu - li) > 1:
        mid = np.int32((li + hu) // 2)
        if pred(mid.view(F32)):
            li = int(mid)
        else:
            hu = int(mid)
    return np.int32(li).view(F32), np.int32(hu).view(F32)


def d2_gate_cases(state, transform):
    """d2[4] at exactly 5.0f (kept: the test is > 5) and one float step beyond (dropped). The 5th neighbour sits at
    (2, 1, 0) from the query's float world point; the other four are 0.5-0.875 m away on the same horizontal plane."""
    out = []
    for k, b in enumerate(([16.0, -24.0, 1.5], [-40.0, 40.0, 2.25])):
        # the first body point (stepping x by 1/8 m) whose world point w has w.x + 2 and w.y + 1 exact in float32
        for step in range(256):
            body = np.asarray(b, F32) + np.array([step / 8.0, 0, 0], F32)
            w = transform(state, body[None])[0]
            if F32(w[0] + F32(2)) - w[0] == 2 and F32(w[1] + F32(1)) - w[1] == 1:
                break
        for beyond in (False, True):
            x5 = F32(w[0] + F32(2))
            if beyond:
                x5 = np.nextafter(x5, F32(np.inf))
            ring = w + np.array([[0.5, 0, 0], [0, 0.625, 0], [-0.75, 0, 0], [0, -0.875, 0]], F32)
            pts = np.vstack([ring, np.array([[x5, F32(w[1] + F32(1)), w[2]]], F32)])
            c = case(f"d2_{'beyond' if beyond else 'eq5'}{k}", "gate_d2", pts, query=w, body=body,
                     branches=("d2_beyond" if beyond else "d2_eq5",))
            c["d2"] = sorted_d2(pts, w)
            out.append(c)
    return out


RING = np.array([[0.5, 0, 0], [0, 0.55, 0], [-0.6, 0, 0], [0, -0.65, 0], [0.3, 0.35, 0]], F32)  # distinct distances


def s_gate_cases(state, transform, esti_plane, residual_pass):
    """The s > 0.9 gate: a body point at the sensor origin (bn = 0) with pd2 == 0 and pd2 != 0, tiny body norms, and
    body points a float step either side of 0.9|pd2|/sqrt(bn) = 0.1 (bisected with the oracle's residual pass)."""
    out = []
    # bn == 0: the world point is the pose's translation, rounded. Away from the origin a horizontal plane through it,
    # nudged by float steps, puts pd2 at exactly 0 (at the origin no plane through the point is accepted)
    w0 = transform(state, np.zeros((1, 3), F32))[0]
    if np.any(w0 != 0):
        zero = None
        for scale in (1, 2, 3, 4):
            for k in range(200):
                z = F32(w0[2] + F32((k + 1) // 2 * (1 if k % 2 else -1)) * np.spacing(w0[2]))
                pts = (RING * F32(scale) + np.array([w0[0], w0[1], z], F32)).astype(F32)
                pts[:, 2] = z
                ok, pabcd = esti_plane(by_distance(pts, w0))
                if ok and on_plane(w0[None], pabcd)[0] == 0:
                    zero = pts
                    break
            if zero is not None:
                break
        assert zero is not None, "no horizontal plane with pd2 == 0 at the pose's translation"
        out.append(case("bn0_pd2_zero", "gate_s", zero, query=w0, body=np.zeros(3, F32), branches=("bn0",)))
    out.append(case("bn0_pd2_nonzero", "gate_s", RING + w0 + np.array([0, 0, -0.05], F32), query=w0,
                    body=np.zeros(3, F32), branches=("bn0",)))
    # tiny body norms: the world point is next to the translation, 0.05 sqrt(bn) above a plane (half the gate's margin)
    # or 0.01 m above it
    for k, (s, up) in enumerate(((1e-3, None), (1e-3, 0.01), (1e-6, None), (1e-12, None), (1e-40, None))):
        body = np.array([s, -s, s], F32)
        w = transform(state, body[None])[0]
        up = 0.05 * np.sqrt(np.sqrt(3.0) * s) if up is None else up
        out.append(case(f"tiny_body{k}", "gate_s", RING * F32(2 + k) + w - np.array([0, 0, up], F32), query=w,
                        body=body, branches=("tiny_bn",)))
    # |pd2| across the threshold: the body point rises along z above a fixed world plane
    for k, b in enumerate(([12.0, -30.0, 2.0], [-50.0, -12.0, 1.5])):
        b0 = np.asarray(b, F32)
        pts = (RING * F32(0.8) + transform(state, b0[None])[0]).astype(F32)
        assert esti_plane(pts)[0]

        def selected(bz):
            body = np.array([[b0[0], b0[1], bz]], F32)
            w = transform(state, body)
            sel = np.ones(1, np.uint8)
            residual_pass(state, body, w, by_distance(pts, w[0])[None], sorted_d2(pts, w[0])[None],
                          np.array([5], np.int32), True, sel)
            return bool(sel[0])

        for tag, bz in zip(("in", "out"), _bisect_f32(selected, b0[2], b0[2] + F32(3))):
            body = np.array([b0[0], b0[1], bz], F32)
            out.append(case(f"s_{tag}{k}", "gate_s", pts, query=transform(state, body[None])[0], body=body,
                            branches=(f"s_{tag}",)))
    return out


def small_cluster_maps():
    """cnt < 5: maps of 1-4 points in all (the search is unbounded, so the map itself must be that small)."""
    base = np.array([[20, 10, 1.0], [20.5, 10, 1.0], [20, 10.5, 1.0], [20.5, 10.5, 1.25]], F32)
    return [(k, base[:k].copy(), np.array([20.25, 10.25, 1.0], F32)) for k in range(1, 5)]


# ------------------------------------------------------------------------------------------------ pass sequence
def pass_sequence_scene(rng):
    """Clusters on horizontal planes 30-95 m out with the query 0.5 m above or below each plane (|pd2| = 0.5 passes
    the s gate there: sqrt(30)/9 > 0.6). Pose B lifts the sensor by 1 m: the queries above their plane move to
    |pd2| = 1.5 and fail, the others to 0.5 and pass."""
    out = []
    for k in range(10):
        c = np.array([-80.0 + 20 * (k % 5) * 2, -30.0 + 60 * (k // 5), 0.5 + 0.25 * k])
        p = plane_points(c, [0, 0, 1], rng, 0.4, 0.002)
        q = c + [0.05, -0.05, 0.5 if k % 2 else -0.5]
        out.append(case(f"seq{k}", "sequence", p, query=q))
    state_b = POSE_A.copy()
    state_b[2] += 1.0
    return out, POSE_A.copy(), state_b


# ------------------------------------------------------------------------------------------------ classifier
def classifier_cases(fs):
    """map_incremental classifier cases for filter_size_map_min = fs: queries on voxel faces, at voxel centres, with
    negative coordinates; first neighbours at exactly 0.5*fs from the centre on one, two and three axes (the NoNeed test
    is strict >); a neighbour exactly as far from the centre as the point (the need_add test is strict <).
    Returns a list of (name, cluster points, world query, branch)."""
    fs = float(fs)
    h = 0.5 * fs
    out = []
    sites = [np.array(v, np.float64) for v in ((30, 30, 2), (-30, 30, 2), (30, -30, -2), (-30, -30, -2), (0, 60, 1),
                                                (60, 0, 1), (-60, 0, -1), (0, -60, -1), (60, 60, 3), (-60, -60, 3))]
    it = iter(sites)

    def snap(v):  # voxel corner near v (floor(v / fs) * fs) in double
        return np.floor(v / fs) * fs

    def mid_of(p):
        return (np.floor(p.astype(np.float64) / fs) * fs + h).astype(F32)

    def add(name, pts, q, branch):
        out.append((name, np.asarray(pts, F32), np.asarray(q, F32), branch))

    # query at a voxel centre; neighbours around it at distinct distances
    s = snap(next(it))
    q = s + h
    add("centre", q + np.array([[0.3, 0, 0], [0, 0.35, 0], [0, 0, -0.4], [-0.45, 0, 0], [0, -0.5, 0]]) * fs, q, "centre")
    # query on a voxel face (x exactly on a multiple of fs); negative coordinates go through floor
    s = snap(next(it))
    q = s + [0.0, 0.3 * fs, 0.6 * fs]
    add("face_neg", q + np.array([[0.2, 0.1, 0], [0.5, 0, 0.1], [0, 0.6, 0], [-0.7, 0, 0], [0, 0, 0.8]]) * fs, q, "face")
    # first neighbour at exactly 0.5*fs from the centre on 1, 2 and 3 axes, the other axes beyond
    for nax in (1, 2, 3):
        s = snap(next(it))
        q = s + np.array([0.25, 0.25, 0.25]) * fs
        m = mid_of(q[None].astype(F32))[0]
        off = np.array([h if a < nax else 0.75 * fs for a in range(3)], F32)
        n0 = (m + off).astype(F32)
        far = m + np.array([[1.5, 1.5, 1.5], [-1.5, 1.6, 1.5], [1.7, -1.5, 1.5], [1.5, 1.5, -1.8]]) * fs
        add(f"half_{nax}axes", np.vstack([n0, far]), q, "strict_gt")
    # all three axes beyond 0.5*fs: PointNoNeedDownsample
    s = snap(next(it))
    q = s + np.array([0.5, 0.5, 0.5]) * fs
    m = s + h
    add("beyond_3axes", np.vstack([m + 0.625 * fs, m + np.array([[1.5, 1.5, 1.5], [-1.5, 1.6, 1.5], [1.7, -1.5, 1.5],
                                                                 [1.5, 1.5, -1.8]]) * fs]), q, "nonneed")
    # a neighbour exactly as far from the centre as the point (its mirror image through the centre): not nearer, so the
    # point is still added; the other neighbours are farther from the centre
    s = snap(next(it))
    m = s + h
    d = np.array([0.125, 0.25, -0.125]) * fs
    q = m + d
    mirror = m - d
    add("mirror_tie", np.vstack([mirror, m + d * 3, m - d * 3, m + np.array([0.0, 0.0, 0.5]) * fs,
                                 m + np.array([0.5, -0.5, 0]) * fs]), q, "strict_lt")
    # one neighbour strictly nearer the centre: dropped
    s = snap(next(it))
    m = s + h
    q = m + d
    add("nearer", np.vstack([m + d * 0.5, m + d * 3, m - d * 3, m + np.array([0.0, 0.0, 0.5]) * fs,
                             m + np.array([0.5, -0.5, 0]) * fs]), q, "nearer")
    return out
