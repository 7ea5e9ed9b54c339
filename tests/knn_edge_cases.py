"""Constructed maps and queries for the k-NN search at the places where a hashed-voxel search goes wrong: voxel, block
and coarse-cell faces (where the key floor(fl(x / ds)) and the float face fl(k * ds) disagree by an ulp), the
completeness test of each search phase, exact float ties, overflow chains and the max_dist bound.

Everything here is plain numpy and deterministic.  The answer each case is checked against is `brute`: a float32 brute
force over the whole constructed map with the kernels' distance ((dx*dx + dy*dy) + dz*dz, each operation rounded, no
FMA), ascending, ties in (x, y, z) order, and a neighbour kept when its float d2 <= max_dist * max_dist in double (the
reference ikd-Tree's comparison, ikd_Tree.cpp:872,887).

Phases of the search (knn_kernels.cuh): 0 the 5x5x5 voxel stencil, 1 the block rings 1..8, 2 the 3x3x3 coarse cells,
3 every coarse cell.  `expected_phase` restates, in float32, the test each phase uses to stop: the k-th distance so far
is below the squared distance to the searched region's faces shrunk by the margin
mg = 1e-3 * ds + 4.8e-7 * (|qx| + |qy| + |qz|)."""
import numpy as np

F32 = np.float32
DS_LIST = (0.2, 0.25, 0.1, 0.3, 0.5, 1.0)
K_SCAN = 5          # the scan path's k
MAX_DISTS = (0.1, 0.3, 0.7, 1.3, 1.0, 50.0)
COMPLETENESS = ("stencil", "ring1", "ring2", "ring3", "ring8", "coarse")
# the phase that finishes a query whose k-th neighbour sits at the face of each region
NEXT_PHASE = {"stencil": 1, "ring1": 1, "ring2": 1, "ring3": 1, "ring8": 2, "coarse": 3}


# ------------------------------------------------------------------------------------------------ float emulation
def key(x, ds):
    """voxel_of: floor(__fdiv_rn(x, ds)); numpy's float32 division is correctly rounded, as __fdiv_rn is."""
    return np.floor(np.asarray(x, F32) / F32(ds)).astype(np.int64)


def face(k, ds):
    """The float face of voxel index k: fl(k * ds), as the kernels compute (float)k * ds."""
    return F32(F32(k) * F32(ds))


def step(x, n):
    """x moved by n float steps (n < 0: towards -inf)."""
    x = F32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, F32(np.inf) if n > 0 else F32(-np.inf), dtype=F32)
    return F32(x)


def sqdist(q, p):
    """((dx*dx + dy*dy) + dz*dz) in float32, each operation rounded; q (..., 3), p (..., 3) broadcast."""
    q = np.asarray(q, F32)
    p = np.asarray(p, F32)
    d = (q - p).astype(F32)
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F32)


def margin(q, ds):
    q = np.asarray(q, F32)
    a = (np.abs(q[..., 0]) + np.abs(q[..., 1])).astype(F32) + np.abs(q[..., 2])
    return (F32(F32(1e-3) * F32(ds)) + F32(4.8e-7) * a.astype(F32)).astype(F32)


def cover2(q, lo, hi, mg):
    """Squared distance from q to the nearest face of [lo, hi) shrunk by mg, 0 when not positive (cover2)."""
    q = np.asarray(q, F32)
    lo = np.asarray(lo, F32)
    hi = np.asarray(hi, F32)
    c = F32(min(float(F32(q[j] - lo[j])) if s == 0 else float(F32(hi[j] - q[j])) for j in range(3) for s in (0, 1)))
    c = F32(c - F32(mg))
    return F32(c * c) if c > 0 else F32(0.0)


def max_d2(max_dist):
    """The largest float32 not above (double)max_dist^2: a float d2 passes the reference's double test iff d2 <= it."""
    if max_dist is None or not max_dist > 0:
        return F32(np.inf)
    sq = float(F32(max_dist)) * float(F32(max_dist))
    f = F32(sq)
    return np.nextafter(f, F32(0), dtype=F32) if float(f) > sq else f


# ------------------------------------------------------------------------------------------------ reference answer
def candidates(mp, q, max_dist=None):
    """All map points within max_dist of q, sorted by (d2, x, y, z): (d2[m], xyz[m, 3], index[m])."""
    mp = np.asarray(mp, F32).reshape(-1, 3)
    if len(mp) == 0 or not np.isfinite(np.asarray(q, F32)).all():
        return np.zeros(0, F32), np.zeros((0, 3), F32), np.zeros(0, np.int64)
    d2 = sqdist(q, mp)
    ok = np.nonzero(d2 <= max_d2(max_dist))[0]
    o = ok[np.lexsort((mp[ok, 2], mp[ok, 1], mp[ok, 0], d2[ok]))]
    return d2[o], mp[o], o


def brute(mp, qs, k, max_dist=None):
    """k-NN of every query: xyz [n, k, 3] (NaN past the count), d2 [n, k] (INF past the count), cnt [n]."""
    qs = np.asarray(qs, F32).reshape(-1, 3)
    xyz = np.full((len(qs), k, 3), np.nan, F32)
    d2 = np.full((len(qs), k), np.inf, F32)
    cnt = np.zeros(len(qs), np.int32)
    for i, q in enumerate(qs):
        d, p, _ = candidates(mp, q, max_dist)
        c = min(k, len(d))
        cnt[i] = c
        d2[i, :c] = d[:c]
        xyz[i, :c] = p[:c]
    return xyz, d2, cnt


def _rows(a):
    return [tuple(np.asarray(r, F32).view(np.uint32).tolist()) for r in np.asarray(a, F32).reshape(len(a), -1)]


def check_knn(mp, qs, k, xyz, d2, cnt, max_dist=None, lex=None, extra=None, mp_extra=None):
    """Compare one search's answer with the brute force, stricter than helpers.knn_equal: counts and distances bit-equal;
    every returned point lies at its distance; every group of equal distances is a sub-multiset of ALL the map points
    at that distance (members beyond k included); for the queries in `lex` each tie group is in (x, y, z) order.
    `extra`/`mp_extra`: per-neighbour records (e.g. intensities) and the map's records, compared the same way.
    Returns a list of failure strings (empty when the answer is exact)."""
    qs = np.asarray(qs, F32).reshape(-1, 3)
    mp = np.asarray(mp, F32).reshape(-1, 3)
    bad = []
    for i, q in enumerate(qs):
        d, p, idx = candidates(mp, q, max_dist)
        c = min(k, len(d))
        if int(cnt[i]) != c:
            bad.append(f"q{i}: count {int(cnt[i])} != {c}")
            continue
        if not np.array_equal(np.asarray(d2[i, :c], F32).view(np.uint32), d[:c].view(np.uint32)):
            bad.append(f"q{i}: d2 {d2[i, :c].tolist()} != {d[:c].tolist()}")
            continue
        got = np.asarray(xyz[i, :c], F32)
        if c and not np.array_equal(sqdist(q, got).view(np.uint32), d[:c].view(np.uint32)):
            bad.append(f"q{i}: points not at their distances")
            continue
        for v in np.unique(d[:c]):
            g = np.nonzero(d[:c] == v)[0]
            pool = np.nonzero(d == v)[0]
            mine = got[g] if extra is None else np.concatenate([got[g], np.asarray(extra[i, g], F32).reshape(len(g), -1)], 1)
            full = p[pool] if mp_extra is None else np.concatenate([p[pool], np.asarray(mp_extra, F32).reshape(len(mp), -1)[idx[pool]]], 1)
            avail = _rows(full)
            for r in _rows(mine):
                if r in avail:
                    avail.remove(r)
                else:
                    bad.append(f"q{i}: {np.asarray(r, np.uint32).view(F32).tolist()} not among the points at d2={float(v)!r}")
            if lex is not None and lex[i] and len(g) > 1:
                sub = got[g]
                if not np.array_equal(np.lexsort((sub[:, 2], sub[:, 1], sub[:, 0])), np.arange(len(g))):
                    bad.append(f"q{i}: tie group at d2={float(v)!r} not in (x, y, z) order: {sub.tolist()}")
    return bad


# ------------------------------------------------------------------------------------------------ search phases
def expected_phase(mp, q, ds, k=K_SCAN, max_dist=None, margin_scale=1.0):
    """The phase that finishes query q (K = k), restating each phase's stop test in float32 (see the module doc).
    Rings report 1 with the ring number in the second value.  margin_scale = 0: the same tests without the margin."""
    mp = np.asarray(mp, F32).reshape(-1, 3)
    q = np.asarray(q, F32)
    lim = max_d2(max_dist)
    if not (np.abs(q) < F32(4.0e6) * F32(ds)).all():
        return 0, 0
    mg = F32(margin(q, ds) * F32(margin_scale))
    cv = key(q, ds)
    kp = key(mp, ds) if len(mp) else np.zeros((0, 3), np.int64)
    d2 = sqdist(q, mp) if len(mp) else np.zeros(0, F32)
    within = d2 <= lim

    def kth(sel):
        s = np.sort(d2[sel & within])
        return (F32(s[k - 1]), True) if len(s) >= k else (F32(np.inf), False)

    dk, full = kth((np.abs(kp - cv) <= 2).all(1))
    cov = cover2(q, F32(cv - 2) * F32(ds), F32(cv + 3) * F32(ds), mg)
    if (full and dk < cov) or cov > lim:
        return 0, 0
    qb, qc = cv >> 2, cv >> 5
    kb, kc = kp >> 2, kp >> 5
    bs4 = F32(F32(4.0) * F32(ds))
    any27 = (np.abs(kc - qc) <= 1).all(1).any()
    for r in range(1, 9):
        if r == 3 and not any27:
            break
        dk, full = kth((np.abs(kb - qb) <= r).all(1))
        cov = cover2(q, F32(qb - r) * bs4, F32(qb + r + 1) * bs4, mg)
        if (full and dk < cov) or cov > lim:
            return 1, r
    cs32 = F32(F32(32.0) * F32(ds))
    dk, full = kth((np.abs(kc - qc) <= 1).all(1) | (np.abs(kb - qb) <= 8).all(1))
    cov = cover2(q, F32(qc - 1) * cs32, F32(qc + 2) * cs32, mg)
    if (full and dk < cov) or cov > lim:
        return 2, 0
    return 3, 0


# ------------------------------------------------------------------------------------------------ case families
def _case(name, ds, mp, qs, **kw):
    c = dict(name=name, ds=float(ds), map=np.asarray(mp, F32).reshape(-1, 3), queries=np.asarray(qs, F32).reshape(-1, 3),
             max_dist=None)
    c.update(kw)
    return c


def outside_keyed_faces(ds, kmax=400):
    """Faces k (1 <= k < kmax) of voxel size ds with a point keyed to the far side of the face while its coordinate lies
    on the near side: (k, x, side) where side = +1: x < fl(k ds) but key(x) == k (a region ending at face k holds it by
    coordinate, not by key); side = -1: x >= fl(k ds) but key(x) == k - 1."""
    out = []
    for k in range(1, kmax):
        f = face(k, ds)
        for n in (1, 2, 3):
            x = step(f, -n)
            if key(x, ds) == k:
                out.append((k, x, +1))
                break
        for n in (0, 1, 2, 3):
            x = step(f, n)
            if key(x, ds) == k - 1:
                out.append((k, x, -1))
                break
    return out


def face_cases(ds, seed=0):
    """Points and queries at voxel, block and coarse faces fl(k ds) and up to three float steps either side, both
    signs, with 0, -0.0 and subnormals around the origin."""
    rng = np.random.default_rng(seed + int(ds * 1000))
    ks = sorted({1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 64, 96} | {int(k) for k in rng.integers(1, 300, 6)})
    coords = [F32(0.0), F32(-0.0), F32(1e-45), F32(-1e-45), F32(1e-40), F32(-1e-40), F32(1.2e-38)]
    for k in ks:
        for s in (1, -1):
            f = face(s * k, ds)
            coords += [step(f, n) for n in range(-3, 4)]
    coords = np.array(coords, F32)
    out = []
    for tag, lo, hi in (("near", 0, None),):
        pts = coords[rng.integers(0, len(coords), (700, 3))]
        # keep it small enough for the brute force; many points share coordinates along an axis (exact ties)
        pts = np.unique(pts.view(np.uint32), axis=0).view(F32)
        qs = np.concatenate([coords[rng.integers(0, len(coords), (150, 3))],
                             np.array([[0, 0, 0], [-0.0, -0.0, -0.0], [1e-45, -1e-45, 0]], F32)])
        out.append(_case(f"faces_{tag}_ds{ds}", ds, pts, qs))
    return out


def _fill(q, ds, n):
    """n filler points within 0.3 voxel of q (distinct, inside the stencil): the K-1 nearest neighbours."""
    offs = np.array([[0.1, 0.05, 0.0], [-0.12, 0.0, 0.06], [0.0, -0.14, -0.03], [0.02, 0.11, -0.13], [-0.05, -0.08, 0.15],
                     [0.16, -0.1, 0.04], [-0.15, 0.12, -0.1]], np.float64)[:n]
    return (np.asarray(q, np.float64) + offs * ds).astype(F32)


def _match_d2(q, target, along, start, ds):
    """The point q + t * e_along (t near start), nudged along the next axis by a small offset whose square fills the
    gap, whose float d2 is nearest above and nearest below target: ((d2, point), (d2, point))."""
    best_hi = best_lo = None
    x0 = F32(q[along] + F32(start))
    side = (along + 1) % 3
    for n in range(-40, 41):
        p = np.array(q, F32)
        p[along] = step(x0, n)
        base = float(sqdist(q, p))
        ys = [q[side]]
        for want in (step(target, -1), step(target, 1)):
            gap = float(want) - base
            if gap > 0:
                y0 = F32(q[side] + F32(np.sqrt(gap)))
                ys += [step(y0, m) for m in range(-4, 5)]
        for y in ys:
            p2 = p.copy()
            p2[side] = y
            d = sqdist(q, p2)
            if d > target and (best_hi is None or d < best_hi[0]):
                best_hi = (d, p2)
            if d < target and (best_lo is None or d > best_lo[0]):
                best_lo = (d, p2)
    return best_hi, best_lo


def completeness_cases(ds, region):
    """The query's K-th neighbour inside `region` sits at the distance c of the region's +x face (within the margin),
    and a competitor keyed outside the region but lying inside its float face (an outside_keyed_faces point, or the
    face itself for the binary ds) is one float step nearer ("near") or farther ("far").  The region's stop test must
    fail, or the nearer competitor is lost."""
    dsf = F32(ds)
    # query position along x in voxels relative to the voxel/block/cell that ends at the face; y and z sit in voxel 17 of
    # coarse cell 0 (block 4), far enough from every y/z face that the +x face is the nearest one of the region
    if region == "stencil":
        unit, back, yz = 1, 2.3, 17.5
    elif region.startswith("ring"):
        r = int(region[4:])
        unit, back, yz = 4, 4 * r + 0.7, 17.5
    else:  # the 3x3x3 coarse cells: the query in the middle of its cell so that ring 8 ends before them
        unit, back, yz = 32, 47.7, 16.1
    # (a ring's face must not be a coarse face too: the 3x3x3 coarse cells would then end there as well)
    cands = [(k, x, s) for k, x, s in outside_keyed_faces(ds, 4000)
             if s == +1 and k % unit == 0 and k >= 64 and (unit != 4 or k % 32)]
    if not cands:   # binary ds: fl(k ds) is exact, the competitor sits on the face itself (keyed outside)
        k = 132 if unit < 32 else 160
        cands = [(k, face(k, ds), 0)]
    out = []
    for j, (k, xo, _) in enumerate(cands[:2]):
        qx = F32((k - back) * float(dsf))
        q = np.array([qx, F32(yz * float(dsf)), F32(yz * float(dsf))], F32)
        comp = np.array([xo, q[1], q[2]], F32)
        dc = sqdist(q, comp)
        hi, lo = _match_d2(q, dc, 0, -float(F32(xo - qx)), ds)   # the K-th neighbour in -x, the mirror of the competitor
        for tag, m in (("near", hi), ("far", lo)):
            pts = np.concatenate([_fill(q, ds, K_SCAN - 1), m[1][None], comp[None]])
            out.append(_case(f"complete_{region}_{tag}{j}_ds{ds}", ds, pts, q[None], region=region, variant=tag,
                             comp=comp, kth=m[1], face_k=k))
    return out


def tie_cases(ds):
    """Exact float ties: (a) eight points at one distance around a query inside the stencil (the stencil resolves it;
    its ties keep arrival order, compare as sets), straddling position K; (b) a tie between a point of ring 1 and a
    lexicographically smaller point of ring 2 at the K-th position (the exact kernel resolves it: the (x, y, z) rule
    must pick the ring-2 point, which arrives after the bound has reached the tie distance); and its mirror."""
    out = []
    g = 1.0 / 64.0
    dsf = float(F32(ds))
    # (a)
    c = np.round(np.array([10.5, 17.5, 17.5]) * dsf / g) * g
    a = np.round(0.9 * dsf / g) * g
    dirs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 1, 0], [-1, -1, 0]], np.float64)
    lens = np.array([a] * 6 + [np.round(a / np.sqrt(2) / g) * g] * 2)
    pts = (c + dirs * lens[:, None]).astype(F32)
    pts = pts[:6]   # the six axis points are tied exactly
    pts = np.concatenate([pts, _fill(c, ds, 2)])
    out.append(_case(f"tie_stencil_ds{ds}", ds, pts, c[None], lex_exact=False))
    # (b) query at local (x=0.5, y=1.5, z=1.5) voxels of block 8: ring 1 ends 4.5 voxels away in -x, more elsewhere.
    # A (ring 1, +y) arrives first and sets the bound to D^2; B (ring 2, -x) has the smaller x.  The mirror negates the
    # scene: the ring-1 point is then the smaller one, so the other answer occurs.
    for sgn in (1.0, -1.0):
        q = np.round(np.array([32.5, 33.5, 33.5]) * dsf / g) * g
        D = np.round(5.6 * dsf / g) * g
        A = q + np.array([0.0, D, 0.0])
        B = q + np.array([-D, 0.0, 0.0])
        q, A, B = sgn * q, sgn * A, sgn * B
        pts = np.concatenate([_fill(q, ds, K_SCAN - 1), np.array([A, B], F32)]).astype(F32)
        out.append(_case(f"tie_rings{'_mirror' if sgn < 0 else ''}_ds{ds}", ds, pts, q[None].astype(F32), lex_exact=True,
                         ring1=A.astype(F32), ring2=B.astype(F32)))
    return out


def sparse_far_cases(ds, seed=1):
    """Maps of 0-4 points; queries with fewer than K points within max_dist; maps translated to 1e4 m, 1e5 m and just
    inside the coordinate bound 4e6 ds."""
    rng = np.random.default_rng(seed + int(ds * 1000))
    out = []
    for n in range(5):
        mp = (rng.normal(0, 2.0, (n, 3))).astype(F32)
        qs = np.concatenate([rng.normal(0, 3.0, (6, 3)), rng.normal(0, 40.0, (2, 3))]).astype(F32)
        out.append(_case(f"sparse{n}_ds{ds}", ds, mp, qs))
        out.append(_case(f"sparse{n}_md_ds{ds}", ds, mp, qs, max_dist=F32(2.5)))
    for off in (1e4, 1e5, 0.999 * 4e6 * float(F32(ds))):
        base = np.array([off, -off * 0.5, off * 0.25])
        mp = (base + rng.normal(0, 1.0, (60, 3))).astype(F32)
        qs = (base + np.concatenate([rng.normal(0, 1.0, (20, 3)), rng.normal(0, 30.0, (4, 3))])).astype(F32)
        out.append(_case(f"far{int(off)}_ds{ds}", ds, mp, qs))
    return out


def out_of_range_queries(ds):
    """Queries at and beyond the stencil's bound 4e6 ds and NaN queries: the search returns no neighbours for them
    (the reference searches them; see DESIGN.md section 5)."""
    lim = F32(4.0e6) * F32(ds)
    return np.array([[lim, 0, 0], [0, -lim, 0], [0, 0, step(lim, 1)], [np.inf, 0, 0], [np.nan, 0, 0], [0, np.nan, 1]], F32)


def _hit_d2(target, axis):
    """A point p with sqdist(0, p) == target exactly (p on `axis`, plus a small second coordinate when needed)."""
    t = float(target)
    x0 = F32(np.sqrt(t))
    ulp = float(np.spacing(F32(target)))
    for y in [F32(0.0)] + [F32(np.sqrt(j * ulp)) for j in (0.75, 1.0, 1.25, 1.5, 2.0, 2.5, 3.0)]:
        for n in range(-60, 61):
            p = np.zeros(3, F32)
            p[axis] = step(x0, n)
            p[(axis + 1) % 3] = y
            if sqdist(np.zeros(3, F32), p) == target:
                return p
    return None


def max_dist_cases():
    """Neighbours of a query at the origin at d2 equal to the float square fl(md * md), to the largest float not above
    the exact double square, and one float step either side of each, for each max_dist (a float32 value)."""
    out = []
    for md in MAX_DISTS:
        m = F32(md)
        fsq = F32(m * m)
        dsq = max_d2(m)
        targets = sorted({float(v) for v in (fsq, step(fsq, -1), step(fsq, 1), dsq, step(dsq, -1), step(dsq, 1))})
        pts = []
        for j, t in enumerate(targets):
            p = _hit_d2(F32(t), j % 3)
            assert p is not None, (md, t)
            pts.append(p * (1 if j % 2 else -1))
        pts = np.array(pts, F32)
        out.append(_case(f"max_dist_{md}", 0.2, pts, np.zeros((1, 3), F32), max_dist=m, fsq=fsq, dsq=dsq))
    return out


def chain_ops(seed=2, ds=0.2):
    """Overflow chains from a verbatim Build and Add_Points(..., False): several points per voxel, then Delete_Points of
    chain heads, middles and tails (the chains are no longer contiguous), then a verbatim insert that reuses the freed
    nodes.  Returns (ops, final content [n, 4] xyz + intensity, queries)."""
    rng = np.random.default_rng(seed)
    dsf = float(F32(ds))
    vox = rng.integers(-6, 6, (24, 3))
    pts = []
    for v in vox:
        m = int(rng.integers(2, 9))
        pts.append((v + rng.uniform(0.05, 0.95, (m, 3))) * dsf)
    pts = np.concatenate(pts).astype(F32)
    inten = np.arange(len(pts), dtype=F32)
    build = np.concatenate([pts, inten[:, None]], 1)
    # delete: in every voxel with >= 3 points its first, a middle and its last point (insert order = Build order)
    kv = key(pts, ds)
    dele = []
    for v in np.unique(kv, axis=0):
        idx = np.nonzero((kv == v).all(1))[0]
        if len(idx) >= 3:
            dele += [idx[0], idx[len(idx) // 2], idx[-1]]
        elif len(idx) == 2:
            dele.append(idx[1])
    dele = np.array(sorted(set(dele)))
    keep = np.setdiff1d(np.arange(len(pts)), dele)
    add = ((vox[:12] + rng.uniform(0.05, 0.95, (12, 3))) * dsf).astype(F32)
    add = np.concatenate([add, add[:4] + F32(0.01 * dsf)]).astype(F32)
    add4 = np.concatenate([add, (1000 + np.arange(len(add)))[:, None].astype(F32)], 1)
    ops = [("build", build), ("delete", pts[dele]), ("add", add4)]
    final = np.concatenate([build[keep], add4])
    qs = np.concatenate([((vox + 0.5) * dsf), ((vox[:8] + rng.uniform(0, 1, (8, 3))) * dsf)]).astype(F32)
    return ops, final, qs


def duplicate_points(seed=3, ds=0.2):
    """A verbatim Build with duplicated coordinates carrying distinct intensities (2-4 copies per point)."""
    rng = np.random.default_rng(seed)
    base = (rng.uniform(-1.0, 1.0, (10, 3))).astype(F32)
    rows = []
    for j, p in enumerate(base):
        for c in range(1 + (j % 4)):
            rows.append([p[0], p[1], p[2], F32(10 * j + c)])
    pts4 = np.array(rows, F32)
    qs = np.concatenate([base, base[:3] + F32(0.05)]).astype(F32)
    return pts4, qs


def pool_end_points(ds=0.2):
    """A map for max_points = 2048 (overflow pool of 1024 nodes) whose Build uses every overflow node: 64 voxels of 17
    points each (64 heads + 1024 chain nodes)."""
    rng = np.random.default_rng(4)
    dsf = float(F32(ds))
    vox = np.array([[i % 4, (i // 4) % 4, i // 16] for i in range(64)]) * 2
    pts = np.concatenate([(v + rng.uniform(0.05, 0.95, (17, 3))) * dsf for v in vox]).astype(F32)
    qs = np.concatenate([(vox + 0.5) * dsf, rng.uniform(-0.5, 8 * dsf, (24, 3))]).astype(F32)
    return pts, qs


def search_cases():
    """Every case whose map is a plain Build of its points."""
    out = []
    for ds in DS_LIST:
        out += face_cases(ds)
        for region in COMPLETENESS:
            out += completeness_cases(ds, region)
        out += tie_cases(ds)
        out += sparse_far_cases(ds)
    out += max_dist_cases()
    return out
