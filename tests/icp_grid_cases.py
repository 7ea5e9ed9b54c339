"""Constructed targets and queries for the registrations' grid nearest-neighbour search (icp_kernels.cuh, shared by
flb_keyframes_icp, _fricp, _sicp, _aaicp and _icp_batch), with a float32 restatement of the grid and a brute-force 1-NN
under the search's contract: float d² = (dx*dx + dy*dy) + dz*dz, ties to the lower target index.

The restatements follow the operation order of icp_host.cuh / icp_kernels.cuh with no FMA:
  grid(lo, hi, n)     icp_grid: double sizing, the cap loop, then the float casts of e, inv_e and slack;
  cells(g, p)         icp_cell1: floor((p - o) * inv_e) in float, clamped to the grid;
  face(g, a, k)       o + k * e in float (a cell's lower face along axis a);
  ring_lb / ring_done icp_ring_lb / icp_ring_done for a fine ring.
Every case records what it claims to exercise (Case.claims); tests/test_icp_grid_cpu.py checks each claim with these
restatements, and tests/test_gpu_icp_grid.py runs the cases through the device search.  All cases are deterministic.

What the slack and the ring margin each guard.  The slack (1e-3 e + 4e-6 (max |coordinate| + extent)) covers the float
cell assignment: the slack-trap queries of families a and b (_slack_traps) have a nearest target that the assignment
puts one cell across a face, and the restated search with slack 0 returns a wrong answer on every one of them.  The
1 - 1e-6 margin of icp_ring_done covers the float rounding of d² (a few 1e-8 relative).  For a query inside the box it
cannot change a result while the slack is in place: a ring's bound lb is below the true distance by at least the slack,
and slack / lb >= 1e-3 e / (1024 sqrt(3) e), about 5.6e-7, already more than the margin.  Only a query far outside the
box (roughly 10 km for these boxes), where lb grows and the slack does not, could make the margin observable; no case
here goes that far, so removing the margin is not expected to fail these tests.

The face placements of families a and b hold on the float grid of the raw target.  fricp normalises the clouds
(p / scale - mu) and builds its grid over that, so on the double path these cases are exactness checks on near-tied
and tied clouds, not face cases."""
import math
from dataclasses import dataclass, field

import numpy as np

F = np.float32
ICP_C = 8
ICP_RINGS = 2
CELLS_PER_POINT = 8.0
MAX_CELLS = 134217728.0
LATTICE_N, LATTICE_PITCH = 256, 0.125   # family h: 256³ points at 0.125 m


# ------------------------------------------------------------------------------------------------ restatements
@dataclass
class Grid:
    o: np.ndarray        # (3,) float32 origin (the finite minimum)
    e: np.float32
    inv_e: np.float32
    slack: np.float32
    dims: tuple          # fine cells per axis, multiples of 8
    e_double: float      # the double edge before the cast
    cap_steps: int       # e *= 1.25 steps of the ICP_MAX_CELLS loop
    ext_over_e: tuple    # ext[a] / e in double, as the sizing computes it


def grid(lo, hi, n_fin):
    lo, hi = np.asarray(lo, F), np.asarray(hi, F)
    ext = [float(hi[a]) - float(lo[a]) for a in range(3)]
    L = max(0.0, *ext)
    amax = max(0.0, *[max(abs(float(lo[a])), abs(float(hi[a]))) for a in range(3)])
    e = 1.0
    if L > 0.0:
        floor_e = L / 1024.0
        V = 1.0
        for a in range(3):
            V *= max(ext[a], floor_e)
        e = max(math.cbrt(V / (CELLS_PER_POINT * n_fin)), floor_e)
    steps = 0
    while True:
        dims = tuple((int(math.floor(ext[a] / e)) + 1 + ICP_C - 1) // ICP_C * ICP_C for a in range(3))
        if float(dims[0]) * dims[1] * dims[2] <= MAX_CELLS:
            break
        e *= 1.25
        steps += 1
    e32 = F(e)
    with np.errstate(over="ignore"):
        slack = F(F(1e-3) * e32) + F(F(4e-6) * F(amax + L))
    return Grid(lo.copy(), e32, F(F(1.0) / e32), F(slack), dims, e, steps, tuple(x / e for x in ext))


def grid_of(tgt):
    fin = np.isfinite(tgt[:, :3]).all(1)
    t = tgt[fin, :3].astype(F)
    return grid(t.min(0), t.max(0), int(fin.sum()))


def raw_cells(g, p):
    """floor((p - o) * inv_e) in float, before the clamp (int64, may lie outside the grid)."""
    p = np.asarray(p, F).reshape(-1, 3)
    with np.errstate(over="ignore", invalid="ignore"):
        f = np.floor((p - g.o) * g.inv_e)
    f = np.clip(np.nan_to_num(f, nan=0.0, posinf=2.0 ** 40, neginf=-2.0 ** 40), -2.0 ** 40, 2.0 ** 40)
    return f.astype(np.int64)


def cells(g, p):
    return np.clip(raw_cells(g, p), 0, np.array(g.dims) - 1)


def exact_cells(g, p):
    """The cell each coordinate lies in, in exact arithmetic: the largest k with o + k e <= p (x, o, e are floats, so
    p - o and k e are exact in double)."""
    d = np.asarray(p, F).reshape(-1, 3).astype(np.float64) - g.o.astype(np.float64)
    e = float(g.e)
    k = np.floor(d / e)
    k = np.where(k * e > d, k - 1, k)
    k = np.where((k + 1) * e <= d, k + 1, k)
    return k.astype(np.int64)


def face(g, a, k):
    return F(g.o[a] + F(F(k) * g.e))


def ring_lb(g, q, c, r):
    """icp_ring_lb for fine ring r >= 1 around cell c (span 1): float distance, inf when the ring has no cell."""
    lb = F(np.inf)
    for a in range(3):
        if c[a] - r >= 0:
            lb = min(lb, max(F(q[a] - F(F(g.o[a] + F(F(c[a] - r + 1) * g.e)) + g.slack)), F(0)))
        if c[a] + r < g.dims[a]:
            lb = min(lb, max(F(F(F(g.o[a] + F(F(c[a] + r) * g.e)) - g.slack) - q[a]), F(0)))
    return lb


def ring_done(g, q, c, r, best):
    lb = ring_lb(g, q, c, r)
    return bool(lb == np.inf or float(lb) * float(lb) * (1.0 - 1e-6) > float(best))


def cell_index(g, tgt):
    """The finite targets by their (clamped) cell: {(ix, iy, iz): ascending target indices}."""
    fin = np.flatnonzero(np.isfinite(tgt[:, :3]).all(1))
    out = {}
    for i, c in zip(fin, map(tuple, cells(g, tgt[fin]))):
        out.setdefault(c, []).append(i)
    return out


def fine_search(g, tgt, q, index, slack=None, rings=ICP_RINGS):
    """icp_fine_rings with icp_scan for one float query, in the kernel's cell order, on the grid g with its slack (or
    the given one): (closed, index, d²).  The fine rings' result is the device's result whenever they close."""
    g = g if slack is None else Grid(g.o, g.e, g.inv_e, F(slack), g.dims, g.e_double, g.cap_steps, g.ext_over_e)
    q = np.asarray(q, F)
    c = cells(g, q[None])[0]
    best, bi = F(np.inf), np.iinfo(np.int32).max

    def lb2(ix, iy, iz):
        acc = []
        for a, k in enumerate((ix, iy, iz)):
            lo = F(F(g.o[a] + F(F(k) * g.e)) - g.slack)
            hi = F(F(g.o[a] + F(F(k + 1) * g.e)) + g.slack)
            acc.append(max(max(F(lo - q[a]), F(q[a] - hi)), F(0)))
        return F(F(F(acc[0] * acc[0]) + F(acc[1] * acc[1])) + F(acc[2] * acc[2]))

    with np.errstate(over="ignore"):
        for r in range(rings + 2):
            if r > 0 and ring_done(g, q, c, r, best):
                return True, int(bi), best
            if r == rings + 1:
                break
            for dz in range(-r, r + 1):
                for dy in range(-r, r + 1):
                    face_row = abs(dz) == r or abs(dy) == r
                    for dx in (range(-r, r + 1) if face_row or r == 0 else (-r, r)):
                        k = (c[0] + dx, c[1] + dy, c[2] + dz)
                        if not all(0 <= k[a] < g.dims[a] for a in range(3)) or not lb2(*k) <= best:
                            continue
                        for i in index.get(k, ()):
                            d = tgt[i, :3] - q
                            d2 = F(F(F(d[0] * d[0]) + F(d[1] * d[1])) + F(d[2] * d[2]))
                            if d2 < best or (d2 == best and i < bi):
                                best, bi = d2, i
    return False, int(bi), best


# ------------------------------------------------------------------------------------------------ reference
def brute_nn(q, tgt, chunk=None, ties=False):
    """Exact 1-NN of every query over the finite targets: (index, float d²) and, with ties, the number of targets at
    that d² and the smallest d² of the other targets.  Index -1 / d² inf for a non-finite query or no finite target; a query whose every d² overflows takes the
    lowest finite index."""
    q = np.asarray(q, F)[:, :3]
    t = np.asarray(tgt, F)[:, :3]
    fin = np.flatnonzero(np.isfinite(t).all(1))
    tf = t[fin]
    m = len(q)
    idx = np.full(m, -1, np.int32)
    d2 = np.full(m, np.inf, F)
    cnt = np.zeros(m, np.int32)
    second = np.full(m, np.inf, F)
    if len(fin) == 0 or m == 0:
        return (idx, d2, cnt, second) if ties else (idx, d2)
    chunk = chunk or max(1, (1 << 24) // max(len(tf), 1))
    with np.errstate(over="ignore", invalid="ignore"):
        for b in range(0, m, chunk):
            qq = q[b:b + chunk]
            dx = tf[None, :, 0] - qq[:, None, 0]
            dy = tf[None, :, 1] - qq[:, None, 1]
            dz = tf[None, :, 2] - qq[:, None, 2]
            d = (dx * dx + dy * dy) + dz * dz
            j = np.argmin(d, axis=1)   # the first minimum: the lowest finite index
            best = d[np.arange(len(qq)), j]
            ok = np.isfinite(qq).all(1)
            idx[b:b + chunk] = np.where(ok, fin[j], -1)
            d2[b:b + chunk] = np.where(ok, best, np.inf)
            if ties:
                cnt[b:b + chunk] = np.where(ok, (d == best[:, None]).sum(1), 0)
                d[np.arange(len(qq)), j] = np.inf
                second[b:b + chunk] = d.min(1) if d.shape[1] else np.inf
    return (idx, d2, cnt, second) if ties else (idx, d2)


def lattice_keyframe(k):
    """Key frame k (0..15) of the family-h lattice: points i = k 2^20 .. (k+1) 2^20 - 1 of the 256³ lattice, index
    i = (iz 256 + iy) 256 + ix, coordinates i_a * 0.125."""
    i = np.arange(k << 20, (k + 1) << 20, dtype=np.int64)
    n = LATTICE_N
    return (np.stack([i % n, (i // n) % n, i // (n * n)], 1) * LATTICE_PITCH).astype(F)


def lattice_queries(m=1 << 20, seed=11):
    """Queries on the 2^-6 m grid in and up to 1 m around the lattice box: every coordinate difference to a lattice
    point and every d² below 3 * 33² is exact in float, and 1/8 of the coordinates sit on a lattice mid-plane."""
    rng = np.random.default_rng(seed)
    return (rng.integers(-64, 64 * 33, size=(m, 3)) / 64.0).astype(F)


def lattice_nn(q):
    """The analytic 1-NN on the lattice: each coordinate rounded to the lattice, a mid-plane tie to the lower index."""
    q = np.asarray(q, F)[:, :3].astype(np.float64)
    k = np.clip(np.ceil(q / LATTICE_PITCH - 0.5), 0, LATTICE_N - 1).astype(np.int64)   # x.5 rounds down
    p = (k * LATTICE_PITCH).astype(F)
    qf = q.astype(F)
    d = p - qf
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    return ((k[:, 2] * LATTICE_N + k[:, 1]) * LATTICE_N + k[:, 0]).astype(np.int64), d2.astype(F)


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    name: str
    family: str
    tgt: np.ndarray                      # (n, 3) float32, NaN rows allowed
    qry: np.ndarray                      # (m, 3) float32
    claims: dict = field(default_factory=dict)
    max_dist: float = 200.0
    double_path: bool = True             # also run through fricp's double search
    knn7: bool = False                   # a 7-NN family (nu_end decided by the self-query)


def _ulps(x, k):
    """x moved by k float steps."""
    x = F(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F(np.inf) if k > 0 else F(-np.inf))
    return x


def _boxed(rng, lo, hi, n, inner):
    """n targets in [lo, hi]: the two corners (so the box and the grid are fixed before the rest is placed), then inner."""
    pts = np.empty((n, 3), F)
    pts[0], pts[1] = lo, hi
    pts[2:2 + len(inner)] = inner
    rest = n - 2 - len(inner)
    pts[2 + len(inner):] = rng.uniform(lo, hi, size=(rest, 3)).astype(F)
    return pts


def _faces_case(lo, hi, n, step, seed, n_grid=None):
    """n targets on faces o + k e (k a multiple of step) and 1-4 float steps either side of them, and queries on the
    faces between mirrored target pairs (exact ties) and between pairs one float step apart; the grid is the one of
    n_grid (>= n) targets in the box."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, F), np.asarray(hi, F)
    g = grid(lo, hi, n_grid or n)
    inner, qry = [], []
    for j in range(n // 6):
        a = j % 3
        k = int(rng.integers(1, g.dims[a] // step - 1)) * step if step > 1 else int(rng.integers(1, int(g.ext_over_e[a])))
        f = face(g, a, k)
        if not lo[a] < f < hi[a]:
            continue
        p = rng.uniform(lo, hi).astype(F)
        p[a] = _ulps(f, int(rng.integers(-4, 5)))
        inner.append(p)
    for j in range(n // 6):   # mirrored pairs across a face: the query on the face
        a = j % 3
        k = int(rng.integers(1, g.dims[a] // step - 1)) * step if step > 1 else int(rng.integers(1, int(g.ext_over_e[a])))
        f = face(g, a, k)
        d = F(float(g.e) * rng.uniform(0.01, 0.4))
        lo_p, hi_p = F(f - d), F(f + d)
        if not (lo[a] < lo_p and hi_p < hi[a]) or F(f - lo_p) != F(hi_p - f):
            continue
        base = rng.uniform(lo + 0.1 * (hi - lo), hi - 0.1 * (hi - lo)).astype(F)
        t0, t1, q = base.copy(), base.copy(), base.copy()
        t0[a], t1[a] = lo_p, hi_p
        if j % 2:
            t1[a] = _ulps(hi_p, 1)   # one float step farther: no tie, d² one or two steps apart
        inner += [t0, t1]
        q[(a + 1) % 3] = F(q[(a + 1) % 3] + F(0.03 * float(g.e)))
        q[a] = f
        qry.append(q)
    tgt = _boxed(rng, lo, hi, n, np.array(inner, F))
    qry = np.concatenate([np.array(qry, F), rng.uniform(lo, hi, size=(500, 3)).astype(F)])
    perm = rng.permutation(n)
    return tgt[perm], qry, g


def _binned_across_faces(g, step=1):
    """The number of faces o + k e (k a multiple of step) with a coordinate within 8 float steps of it that the float cell assignment puts on
    the other side."""
    n = 0
    for a in range(3):
        f = np.array([face(g, a, k) for k in range(2, int(g.ext_over_e[a]) - 1)], F)
        k = np.arange(2, int(g.ext_over_e[a]) - 1)
        hit = np.zeros(len(f), bool)
        for dirn in (-np.inf, np.inf):
            p = f.copy()
            for _ in range(8):
                pts = np.zeros((len(p), 3), F) + g.o
                pts[:, a] = p
                hit |= raw_cells(g, pts)[:, a] != exact_cells(g, pts)[:, a]
                p = np.nextafter(p, F(dirn))
        n += int(hit[k % step == 0].sum())
    return n


def _rounding_box(lo, hi, n, want, want_coarse=0):
    """hi with its z raised by the smallest of 0, 1, 2, ... mm for which the grid of n points in [lo, hi] has at least
    `want` faces (and `want_coarse` coarse faces) with binned-across coordinates (the float cell assignment errs near a
    face only for some edges e)."""
    for t in range(200):
        h = np.array(hi, F)
        h[2] = F(float(hi[2]) + 1e-3 * t)
        g = grid(lo, h, n)
        if _binned_across_faces(g) >= want and _binned_across_faces(g, ICP_C) >= want_coarse:
            return h
    raise AssertionError("no box with binned-across faces")


def _slack_traps(tgt, g, qry, rng, n, delta):
    """Queries whose answer only the slack protects.  A target p within a few float steps of a cell face, on the side of
    the face its coordinate lies, but binned by the float cell assignment into the cell across the face; the query delta
    from p on its own side (so one cell away from p's bin); a competitor mirrored through the query along that axis,
    nudged sideways so that its d² lies strictly between p's and the squared distance to the face.  With slack 0 the
    fine rings find the competitor in the query's cell, bound p's cell by the face and close without visiting it: the
    wrong answer.  Trap points overwrite targets that do not span the box (the count, the box and so the grid stay),
    and targets near a trap query move elsewhere in the box.  Only triples whose brute-force answer is p and on which
    the restated slack-0 search (fine_search) returns the competitor are kept.  Returns the target and the queries with
    the kept trap queries appended, and their count."""
    tgt = tgt.copy()
    lo, hi = tgt.min(0), tgt.max(0)
    cand = []
    with np.errstate(over="ignore"):
        for a in range(3):
            b = (a + 1) % 3
            for k in range(2, int(g.ext_over_e[a]) - 1):
                f = face(g, a, k)
                for s in (-1, 1):   # p below the face binned above it, or above the face binned below it
                    for j in range(1 if s > 0 else 1, 9):
                        p = np.array([F(face(g, m, int(rng.integers(2, max(3, int(g.ext_over_e[m]) - 2)))) + F(0.5 * float(g.e)))
                                      for m in range(3)], F)
                        p[a] = _ulps(f, s * j if s < 0 else j - 1)
                        raw, ex = raw_cells(g, p[None])[0, a], exact_cells(g, p[None])[0, a]
                        if raw == ex:
                            continue
                        q = p.copy()
                        q[a] = F(p[a] + F(s * delta))
                        d = F(p[a] - q[a])
                        c = q.copy()
                        c[a] = F(q[a] - d)
                        if F(q[a] - c[a]) != d:
                            break
                        gap = (float(f) - float(q[a])) ** 2 - float(d) ** 2   # face² - p², in double
                        c[b] = F(c[b] + F(math.sqrt(max(gap, 0.0) / 4.0)))
                        if (cells(g, c[None]) == cells(g, q[None])).all() and (lo < c).all() and (c < hi).all():
                            cand.append((p, q, c))
                        break
    order = rng.permutation(len(cand))
    cand = [cand[i] for i in order[:4 * n]]
    if not cand:
        return tgt, qry, 0
    span = (tgt == lo).any(1) | (tgt == hi).any(1)
    free = rng.permutation(np.flatnonzero(~span))[:2 * len(cand)]
    for m, (p, q, c) in enumerate(cand):
        tgt[free[2 * m]], tgt[free[2 * m + 1]] = p, c
    qs = np.array([q for _, q, _ in cand], F)
    keep_rows = set(free.tolist())

    def crowded(p):
        return (np.abs(p[:, None, :].astype(np.float64) - qs[None]).max(2) < 4 * delta).any(1)
    bad = np.array([i for i in np.flatnonzero(crowded(tgt)) if i not in keep_rows and not span[i]], np.int64)
    while len(bad):
        tgt[bad] = rng.uniform(lo, hi, size=(len(bad), 3)).astype(F)
        bad = bad[crowded(tgt[bad])]
    index = cell_index(g, tgt)
    bi, _ = brute_nn(qs, tgt)
    kept = [m for m in range(len(cand)) if bi[m] == free[2 * m]
            and fine_search(g, tgt, qs[m], index, slack=0.0)[:2] == (True, int(free[2 * m + 1]))][:n]
    return tgt, np.concatenate([qry, qs[kept]]), len(kept)


def _family_a():
    tgt, qry, g = _faces_case((-3.7, 1.3, 0.45), (6.1, 9.9, 4.05), 6000, 1, 1)
    m0 = len(qry)
    tgt, qry, n = _slack_traps(tgt, g, qry, np.random.default_rng(10), 24, 0.05)
    return Case("a: fine faces", "a", tgt, qry, {"binned_across": 1, "tie_across_cells": 20, "one_step_apart": 20,
                                                 "slack_traps": (m0, n, 12)})


def _family_b():
    n_hand = 24
    hi = _rounding_box(np.array((100.3, -250.7, 3.1), F), np.array((131.9, -219.2, 9.7), F), 20000, 24, 1)
    tgt, qry, g = _faces_case((100.3, -250.7, 3.1), hi, 20000 - 2 * n_hand, ICP_C, 2, n_grid=20000)
    # the handoff: lone queries in cleared regions, the nearest target at fine ring 2 or 3, a competitor at the mirrored
    # position one float step nearer or farther
    rng = np.random.default_rng(20)
    lo, hi = tgt.min(0), tgt.max(0)
    e = float(g.e)
    centres = []
    while len(centres) < n_hand:
        c = np.array([int(rng.integers(8, g.dims[0] - 8)), int(rng.integers(8, int(g.ext_over_e[1]) - 8)),
                      int(rng.integers(6, int(g.ext_over_e[2]) - 6))])
        if all(np.abs(c - cc).max() >= 12 for cc in centres):
            centres.append(c)
    centres = np.array(centres)

    def crowded(p):
        return (np.abs(cells(g, p)[:, None, :] - centres[None]).max(2) <= 5).any(1)
    bad = np.flatnonzero(crowded(tgt))
    bad = bad[(tgt[bad] != lo).any(1) & (tgt[bad] != hi).any(1)]
    while len(bad):   # move the points of the cleared regions elsewhere, so the count (and the grid) stays
        tgt[bad] = rng.uniform(lo, hi, size=(len(bad), 3)).astype(F)
        bad = bad[crowded(tgt[bad])]
    extra, hq = [], []
    for j, c in enumerate(centres):
        q = np.array([F(face(g, a, c[a]) + F(0.5 * e)) for a in range(3)], F)
        cq = cells(g, q[None])[0]
        ring, a = 2 + j % 2, j % 3
        t0 = q.copy()
        t0[a] = F(face(g, a, cq[a] + ring) + F(0.02 * e))    # inside ring `ring`
        t1 = q.copy()
        t1[a] = _ulps(F(q[a] - F(t0[a] - q[a])), (-1) ** (j // 2))   # mirrored, one float step farther or nearer
        extra += [t0, t1]
        hq.append(q)
    tgt = np.concatenate([tgt, np.array(extra, F)])
    tgt = tgt[np.random.default_rng(21).permutation(len(tgt))]
    qry = np.concatenate([qry, np.array(hq, F)])
    m0 = len(qry)
    tgt, qry, n = _slack_traps(tgt, g, qry, np.random.default_rng(22), 24, 0.08)
    return Case("b: coarse faces and the fine-to-coarse handoff", "b", tgt, qry,
                {"binned_across_coarse": 1, "tie_across_cells": 20, "ring2": 8, "ring3": 8, "slack_traps": (m0, n, 2)})


def _family_c():
    rng = np.random.default_rng(3)
    p = 0.25   # dyadic: every coordinate, difference and d² below is exact
    n = 14
    ijk = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = (ijk * p + np.array([-1.5, 2.0, 0.75])).astype(F)
    base = ijk[rng.choice(len(ijk), 3000)].astype(np.float64)
    base = base[(base < n - 1).all(1)]
    q = []
    for j, b in enumerate(base):   # edge, face and cube midpoints: 2, 4 and 8 equidistant targets
        off = np.zeros(3)
        kind = j % 3
        axes = rng.permutation(3)[:kind + 1]
        off[axes] = 0.5
        q.append((b + off) * p + np.array([-1.5, 2.0, 0.75]))
    qry = np.array(q, F)
    tgt = lat[rng.permutation(len(lat))]
    # ties between a candidate in the fine rings and one only the far path reaches: sparse dyadic pairs in a large box
    g_lo, g_hi = np.array([0.0, 0.0, 0.0], F), np.array([64.0, 64.0, 16.0], F)
    far_t, far_q = [g_lo, g_hi], []
    gg = grid(g_lo, g_hi, 2 + 2 * 40 + 2000)
    e = float(gg.e)
    for j in range(40):
        a = j % 2
        c = np.array([4 + (j % 6) * 6, 4 + (j // 6) * 4, 2]) + 0.9
        qq = (np.floor(c * e * 256) / 256).astype(F)
        D = F(np.floor(2.5 * e * 256) / 256)
        t0, t1 = qq.copy(), qq.copy()
        t0[a], t1[a] = F(qq[a] - D), F(qq[a] + D)
        far_t += [t0, t1]
        far_q.append(qq)
    fill = np.random.default_rng(30).uniform([0, 0, 12], [64, 64, 16], size=(2000, 3)).astype(F)   # keeps e small, away from the pairs
    ft = np.concatenate([np.array(far_t, F), fill])
    ft = ft[np.random.default_rng(31).permutation(len(ft))]
    return [Case("c: exact ties on a dyadic lattice", "c", tgt, qry, {"ties": (2, 4, 8)}),
            Case("c: ties between the fine rings and the far path", "c", ft, np.array(far_q, F), {"far_ties": 15})]


def _family_d():
    rng = np.random.default_rng(4)
    a = rng.uniform(0, 5, size=(50000, 3))
    b = rng.uniform(395, 400, size=(50000, 3))
    tgt = np.concatenate([a, b]).astype(F)
    tgt = tgt[rng.permutation(len(tgt))]
    qry = rng.uniform(120, 280, size=(3000, 3)).astype(F)
    return Case("d: two corner clusters, queries in the empty middle", "d", tgt, qry, {"min_coarse_ring": 3})


def _family_e():
    rng = np.random.default_rng(5)
    lo, hi = np.array([-7.3, 2.1, -0.6], F), np.array([12.9, 30.4, 5.5], F)
    tgt = rng.uniform(lo, hi, size=(8000, 3)).astype(F)
    tgt[0] = np.nan   # the lowest finite index is 1
    tgt[1], tgt[2] = lo, hi
    g = grid(lo, hi, len(tgt) - 1)
    q = []
    mid = ((lo.astype(np.float64) + hi) / 2).astype(F)
    for a in range(3):
        for side in (lo, hi):
            s = -1 if side is lo else 1
            for off in (_ulps(side[a], s) - side[a], F(s * float(g.e)), F(s * 1000.0)):
                for k in range(20):
                    p = rng.uniform(lo, hi).astype(F)
                    p[a] = F(side[a] + F(off))
                    q.append(p)
    for d in np.array([[1, 1, 1], [-1, 1, -1], [1, -1, -1], [-1, -1, 1]], np.float64):
        for k in range(20):
            q.append((mid + d * 1000.0 + rng.uniform(-5, 5, 3)).astype(F))
    over = []
    for d in np.array([[1, 0, 0], [0, -1, 0], [0, 0, 1], [1, 1, 1], [-1, -1, -1]], np.float64):
        over.append((d * 3e19).astype(F))   # (3e19)² overflows: every d² is inf
    qry = np.concatenate([np.array(q, F), np.array(over, F)])
    return Case("e: queries outside the target box", "e", tgt, qry, {"outside": len(q), "overflow": len(over)},
                double_path=False)


def _mult8_boxes():
    """Cubes [0, L]³ with 64 points, L near 1, where ext / e is within a few ulps of 8: floor(ext/e) + 1 lands on 8
    (a whole 8-cell axis) or 9 (one past: 16 cells)."""
    found = {}
    L = F(1.0)
    for _ in range(4000):
        L = _ulps(L, 1)
        g = grid((0, 0, 0), (L, L, L), 64)
        r = g.ext_over_e[0]
        k = int(math.floor(r)) + 1
        if abs(r - 8.0) < 1e-12 and k in (8, 9) and k not in found:
            found[k] = L
        if len(found) == 2:
            break
    return found


def _family_f():
    rng = np.random.default_rng(6)
    out = []
    q = rng.uniform(-3, 3, size=(400, 3)).astype(F)
    out.append(Case("f: one target point", "f", np.array([[0.5, -1.25, 2.0]], F), q, {"n_fin": 1}, double_path=False))
    same = np.tile(np.array([[1.5, 2.5, -0.5]], F), (300, 1))
    out.append(Case("f: all targets identical", "f", same, q, {"zero_extent": 3}))
    t = np.zeros((2000, 3), F)
    t[:, 0] = rng.uniform(-20, 20, 2000)
    t[:, 1], t[:, 2] = 3.0, -1.0
    out.append(Case("f: collinear targets", "f", t, rng.uniform([-25, 0, -4], [25, 6, 2], size=(2000, 3)).astype(F),
                    {"zero_extent": 2}))
    t = rng.uniform([-30, -30, 0], [30, 30, 0], size=(20000, 3)).astype(F)
    t[:, 2] = -1.8
    out.append(Case("f: coplanar targets (flat ground)", "f", t, rng.uniform([-35, -35, -3], [35, 35, 2], size=(4000, 3)).astype(F),
                    {"zero_extent": 1, "gz": 8}))
    t = (np.array([1.0, 2.0, 3.0]) + rng.uniform(0, 1e-6, size=(500, 3))).astype(F)
    out.append(Case("f: a 1e-6 m extent", "f", t, (np.array([1.0, 2.0, 3.0]) + rng.uniform(-3e-6, 4e-6, size=(1000, 3))).astype(F),
                    {"tiny": 1e-6}))
    for k, L in sorted(_mult8_boxes().items()):
        t = rng.uniform(0, float(L), size=(64, 3)).astype(F)
        t[0], t[1] = 0.0, L
        t[2:10] = np.array([[float(L) * ((j >> b) & 1) for b in range(3)] for j in range(8)], F)   # every corner, so the
        t[10:20, 0] = L                                                                           # last cell holds points
        qq = rng.uniform(-0.1, float(L) + 0.1, size=(3000, 3)).astype(F)
        out.append(Case(f"f: floor(ext/e) + 1 = {k}", "f", t, qq, {"mult8": k}))
    return out


def _family_g():
    rng = np.random.default_rng(7)
    local = rng.uniform([-10, -10, -2], [10, 10, 4], size=(20000, 3))
    out = []
    for shift, claim in (((1e4, 1e4, 1e4), "slack_from_coordinates"), ((4e5, 4e6, 10.0), "open_after_fine_rings")):
        t = (local + np.array(shift)).astype(F)
        qq = (rng.uniform([-11, -11, -3], [11, 11, 5], size=(4000, 3)) + np.array(shift)).astype(F)
        out.append(Case(f"g: local scene at {shift}", "g", t, qq, {claim: True}))
    return out


def _family_i():
    """Isolated query-target pairs whose float d² is the largest float not above (double) max_dist², and one float step
    either side."""
    md = 0.7
    M = md * md
    F0 = F(M)
    if float(F0) > M:
        F0 = _ulps(F0, -1)
    want = {-1: _ulps(F0, -1), 0: F0, 1: _ulps(F0, 1)}
    dx = F(0.6875)   # dyadic: c + dx is exact below
    sx = F(dx * dx)
    pairs = {}
    dy = F(math.sqrt(max(float(want[-1]) - float(sx), 0.0)) * 0.999)
    for _ in range(20000):
        d2 = F(F(F(dx * dx) + F(dy * dy)) + F(0))
        for k, v in want.items():
            if d2 == v and k not in pairs:
                pairs[k] = (dx, dy)
        if len(pairs) == 3:
            break
        dy = _ulps(dy, 1)
    assert len(pairs) == 3
    t, q = [], []
    for j in range(30):
        k = (-1, 0, 1)[j % 3]
        ddx, ddy = pairs[k]
        c = np.array([j * 10.0, 0.0, 0.0], F)
        t.append(c)
        q.append(np.array([F(c[0] + ddx), ddy, F(0)], F))
    qq = np.array(q, F)
    # the offsets must survive the addition to c: keep only x where c + dx - c == dx
    assert all(F(qq[j, 0] - t[j][0]) == pairs[(-1, 0, 1)[j % 3]][0] for j in range(30))
    return Case("i: the max_correspondence_distance gate", "i", np.array(t, F), qq, {"gate": (md, 10, 10, 10)}, max_dist=md,
                double_path=False)


def _knn7_clusters():
    """Isolated clusters of 2-6 points on a jittered 10 m grid, all within 0.5 m of one plane (so the fine edge is far
    below the cluster spacing): every point's 7th neighbour lies in another cluster."""
    rng = np.random.default_rng(8)
    pts = []
    for i in range(20):
        for j in range(20):
            c = np.array([10.0 * i, 10.0 * j, 0.0]) + rng.uniform([-2, -2, 0], [2, 2, 0.4])
            pts.append(c + rng.uniform(-0.05, 0.05, size=(int(rng.integers(2, 7)), 3)))
    t = np.concatenate(pts).astype(F)
    return Case("7-NN: isolated clusters of 2-6 points", "knn7", t[rng.permutation(len(t))], t[::3].copy(), {"knn7_outside": 0.5},
                knn7=True)


def _knn7_lattice():
    """A planar dyadic lattice (0.5 m pitch, 64 x 64): four equal nearest distances and two equal diagonal ones."""
    rng = np.random.default_rng(9)
    ij = np.stack(np.meshgrid(np.arange(64), np.arange(64), indexing="ij"), -1).reshape(-1, 2)
    t = np.column_stack([ij * 0.5, np.full(len(ij), 1.25)]).astype(F)
    return Case("7-NN: tie-heavy planar lattice", "knn7", t[rng.permutation(len(t))], t[::5].copy(), {"knn7_outside": 0.5},
                knn7=True)


def cases():
    """Every constructed case but the 2^24-point lattice (family h, lattice_*)."""
    return ([_family_a(), _family_b()] + _family_c() + [_family_d(), _family_e()] + _family_f() + _family_g() +
            [_family_i(), _knn7_clusters(), _knn7_lattice()])


# ------------------------------------------------------------------------------------------------ fricp's frame
def normalised_target(c):
    """The target as fricp normalises it (p / scale - mu, scale = the larger box diagonal of source and target) and its
    float rounding, the input of the index build."""
    def diag(p):
        p = p[np.isfinite(p).all(1)]
        e = [float(p[:, a].max()) - float(p[:, a].min()) for a in range(3)]
        return math.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
    scale = max(diag(c.tgt), diag(c.qry)) or 1.0
    t = c.tgt[np.isfinite(c.tgt).all(1)].astype(np.float64) / scale
    t = t - t.mean(0)
    return t, t.astype(F)


def knn7_outside_fraction(c):
    """The fraction of target points whose 7th nearest target (itself included) lies outside the 5x5x5 fine cells
    around its own cell, on the grid of the normalised target."""
    t, tf = normalised_target(c)
    g = grid_of(tf)
    cl = cells(g, tf)
    out = 0
    for b in range(0, len(t), 512):
        d = ((t[b:b + 512, None, :] - t[None, :, :]) ** 2).sum(-1)
        j7 = np.argsort(d, axis=1, kind="stable")[:, 6]
        out += int((np.abs(cl[j7] - cl[b:b + 512]).max(1) > 2).sum())
    return out / len(t)
