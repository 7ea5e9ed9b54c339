"""Scenario generators of the map lifecycle tests: the map driven as a node drives it for a long run, a sliding window
that inserts ahead and deletes behind, scan after scan (lasermap_fov_segment + map_incremental, laserMapping.cpp).

Every generated point keeps at least FACE_MARGIN * ds from every voxel face (tested in float64 on the float32 value), so
the device map's integer voxel keys and the reference's float box tests agree on every point (DESIGN.md §5, deviation 2).
"""
import numpy as np

from better_fastlio2_b200 import synth

DS = 0.2
FACE_MARGIN = 0.01
COARSE = 32 * DS          # a coarse cell is 8 x 8 x 8 blocks of 4 x 4 x 4 voxels: 6.4 m at ds = 0.2
BIG = 1.0e4               # "everything" along an axis a delete box does not bound


def face_ok(pts, ds=DS, margin=FACE_MARGIN):
    """Rows whose three coordinates all lie at least margin * ds from a voxel face, tested in float64 on the float32
    values against the float32 voxel size the map uses."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    f = p / np.float64(np.float32(ds))
    r = f - np.floor(f)
    return ((r >= margin) & (r <= 1.0 - margin)).all(1)


def face_filter(pts, ds=DS):
    pts = np.asarray(pts, np.float32)
    return pts[face_ok(pts, ds)]


def coarse_keys(pts, ds=DS):
    """(coarse cell, block) integer keys of each point, computed the way the device map keys them (float32 floor(x/ds))."""
    v = np.floor(np.asarray(pts, np.float32) / np.float32(ds)).astype(np.int64)
    b = v >> 2
    return b >> 3, b


def n_unique_rows(a):
    return len(np.unique(a, axis=0)) if len(a) else 0


# ---------------------------------------------------------------------------------------------- (a) sparse corridor
class Corridor:
    """Each step adds PER_STEP points, each alone in its own coarse cell of the x column `step` (an 8 x 8 grid of cells in
    y, z), and then deletes, with one half-open box, every column more than `window` steps behind.  Cells are one block
    each, so every delete empties whole coarse cells: the regime in which the coarse level only grows between rehashes."""
    PER_STEP = 64

    def __init__(self, window=8, seed=0):
        self.window = window
        self.rng = np.random.default_rng(seed)

    def points(self, step):
        j = np.arange(self.PER_STEP)
        return _one_per_cell(np.stack([np.full(self.PER_STEP, step), j % 8, j // 8], 1), self.rng)

    def delete_box(self, step):
        """Everything in the columns < step - window + 1 (None while the window is filling)."""
        cut = step - self.window + 1
        if cut <= 0:
            return None
        return np.array([-BIG, -BIG, -BIG, cut * COARSE, BIG, BIG], np.float32)

    def live_cells(self, step):
        return self.PER_STEP * min(step + 1, self.window)

    def queries(self, step, rng, n_near=256, n_far=64):
        """Near queries inside the live window and far ones tens of metres off it (no coarse cell of the map within the
        3 x 3 x 3 around them, so their search goes through every coarse cell of the map)."""
        x0 = max(0, step - self.window + 1) * COARSE
        x1 = (step + 1) * COARSE
        near = np.stack([rng.uniform(x0, x1, n_near), rng.uniform(0, 8 * COARSE, n_near), rng.uniform(0, 8 * COARSE, n_near)], 1)
        far = np.stack([rng.uniform(x0 - 20, x1 + 20, n_far), rng.uniform(-60, -30, n_far), rng.uniform(-10, 90, n_far)], 1)
        return face_filter(near.astype(np.float32)), face_filter(far.astype(np.float32))


def distinct_cells(n, seed=0):
    """n points, each alone in its own coarse cell (a 3-D grid of cells, one point per cell)."""
    side = int(np.ceil(n ** (1.0 / 3.0)))
    idx = np.arange(n)
    return _one_per_cell(np.stack([idx % side, (idx // side) % side, idx // (side * side)], 1) - side // 2,
                         np.random.default_rng(seed))


def _one_per_cell(cells, rng):
    """One random point inside each given coarse cell, away from the cell's faces and from every voxel face."""
    cells = np.asarray(cells, np.float64)
    pts = np.empty((len(cells), 3), np.float32)
    todo = np.ones(len(cells), bool)
    while todo.any():   # redraw the few points that land near a voxel face
        sel = np.nonzero(todo)[0]
        p = ((cells[sel] + rng.uniform(0.05, 0.95, (len(sel), 3))) * COARSE).astype(np.float32)
        ok = face_ok(p)
        pts[sel[ok]] = p[ok]
        todo[sel[ok]] = False
    return pts


# ---------------------------------------------------------------------------------------------- (b) driven route
class Route:
    """VLP-16 scans (every `ray_step`-th ray) along synth.trajectory_state through synth.city_world at 10 m/s, their world
    points from the true pose (face-filtered), the 0.5 m voxel-filtered cloud map_incremental would insert and a verbatim
    batch of scan points (they land in voxels that already hold a point: overflow chains form and are freed again)."""

    def __init__(self, n_steps, seed=3, ray_step=2, max_range=55.0, n_verbatim=200):
        self.n_steps = n_steps
        self.seed = seed
        self.world = synth.city_world(half_extent=n_steps * 1.0 + 2 * max_range, seed=seed)
        self.dirs = synth.lidar_dirs("vlp16")[::ray_step]
        self.max_range = max_range
        self.n_verbatim = n_verbatim

    def truth(self, k):
        return synth.trajectory_state(k)

    def step(self, k):
        """(body scan, downsampled world points, verbatim world points) of scan k, deterministic in (seed, k)."""
        rng = np.random.default_rng((self.seed, k))
        st = self.truth(k)
        body = synth.scan_from_pose(self.world, st, self.dirs, rng, max_range=self.max_range)
        world = synth.body_to_world_np(st, body)
        down = face_filter(synth.voxel_downsample(world, 0.5))
        verb = face_filter(world[rng.choice(len(world), min(self.n_verbatim, len(world)), replace=False)])
        return body, down, verb

    @staticmethod
    def pos_lid(state):
        R = synth.quat_to_mat(state[3:7])
        return state[0:3] + R @ state[11:14]

    def far_queries(self, k, rng, n=32):
        x = self.truth(k)[0]
        q = np.stack([rng.uniform(x - 40, x + 40, n), rng.choice([-1.0, 1.0], n) * rng.uniform(90, 120, n),
                      rng.uniform(-5, 60, n)], 1)
        return face_filter(q.astype(np.float32))


# ---------------------------------------------------------------------------------------------- exact k-NN reference
def brute_knn(points, queries, k=5, chunk=64):
    """Exact k-NN over `points` in float32 with the map's distance, (dx*dx + dy*dy) + dz*dz, returning for each query
    every point at a distance <= the k-th one, in the order (distance, x, y, z): (d2[nq, k], cands) with cands[i] the
    (m_i, 4) array of (d2, x, y, z) rows (m_i >= k when ties reach past the k-th)."""
    p = np.asarray(points, np.float32)
    q = np.asarray(queries, np.float32)
    d2k = np.full((len(q), k), np.inf, np.float32)
    cands = []
    for a in range(0, len(q), chunk):
        qq = q[a:a + chunk]
        d = ((p[None, :, 0] - qq[:, None, 0]) * (p[None, :, 0] - qq[:, None, 0]) +
             (p[None, :, 1] - qq[:, None, 1]) * (p[None, :, 1] - qq[:, None, 1])) + \
            (p[None, :, 2] - qq[:, None, 2]) * (p[None, :, 2] - qq[:, None, 2])
        kk = min(k, p.shape[0])
        part = np.partition(d, kk - 1, axis=1)[:, :kk]
        part.sort(axis=1)
        d2k[a:a + len(qq), :kk] = part
        for i in range(len(qq)):
            sel = np.nonzero(d[i] <= part[i, kk - 1])[0]
            rows = np.concatenate([d[i, sel][:, None], p[sel]], 1)
            rows = rows[np.lexsort((rows[:, 3], rows[:, 2], rows[:, 1], rows[:, 0]))]
            cands.append(rows)
    return d2k, cands


def assert_knn_exact(points, queries, xyz, d2, cnt, k=5):
    """A k-NN answer against brute force over the map's own content: counts and distances bit-equal, and each query's
    neighbours, in the order returned, equal the brute force's first k in the order (distance, x, y, z).  The one
    exception is a query where two DIFFERENT points lie at exactly the same float distance: the stencil pass keeps such
    ties in arrival order (TopKId in knn_kernels.cuh), so there the neighbours nearer than the shared distance must match
    in order and the tied ones must be tied points of the brute force.  Returns the number of such queries."""
    bd2, cands = brute_knn(points, queries, k)
    assert np.array_equal(cnt, np.full(len(queries), min(k, len(points)), np.int32))
    assert np.array_equal(d2, bd2), f"max |dd2| = {np.abs(d2 - bd2).max()}"
    n_tied = 0
    for i in range(len(queries)):
        got = np.concatenate([d2[i][:, None], xyz[i]], 1)
        want = cands[i]
        distinct = np.unique(want, axis=0)   # (the same point held twice is no tie: either copy is the same row)
        if len(np.unique(distinct[:, 0])) == len(distinct):
            assert np.array_equal(got, want[:k]), (i, got, want)
            continue
        n_tied += 1
        for d in np.unique(got[:, 0]):
            g, w = got[got[:, 0] == d], want[want[:, 0] == d]
            if len(np.unique(w, axis=0)) == 1 or (d < want[k - 1, 0] and len(w) == len(g) == 1):
                assert np.array_equal(g, w[:len(g)]), (i, got, want)
                continue
            for r in g:   # tied distinct points: each returned one is a tied point of the brute force, none twice
                hit = np.nonzero((w == r).all(1))[0]
                assert len(hit), (i, r, want)
                w = np.delete(w, hit[0], 0)
        assert np.array_equal(got[:, 0], want[:k, 0]), i
    return n_tied
