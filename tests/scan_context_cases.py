"""Directed Scan Context inputs and an independent numpy restatement of SCManager::makeScancontext
(include/sc-relo/Scancontext.cpp:195-251), shared by the CPU and GPU Scan Context tests."""
import numpy as np

RINGS, SECTORS, MAX_RADIUS = 20, 60, 80.0
F = np.float32


def _up(v):
    return np.nextafter(F(v), F(np.inf))


def _down(v):
    return np.nextafter(F(v), F(-np.inf))


def edge_points(lidar_height=1.5):
    """(n,4) float32 x, y, z, intensity: the axes, signed zeros, the origin, NaN / Inf in every coordinate, the 80 m
    edge and heights at, just below and just above -1000 after adding lidar_height."""
    h = lidar_height
    z_at = F(-1000.0 - h)                    # pt.z == -1000 exactly (for the heights used here)
    rows = [
        # axes
        (5, 0, 1), (0, 5, 2), (-5, 0, 3), (0, -5, 4), (30, 0, 0.5), (0, 30, 0.25), (-30, 0, 0.75), (0, -30, 0.125),
        # signed zeros: x = -0, y > 0 is -90 degrees (sector 1); x = ±0, y = 0 is NaN (sector 1)
        (0.0, 7, 5), (-0.0, 7, 6), (0.0, -7, 7), (-0.0, -7, 8), (-0.0, 0.0, 9), (0.0, -0.0, 10), (-0.0, -0.0, 11),
        # the origin
        (0, 0, 12),
        # NaN / Inf in x, y, z
        (np.nan, 3, 13), (3, np.nan, 14), (3, 4, np.nan), (np.inf, 0, 15), (0, np.inf, 16), (-np.inf, 2, 17),
        (3, 4, np.inf), (3, 4, -np.inf), (np.nan, np.nan, 18), (np.inf, np.nan, 19),
        # 80 m exactly (kept) and one ulp above (skipped)
        (80, 0, 20), (0, -80, 21), (48, 64, 22), (-48, -64, 23), (_up(80), 0, 24), (0, -_up(80), 25),
        # heights at, below and just above -1000 once lidar_height is added
        (10, 10, z_at), (10, 10, _down(z_at)), (-10, 10, z_at), (-10, 10, _up(z_at)), (-10, -10, -5000),
        # same bin, several heights (the maximum wins whatever the order)
        (12, 1, 0.5), (12, 1.01, 2.5), (12, 1.02, 1.5),
    ]
    p = np.array([(x, y, z, i) for i, (x, y, z) in enumerate(rows)], dtype=np.float64)
    return p.astype(np.float32)


def np_scan_context(pts, lidar_height=1.5):
    """makeScancontext, restated with numpy in the reference's types (float32 point, float64 desc)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, pts.shape[1] if np.ndim(pts) == 2 else 3)
    desc = np.full((RINGS, SECTORS), -1000.0)
    if len(p) == 0:
        return np.zeros((RINGS, SECTORS))
    x, y = p[:, 0], p[:, 1]
    z = (p[:, 2].astype(np.float64) + lidar_height).astype(np.float32)
    r2d = 180 / np.pi
    with np.errstate(all="ignore"):
        rng = np.sqrt(x * x + y * y)                               # float32 products, sum and root
        ang = np.empty(len(p), np.float64)
        c1 = (x >= 0) & (y >= 0)
        c2 = (x < 0) & (y >= 0)
        c3 = (x < 0) & (y < 0)
        c4 = ~(c1 | c2 | c3)
        ang[c1] = r2d * np.arctan((y[c1] / x[c1]).astype(np.float64))
        ang[c2] = 180 - r2d * np.arctan((y[c2] / (-x[c2])).astype(np.float64))
        ang[c3] = 180 + r2d * np.arctan((y[c3] / x[c3]).astype(np.float64))
        ang[c4] = 360 - r2d * np.arctan(((-y[c4]) / x[c4]).astype(np.float64))
        ang = ang.astype(np.float32)
        ring_f = np.ceil((rng.astype(np.float64) / MAX_RADIUS) * RINGS)
        sect_f = np.ceil((ang.astype(np.float64) / 360.0) * SECTORS)
    keep = ~(rng.astype(np.float64) > MAX_RADIUS)
    # int(NaN): INT_MIN on x86, 0 on the device; either way the clamp gives 1
    ring = np.where(np.isnan(ring_f), 1, np.clip(np.nan_to_num(ring_f), 1, RINGS)).astype(int)
    sect = np.where(np.isnan(sect_f), 1, np.clip(np.nan_to_num(sect_f), 1, SECTORS)).astype(int)
    for i in np.nonzero(keep)[0]:
        r, s = ring[i] - 1, sect[i] - 1
        if desc[r, s] < z[i]:
            desc[r, s] = z[i]
    desc[desc == -1000.0] = 0.0
    return desc


def sector_key(sc):
    return sc.mean(axis=0)


def sc_distance(sc1, sc2, search_ratio=0.2):
    """SCManager::distanceBtnScanContext (Scancontext.cpp:143-181): sector-key pre-alignment, then the column-wise
    cosine distance over the shifts around it.  Returns (distance, shift)."""
    v1, v2 = sector_key(sc1), sector_key(sc2)
    diffs = [np.linalg.norm(v1 - np.roll(v2, s)) for s in range(SECTORS)]
    arg = int(np.argmin(diffs))
    radius = int(round(0.5 * search_ratio * SECTORS))
    space = sorted({(arg + d) % SECTORS for d in range(-radius, radius + 1)})
    best, best_shift = 1e7, 0
    for s in space:
        sc2s = np.roll(sc2, s, axis=1)
        n1, n2 = np.linalg.norm(sc1, axis=0), np.linalg.norm(sc2s, axis=0)
        ok = (n1 != 0) & (n2 != 0)
        sim = (sc1[:, ok] * sc2s[:, ok]).sum(axis=0) / (n1[ok] * n2[ok])
        d = 1.0 - sim.sum() / ok.sum()
        if d < best:
            best, best_shift = d, s
    return best, best_shift
