"""Driver-record cases of the preprocessing contract (flb_frontend_preprocess), shared by the oracle tests on the CPU and
the device parity tests.  Each case is (records: numpy structured array in message order, cfg: preprocess_config kwargs)."""
import numpy as np

from better_fastlio2_b200 import capi, synth

VELO = synth.VELO_DTYPE
VELO_NT = synth.VELO_DTYPE_NO_TIME
OUSTER = synth.OUSTER_DTYPE
LIVOX = synth.LIVOX_DTYPE
# time field value per unit for a 0..100 ms sweep (SEC, MS, US, NS)
_UNIT = {capi.SEC: 1e-3, capi.MS: 1.0, capi.US: 1e3, capi.NS: 1e6}


def _records(dtype, xyz, **fields):
    rec = np.zeros(len(xyz), dtype)
    for k, c in enumerate("xyz"):
        rec[c] = np.asarray(xyz, np.float32)[:, k] if len(xyz) else []
    for k, v in fields.items():
        rec[k] = v
    return rec


def _spin(rng, n_rings=4, n_cols=200, step_deg=2.0, start_deg=10.0, r=(2.0, 30.0)):
    """Column-major firing of n_rings rings, azimuth decreasing by step_deg per column (clockwise)."""
    az = np.deg2rad(start_deg - np.arange(n_cols) * step_deg)
    el = np.deg2rad(np.linspace(-10, 10, n_rings))
    A, E = np.meshgrid(az, el, indexing="ij")
    rng_m = rng.uniform(*r, A.size)
    xyz = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3) * rng_m[:, None]
    ring = np.tile(np.arange(n_rings), n_cols)
    frac = np.repeat(np.arange(n_cols) / n_cols, n_rings)
    return xyz.astype(np.float32), ring, frac


def cases():
    """name -> (records, cfg)"""
    rng = np.random.default_rng(2024)
    out = {}
    xyz, ring, frac = _spin(rng)
    inten = rng.uniform(0, 255, len(xyz)).astype(np.float32)
    for unit, scale in _UNIT.items():
        t = (frac * 100.0 * scale).astype(np.float32)
        out[f"velo_time_unit{unit}"] = (_records(VELO, xyz, intensity=inten, ring=ring, time=t),
                                        dict(lidar_type=capi.VELO16, n_scans=4, time_unit=unit, blind=4.0))
        out[f"ouster_time_unit{unit}"] = (_records(OUSTER, xyz, intensity=inten, ring=ring, t=(frac * 1e8).astype(np.uint32)),
                                          dict(lidar_type=capi.OUST64, n_scans=4, time_unit=unit, blind=4.0))
    t_s = (frac * 0.1).astype(np.float32)
    for pfn in (1, 3, 4):
        out[f"velo_pfn{pfn}"] = (_records(VELO, xyz, intensity=inten, ring=ring, time=t_s),
                                 dict(lidar_type=capi.VELO16, n_scans=4, time_unit=capi.SEC, point_filter_num=pfn, blind=2.0))
        out[f"velo_notime_pfn{pfn}"] = (_records(VELO_NT, xyz, intensity=inten, ring=ring),
                                        dict(lidar_type=capi.VELO16, n_scans=4, point_filter_num=pfn, blind=2.0))
        out[f"ouster_pfn{pfn}"] = (_records(OUSTER, xyz, intensity=inten, t=(frac * 1e8).astype(np.uint32)),
                                   dict(lidar_type=capi.OUST64, n_scans=4, time_unit=capi.NS, point_filter_num=pfn, blind=2.0))
    # 200 columns x 2 deg = 400 deg: every ring's synthesised time wraps past its first point's azimuth
    out["velo_notime_wrap"] = (_records(VELO_NT, xyz, intensity=inten, ring=ring),
                               dict(lidar_type=capi.VELO16, n_scans=4, scan_rate=10, blind=0.01))
    out["velo_notime_scan_rate20_nscans8"] = (_records(VELO_NT, xyz, intensity=inten, ring=ring),
                                              dict(lidar_type=capi.VELO16, n_scans=8, scan_rate=20, blind=0.01))
    # the time field is present but the LAST record's time is 0: the times are synthesised
    t0 = t_s.copy()
    t0[-1] = 0.0
    out["velo_last_time_zero"] = (_records(VELO, xyz, intensity=inten, ring=ring, time=t0),
                                  dict(lidar_type=capi.VELO16, n_scans=4, time_unit=capi.SEC, blind=0.01))
    # a NaN return in ring 1 (column 179) just before the azimuth passes the ring's first point (column 180): the wrap
    # test compares with a NaN time_last, fails, and ring 1 never wraps afterwards
    xn = xyz.copy()
    xn[4 * 179 + 1] = np.nan
    out["velo_notime_nan_mid_ring"] = (_records(VELO_NT, xn, intensity=inten, ring=ring),
                                       dict(lidar_type=capi.VELO16, n_scans=4, blind=0.01))
    xn2 = xyz.copy()
    xn2[4 * 3 + 2, 1] = np.nan
    xn2[4 * 120 + 2] = 0.0
    out["ouster_nan_zero"] = (_records(OUSTER, xn2, intensity=inten, t=(frac * 1e8).astype(np.uint32)),
                              dict(lidar_type=capi.OUST64, n_scans=4, time_unit=capi.NS, blind=1.0))
    # points at exactly blind (3-4-0 triangle, blind 5): Velodyne drops them (r^2 > blind^2 fails), Ouster keeps them
    ex = np.array([[3, 4, 0], [0, 3, 4], [6, 0, 0], [3, 4, 0], [1, 1, 1], [0, 0, 5]], np.float32)
    out["velo_exact_blind"] = (_records(VELO, ex, intensity=np.arange(6), ring=np.zeros(6), time=np.arange(1, 7) * 1e-3),
                               dict(lidar_type=capi.VELO16, n_scans=1, time_unit=capi.SEC, blind=5.0))
    out["ouster_exact_blind"] = (_records(OUSTER, ex, intensity=np.arange(6), t=np.arange(1, 7) * 1000),
                                 dict(lidar_type=capi.OUST64, n_scans=1, time_unit=capi.NS, blind=5.0))
    out["livox_quirks"] = livox_quirks()
    lv = np.zeros(500, LIVOX)
    lv["x"] = rng.uniform(-20, 20, 500)
    lv["y"] = rng.uniform(-20, 20, 500)
    lv["z"] = rng.uniform(-2, 2, 500)
    lv["offset_time"] = np.sort(rng.integers((1 << 24) + 1, 100_000_000, 500)).astype(np.uint32)   # > 2^24: float rounds
    lv["reflectivity"] = rng.integers(0, 256, 500)
    lv["tag"] = rng.choice([0x00, 0x10, 0x20, 0x30, 0x01], 500)
    lv["line"] = rng.integers(0, 6, 500)
    for pfn in (1, 3, 4):
        out[f"livox_big_offset_time_pfn{pfn}"] = (lv, dict(lidar_type=capi.LIVOX, n_scans=4, point_filter_num=pfn, blind=10.0))
    # empty and one-record messages
    one = np.array([[5.0, -1.0, 0.5]], np.float32)
    for name, dt, cfg, extra in (("velo", VELO, dict(lidar_type=capi.VELO16, n_scans=1, time_unit=capi.SEC), dict(time=[0.01])),
                                 ("velo_notime", VELO_NT, dict(lidar_type=capi.VELO16, n_scans=1), {}),
                                 ("ouster", OUSTER, dict(lidar_type=capi.OUST64, n_scans=1, time_unit=capi.NS), dict(t=[7])),
                                 ("livox", LIVOX, dict(lidar_type=capi.LIVOX, n_scans=1), dict(offset_time=[9]))):
        out[f"{name}_empty"] = (np.zeros(0, dt), cfg)
        out[f"{name}_one"] = (_records(dt, one, **extra), cfg)
    return out


def livox_quirks():
    """Hand-made CustomMsg (n_scans 4, blind 0.5, point_filter_num 1) exercising record 0, tag/line filtering, the
    `||`/`&&` precedence of the keep test and the zero pl_full[i-1] after an unfilled record."""
    rows = [
        # x,    y,    z,   tag,  line
        (9.0, 9.0, 9.0, 0x00, 0),    # 0: never used (the loop starts at 1)
        (0.0, 0.0, 0.3, 0x00, 0),    # 1: prev = zero point (record 0 is not filled): only dz differs, inside blind -> drop
        (0.0, 0.0, 0.4, 0x10, 1),    # 2: prev = record 1 (filled): only dz differs, inside blind -> drop
        (0.1, 0.0, 0.4, 0x00, 2),    # 3: dx differs, inside blind -> KEEP (the blind cut only binds when x and y repeat)
        (0.1, 0.0, 2.0, 0x00, 3),    # 4: only dz differs, outside blind -> keep
        (0.1, 0.0, 2.0, 0x00, 3),    # 5: exact repeat -> drop
        (5.0, 5.0, 5.0, 0x20, 0),    # 6: second return (tag 0x20) -> invalid
        (5.0, 5.0, 5.0, 0x30, 0),    # 7: tag 0x30 -> invalid
        (0.1, 0.0, 2.0, 0x00, 4),    # 8: line >= n_scans -> invalid
        (0.0, 0.0, 0.2, 0x00, 0),    # 9: prev (8) unfilled -> zero point; only dz differs, inside blind -> drop
        (0.0, 0.0, 0.0, 0x00, 0),    # 10: prev = record 9 (filled): dz differs by 0.2, r = 0 -> drop
        (0.0, 0.0, 0.0, 0x11, 0),    # 11: tag & 0x30 == 0x10 with low bits set: valid; repeat -> drop
        (7.0, 0.0, 0.0, 0x04, 1),    # 12: keep
    ]
    rec = np.zeros(len(rows), LIVOX)
    for i, (x, y, z, tag, line) in enumerate(rows):
        rec[i] = (1000 * i, x, y, z, 10 + i, tag, line)
    return rec, dict(lidar_type=capi.LIVOX, n_scans=4, point_filter_num=1, blind=0.5)


def synthetic(model, with_time=True, seed=3, half_extent=100.0):
    """A full sweep of driver records from synth.driver_records and the BASELINE-like configuration of its sensor."""
    rng = np.random.default_rng(seed)
    world = synth.city_world(half_extent=half_extent, seed=seed)
    rec = synth.driver_records(model, world, synth.trajectory_state(0), rng, with_time=with_time)
    return rec, dict(SENSOR_CFG[model])


# preprocess parameters of the sensors (config/velodyne16.yaml, mulran.yaml, hap_livox.yaml; time units of the layouts)
SENSOR_CFG = {
    "vlp16": dict(lidar_type=capi.VELO16, n_scans=16, scan_rate=10, point_filter_num=4, time_unit=capi.SEC, blind=2.0),
    "hdl64": dict(lidar_type=capi.VELO16, n_scans=64, scan_rate=10, point_filter_num=1, time_unit=capi.SEC, blind=4.0),
    "os64": dict(lidar_type=capi.OUST64, n_scans=64, point_filter_num=1, time_unit=capi.NS, blind=4.0),
    "hap": dict(lidar_type=capi.LIVOX, n_scans=4, point_filter_num=3, blind=0.5),
}
