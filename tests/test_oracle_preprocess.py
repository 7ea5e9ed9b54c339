"""CPU tests of the preprocessing contract (flb_frontend_preprocess): the C++ oracle (tests/cpp/preprocess_oracle.cpp)
against an independent plain-Python transliteration of Preprocess::process (src/preprocess.cpp, feature extraction off)
that uses math.atan2 and np.float32 scalars; the C-ABI argument checks, which run before any device work; the struct
layouts against their ctypes mirrors; and a compile of the preprocess facade smoke."""
import ctypes
import math
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from better_fastlio2_b200 import capi
from tests import preprocess_cases as pc
from tests import preprocess_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


# ------------------------------------------------------------------------------------------------ transliteration
class _Rec:
    def __init__(self, records, lay):
        self.b = np.ascontiguousarray(records).tobytes()
        self.lay = lay

    def get(self, i, field, fmt):
        off = getattr(self.lay, "off_" + field)
        if off < 0:
            return 0
        return struct.unpack_from("<" + fmt, self.b, i * self.lay.stride + off)[0]


def _scale(unit):
    return {0: f32(1e3), 1: f32(1.0), 2: f32(1e-3), 3: f32(1e-6)}.get(unit, f32(1.0))


def transliterate(records, cfg):
    """pl_surf as a list of (x, y, z, intensity, curvature) np.float32 tuples; raises IndexError for ring >= n_scans."""
    c = capi.preprocess_config(**cfg)
    lay = capi.raw_layout(records.dtype)
    r = _Rec(records, lay)
    n = len(records)
    out = []
    blind2 = c.blind * c.blind
    with np.errstate(all="ignore"):
        if c.lidar_type == capi.LIVOX:
            full = [(f32(0), f32(0), f32(0))] * n
            valid_num = 0
            for i in range(1, n):
                tag = r.get(i, "tag", "B")
                if r.get(i, "line", "B") < c.n_scans and ((tag & 0x30) == 0x10 or (tag & 0x30) == 0x00):
                    valid_num += 1
                    if valid_num % c.point_filter_num == 0:
                        x, y, z = (f32(r.get(i, k, "f")) for k in "xyz")
                        full[i] = (x, y, z)
                        px, py, pz = full[i - 1]
                        r2 = x * x + y * y + z * z
                        if (float(abs(x - px)) > 1e-7 or float(abs(y - py)) > 1e-7
                                or (float(abs(z - pz)) > 1e-7 and float(r2) > blind2)):
                            out.append((x, y, z, f32(r.get(i, "intensity", "B")), f32(r.get(i, "time", "I")) / f32(1e6)))
        elif c.lidar_type == capi.OUST64:
            for i in range(n):
                if i % c.point_filter_num != 0:
                    continue
                x, y, z = (f32(r.get(i, k, "f")) for k in "xyz")
                if float(x * x + y * y + z * z) < blind2:
                    continue
                out.append((x, y, z, f32(r.get(i, "intensity", "f")), f32(r.get(i, "time", "I")) * _scale(c.time_unit)))
        else:
            if n == 0:
                return out
            omega = 0.361 * c.scan_rate
            given = f32(r.get(n - 1, "time", "f")) > 0
            first = [True] * c.n_scans
            yaw_fp = [0.0] * c.n_scans
            time_last = [f32(0)] * c.n_scans
            for i in range(n):
                x, y, z = (f32(r.get(i, k, "f")) for k in "xyz")
                cur = f32(r.get(i, "time", "f")) * _scale(c.time_unit)
                if not given:
                    layer = r.get(i, "ring", "H")
                    if layer >= c.n_scans:
                        raise IndexError(layer)
                    yaw = math.atan2(float(y), float(x)) * 57.2957
                    if first[layer]:
                        first[layer] = False
                        yaw_fp[layer] = yaw
                        time_last[layer] = f32(0)
                        continue
                    cur = f32((yaw_fp[layer] - yaw) / omega) if yaw <= yaw_fp[layer] else f32((yaw_fp[layer] - yaw + 360.0) / omega)
                    if cur < time_last[layer]:
                        cur = f32(float(cur) + 360.0 / omega)
                    time_last[layer] = cur
                if i % c.point_filter_num == 0 and float(x * x + y * y + z * z) > blind2:
                    out.append((x, y, z, f32(r.get(i, "intensity", "f")), cur))
    return out


def bits_equal(a, b):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


CASES = pc.cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_transliteration(name):
    rec, cfg = CASES[name]
    ref = transliterate(rec, cfg)
    xyzi, cur, last = po.preprocess(rec, cfg)
    assert len(xyzi) == len(ref)
    if ref:
        t = np.array(ref, np.float32)
        assert bits_equal(xyzi, t[:, :4]) and bits_equal(cur, t[:, 4])
        assert bits_equal(last, t[-1, 4])
    else:
        assert last == 0


def test_case_properties():
    """The cases exercise what they are named after."""
    def run(name):
        return po.preprocess(*CASES[name])
    # Velodyne without time: the first record of each of the 4 rings is dropped, times wrap once per ring
    xyzi, cur, _ = run("velo_notime_wrap")
    assert len(xyzi) == len(CASES["velo_notime_wrap"][0]) - 4
    assert (cur >= 0).all() and cur.max() > 360.0 / (0.361 * 10) * 0.99
    first = CASES["velo_notime_wrap"][0][:4]
    assert not any((xyzi[:, 0] == p["x"]).any() for p in first)
    # last time 0 -> synthesised (not the field's 0..0.1 s * 1e3)
    _, cur, _ = run("velo_last_time_zero")
    assert cur.max() > 100.0
    # NaN record 717 in ring 1: dropped by the blind test (NaN > blind^2 is false) but its NaN time_last stops ring 1's
    # wrap; records 796 / 797 (rings 0 / 1 of the last column) are outputs 791 / 792 after the 4 ring heads and the NaN
    _, cur, _ = run("velo_notime_nan_mid_ring")
    assert len(cur) == 800 - 5 and not np.isnan(cur).any()
    assert cur[791] > 99.0 and cur[792] < 20.0
    # exact blind: Velodyne drops the r == blind points, Ouster keeps them
    v, _, _ = run("velo_exact_blind")
    o, _, _ = run("ouster_exact_blind")
    assert len(v) == 1 and len(o) == 5
    # Ouster keeps NaN returns, drops zero returns
    o, _, _ = run("ouster_nan_zero")
    assert np.isnan(o[:, 1]).sum() == 1 and not (o[:, :3] == 0).all(1).any()
    # Livox: exactly records 3, 4 and 12 survive
    xyzi, cur, last = run("livox_quirks")
    assert np.array_equal(xyzi[:, 3], np.array([13, 14, 22], np.float32))
    assert np.array_equal(cur, np.array([3000, 4000, 12000], np.float32) / np.float32(1e6)) and last == cur[-1]
    # offset_time > 2^24 rounds to float before the division
    rec, cfg = CASES["livox_big_offset_time_pfn1"]
    _, cur, _ = po.preprocess(rec, cfg)
    assert (cur > 16.77e-3).all()
    assert len(run("velo_notime_one")[0]) == 0 and len(run("velo_one")[0]) == 1 and len(run("livox_one")[0]) == 0
    for s in ("velo", "velo_notime", "ouster", "livox"):
        assert len(run(f"{s}_empty")[0]) == 0


def test_ring_out_of_range_rejected_by_oracle():
    rec, cfg = CASES["velo_notime_wrap"]
    with pytest.raises(ValueError):
        po.preprocess(rec, dict(cfg, n_scans=3))
    with pytest.raises(IndexError):
        transliterate(rec, dict(cfg, n_scans=3))
    # with per-point time the ring is never read
    rec, cfg = CASES["velo_pfn1"]
    assert len(po.preprocess(rec, dict(cfg, n_scans=1))[0]) > 0


@pytest.mark.parametrize("model,with_time", [("vlp16", True), ("vlp16", False), ("os64", True), ("hap", True)])
def test_oracle_on_synthetic_sweeps(model, with_time):
    rec, cfg = pc.synthetic(model, with_time=with_time, half_extent=60.0)
    rec = rec[:6000]
    ref = np.array(transliterate(rec, cfg), np.float32).reshape(-1, 5)
    xyzi, cur, last = po.preprocess(rec, cfg)
    assert len(xyzi) == len(ref) > 100
    assert bits_equal(xyzi, ref[:, :4]) and bits_equal(cur, ref[:, 4])


# ------------------------------------------------------------------------------------------------ C ABI, no GPU
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    L = ctypes.CDLL(capi.LIB_PATH)
    L.flb_last_error.restype = ctypes.c_char_p
    vp, ip = ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)
    L.flb_frontend_preprocess.argtypes = [vp, ctypes.POINTER(capi.PreprocessConfig), ctypes.POINTER(capi.RawLayout), vp,
                                          ctypes.c_int, ip, ctypes.POINTER(ctypes.c_float)]
    return L


def test_preprocess_rejects_bad_arguments(lib):
    """Argument validation runs before any device work; with a null front end the first argument problem is reported."""
    rec = np.zeros(8, pc.VELO)
    good_cfg = dict(lidar_type=capi.VELO16, n_scans=16)

    def call(cfg=good_cfg, lay=None, n=8, records=rec, handle=None):
        c = capi.preprocess_config(**cfg) if cfg is not None else None
        L = lay if lay is not None else capi.raw_layout(pc.VELO)
        n_out, last = ctypes.c_int(-5), ctypes.c_float(-5)
        rc = lib.flb_frontend_preprocess(handle, ctypes.byref(c) if c is not None else None, ctypes.byref(L),
                                         records.ctypes.data if records is not None else None, n, ctypes.byref(n_out),
                                         ctypes.byref(last))
        return rc, lib.flb_last_error().decode()

    def lay(**kw):
        L = capi.raw_layout(pc.VELO)
        for k, v in kw.items():
            setattr(L, k, v)
        return L

    rc, msg = call()
    assert rc != 0 and "null front end" in msg
    for cfg, what in ((dict(good_cfg, lidar_type=0), "lidar_type"), (dict(good_cfg, lidar_type=4), "lidar_type"),
                      (dict(good_cfg, point_filter_num=0), "point_filter_num"), (dict(good_cfg, n_scans=0), "n_scans")):
        rc, msg = call(cfg=cfg)
        assert rc != 0 and what in msg, msg
    rc, msg = call(cfg=None)
    assert rc != 0 and "null config" in msg
    for L, what in ((lay(off_x=-1), "field x is required"), (lay(off_z=-1), "field z is required"),
                    (lay(off_time=19), "field time"), (lay(off_ring=21), "field ring"), (lay(off_intensity=20), "intensity"),
                    (lay(stride=0), "stride")):
        rc, msg = call(lay=L)
        assert rc != 0 and what in msg, msg
    rc, msg = call(records=None)
    assert rc != 0 and "null records" in msg
    rc, msg = call(n=-1)
    assert rc != 0 and "records" in msg
    # a Livox reflectivity is one byte: offset stride-1 is inside the record
    lv = capi.raw_layout(pc.LIVOX)
    lv.off_intensity = 19
    rc, msg = call(cfg=dict(lidar_type=capi.LIVOX, n_scans=4), lay=lv, records=np.zeros(8, pc.LIVOX))
    assert "null front end" in msg
    lv.off_line = 20
    rc, msg = call(cfg=dict(lidar_type=capi.LIVOX, n_scans=4), lay=lv, records=np.zeros(8, pc.LIVOX))
    assert "field line" in msg


def test_preprocess_structs_match_header():
    prog = r'''
#include <stddef.h>
#include <stdio.h>
#include "fastlio_b200.h"
int main(){printf("%zu %zu %zu %zu %zu %zu\n", sizeof(flb_preprocess_config), sizeof(flb_raw_layout),
 offsetof(flb_preprocess_config, time_unit), offsetof(flb_preprocess_config, blind), offsetof(flb_raw_layout, off_ring),
 offsetof(flb_raw_layout, off_line));return 0;}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    P, R = capi.PreprocessConfig, capi.RawLayout
    mine = [ctypes.sizeof(P), ctypes.sizeof(R), P.time_unit.offset, P.blind.offset, R.off_ring.offset, R.off_line.offset]
    assert got == mine, (got, mine)


def build_facade_smoke(out_dir):
    """g++ build of tests/cpp/preprocess_facade_smoke.cpp against the library (the header needs neither ROS nor PCL)."""
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    libdir = os.path.dirname(capi.LIB_PATH)
    exe = os.path.join(out_dir, "preprocess_facade_smoke")
    cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "preprocess_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
           f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_preprocess_facade_compiles():
    with tempfile.TemporaryDirectory() as d:
        exe = build_facade_smoke(d)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, (out.stdout, out.stderr)
        assert "NO_GPU compile-only ok" in out.stdout or "PREPROCESS_FACADE_OK" in out.stdout
