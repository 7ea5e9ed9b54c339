"""ctypes loader of the Scan Context oracle (tests/cpp/scan_context_oracle.cpp), compiled with g++ into a temporary
directory on first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "scan_context_oracle.cpp")
RINGS, SECTORS = 20, 60
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_sc_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libsc_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        L.orc_scan_context.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def scan_context(pts, lidar_height=1.5):
    """makeScancontext of an (n,3) or (n,4) float32 cloud: (desc (20,60) float64, sensitive (n,) bool per point,
    mask (20,60) bool of the bins an atan-sensitive point could reach)."""
    p = np.ascontiguousarray(pts, np.float32)
    n = len(p)
    stride = p.shape[1] if p.ndim == 2 else 3
    desc = np.empty((RINGS, SECTORS), np.float64)
    sens = np.zeros(max(n, 1), np.uint8)
    mask = np.zeros((RINGS, SECTORS), np.uint8)
    rc = lib().orc_scan_context(p.ctypes.data if n else None, n, stride, float(lidar_height), desc.ctypes.data, sens.ctypes.data,
                                mask.ctypes.data)
    if rc:
        raise ValueError(f"orc_scan_context rc={rc}")
    return desc, sens[:n].astype(bool), mask.astype(bool)
