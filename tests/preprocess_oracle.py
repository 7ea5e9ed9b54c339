"""ctypes loader of the preprocess oracle (tests/cpp/preprocess_oracle.cpp), compiled with g++ into a temporary
directory on first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from better_fastlio2_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "preprocess_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_pp_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libpp_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                        "-I", os.path.join(ROOT, "include"), SRC, "-o", so], check=True)
        L = C.CDLL(so)
        L.orc_preprocess.argtypes = [C.POINTER(capi.PreprocessConfig), C.POINTER(capi.RawLayout), C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float)]
        _lib = L
    return _lib


def preprocess(records, cfg, layout=None):
    """The oracle's pl_surf for a numpy structured array of driver records: (xyzi (m,4), curvature (m,), last_curvature).
    Raises ValueError for a Velodyne ring >= n_scans (rc 2) or bad arguments (rc 1)."""
    rec, c, lay = capi._preprocess_args(records, cfg, layout)
    n = len(rec)
    xyzi = np.empty((max(n, 1), 4), np.float32)
    cur = np.empty(max(n, 1), np.float32)
    m, last = C.c_int(0), C.c_float(0)
    rc = lib().orc_preprocess(C.byref(c), C.byref(lay), rec.ctypes.data if n else None, n, xyzi.ctypes.data, cur.ctypes.data,
                              C.byref(m), C.byref(last))
    if rc:
        raise ValueError(f"orc_preprocess rc={rc}")
    return xyzi[:m.value].copy(), cur[:m.value].copy(), np.float32(last.value)
