"""ctypes loader of the loop-closure ICP oracle (tests/cpp/icp_oracle.cpp), compiled with g++ into a temporary directory on
first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "icp_oracle.cpp")
STATES = ["NOT_CONVERGED", "ITERATIONS", "TRANSFORM", "ABS_MSE", "REL_MSE", "NO_CORRESPONDENCES"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_icp_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libicp_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_icp.argtypes = [vp, C.c_int, vp, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, vp, vp, vp, vp, vp, vp]
        L.orc_nn.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]
        _lib = L
    return _lib


def _p4(a):
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim != 2 or a.shape[1] not in (3, 4):
        raise ValueError("points must be (n,3) or (n,4) float32")
    if a.shape[1] == 3:
        a = np.ascontiguousarray(np.column_stack([a, np.zeros(len(a), np.float32)]))
    return a


def icp(src, tgt, max_correspondence_distance=200.0, max_iterations=100, transformation_epsilon=1e-6,
        euclidean_fitness_epsilon=1e-6):
    """The contract on host clouds (the source already pre-transformed).  Returns (result dict as KeyFrameStore.icp,
    corr_idx, corr_d2, log (iterations, 4): cos_angle, |t|², mse, previous mse per iteration)."""
    s, t = _p4(src), _p4(tgt)
    n = len(s)
    T = np.empty(16, np.float32)
    info = np.zeros(4, np.int32)
    fit = np.zeros(1, np.float64)
    idx = np.empty(max(n, 1), np.int32)
    d2 = np.empty(max(n, 1), np.float32)
    rows = max(int(max_iterations), 1)
    log = np.full((rows, 4), np.nan)
    lib().orc_icp(s.ctypes.data, n, t.ctypes.data, len(t), float(max_correspondence_distance), int(max_iterations),
                  float(transformation_epsilon), float(euclidean_fitness_epsilon), T.ctypes.data, info.ctypes.data, fit.ctypes.data,
                  idx.ctypes.data, d2.ctypes.data, log.ctypes.data)
    res = {"final_transformation": T.reshape(4, 4), "converged": bool(info[0]), "iterations": int(info[1]), "state": int(info[2]),
           "state_name": STATES[int(info[2])], "n_source": n, "n_target": len(t), "n_correspondences": int(info[3]),
           "fitness_score": float(fit[0])}
    return res, idx[:n].copy(), d2[:n].copy(), log[:max(int(info[1]), 0)].copy()


def nearest(q, tgt):
    """Exact 1-NN of every query under the contract's rule: (index, float d²)."""
    a, t = _p4(q), _p4(tgt)
    idx = np.empty(max(len(a), 1), np.int32)
    d2 = np.empty(max(len(a), 1), np.float32)
    lib().orc_nn(a.ctypes.data, len(a), t.ctypes.data, len(t), idx.ctypes.data, d2.ctypes.data)
    return idx[:len(a)].copy(), d2[:len(a)].copy()
