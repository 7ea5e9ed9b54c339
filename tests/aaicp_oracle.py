"""ctypes loader of the relocalisation AA-ICP oracle (tests/cpp/aaicp_oracle.cpp), compiled with g++ into a temporary
directory on first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from tests.fricp_oracle import _p4

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "aaicp_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_aaicp_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libaaicp_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_aaicp.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, C.c_double, C.c_double, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
        L.orc_aa_euler.argtypes = [vp, vp]
        L.orc_aa_euler.restype = None
        L.orc_aa_mat4.argtypes = [vp, vp]
        L.orc_aa_mat4.restype = None
        L.orc_aa_inv4.argtypes = [vp, vp]
        L.orc_aa_inv4.restype = None
        L.orc_aa_qr_solve.argtypes = [vp, C.c_int, vp, vp]
        _lib = L
    return _lib


def aaicp(src, tgt, max_icp=100, stop=1e-5, error_overflow_threshold=0.05, norm=None, log_cap=100000):
    """AA-ICP (regMode 1) on host clouds (the source already pre-transformed).  norm = (scale, mu_s (3,), mu_t (3,))
    replaces the oracle's own normalisation.  Returns (result dict with the keys of KeyFrameStore.aaicp that the oracle
    knows, and anderson_ms: the wall time of its Euler / QR / mixing work; corr, resid, log (k, 6): energy, prev_energy
    before the test, outcome (-1 first, 1 accepted, 0 reset), α count, stop2, smallest alphas_cond margin)."""
    s, t = _p4(src), _p4(tgt)
    n = len(s)
    res = np.zeros(12)
    info = np.zeros(7, np.int32)
    dinfo = np.zeros(9)
    corr = np.empty(max(n, 1), np.int32)
    resid = np.empty(max(n, 1))
    log = np.zeros((max(log_cap, 1), 6))
    log_n = np.zeros(1, np.int32)
    nb = None
    if norm is not None:
        nb = np.ascontiguousarray(np.r_[norm[0], np.asarray(norm[1], float), np.asarray(norm[2], float)], np.float64)
    lib().orc_aaicp(s.ctypes.data, n, t.ctypes.data, len(t), int(max_icp), float(stop), float(error_overflow_threshold),
                    None if nb is None else nb.ctypes.data, res.ctypes.data, info.ctypes.data, dinfo.ctypes.data,
                    corr.ctypes.data, resid.ctypes.data, log.ctypes.data, int(log_cap), log_n.ctypes.data)
    T = np.eye(4)
    T[:3] = res.reshape(3, 4)
    out = {"res_trans": T, "status": int(info[0]), "iterations": int(info[1]), "accepted": int(info[2]),
           "resets": int(info[3]), "history": int(info[4]), "n_source_finite": int(info[5]), "n_target_finite": int(info[6]),
           "scale": dinfo[0], "mu_source": dinfo[1:4].copy(), "mu_target": dinfo[4:7].copy(), "energy": dinfo[7], "anderson_ms": dinfo[8]}
    return out, corr[:n].copy(), resid[:n].copy(), log[:int(log_n[0])].copy()


def euler(R):
    """Matrix3::eulerAngles(0, 1, 2) of a 3x3 rotation."""
    m = np.ascontiguousarray(R, np.float64).reshape(9)
    e = np.zeros(3)
    lib().orc_aa_euler(m.ctypes.data, e.ctypes.data)
    return e


def mat4(v):
    """Vector62Matrix4: AngleAxis X * AngleAxis Y * AngleAxis Z as quaternions, the translation v[3:]."""
    a = np.ascontiguousarray(v, np.float64).reshape(6)
    T = np.zeros(16)
    lib().orc_aa_mat4(a.ctypes.data, T.ctypes.data)
    return T.reshape(4, 4)


def inv4(A):
    a = np.ascontiguousarray(A, np.float64).reshape(16)
    out = np.zeros(16)
    lib().orc_aa_inv4(a.ctypes.data, out.ctypes.data)
    return out.reshape(4, 4)


def qr_solve(A, b):
    """ColPivHouseholderQR(A).solve(b) for a 6 x n A.  Returns (x, rank)."""
    A = np.asarray(A, np.float64)
    a = np.ascontiguousarray(A.T).reshape(-1)   # column-major
    bb = np.ascontiguousarray(b, np.float64).reshape(6)
    x = np.zeros(A.shape[1])
    r = lib().orc_aa_qr_solve(a.ctypes.data, A.shape[1], bb.ctypes.data, x.ctypes.data)
    return x, r
