"""ctypes loader of the relocalisation registration oracle (tests/cpp/fricp_oracle.cpp), compiled with g++ into a temporary
directory on first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "fricp_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_fricp_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libfricp_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_fricp.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double,
                                C.c_double, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
        L.orc_se3_log.argtypes = [vp, vp]
        L.orc_se3_exp.argtypes = [vp, vp]
        L.orc_median.argtypes = [vp, C.c_int]
        L.orc_median.restype = C.c_double
        L.orc_anderson.argtypes = [C.c_int, vp, C.c_int, vp, vp, vp]
        _lib = L
    return _lib


def _p4(a):
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim != 2 or a.shape[1] not in (3, 4):
        raise ValueError("points must be (n,3) or (n,4) float32")
    if a.shape[1] == 3:
        a = np.ascontiguousarray(np.column_stack([a, np.zeros(len(a), np.float32)]))
    return a


def fricp(src, tgt, mode=4, max_icp=100, stop=1e-5, anderson_m=5, nu_begin_k=3.0, nu_end_k=1.0 / (3.0 * np.sqrt(3.0)),
          nu_alpha=0.5, norm=None, log_cap=100000):
    """The contract on host clouds (the source already pre-transformed).  norm = (scale, mu_s (3,), mu_t (3,)) replaces the
    oracle's own normalisation.  Returns (result dict with the keys of KeyFrameStore.fricp, corr, resid, log (k, 5):
    stage, energy, previous last_energy, |T - T_prev|_F, accepted)."""
    s, t = _p4(src), _p4(tgt)
    n = len(s)
    res = np.zeros(12)
    info = np.zeros(6, np.int32)
    dinfo = np.zeros(10)
    corr = np.empty(max(n, 1), np.int32)
    resid = np.empty(max(n, 1))
    log = np.zeros((max(log_cap, 1), 5))
    log_n = np.zeros(1, np.int32)
    nb = None
    if norm is not None:
        nb = np.ascontiguousarray(np.r_[norm[0], np.asarray(norm[1], float), np.asarray(norm[2], float)], np.float64)
    lib().orc_fricp(s.ctypes.data, n, t.ctypes.data, len(t), int(mode), int(max_icp), float(stop), int(anderson_m),
                    float(nu_begin_k), float(nu_end_k), float(nu_alpha), None if nb is None else nb.ctypes.data, res.ctypes.data,
                    info.ctypes.data, dinfo.ctypes.data, corr.ctypes.data, resid.ctypes.data, log.ctypes.data, int(log_cap),
                    log_n.ctypes.data)
    T = np.eye(4)
    T[:3] = res.reshape(3, 4)
    out = {"res_trans": T, "status": int(info[0]), "stages": int(info[1]), "iterations": int(info[2]),
           "rejections": int(info[3]), "n_source_finite": int(info[4]), "n_target_finite": int(info[5]), "scale": dinfo[0],
           "mu_source": dinfo[1:4].copy(), "mu_target": dinfo[4:7].copy(), "nu_begin": dinfo[7], "nu_end": dinfo[8],
           "energy": dinfo[9]}
    return out, corr[:n].copy(), resid[:n].copy(), log[:int(log_n[0])].copy()


def se3_log(T):
    """Closed-form log of a 4x4 rigid transform: the 4x4 log matrix."""
    T12 = np.ascontiguousarray(np.asarray(T, np.float64)[:3].reshape(12))
    L = np.zeros(16)
    lib().orc_se3_log(T12.ctypes.data, L.ctypes.data)
    return L.reshape(4, 4).T.copy()   # column-major in the oracle


def se3_exp(L):
    Lc = np.ascontiguousarray(np.asarray(L, np.float64).T.reshape(16))
    T12 = np.zeros(12)
    lib().orc_se3_exp(Lc.ctypes.data, T12.ctypes.data)
    T = np.eye(4)
    T[:3] = T12.reshape(3, 4)
    return T


def median(v):
    v = np.ascontiguousarray(v, np.float64)
    return lib().orc_median(v.ctypes.data, len(v))


def anderson(m, u0, ops, g):
    """Runs ops (0 compute, 1 replace, 2 reset) with the 16-vectors g[k]; returns the current u after every op."""
    u0 = np.ascontiguousarray(u0, np.float64)
    ops = np.ascontiguousarray(ops, np.int32)
    g = np.ascontiguousarray(g, np.float64).reshape(len(ops), 16)
    out = np.zeros((len(ops), 16))
    lib().orc_anderson(int(m), u0.ctypes.data, len(ops), ops.ctypes.data, g.ctypes.data, out.ctypes.data)
    return out
