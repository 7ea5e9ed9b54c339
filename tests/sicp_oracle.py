"""ctypes loader of the relocalisation Sparse ICP oracle (tests/cpp/sicp_oracle.cpp), compiled with g++ into a temporary
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
SRC = os.path.join(ROOT, "tests", "cpp", "sicp_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_sicp_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libsicp_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_sicp.argtypes = [vp, C.c_int, vp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int,
                               C.c_double, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
        L.orc_sicp_shrink.argtypes = [C.c_double] * 5
        L.orc_sicp_shrink.restype = C.c_double
        L.orc_sicp_thresholds.argtypes = [C.c_double, C.c_double, vp]
        L.orc_sicp_thresholds.restype = None
        _lib = L
    return _lib


def sicp(src, tgt, p=0.4, mu=10.0, alpha=1.2, max_mu=1e5, max_icp=100, max_outer=100, stop=1e-5, norm=None, log_cap=100000):
    """Sparse ICP (regMode 7) on host clouds (the source already pre-transformed).  norm = (scale, mu_s (3,), mu_t (3,))
    replaces the oracle's own normalisation.  Returns (result dict with the keys of KeyFrameStore.sicp that the oracle
    knows, corr, resid, log (k, 5): ADMM iterations, primal, dual, stop, μ at exit)."""
    s, t = _p4(src), _p4(tgt)
    n = len(s)
    res = np.zeros(12)
    info = np.zeros(5, np.int32)
    dinfo = np.zeros(11)
    corr = np.empty(max(n, 1), np.int32)
    resid = np.empty(max(n, 1))
    log = np.zeros((max(log_cap, 1), 5))
    log_n = np.zeros(1, np.int32)
    nb = None
    if norm is not None:
        nb = np.ascontiguousarray(np.r_[norm[0], np.asarray(norm[1], float), np.asarray(norm[2], float)], np.float64)
    lib().orc_sicp(s.ctypes.data, n, t.ctypes.data, len(t), float(p), float(mu), float(alpha), float(max_mu), int(max_icp),
                         int(max_outer), float(stop), None if nb is None else nb.ctypes.data, res.ctypes.data, info.ctypes.data,
                         dinfo.ctypes.data, corr.ctypes.data, resid.ctypes.data, log.ctypes.data, int(log_cap), log_n.ctypes.data)
    T = np.eye(4)
    T[:3] = res.reshape(3, 4)
    out = {"res_trans": T, "status": int(info[0]), "iterations": int(info[1]), "admm_iterations": int(info[2]),
           "n_source_finite": int(info[3]), "n_target_finite": int(info[4]), "scale": dinfo[0], "mu_source": dinfo[1:4].copy(),
           "mu_target": dinfo[4:7].copy(), "primal": dinfo[7], "dual": dinfo[8], "stop": dinfo[9], "mu_exit": dinfo[10]}
    return out, corr[:n].copy(), resid[:n].copy(), log[:int(log_n[0])].copy()


def sicp_shrink(n, mu, p, Ba, ha):
    """The factor shrink<3> multiplies Z_i by."""
    return lib().orc_sicp_shrink(float(n), float(mu), float(p), float(Ba), float(ha))


def sicp_thresholds(mu, p):
    """(Ba, ha) of shrink<3> at mu."""
    out = np.zeros(2)
    lib().orc_sicp_thresholds(float(mu), float(p), out.ctypes.data)
    return out[0], out[1]
