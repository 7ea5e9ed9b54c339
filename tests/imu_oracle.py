"""ctypes loader of the IMU propagation oracle (tests/cpp/imu_oracle.cpp), compiled with g++ into a temporary directory on
first use, so the repository tree is never written.  OracleImu keeps ImuProcess's persistent members in a flat array."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "imu_oracle.cpp")
_lib = None

# slots of the flat state (see the enum in imu_oracle.cpp)
S_MEAN_ACC, S_MEAN_GYR, S_COV_ACC, S_COV_GYR, S_QD, S_ANGVEL, S_ACC_S, S_LAST_IMU = 24, 27, 30, 33, 36, 48, 51, 54
S_LAST_END, S_INIT_ITER, S_NEED_INIT, S_FIRST, S_NPOSES = 61, 62, 63, 64, 65


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_imu_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libimu_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_imu_state_size.restype = C.c_int
        L.orc_imu_new.argtypes = [vp, vp]
        L.orc_imu_new.restype = None
        L.orc_imu_reset.argtypes = [vp]
        L.orc_imu_reset.restype = None
        L.orc_imu_predict.argtypes = [vp, vp, vp, vp, vp, C.c_double]
        L.orc_imu_predict.restype = None
        L.orc_imu_process.argtypes = [vp, vp, C.c_int, C.c_double, C.c_double, vp, vp, vp]
        L.orc_imu_process.restype = C.c_int
        _lib = L
    return _lib


def config_vector(T=(0, 0, 0), R=np.eye(3), gyr=(0.1,) * 3, acc=(0.1,) * 3, bias_gyr=(1e-4,) * 3, bias_acc=(1e-4,) * 3):
    return np.ascontiguousarray(np.concatenate([np.asarray(T, float), np.asarray(R, float).reshape(9), gyr, acc, bias_gyr,
                                                bias_acc]), np.float64)


def predict(x, P, q_diag, in_acc, in_gyr, dt):
    """One esekf::predict; returns new (x, P)."""
    x = np.array(x, np.float64, copy=True)
    P = np.ascontiguousarray(np.array(P, np.float64, copy=True).reshape(23, 23))
    q = np.ascontiguousarray(q_diag, np.float64)
    a = np.ascontiguousarray(in_acc, np.float64)
    g = np.ascontiguousarray(in_gyr, np.float64)
    lib().orc_imu_predict(x.ctypes.data, P.ctypes.data, q.ctypes.data, a.ctypes.data, g.ctypes.data, float(dt))
    return x, P


class OracleImu:
    def __init__(self, cfg=None):
        self.s = np.zeros(lib().orc_imu_state_size())
        c = config_vector() if cfg is None else np.ascontiguousarray(cfg, np.float64)
        lib().orc_imu_new(c.ctypes.data, self.s.ctypes.data)
        self.last_poses = np.zeros((0, 22))

    def reset(self):
        lib().orc_imu_reset(self.s.ctypes.data)

    def process(self, imu7, beg, end, state26, P):
        """Returns (status, state26, P, IMUpose)."""
        a = np.ascontiguousarray(np.asarray(imu7, np.float64).reshape(-1, 7))
        x = np.array(state26, np.float64, copy=True)
        Pm = np.ascontiguousarray(np.array(P, np.float64, copy=True).reshape(23, 23))
        poses = np.zeros((256, 22))
        st = lib().orc_imu_process(self.s.ctypes.data, a.ctypes.data if len(a) else None, len(a), float(beg), float(end),
                                   x.ctypes.data, Pm.ctypes.data, poses.ctypes.data)
        if st == 2:
            self.last_poses = poses[:int(self.s[S_NPOSES])].copy()
        return st, x, Pm, self.last_poses if st == 2 else np.zeros((0, 22))

    def info(self):
        s = self.s
        return dict(mean_acc=s[S_MEAN_ACC:S_MEAN_ACC + 3].copy(), mean_gyr=s[S_MEAN_GYR:S_MEAN_GYR + 3].copy(),
                    cov_acc=s[S_COV_ACC:S_COV_ACC + 3].copy(), cov_gyr=s[S_COV_GYR:S_COV_GYR + 3].copy(),
                    Qd=s[S_QD:S_QD + 12].copy(), angvel_last=s[S_ANGVEL:S_ANGVEL + 3].copy(),
                    acc_s_last=s[S_ACC_S:S_ACC_S + 3].copy(), last_imu=s[S_LAST_IMU:S_LAST_IMU + 7].copy(),
                    last_lidar_end_time=s[S_LAST_END], init_iter_num=int(s[S_INIT_ITER]), imu_need_init=int(s[S_NEED_INIT]),
                    b_first_frame=int(s[S_FIRST]), n_poses=int(s[S_NPOSES]))
