"""ctypes loader of the camera-colour / IMU-frame publishing oracle (tests/cpp/color_oracle.cpp), compiled with g++ into a
temporary directory on first use, so the repository tree is never written."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "color_oracle.cpp")
W_MAX, H_MAX = 1280, 720   # the reference's Wmax x Hmax
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="flb_color_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libcolor_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.orc_projection.argtypes = [vp, vp, vp]
        L.orc_projection.restype = None
        L.orc_colorize.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
        L.orc_colorize.restype = C.c_int
        L.orc_to_imu.argtypes = [vp, C.c_int, vp, vp]
        L.orc_to_imu.restype = None
        L.orc_copy_image.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp]
        L.orc_copy_image.restype = None
        _lib = L
    return _lib


def _p4(a):
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim != 2 or a.shape[1] not in (3, 4):
        raise ValueError("points must be (n,3) or (n,4) float32")
    if a.shape[1] == 3:
        a = np.ascontiguousarray(np.column_stack([a, np.zeros(len(a), np.float32)]))
    return a


def projection(cam_ex, cam_in):
    ex = np.ascontiguousarray(cam_ex, np.float64).reshape(16)
    ki = np.ascontiguousarray(cam_in, np.float64).reshape(12)
    M = np.empty(12, np.float64)
    lib().orc_projection(ex.ctypes.data, ki.ctypes.data, M.ctypes.data)
    return M.reshape(3, 4)


def colorize(cam_ex, cam_in, img, pts, state26, width=W_MAX, height=H_MAX):
    """The contract on a host cloud: (world xyzi (k,4) float32, bgra (k,) uint32, source indices (k,) int32).
    img: (height, width, 3) uint8, or None for the all-zero image."""
    ex = np.ascontiguousarray(cam_ex, np.float64).reshape(16)
    ki = np.ascontiguousarray(cam_in, np.float64).reshape(12)
    im = np.zeros((height, width, 3), np.uint8) if img is None else np.ascontiguousarray(img[:height, :width], np.uint8)
    assert im.shape == (height, width, 3)
    p = _p4(pts)
    st = np.ascontiguousarray(state26, np.float64)
    n = len(p)
    xyzi = np.empty((max(n, 1), 4), np.float32)
    bgra = np.empty(max(n, 1), np.uint32)
    idx = np.empty(max(n, 1), np.int32)
    k = lib().orc_colorize(ex.ctypes.data, ki.ctypes.data, width, height, im.ctypes.data, p.ctypes.data, n, st.ctypes.data,
                           xyzi.ctypes.data, bgra.ctypes.data, idx.ctypes.data)
    return xyzi[:k].copy(), bgra[:k].copy(), idx[:k].copy()


def to_imu(pts, state26):
    p = _p4(pts)
    st = np.ascontiguousarray(state26, np.float64)
    out = np.empty((max(len(p), 1), 4), np.float32)
    lib().orc_to_imu(p.ctypes.data, len(p), st.ctypes.data, out.ctypes.data)
    return out[:len(p)].copy()


def forward_camera(fx=900.0, fy=900.0, width=W_MAX, height=H_MAX, t=(0.0, 0.0, 0.0)):
    """A camera looking along lidar +x: the extrinsic maps lidar (x, y, z) to camera (−y, −z, x) + t; the intrinsic has
    its principal point at the image centre.  Returns (cam_ex 16, cam_in 12) row-major."""
    ex = np.array([[0, -1, 0, t[0]], [0, 0, -1, t[1]], [1, 0, 0, t[2]], [0, 0, 0, 1]], np.float64)
    ki = np.array([[fx, 0, width / 2.0, 0], [0, fy, height / 2.0, 0], [0, 0, 1, 0]], np.float64)
    return ex.reshape(-1), ki.reshape(-1)
