"""CPU tests of the key-frame store's C ABI: every entry point rejects null handles and invalid arguments before any
device work, without a device there is no map to create a store on (no CPU fallback), and the C++ facade compiles as
src/laserMapping.cpp would use it."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def _err(L):
    return L.flb_last_error().decode()


def test_null_handles_are_rejected(L):
    n, idx, nll = C.c_int(-7), C.c_int(-7), C.c_longlong(0)
    h = C.c_void_p(1234)
    assert L.flb_keyframes_create(None, 1000, 10, C.byref(h)) != 0 and "null" in _err(L)
    assert L.flb_keyframes_append_frontend(None, None, C.byref(idx)) != 0 and "null" in _err(L)
    assert L.flb_keyframes_append(None, None, 0, 48, 32, 36, C.byref(idx)) != 0 and "null" in _err(L)
    assert L.flb_keyframes_download(None, 0, None, None, 0, C.byref(n)) != 0 and "null" in _err(L)
    assert L.flb_keyframes_info(None, C.byref(n), C.byref(nll), C.byref(nll), C.byref(nll)) != 0 and "null" in _err(L)
    assert L.flb_map_release_keyframe_scratch(None) != 0 and "null map" in _err(L)
    assert L.flb_keyframes_size(None, 0) == -1 and "null" in _err(L)
    assert L.flb_map_reconstruct_from_keyframes(None, None, None, 0, None, C.c_float(0.2), None, 0, C.byref(n)) != 0
    assert "null" in _err(L)
    assert L.flb_keyframes_assemble(None, None, 0, 0, None, C.c_float(0.0), None, None, 0, C.byref(n)) != 0
    assert "null" in _err(L)
    assert idx.value == -7          # nothing was written on failure
    L.flb_keyframes_destroy(None)   # destroying a null handle is a no-op


def test_no_store_without_a_device(L):
    """A store needs a map, and without a CUDA device map creation fails loudly (no CPU fallback); a store cannot be
    created without a map either (test_null_handles_are_rejected)."""
    from better_fastlio2_b200 import capi
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(capi.FlbError, match="no CUDA device"):
        capi.KDTree(voxel_size=0.2)


def test_python_layer_checks_transform_shapes():
    from better_fastlio2_b200 import capi

    class _FakeStore(capi.KeyFrameStore):
        def __init__(self):
            self.h = None

        def size(self, k):
            return 3

    s = _FakeStore()
    with pytest.raises(ValueError):
        s.assemble([0, 1], poses6=[[0] * 6])             # one transform per key frame
    with pytest.raises(ValueError):
        s.assemble([0], poses6=[[0] * 6], affines=[[0] * 12])
    with pytest.raises(ValueError):
        s.reconstruct([0, 1], [[0] * 6], 0.2)


def test_header_documents_the_store():
    src = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for name in ("flb_keyframes_create", "flb_keyframes_append_frontend", "flb_keyframes_assemble",
                 "flb_map_reconstruct_from_keyframes", "FLB_KF_POSE6", "FLB_KF_AFFINE"):
        assert name in src
    for cite in ("laserMapping.cpp:756-758", "correctPoses :780-795", ":856-883"):
        assert cite in src, cite


def test_keyframe_facade_compiles(L):
    from better_fastlio2_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "keyframe_facade_smoke")
        cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", "keyframe_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
               f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "NO_GPU compile-only ok" in out.stdout or "KEYFRAME_FACADE_OK" in out.stdout
