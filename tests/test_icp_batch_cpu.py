"""CPU tests of the inter-session registration (flb_keyframes_icp_batch): argument checking before any device work, with
the error naming the pair and the field; the stats struct's layout; the header's documentation; and the C++ facade
compiled as the multi-session mapper would use it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from better_fastlio2_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return capi.lib()


def test_stats_layout_matches_the_c_compiler():
    from better_fastlio2_b200 import capi
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "fastlio_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu\n", sizeof(flb_icp_batch_stats), offsetof(flb_icp_batch_stats, rounds),
         offsetof(flb_icp_batch_stats, setup_syncs), offsetof(flb_icp_batch_stats, iteration_syncs));
  return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "layout.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "layout")
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    s = capi.IcpBatchStats
    assert got == [C.sizeof(s), s.rounds.offset, s.setup_syncs.offset, s.iteration_syncs.offset]


def test_invalid_arguments_are_rejected_with_a_message(L):
    """Every check that needs no store runs before the store is touched: a null store behind otherwise valid arguments
    reaches the store check last, so each earlier message proves its check came first.  The ids' range needs a store and
    is checked on the GPU (tests/test_gpu_icp_batch.py)."""
    from better_fastlio2_b200 import capi
    p = capi._p
    off = np.array([0, 1, 2], np.int32)
    ids = np.array([0, 1], np.int32)
    p6 = np.zeros(12, np.float32)
    good = capi.IcpConfig(30.0, 10, 1e-6, 1e-6)
    res = (capi.IcpResult * 2)()
    res[0].iterations = 77
    st = capi.IcpBatchStats(5, 6, 7)

    def cfg(**kw):
        c = capi.IcpConfig(30.0, 10, 1e-6, 1e-6)
        for k, v in kw.items():
            setattr(c, k, v)
        return C.byref(c)

    f = L.flb_keyframes_icp_batch
    g, s = C.byref(good), C.byref(st)

    def call(n=2, so=off, si=ids, sp=p6, to=off, ti=ids, tp=p6, leaf=0.2, c=g, o=res):
        return f(None, n, p(so), p(si), p(sp), p(to), p(ti), p(tp), leaf, c, o, s)

    cases = [
        (lambda: call(n=-1), "negative n_pairs"),
        (lambda: call(o=None), "null result"),
        (lambda: call(c=None), "null config"),
        (lambda: call(c=cfg(max_iterations=-1)), "max_iterations >= 0"),
        (lambda: call(c=cfg(max_correspondence_distance=-1.0)), "max_correspondence_distance >= 0"),
        (lambda: call(c=cfg(transformation_epsilon=float("inf"))), "finite"),
        (lambda: call(c=cfg(euclidean_fitness_epsilon=float("nan"))), "finite"),
        (lambda: call(leaf=-0.1), "leaf_size must be finite and >= 0"),
        (lambda: call(leaf=float("nan")), "leaf_size must be finite and >= 0"),
        (lambda: call(leaf=float("inf")), "leaf_size must be finite and >= 0"),
        (lambda: call(so=None), "null src_offsets"),
        (lambda: call(to=None), "null tgt_offsets"),
        (lambda: call(so=np.array([1, 1, 2], np.int32)), "src_offsets[0] is 1, must be 0"),
        (lambda: call(to=np.array([0, 2, 1], np.int32)), "pair 1: tgt_offsets decrease (1 after 2)"),
        (lambda: call(si=None), "null src_ids or src_poses6"),
        (lambda: call(tp=None), "null tgt_ids or tgt_poses6"),
        (lambda: call(sp=np.r_[np.zeros(6), [0, 0, np.nan, 0, 0, 0]].astype(np.float32)), "pair 1: src_poses6 entry 1 is not finite"),
        (lambda: call(tp=np.r_[[np.inf], np.zeros(11)].astype(np.float32)), "pair 0: tgt_poses6 entry 0 is not finite"),
        (lambda: call(), "null key-frame store"),
    ]
    for fn, msg in cases:
        assert fn() != 0
        assert msg in L.flb_last_error().decode(), (msg, L.flb_last_error().decode())
    assert res[0].iterations == 77 and (st.rounds, st.setup_syncs, st.iteration_syncs) == (5, 6, 7)   # nothing written
    # n_pairs == 0 does nothing, whatever else is passed
    assert f(None, 0, None, None, None, None, None, None, -1.0, None, None, s) == 0
    assert (st.rounds, st.setup_syncs, st.iteration_syncs) == (0, 0, 0)


def test_python_layer_checks_pose_shapes():
    from better_fastlio2_b200 import capi

    class _FakeStore(capi.KeyFrameStore):
        def __init__(self):
            self.h = None

    s = _FakeStore()
    with pytest.raises(ValueError):
        s.icp_batch([([0, 1], [[0] * 6], [0], [[0] * 6])])
    with pytest.raises(ValueError):
        s.icp_batch([([0], [[0] * 6], [0, 1], [[0] * 6])])


def test_header_documents_icp_batch():
    src = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for name in ("flb_keyframes_icp_batch", "flb_icp_batch_stats", "rounds", "setup_syncs", "iteration_syncs", "2^27"):
        assert name in src, name


def test_icp_batch_facade_compiles_and_fails_loudly_without_a_gpu(L):
    from better_fastlio2_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "icp_batch_facade_smoke")
        cmd = ["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", "icp_batch_facade_smoke.cpp"), "-L", libdir, "-lfastlio_b200",
               f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    if capi.device_count() > 0:
        assert out.returncode == 0 and "ICP_BATCH_FACADE_OK" in out.stdout, (out.returncode, out.stdout, out.stderr)
    else:   # no device: the store cannot be attached, and the facade says so on stderr
        assert out.returncode == 2 and "NO_GPU" in out.stdout and "KeyFrameStore::attach" in out.stderr, (out.stdout, out.stderr)
