"""GPU test of the multi-process re-page primitives on ONE device: W = 2^k 'ranks' are W engines over external pages of the same GPU
(the peer mappings of the real thing are then plain device pointers), so the pull-mode exchange — fused into the first sweep
(k_fused_sweep<PULL>) or as the plain gather kernel — and the push kernel run in the driver's single-GPU `pytest -m gpu` pass.
The multi-process form over CUDA IPC + NCCL is tests/test_sharded_gpu.py (needs >= 2 GPUs)."""
import ctypes
import random

import numpy as np
import pytest

from qrack_b200 import _abi

import npref
import util
from test_fused_emulation import _random_gate_arrays

pytestmark = pytest.mark.gpu


def _pages(lib, n, nbytes):
    out = []
    for _ in range(n):
        p = ctypes.c_void_p()
        _abi.check(lib, lib.b200sv_alloc_page(0, nbytes, ctypes.byref(p)))
        out.append(p.value)
    return out


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("k,nl,n_gates", [(1, 16, 40), (2, 17, 70), (3, 16, 50), (3, 18, 0), (2, 15, 0)])
def test_exchange_pull_and_push_on_one_device(prec, k, nl, n_gates):
    from qrack_b200.qengine import QEngineCUDA
    lib = _abi.load()
    W = 1 << k
    rng = random.Random(31 * k + nl + prec)
    nrng = np.random.default_rng(5 * k + nl)
    cplx = np.complex64 if prec == 32 else np.complex128
    nbytes = (1 << nl) * (8 if prec == 32 else 16)
    cur, nxt, psh = _pages(lib, W, nbytes), _pages(lib, W, nbytes), _pages(lib, W, nbytes)
    host = [((nrng.standard_normal(1 << nl) + 1j * nrng.standard_normal(1 << nl)) / np.sqrt(2.0 ** (nl + 1))).astype(cplx)
            for _ in range(W)]
    eng = [QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1)) for r in range(W)]
    try:
        for r in range(W):
            eng[r].be.set_state(host[r])
            eng[r].Finish()
        lo = 1 if prec == 32 else 0
        vb = rng.sample(range(lo, nl), k)
        vbc = (ctypes.c_int * k)(*vb)
        g, o1, o2, pm, mats = _random_gate_arrays(nl, n_gates, rng)
        # --- push kernel first (into a third set of pages; the sources stay untouched) ---
        for r in range(W):
            _abi.check(lib, lib.b200sv_exchange_scatter(eng[r].be.h, k, vbc, r, (ctypes.c_void_p * W)(*psh)))
        for r in range(W):
            eng[r].Finish()
        pushed = []
        for r in range(W):
            chk = QEngineCUDA.over_buffer(psh[r], nl, 0, prec, random.Random(1))
            pushed.append(chk.be.get_state())
            del chk
        # --- pull mode: declare, queue the window's gates, read back (the flush carries the re-page) ---
        src = (ctypes.c_void_p * W)(*cur)
        for r in range(W):
            _abi.check(lib, lib.b200sv_exchange_pull(eng[r].be.h, k, vbc, r, src, ctypes.c_void_p(nxt[r])))
            if g:
                eng[r].be.apply_gates(g, o1, o2, pm, mats)
        got = [eng[r].be.get_state() for r in range(W)]
        for r in range(W):
            want = npref.exchange(host, k, vb, r)
            assert np.array_equal(pushed[r], want), ("push", r, vb)
            st = eng[r].be.stats()
            if g:
                _abi.check(lib, lib.b200sv_emulate_fused(nl, prec, g, o1, o2, pm, mats, want.ctypes.data_as(ctypes.c_void_p)))
                d = float(np.abs(got[r].astype(np.complex128) - want.astype(np.complex128)).max())
                assert d <= util.AMP_TOL[prec], ("pull + sweeps", r, vb, d)
                assert st["pull_sweeps"] == 1
            else:
                assert np.array_equal(got[r], want), ("pull as a gather", r, vb)
                assert st["pull_sweeps"] == 0
        # the sources were only read
        for r in range(W):
            chk = QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1))
            assert np.array_equal(chk.be.get_state(), host[r])
            del chk
        # a second exchange back with the same victims restores the original pages (re-page twice = identity)
        src2 = (ctypes.c_void_p * W)(*nxt)
        if not g:
            for r in range(W):
                _abi.check(lib, lib.b200sv_exchange_pull(eng[r].be.h, k, vbc, r, src2, ctypes.c_void_p(cur[r])))
            back = [eng[r].be.get_state() for r in range(W)]
            for r in range(W):
                assert np.array_equal(back[r], host[r]), ("round trip", r)
    finally:
        for e in eng:
            e.Finish()
        del eng
        for p in cur + nxt + psh:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))


def test_exchange_pull_argument_checks():
    from qrack_b200.qengine import QEngineCUDA
    lib = _abi.load()
    q = QEngineCUDA(10, 0, random.Random(1), 1.0 + 0j, False, False, deviceId=0, precision=32)
    vb = (ctypes.c_int * 1)(3)
    two = _pages(lib, 2, 8 << 10)
    try:
        src = (ctypes.c_void_p * 2)(*two)
        # an engine that owns its buffer cannot be re-paged
        assert lib.b200sv_exchange_pull(q.be.h, 1, vb, 0, src, ctypes.c_void_p(two[1])) == _abi.B200SV_EINVAL
        e = QEngineCUDA.over_buffer(two[0], 10, 0, 32, random.Random(1))
        assert lib.b200sv_exchange_pull(e.be.h, 1, vb, 0, src, ctypes.c_void_p(two[1])) == _abi.B200SV_EINVAL   # out aliases a source
        assert lib.b200sv_exchange_pull(e.be.h, 4, vb, 0, src, None) == _abi.B200SV_EINVAL
        bad = (ctypes.c_int * 1)(0)
        assert lib.b200sv_exchange_pull(e.be.h, 1, bad, 0, src, None) == _abi.B200SV_EINVAL                       # inside the 16-byte chunk / null out
        del e
    finally:
        for p in two:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))
