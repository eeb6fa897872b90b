"""The QAlu kernels (k_alu_map, k_phase_flip_if_less) and the re-page kernels (k_exchange_scatter, k_exchange_gather and the
PULL fused sweep) against the float64 NumPy reference (tests/npref.py), both precisions.

Every QAlu map is a permutation, a selection or a sign flip of the amplitudes, and a re-page is a selection, so those
results must equal the reference exactly; only the gates of a pull sweep round (REL_TOL / util.AMP_TOL).  The reference is
always fed the state read back from the engine."""
import ctypes
import random

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi

import npref
from test_kernels_vs_numpy_gpu import amp_close, rel_close

pytestmark = pytest.mark.gpu


def dense(rng, n, prec):
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def engine(n, prec, psi=None):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    if psi is not None:
        q.be.set_state(psi)
    return q


def exact(got, want, what):
    assert np.array_equal(got, want), "%s: %d amplitudes differ" % (what, int(np.sum(got != want)))


def run_alu_cases(n, prec, cases, seed):
    q = engine(n, prec, dense(np.random.default_rng(seed), n, prec))
    psi = q.be.get_state()
    for name, args in cases:
        q.be.set_state(psi)
        getattr(q.be, "alu_" + name)(*args)
        exact(q.be.get_state(), getattr(npref, name)(psi, *args), "%s%r at %dq" % (name, args[:7], n))


# ---------------------------------------------------------------------------------------------------------------
# QAlu maps
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_edge_grid(prec):
    """Every map at the edges of its arguments (npref.alu_grid): register lengths 1, 2 and n, registers at qubit 0 and at
    the top, carries and flags below and above, controls on both sides, 1- and 2-byte table entries."""
    run_alu_cases(13, prec, npref.alu_grid(13), 13 + prec)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [20, 24])
def test_qalu_wide_registers(n, prec):
    """One call per map with registers as wide as the state allows (npref.alu_wide), and the indexed maps with 2- and 3-byte
    table entries and 10 index bits.  The grid is capped at SMs x 16 blocks of 256 threads, so from 20 qubits up every
    thread loops over several amplitudes."""
    run_alu_cases(n, prec, npref.alu_wide(n), n + prec)


@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_calls_in_a_row(prec):
    """Five out-of-place maps back to back on one engine: each adopts the previous call's buffer as its output (the spare
    buffer ping-pong), with nothing read back in between."""
    n = 14
    rng = random.Random(prec)
    calls = [("rol", (3, 2, 9)),
             ("inc", (77, 1, 10, 1 << 13)),
             ("incs", (5, 0, 6, 12)),
             ("hash", (3, 9, npref._perm_table(rng, 9))),
             ("incdecc", (9, 4, 5, 0))]
    q = engine(n, prec, dense(np.random.default_rng(prec), n, prec))
    want = q.be.get_state()
    for name, args in calls:
        getattr(q.be, "alu_" + name)(*args)
        want = getattr(npref, name)(want, *args)
    exact(q.be.get_state(), want, "five calls")


@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_after_compose_and_dispose(prec):
    """Compose and Dispose change the state's size: the spare buffer of the previous map no longer fits and is replaced."""
    nrng = np.random.default_rng(3 + prec)
    q = engine(11, prec, dense(nrng, 11, prec))
    psi = q.be.get_state()
    q.be.alu_rol(4, 1, 9)
    exact(q.be.get_state(), npref.rol(psi, 4, 1, 9), "rol at 11q")
    q.Compose(engine(2, prec, dense(nrng, 2, prec)), 5)
    psi = q.be.get_state()
    assert psi.size == 1 << 13
    q.be.alu_inc(1000, 2, 11, 1)
    exact(q.be.get_state(), npref.inc(psi, 1000, 2, 11, 1), "inc after Compose")
    q.Dispose(3, 4, 9)
    psi = q.be.get_state()
    assert psi.size == 1 << 9
    table = npref._perm_table(random.Random(1), 5)
    q.be.alu_hash(4, 5, table)
    exact(q.be.get_state(), npref.hash(psi, 4, 5, table), "hash after Dispose")


@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_between_fused_gates(prec):
    """Gates queued for a fused sweep, a map, more gates: the map flushes the queue and swaps the state's buffer in the
    middle of the gate stream."""
    n = 14
    rng = random.Random(21 + prec)
    g1, g2 = npref.gate_family("full", n, rng), npref.gate_family("light", n, rng)
    q = engine(n, prec, dense(np.random.default_rng(prec), n, prec))
    psi = q.be.get_state()
    q.be.reset_stats()
    q.be.apply_gates(*npref.pack_gates(g1))
    q.be.alu_muldiv(0, 5, 8, 0, 3, 1 << 13)
    q.be.apply_gates(*npref.pack_gates(g2))
    got = q.be.get_state()
    st = q.be.stats()
    assert st["fused_sweeps"] >= 2 and st["single_launches"] == 0, st
    want = npref.apply_gates(npref.muldiv(npref.apply_gates(psi, g1, prec), 0, 5, 8, 0, 3, 1 << 13), g2, prec)
    amp_close(got, want, prec, "gates, MUL, gates")
    rel_close(got, want, prec, "gates, MUL, gates")


@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_over_an_external_buffer(prec):
    """A state over a caller's buffer keeps living there: the map's result is copied back, so a second view of the same
    buffer sees it."""
    n = 12
    lib = _abi.load()
    page = ctypes.c_void_p()
    _abi.check(lib, lib.b200sv_alloc_page(0, (1 << n) * (8 if prec == 32 else 16), ctypes.byref(page)))
    e = view = None
    try:
        e = QEngineCUDA.over_buffer(page.value, n, 0, prec, random.Random(1))
        e.be.set_state(dense(np.random.default_rng(prec), n, prec))
        psi = e.be.get_state()
        want = psi
        for name, args in (("rol", (5, 0, 12)), ("incdecsc", (6, 2, 7, 0, 1)), ("phase_flip_if_less", (40, 3, 7, -1))):
            getattr(e.be, "alu_" + name)(*args)
            e.Finish()
            want = getattr(npref, name)(want, *args)
            view = QEngineCUDA.over_buffer(page.value, n, 0, prec, random.Random(1))
            exact(view.be.get_state(), want, "%s through a second view" % name)
            view = None
        exact(e.be.get_state(), want, "the engine itself")
    finally:
        del e, view
        lib.b200sv_free_page(0, page)


@pytest.mark.parametrize("prec", [32, 64])
def test_qalu_zero_state_and_empty_registers(prec):
    """The zero state stays the zero state under every map, and a register of length 0 leaves a dense state alone."""
    n = 8
    z = engine(n, prec)
    z.be.zero()
    for name, args in npref.alu_grid(n):
        getattr(z.be, "alu_" + name)(*args)
        assert z.be.is_zero(), (name, args[:7])
    q = engine(n, prec, dense(np.random.default_rng(8), n, prec))
    psi = q.be.get_state()
    for name, args in (("rol", (3, 2, 0)), ("inc", (5, 2, 0, 0)), ("incdecc", (5, 2, 0, 1)), ("incs", (5, 2, 0, 1)),
                       ("incdecsc", (5, 2, 0, -1, 1)), ("incdecsc", (5, 2, 0, 0, 1)), ("muldiv", (0, 3, 2, 5, 0, 0)),
                       ("muldiv", (1, 3, 2, 5, 0, 0)), ("modnout", (0, 3, 5, 2, 5, 0, 0)), ("modnout", (1, 3, 5, 2, 5, 0, 0)),
                       ("modnout", (2, 3, 5, 2, 5, 0, 0)), ("hash", (2, 0, b"\x00"))):
        getattr(q.be, "alu_" + name)(*args)
        exact(q.be.get_state(), psi, "%s with length 0" % name)


def test_qalu_argument_errors():
    """Every argument check of the QAlu ABI returns B200SV_EINVAL and leaves the state as it was."""
    lib = _abi.load()
    n = 8
    q = engine(n, 64, dense(np.random.default_rng(1), n, 64))
    psi = q.be.get_state()
    h = q.be.h
    tab = bytes(8)
    bad = [
        ("rol", (1, 5, 4)), ("rol", (1, -1, 2)), ("rol", (-1, 0, 4)),
        ("inc", (1, 6, 3, 0)), ("inc", (1, 0, 3, 1 << n)),
        ("incdecc", (1, 6, 3, 0)), ("incdecc", (1, 0, 3, -1)), ("incdecc", (1, 0, 3, n)),
        ("incs", (1, 6, 3, 0)), ("incs", (1, 0, 3, -1)), ("incs", (1, 0, 3, n)),
        ("incdecsc", (1, 6, 3, -1, 0)), ("incdecsc", (1, 0, 3, -1, -1)), ("incdecsc", (1, 0, 3, -1, n)),
        ("incdecsc", (1, 0, 3, n, 4)),
        ("muldiv", (0, 3, 6, 0, 3, 0)), ("muldiv", (0, 3, 0, 6, 3, 0)), ("muldiv", (1, 3, 0, 3, 3, 1 << n)),
        ("modnout", (0, 3, 5, 6, 0, 3, 0)), ("modnout", (0, 3, 5, 0, 6, 3, 0)), ("modnout", (0, 3, 5, 0, 3, 3, 1 << n)),
        ("modnout", (-1, 3, 5, 0, 3, 3, 0)), ("modnout", (3, 3, 5, 0, 3, 3, 0)), ("modnout", (0, 3, 0, 0, 3, 3, 0)),
        ("indexed", (0, 6, 3, 0, 3, 0, 0, tab)), ("indexed", (0, 0, 3, 6, 3, 0, 0, tab)), ("indexed", (-1, 0, 3, 3, 3, 0, 0, tab)),
        ("indexed", (3, 0, 3, 3, 3, 0, 0, tab)), ("indexed", (0, 0, 3, 3, 3, 0, 0, None)),
        ("indexed", (1, 0, 3, 3, 3, -1, 0, tab)), ("indexed", (2, 0, 3, 3, 3, n, 0, tab)),
        ("hash", (6, 3, tab)), ("hash", (0, 3, None)),
        ("phase_flip_if_less", (5, 6, 3, -1)), ("phase_flip_if_less", (5, 0, 3, n)),
    ]
    for name, args in bad:
        assert getattr(lib, "b200sv_" + name)(h, *args) == _abi.B200SV_EINVAL, (name, args)
    exact(q.be.get_state(), psi, "after the refused calls")


# ---------------------------------------------------------------------------------------------------------------
# re-page: W = 2^k engines over pages of one device stand in for the ranks
# ---------------------------------------------------------------------------------------------------------------

def alloc_pages(lib, count, nbytes):
    out = []
    for _ in range(count):
        p = ctypes.c_void_p()
        _abi.check(lib, lib.b200sv_alloc_page(0, nbytes, ctypes.byref(p)))
        out.append(p.value)
    return out


def victim_classes(nl, prec):
    """page-index bits where the re-page kernels change behaviour: the lowest one allowed (the 16-byte chunk holds 2 fp32
    amplitudes), one among chunk bits 0..2, chunk bit 11 (the last bit of a 2^12-chunk tile of the fused sweep), chunk
    bit 12 (the first above it) and the top bit"""
    lo = 1 if prec == 32 else 0
    out = []
    for b in (lo, lo + 2, lo + 11, lo + 12, nl - 1):
        if b < nl and b not in out:
            out.append(b)
    return out


def victim_sets(nl, prec, k):
    """windows of k classes, together covering every class; every other window in reverse order"""
    cls = victim_classes(nl, prec)
    for j, s in enumerate(range(0, len(cls), k)):
        vb = [cls[(s + i) % len(cls)] for i in range(k)]
        yield vb[::-1] if j % 2 else vb


def host_pages(nl, prec, count, seed):
    nrng = np.random.default_rng(seed)
    return [dense(nrng, nl, prec) for _ in range(count)]


def read_page(ptr, nl, prec):
    v = QEngineCUDA.over_buffer(ptr, nl, 0, prec, random.Random(1))
    out = v.be.get_state()
    del v
    return out


def scatter_all(lib, eng, k, vb, dst):
    vbc = (ctypes.c_int * k)(*vb)
    for r, e in enumerate(eng):
        _abi.check(lib, lib.b200sv_exchange_scatter(e.be.h, k, vbc, r, (ctypes.c_void_p * len(dst))(*dst)))
    for e in eng:
        e.Finish()


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("nl", [6, 16, 0], ids=["partial_tile", "tiles", "loop_wrap"])
def test_scatter_and_gather_match_the_reference(nl, k, prec):
    """The push kernel (k_exchange_scatter) and the pull re-page without a sweep to carry it (k_exchange_gather) give
    exactly npref.exchange, for victim bits of every class, on a page below one fused-sweep tile, on several tiles, and
    at 2^23 (fp32) / 2^22 (fp64) amplitudes, where each thread's 4-chunk loop wraps."""
    nl = nl or (23 if prec == 32 else 22)
    lib = _abi.load()
    W = 1 << k
    nbytes = (1 << nl) * (8 if prec == 32 else 16)
    cur, nxt, psh = alloc_pages(lib, W, nbytes), alloc_pages(lib, W, nbytes), alloc_pages(lib, W, nbytes)
    host = host_pages(nl, prec, W, 100 * k + nl)
    try:
        for r in range(W):
            e = QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1))
            e.be.set_state(host[r])
            e.Finish()
            del e
        host = [read_page(p, nl, prec) for p in cur]
        for vb in victim_sets(nl, prec, k):
            eng = [QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1)) for r in range(W)]
            scatter_all(lib, eng, k, vb, psh)
            vbc = (ctypes.c_int * k)(*vb)
            src = (ctypes.c_void_p * W)(*cur)
            for r in range(W):
                _abi.check(lib, lib.b200sv_exchange_pull(eng[r].be.h, k, vbc, r, src, ctypes.c_void_p(nxt[r])))
            pulled = [e.be.get_state() for e in eng]
            for r in range(W):
                want = npref.exchange(host, k, vb, r)
                exact(read_page(psh[r], nl, prec), want, "scatter, rank %d, victims %r" % (r, vb))
                exact(pulled[r], want, "gather, rank %d, victims %r" % (r, vb))
                assert eng[r].be.stats()["pull_sweeps"] == 0
            del eng
            for r in range(W):
                exact(read_page(cur[r], nl, prec), host[r], "source page %d after victims %r" % (r, vb))
    finally:
        for p in cur + nxt + psh:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("k", [4, 8])
def test_scatter_to_many_pages(k, prec):
    """The push kernel takes up to k = 8 (256 destination pages, its argument block staged in shared memory)."""
    nl = 10
    lib = _abi.load()
    W = 1 << k
    nbytes = (1 << nl) * (8 if prec == 32 else 16)
    lo = 1 if prec == 32 else 0
    vb = random.Random(k + prec).sample(range(lo, nl), k)
    cur, psh = alloc_pages(lib, W, nbytes), alloc_pages(lib, W, nbytes)
    host = host_pages(nl, prec, W, k + prec)
    eng = []
    try:
        for r in range(W):
            eng.append(QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1)))
            eng[r].be.set_state(host[r])
        scatter_all(lib, eng, k, vb, psh)
        for r in range(W):
            exact(read_page(psh[r], nl, prec), npref.exchange(host, k, vb, r), "rank %d, victims %r" % (r, vb))
    finally:
        del eng
        for p in cur + psh:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))


def test_scatter_rejects_a_rank_outside_the_exchange():
    lib = _abi.load()
    nl, k = 8, 2
    pages = alloc_pages(lib, 5, (1 << nl) * 8)
    try:
        e = QEngineCUDA.over_buffer(pages[4], nl, 0, 32, random.Random(1))
        e.be.set_state(dense(np.random.default_rng(1), nl, 32))
        vb = (ctypes.c_int * k)(3, 5)
        dst = (ctypes.c_void_p * 4)(*pages[:4])
        for rank in (-1, 4, 7):
            assert lib.b200sv_exchange_scatter(e.be.h, k, vb, rank, dst) == _abi.B200SV_EINVAL, rank
        assert lib.b200sv_exchange_scatter(e.be.h, k, vb, 3, dst) == _abi.B200SV_OK
        e.Finish()
        del e
    finally:
        for p in pages:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("family", ["light", "rotation", "full"])
@pytest.mark.parametrize("path", ["staged", "direct"])
@pytest.mark.parametrize("nl,k", [(13, 1), (16, 2)])
def test_pull_sweep_matches_the_reference(nl, k, path, family, prec):
    """A pull re-page carried by the first fused sweep (k_fused_sweep<..., PULL>), then the gates of the window, against
    npref.apply_gates(npref.exchange(...)).  npref.pull_gate_lists gives one list whose first pass stages its tiles through
    shared memory (stage_in_pull) and one whose first pass loads straight from the source pages (pull_src);
    test_npref_pin.py checks on the planner's listing that each takes its path."""
    lib = _abi.load()
    W = 1 << k
    lo = 1 if prec == 32 else 0
    vb = [lo + 12, lo + 2] if k == 2 else [nl - 1 if path == "staged" else lo]
    gates = npref.pull_gate_lists(family, nl, prec)[0 if path == "staged" else 1]
    nbytes = (1 << nl) * (8 if prec == 32 else 16)
    cur, nxt = alloc_pages(lib, W, nbytes), alloc_pages(lib, W, nbytes)
    host = host_pages(nl, prec, W, nl + k + prec)
    eng = []
    try:
        for r in range(W):
            eng.append(QEngineCUDA.over_buffer(cur[r], nl, 0, prec, random.Random(1)))
            eng[r].be.set_state(host[r])
            eng[r].Finish()
        host = [e.be.get_state() for e in eng]
        vbc = (ctypes.c_int * k)(*vb)
        src = (ctypes.c_void_p * W)(*cur)
        packed = npref.pack_gates(gates)
        for r in range(W):
            eng[r].be.reset_stats()
            _abi.check(lib, lib.b200sv_exchange_pull(eng[r].be.h, k, vbc, r, src, ctypes.c_void_p(nxt[r])))
            eng[r].be.apply_gates(*packed)
        got = [e.be.get_state() for e in eng]
        for r in range(W):
            assert eng[r].be.stats()["pull_sweeps"] == 1
            want = npref.apply_gates(npref.exchange(host, k, vb, r), gates, prec)
            what = "%s %s, rank %d, victims %r" % (family, path, r, vb)
            amp_close(got[r], want, prec, what)
            rel_close(got[r], want, prec, what)
    finally:
        del eng
        for p in cur + nxt:
            lib.b200sv_free_page(0, ctypes.c_void_p(p))
