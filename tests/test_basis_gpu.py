"""The per-qubit-basis moments sweep on the GPU (b200sv_moments_basis) against the float64 NumPy reference
(tests/npref_basis.py) at the shapes where its code path changes, its argument errors, what it leaves alone (the state, the
memoised marginals), the mirror's ExpVarUnitaryAll against the compiled reference's fixtures (values and the U3-form
post-state) and its gate route past 12 qubits, and the C++ drop-in against the same fixtures.

NumPy is fed the state the kernel read, read back in the engine's precision.  Every product and sum of the kernel is in double,
so only the order of the operations differs from NumPy: the bar is 1e-12 of each output's scale."""
import ctypes
import math
import os
import random
import subprocess

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi, qscript

import npref_basis as nb
import oracle_observables
import test_basis_cpu as tcpu
import util

pytestmark = pytest.mark.gpu

TOL = 1e-12


def engine(n, prec, psi=None, normalize=False):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    if psi is not None:
        q.SetQuantumState(psi)
    return q


def dense(n, prec, seed=0):
    rng = np.random.default_rng(1000 * n + seed)
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def rand_mats(rng, k):
    return [np.eye(2) + 0.7 * (rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2))) for _ in range(k)]


def check(q, bits, mats, weights, center, what=""):
    psi = q.be.get_state()
    got = q.be.moments_basis(bits, [m.reshape(-1).tolist() for m in mats], weights, center)
    want, scale = nb.moments_basis(psi, bits, mats, weights, center)
    assert np.allclose(got, want, rtol=0, atol=TOL * scale), (what, bits, got, want)


def bit_sets(n, rng, ks):
    """k in ks (those <= n), each with qubit 0 listed and not (both fp32 chunk layouts; at k = 12 < n without
    qubit 0 an fp32 chunk straddles two slabs), led by the top qubit, in shuffled order"""
    out = []
    for k in ks:
        if k > n:
            continue
        for with0 in (True, False):
            if not with0 and k == n:
                continue
            rest = [b for b in range(1, n) if b != n - 1]
            pick = ([0] if with0 else []) + ([n - 1] if n - 1 > 0 else [])
            pick += [int(b) for b in rng.choice(rest, k - len(pick), replace=False)] if k > len(pick) else []
            pick = pick[:k]
            rng.shuffle(pick)
            out.append(pick)
    return out


# n < 12: one slab smaller than the shared buffer; 12: one slab; 13: two; 17 .. 26: many slabs per CTA.  k = 12 is one block
# per slab, smaller k many (k = 3: the last butterfly round is a full one; 5: a partial one)
@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [1, 3, 5, 12, 13, 17, 22, 26])
def test_moments_basis_vs_numpy(n, prec):
    rng = np.random.default_rng(n)
    q = engine(n, prec, dense(n, prec))
    for bits in bit_sets(n, rng, (1, 2, 3, 5, 12) if n <= 17 else (2, 12)):
        k = len(bits)
        mats = rand_mats(rng, k)
        weights = rng.uniform(-1.5, 1.5, 2 * k).tolist()
        check(q, bits, mats, weights, 0.0, (n, prec))
        if k <= 2:
            check(q, bits, mats, weights, 0.375, (n, prec, "centred"))


@pytest.mark.parametrize("prec", [32, 64])
def test_read_only_launches_and_marginals(prec):
    n = 14
    psi = dense(n, prec, 1)
    q = engine(n, prec, psi)
    rng = np.random.default_rng(3)
    mats = [m.reshape(-1).tolist() for m in rand_mats(rng, 4)]
    p3 = q.Prob(3)
    q.be.reset_stats()
    e = q.ExpectationUnitaryAll([0, 3, 9, 13], mats)
    assert q.be.stats()["kernel_launches"] == 1
    assert np.array_equal(q.be.get_state(), psi)
    before = q.be.stats()["kernel_launches"]
    assert q.Prob(3) == p3  # the memoised marginal survives
    assert q.be.stats()["kernel_launches"] == before
    assert math.isfinite(e)
    # the zero state: zeros, no launch
    z = engine(n, prec)
    z.be.zero()
    z.be.reset_stats()
    assert z.be.moments_basis([1, 2], mats[:2], [1.0, -1.0] * 2, 0.0) == (0.0, 0.0, 0.0)
    assert z.be.stats()["kernel_launches"] == 0


@pytest.mark.parametrize("prec", [32, 64])
def test_every_einval(prec):
    q = engine(5, prec, dense(5, prec))
    lib, h = q.be.lib, q.be.h
    bits = (ctypes.c_int * 13)(*range(13))
    m = (ctypes.c_double * (8 * 13))(*([1, 0, 0, 0, 0, 0, 1, 0] * 13))
    w = (ctypes.c_double * 26)(*([1.0, -1.0] * 13))
    out = (ctypes.c_double * 3)()
    fn = lib.b200sv_moments_basis
    assert fn(h, 2, bits, m, w, 0.0, out) == _abi.B200SV_OK
    for args in [(0, bits, m, w), (13, bits, m, w), (-1, bits, m, w), (2, None, m, w), (2, bits, None, w),
                 (2, bits, m, None)]:
        assert fn(h, args[0], args[1], args[2], args[3], 0.0, out) == _abi.B200SV_EINVAL, args[0]
    assert fn(h, 2, bits, m, w, 0.0, None) == _abi.B200SV_EINVAL
    bad = (ctypes.c_int * 2)(1, 5)
    assert fn(h, 2, bad, m, w, 0.0, out) == _abi.B200SV_EINVAL  # out of range
    rep = (ctypes.c_int * 2)(3, 3)
    assert fn(h, 2, rep, m, w, 0.0, out) == _abi.B200SV_EINVAL  # repeated


@pytest.mark.parametrize("prec", [32, 64])
def test_mirror_matches_the_compiled_reference_and_its_post_state(prec):
    psi, queries, results, posts = tcpu._fixture(prec)
    for i, (t, (_, (want,))) in enumerate(zip(queries, results)):
        q = engine(12, prec, psi)
        got = tcpu._call(q, t)
        isExp, bits, form, ops, eig = tcpu.parse_query(t)
        _, scale = nb.exp_var_unitary(psi, isExp, bits, nb.basis_mats(form, bits, ops), eig)
        assert abs(got - want) <= tcpu.REF_REL_TOL[prec] * scale, (t[:2], got, want)
        after = q.GetQuantumState()
        if form == "matrix":
            assert np.array_equal(after, psi)
        elif i in posts:
            assert np.abs(after - posts[i]).max() <= 4 * util.AMP_TOL[prec], t[:2 + len(bits)]


@pytest.mark.parametrize("prec", [32, 64])
def test_gate_route_past_twelve_qubits(prec):
    n, bits = 14, [13, 0, 5, 2, 8, 1, 12, 3, 9, 4, 10, 6, 11]
    psi = dense(n, prec, 2)
    rng = np.random.default_rng(4)
    angles = rng.uniform(-3, 3, 3 * len(bits)).tolist()
    q = engine(n, prec, psi)
    q.be.reset_stats()
    got = q.ExpectationUnitaryAll(bits, angles)
    want, scale = nb.exp_var_unitary(psi, True, bits, nb.basis_mats("u3", bits, angles))
    assert abs(got - want) <= (1e-5 if prec == 32 else 1e-12) * scale
    assert np.abs(q.GetQuantumState() - nb.u3_post_state(psi, bits, angles)).max() <= 20 * util.AMP_TOL[prec]


# ---- the C++ drop-in (dropin/_build, built when the reference sources are present) -------------------------------------
B = os.path.join(util.ROOT, "dropin", "_build")


def test_dropin_matches_the_compiled_reference(tmp_path):
    prec = 32  # dropin/Makefile builds the fp32 harness
    exe = os.path.join(B, "observables_b200_f%d" % prec)
    if not os.path.exists(exe):
        pytest.skip("dropin/_build not built (needs the reference sources: QRACK_REFERENCE)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.join(util.ROOT, "qrack_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    psi, queries, results, posts = tcpu._fixture(prec)
    circ = oracle_observables.observables_circuit()
    script, dump = tmp_path / "q.qs", tmp_path / "s.bin"
    cplx = np.complex64 if prec == 32 else np.complex128

    def run(text):
        script.write_text(text)
        out = subprocess.run([exe, str(script), "--engine", "cuda", "--dump", str(dump)], check=True, capture_output=True,
                             text=True, timeout=600, env=env).stdout
        return out, np.fromfile(str(dump), dtype=cplx)

    _, mine = run(circ)  # the drop-in's state before any query
    for i, (t, (_, (want,))) in enumerate(zip(queries, results)):
        out, after = run(circ + " ".join(t) + "\n")
        (op, (got,)), = qscript.parse_results(out)
        isExp, bits, form, ops, eig = tcpu.parse_query(t)
        _, scale = nb.exp_var_unitary(psi, isExp, bits, nb.basis_mats(form, bits, ops), eig)
        assert op == t[0] and abs(got - want) <= tcpu.REF_REL_TOL[prec] * scale, (t[:2], got, want)
        if form == "matrix":
            assert np.array_equal(after, mine)  # read-only
        elif i in posts:
            assert np.abs(after - posts[i]).max() <= 4 * util.AMP_TOL[prec], t[:2 + len(bits)]
