"""The reduced density matrix sweep on the GPU (b200sv_reduced_density_matrix) against the float64 NumPy reference
(tests/npref_rdm.py) at the shapes where its code path changes, its argument errors, what it leaves alone (the state,
the memoised marginals), the Python mirror against the oracle's literal GetAmplitude loop, a full-size analytic check, and the
C++ drop-in against the compiled reference.

NumPy is fed the state the kernel read, read back in the engine's precision.  Bars are relative to the natural scale of each
entry, s_ij = sum_e |A_ie| |A_je|: 2e-6 (fp32) / 1e-12 (fp64).  Every product and sum of the kernel is in double (an fp32
amplitude converted to double makes each product exact), so only the order of the additions differs from NumPy."""
import ctypes
import math
import os
import random
import subprocess

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi, qscript

import npref_rdm as no
import oracle_rdm as oo
import test_rdm_cpu as tcpu
import util

pytestmark = pytest.mark.gpu

TOL = {32: 2e-6, 64: 1e-12}
SIZES = [1, 2, 5, 13, 17, 22, 24]
KS = [0, 1, 2, 6, 7, 8, 10]  # 6 / 7: one tile / two tiles per side at T = 64


def engine(n, prec, psi=None, normalize=False):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    if psi is not None:
        q.SetQuantumState(psi)
    return q


def dense(n, prec, seed=0, norm2=1.0):
    rng = np.random.default_rng(1000 * n + seed)
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi * math.sqrt(norm2) / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def check(q, qs, prec, what=""):
    """rho of the kernel vs NumPy on the state read back; exactly Hermitian with a real diagonal"""
    psi = q.be.get_state()
    got = q.be.reduced_density_matrix(qs)
    want, scale = no.rdm(psi, qs)
    assert got.shape == want.shape
    err = np.abs(got - want)
    assert (err <= TOL[prec] * scale).all(), (what, qs, float(np.max(err / np.maximum(scale, 1e-300))))
    assert np.array_equal(got, got.conj().T) and not np.diag(got).imag.any(), (what, qs)
    return got


def kept_sets(n, rng):
    """k = 0, and for each other k of KS (and n - 1, n where n <= 13) one set with qubit 0 kept and one without (both fp32
    chunk layouts), led by the top qubit and the byte-boundary qubits 7 / 8 / 15 / 16 where they exist, in shuffled order"""
    ks = sorted({k for k in KS if 0 < k <= n} | ({n - 1, n} - {0} if n <= 13 else set()))
    edge = list(dict.fromkeys(b for b in (n - 1, 7, 8, 15, 16) if 0 < b < n))
    out = [[]]
    for k in ks:
        for with0 in (True, False):
            if not with0 and k == n:
                continue
            first = (([0] if with0 else []) + edge)[:k]
            s = first + rng.sample([b for b in range(1, n) if b not in first], k - len(first))
            rng.shuffle(s)
            out.append(s)
    return out


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_rdm_vs_numpy(n, prec):
    rng = random.Random(n * 13 + prec)
    q = engine(n, prec, dense(n, prec))
    psi = q.GetQuantumState()
    sets = kept_sets(n, rng)
    assert any(0 in s for s in sets) and (n == 1 or any(s and 0 not in s for s in sets))
    for qs in sets:
        check(q, qs, prec, n)
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_unnormalised_trace_zero_state_queued_gates_state_and_marginals(prec):
    n = 11
    # a state of norm^2 0.5: the trace is 0.5, nothing is normalised
    q = engine(n, prec, dense(n, prec, 1, norm2=0.5))
    for qs in ([], [3, 0], [10, 4, 7, 1, 9, 2, 6, 0]):
        rho = check(q, qs, prec, "norm 0.5")
        assert abs(np.trace(rho).real - 0.5) <= 4 * TOL[prec]
    # the zero state: zeros without a launch
    q.ZeroAmplitudes()
    q.be.reset_stats()
    assert not q.be.reduced_density_matrix([2, 5, 1]).any()
    assert q.be.stats()["kernel_launches"] == 0
    # queued, unflushed gates are part of the state the query sees
    q = engine(n, prec, dense(n, prec, 2))
    for b in range(n):
        q.H(b)
        q.T(b)
    got = q.be.reduced_density_matrix([9, 0, 4])
    psi = q.GetQuantumState()
    want, scale = no.rdm(psi, [9, 0, 4])
    assert (np.abs(got - want) <= TOL[prec] * scale).all()
    # the state is bit-identical across the query, and memoised marginals survive it without a new launch
    p3 = q.Prob(3)
    before = q.be.stats()["kernel_launches"]
    q.be.reduced_density_matrix([1, 8])
    assert q.be.stats()["kernel_launches"] == before + 1
    assert q.Prob(3) == p3 and q.Prob(7) >= 0
    assert q.be.stats()["kernel_launches"] == before + 1
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_every_einval(prec):
    n = 9
    q = engine(n, prec, dense(n, prec, 3))
    psi = q.GetQuantumState()
    lib, h = q.be.lib, q.be.h
    E = _abi.B200SV_EINVAL
    out = (ctypes.c_double * (2 << (2 * n)))()

    def rc(k, qs, o=out):
        arr = None if qs is None else (ctypes.c_int * max(len(qs), 1))(*qs)
        return lib.b200sv_reduced_density_matrix(h, k, arr, o)
    assert rc(-1, [0]) == E
    assert rc(n + 1, list(range(n)) + [0]) == E  # k > n
    assert rc(2, None) == E and rc(2, [0, 1], None) == E
    assert rc(2, [0, n]) == E and rc(2, [-1, 3]) == E and rc(3, [4, 2, 4]) == E
    assert rc(0, None) == 0 and out[0] == pytest.approx(1.0, abs=1e-6) and out[1] == 0.0
    big = QEngineCUDA(15, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    assert big.be.lib.b200sv_reduced_density_matrix(big.be.h, 15, (ctypes.c_int * 15)(*range(15)), out) == E
    with pytest.raises(ValueError):
        big.GetReducedDensityMatrix(list(range(15)))
    for bad in ([0, 9], [-1], [2, 2]):
        with pytest.raises(ValueError):
            q.GetReducedDensityMatrix(bad)
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_mirror_matches_the_oracle_loop_without_normalising(prec):
    """doNormalize on and a state made unnormalised by SetAmplitude: the mirror, like the reference's GetAmplitude loop,
    returns rho of the state as it is (trace = sum |psi|^2 != 1)"""
    n = 10
    psi0 = dense(n, prec, 4)
    regs = []
    for cls in (QEngineCUDA, oo.QEngineRestateRdm):
        r = cls(n, 0, random.Random(1), 1.0 + 0j, True, False, precision=prec)
        r.SetQuantumState(psi0)
        r.SetAmplitude(5, 0.3 + 0.2j)
        r.SetAmplitude(700, -0.25j)
        regs.append(r)
    psi = regs[0].be.get_state()
    assert abs(float(np.vdot(psi, psi).real) - 1.0) > 0.05
    for qs in ([], [0], [9, 0, 4], [3, 8, 1, 6, 2]):
        got, want = regs[0].GetReducedDensityMatrix(qs), regs[1].GetReducedDensityMatrix(qs)
        assert got.dtype == regs[0].cplx and got.shape == (1 << len(qs),) * 2
        ref, scale = no.rdm(psi, qs)
        bar = ((1 << (n - len(qs))) + 2) * tcpu.UNIT[prec]
        assert (np.abs(got - want) <= (bar + 2 * TOL[prec]) * scale).all(), qs
        assert abs(np.trace(got).real - float(np.vdot(psi, psi).real)) <= 4 * TOL[prec]


def _bell_model(n, th, ph, kept):
    """rho on `kept` of (x)_{q != 0, top} U3|0> (x) (|00> + |11>) / sqrt 2 on (0, top): the small product system of the kept
    qubits (and the partner of a kept pair member), reduced with NumPy"""
    top = n - 1
    qs = sorted(set(kept) | ({0, top} if set(kept) & {0, top} else set()))
    psi = np.ones(1)
    for q in qs:  # qs ascending: later qubits are the higher index bits
        if q in (0, top):
            continue
        psi = np.kron(np.array([math.cos(th[q]), complex(math.cos(ph[q]), math.sin(ph[q])) * math.sin(th[q])]), psi)
    if 0 in qs:
        # the pair as bits (0 -> index bit 0 of the pair block, top -> the highest bit): insert it around the others
        m = len(qs) - 2
        full = np.zeros(1 << (m + 2), dtype=complex)
        full[np.arange(1 << m) << 1] += psi / math.sqrt(2)
        full[(np.arange(1 << m) << 1) | (1 << (m + 1)) | 1] += psi / math.sqrt(2)
        psi = full
    return no.rdm(psi, [qs.index(q) for q in kept])[0]


@pytest.mark.parametrize("n,prec", [(30, 32), (29, 64)])
def test_full_size_analytic(n, prec):
    """U3 on every qubit but 0 and the top one, H on 0, CNOT(0, top): rho on kept sets that straddle the Bell pair is the
    Kronecker product of single-qubit projectors and the pair's (Bell projector, or I / 2 when only one member is kept)"""
    rng = random.Random(n)
    top = n - 1
    th = [rng.uniform(0.1, 1.4) for _ in range(n)]
    ph = [rng.uniform(-3, 3) for _ in range(n)]
    q = engine(n, prec)
    for b in range(1, top):
        q.U(b, 2 * th[b], ph[b], 0.0)
    q.H(0)
    q.CNOT(0, top)
    for kept in ([0, top], [top, 0], [0], [5, top, 0, 17], [top, 3, 8], [1, 0, 2, 3, top, 7, 15, 16]):
        got = q.GetReducedDensityMatrix(kept).astype(np.complex128)
        tr = np.trace(got).real
        # the fp32 gates round each single-qubit norm by ~2^-24, so the trace drifts by up to ~n 2^-24; the shape is exact to TOL
        assert abs(tr - 1.0) <= (n * 2.0 ** -23 if prec == 32 else 1e-12), (kept, tr)
        want = _bell_model(n, th, ph, kept)
        assert np.abs(got / tr - want).max() <= (1e-6 if prec == 32 else 1e-12), kept


# ---- the C++ drop-in (dropin/_build, built when the reference sources are present) -------------------------------------
B = os.path.join(util.ROOT, "dropin", "_build")


def test_dropin_rdm_matches_the_compiled_reference(tmp_path):
    exe = os.path.join(B, "observables_b200_f32")
    if not os.path.exists(exe):
        pytest.skip("dropin/_build not built (needs the reference sources: QRACK_REFERENCE)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.join(util.ROOT, "qrack_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    circ, full, dump = tmp_path / "c.qs", tmp_path / "q.qs", tmp_path / "s.bin"
    circ.write_text(oo.rdm_circuit())
    full.write_text(oo.rdm_text())
    subprocess.run([exe, str(circ), "--engine", "cuda", "--dump", str(dump)], check=True, timeout=600, env=env)
    out = subprocess.run([exe, str(full), "--engine", "cuda"], check=True, capture_output=True, text=True, timeout=600,
                         env=env).stdout
    mine = np.fromfile(str(dump), dtype=np.complex64)
    psi, rhos = tcpu._fixture(32)
    m, d = np.abs(mine.astype(np.complex128)), np.abs(mine.astype(np.complex128) - psi)
    got = qscript.parse_results(out)
    assert len(got) == len(rhos)
    for (op, vals), qs, ref in zip(got, tcpu._sets(), rhos):
        assert op == "GetReducedDensityMatrix"
        g = np.array(vals).view(np.complex128).reshape(ref.shape)
        want, scale = no.rdm(mine, qs)
        # the drop-in rounds the double sums to real1 (float): one more 2^-24 of each entry
        assert (np.abs(g - want) <= (TOL[32] + 2.0 ** -24) * scale).all(), qs
        moved = no.rdm(m + d, qs)[1] - no.rdm(m, qs)[1]
        assert (np.abs(g - ref) <= (TOL[32] + tcpu.bar(32, len(qs))) * scale + moved).all(), qs
