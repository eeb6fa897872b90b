"""The observable sweeps on the GPU (b200sv_moments_bits / _floats, b200sv_expectation_pauli) against the float64 NumPy
reference (tests/npref_observables.py) at the shapes where their code paths change, their argument errors, what they leave
alone (the state, the memoised marginals), the Python mirror's QInterface methods against the oracle's literal loops, a
full-size analytic check, and the C++ drop-in against the compiled reference.

The reference is fed the state the kernel read, read back in the engine's precision.  Bars are relative to the scale of each
sum: 1e-6 (fp32) / 1e-12 (fp64), since every term is accumulated in double and only the order of the additions differs."""
import ctypes
import math
import os
import random
import re
import subprocess

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi, qscript

import npref_observables as no
import oracle_observables as oo
import test_observables_cpu as tcpu
import util

pytestmark = pytest.mark.gpu

TOL = {32: 1e-6, 64: 1e-12}
SIZES = [1, 2, 7, 8, 9, 15, 16, 17, 22, 24]


def engine(n, prec, psi=None, normalize=False):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    if psi is not None:
        q.SetQuantumState(psi)
    return q


def dense(n, prec, seed=0):
    rng = np.random.default_rng(1000 * n + seed)
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def bit_sets(n, rng):
    """k = 0, 1, 2, 8 and n, with listed qubits on both sides of the byte boundaries where there are any"""
    out = [[], [n - 1]]
    out.append([7, 8] if n > 8 else [0, n - 1] if n > 1 else [0])
    if n >= 8:
        edge = [b for b in (0, 7, 8, 15, 16, 23) if b < n]
        rest = [b for b in range(n) if b not in edge]
        out.append(edge + rng.sample(rest, 8 - len(edge)))
    out.append(rng.sample(range(n), n))
    return [b for i, b in enumerate(out) if len(set(b)) == len(b) and b not in out[:i]]


def _check_moments(got, want, p, w, center, prec, what):
    scales = (1.0, float((p * np.abs(w - center)).sum()) + 1e-300, float((p * (np.abs(w) + abs(center)) ** 2).sum()) + 1e-300)
    for j in range(3):
        assert abs(got[j] - want[j]) <= TOL[prec] * scales[j], (what, j, got, want)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_moments_vs_numpy(n, prec):
    rng = random.Random(n * 7 + prec)
    q = engine(n, prec, dense(n, prec))
    psi = q.GetQuantumState()
    p = np.abs(psi.astype(np.complex128)) ** 2
    for bits in bit_sets(n, rng):
        k = len(bits)
        perms = [rng.randrange(1 << 40) for _ in range(2 * k)]
        offset = rng.randrange(1 << 30)
        w = no.weights_bits(n, bits, perms, offset)
        for center in (0.0, float((p * w).sum())):
            got = q.be.moments_bits(bits, perms, offset, center)
            _check_moments(got, no.moments_bits(psi, bits, perms, offset, center), p, w, center, prec, ("bits", bits, center))
        weights = [rng.uniform(-1.6, 1.6) for _ in range(2 * k)]
        w = no.weights_floats(n, bits, weights)
        for center in (0.0, -0.375):
            got = q.be.moments_floats(bits, weights, center)
            _check_moments(got, no.moments_floats(psi, bits, weights, center), p, w, center, prec, ("floats", bits, center))
    assert np.array_equal(q.GetQuantumState(), psi)


def pauli_cases(n, rng):
    """x masks: bit 0 only, bit 0 + high bits, high bits only, the top qubit (and x = 0); for each every count of Y mod 4
    that fits, with random Z elsewhere, and the pure-Z string"""
    top = n - 1
    xs = {0, 1, 1 << top}
    if n > 2:
        xs |= {1 | (1 << top) | (1 << (n // 2)), (1 << top) | (1 << (n // 2)) | (1 << max(1, n // 3))}
    cases = []
    for x in sorted(xs):
        xb = [b for b in range(n) if (x >> b) & 1]
        others = [b for b in range(n) if not (x >> b) & 1]
        for ny in range(4):
            if ny > len(xb):
                continue
            z = sum(1 << b for b in xb[:ny]) | sum(1 << b for b in others if rng.random() < 0.5)
            cases.append((x, z))
    cases.append((0, (1 << n) - 1))
    return cases


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_pauli_vs_numpy(n, prec):
    rng = random.Random(n * 11 + prec)
    q = engine(n, prec, dense(n, prec, 1))
    psi = q.GetQuantumState()
    for x, z in pauli_cases(n, rng):
        s0, e = q.be.expectation_pauli(x, z)
        w0, we = no.pauli_expectation(psi, x, z)
        assert abs(s0 - w0) <= TOL[prec] and abs(e - we) <= TOL[prec], (n, x, z, (s0, e), (w0, we))
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_zero_state_queued_gates_state_and_marginals(prec):
    n = 10
    q = engine(n, prec)
    q.ZeroAmplitudes()
    q.be.reset_stats()
    assert q.be.moments_bits([1, 2], [0, 1, 2, 3], 5, 1.0) == (0.0, 0.0, 0.0)
    assert q.be.moments_floats([1], [2.0, 3.0], 0.0) == (0.0, 0.0, 0.0)
    assert q.be.expectation_pauli(3, 1) == (0.0, 0.0)
    assert q.be.stats()["kernel_launches"] == 0
    # queued, unflushed gates are part of the state a query sees
    q = engine(n, prec, dense(n, prec, 2))
    for b in range(n):
        q.H(b)
        q.T(b)
    got = q.be.moments_floats([0, 9], [0.5, 2.0, -1.0, 3.0], 0.25)
    gp = q.be.expectation_pauli(0b1000000011, 0b0000000110)
    psi = q.GetQuantumState()
    assert np.allclose(got, no.moments_floats(psi, [0, 9], [0.5, 2.0, -1.0, 3.0], 0.25), rtol=0, atol=4 * TOL[prec])
    assert np.allclose(gp, no.pauli_expectation(psi, 0b1000000011, 0b0000000110), rtol=0, atol=TOL[prec])
    # the state is bit-identical across both queries, and memoised marginals survive them without a new launch
    p3 = q.Prob(3)
    before = q.be.stats()["kernel_launches"]
    q.be.moments_bits([2, 5], [1, 2, 3, 4], 0, 0.0)
    q.be.expectation_pauli(0b10, 0b11)
    assert q.be.stats()["kernel_launches"] == before + 2
    assert q.Prob(3) == p3 and q.Prob(7) >= 0
    assert q.be.stats()["kernel_launches"] == before + 2
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_uint64_limit_and_every_einval(prec):
    n = 9
    q = engine(n, prec, dense(n, prec, 3))
    psi = q.GetQuantumState()
    lib, h = q.be.lib, q.be.h
    top = (1 << 64) - 1
    perms = [1 << 62, (1 << 62) + 7, 3, 1 << 61, 0, 12345]
    offset = top - ((1 << 62) + 7) - (1 << 61) - 12345
    got = q.be.moments_bits([0, 7, 8], perms, offset, 0.0)
    want = no.moments_bits(psi, [0, 7, 8], perms, offset)
    assert abs(got[1] - want[1]) <= TOL[prec] * 2.0 ** 64
    with pytest.raises(ValueError):
        q.be.moments_bits([0, 7, 8], perms, offset + 1, 0.0)

    I3, U6, D6, O3 = (ctypes.c_int * 3)(0, 7, 8), (ctypes.c_uint64 * 6)(*range(6)), (ctypes.c_double * 6)(*range(6)), (ctypes.c_double * 3)()

    def rc(fn, *a):
        return fn(h, *a)
    E = _abi.B200SV_EINVAL
    mb, mf, pa = lib.b200sv_moments_bits, lib.b200sv_moments_floats, lib.b200sv_expectation_pauli
    assert rc(mb, -1, I3, U6, 0, 0.0, O3) == E and rc(mf, -1, I3, D6, 0.0, O3) == E
    assert rc(mb, 3, None, U6, 0, 0.0, O3) == E and rc(mf, 3, None, D6, 0.0, O3) == E
    assert rc(mb, 3, I3, None, 0, 0.0, O3) == E and rc(mf, 3, I3, None, 0.0, O3) == E
    assert rc(mb, 3, I3, U6, 0, 0.0, None) == E and rc(mf, 3, I3, D6, 0.0, None) == E
    for bad in ((0, 9, 1), (0, -1, 1), (4, 2, 4)):
        b = (ctypes.c_int * 3)(*bad)
        assert rc(mb, 3, b, U6, 0, 0.0, O3) == E and rc(mf, 3, b, D6, 0.0, O3) == E
    assert rc(mb, 0, None, None, top, 0.0, O3) == 0 and O3[1] == float(top) * O3[0]
    assert rc(mf, 0, None, None, 0.0, O3) == 0 and O3[1] == O3[0]
    O2 = (ctypes.c_double * 2)()
    assert rc(pa, 1 << n, 0, O2) == E and rc(pa, 0, 1 << n, O2) == E and rc(pa, 1, 1, None) == E
    assert np.array_equal(q.GetQuantumState(), psi)


def _extra_rows(q):
    """k = 0 and k = 1 rows of every method, and the same on the zero state"""
    out = []
    for zero in (False, True):
        if zero:
            q.ZeroAmplitudes()
        out += [q.ExpectationBitsFactorized([], [], 3), q.VarianceBitsFactorized([], [], 3),
                q.ExpectationFloatsFactorized([], []), q.VarianceFloatsFactorized([], []),
                q.ExpectationPauliAll([], []), q.VariancePauliAll([4], [0]),
                q.ExpectationBitsFactorized([4], [3, 9], 2), q.VarianceBitsFactorized([4], [3, 9], 2),
                q.ExpectationFloatsFactorized([8], [0.5, -2.0]), q.VarianceFloatsFactorized([8], [0.5, -2.0]),
                q.ExpectationPauliAll([3, 5], [0, 3]), q.VariancePauliAll([3, 5], [1, 0]),
                q.ExpectationPauliAll([2, 9], [2, 1]), q.VariancePauliAll([2, 9], [3, 1]),
                q.ExpectationBitsAll([1, 9, 8], 7), q.VarianceFloatsFactorized([1, 9], [0.5, 2.0, -1.0, 3.0])]
    return out


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("prec", [32, 64])
def test_mirror_matches_the_oracle_loops(prec, normalize):
    text = oo.observables_text()

    def make(cls):
        return lambda n, p: cls(n, p, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    regs_d, res_d = qscript.run(text, make(QEngineCUDA))
    regs_o, res_o = qscript.run(text, make(oo.QEngineRestateObs))
    psi = util.run_engine(oo.observables_circuit(), QEngineCUDA, prec)[0][0]
    for (gop, (got,)), (wop, (want,)), t in zip(res_d, res_o, tcpu._queries()):
        assert gop == wop == t[0]
        _, scale, psi = no.query_value(psi, t[0], t[1:])
        assert abs(got - want) <= tcpu.REF_REL_TOL[prec] * scale, (t, got, want, scale)
    util.assert_states_close({0: regs_d[0].GetQuantumState()}, {0: regs_o[0].GetQuantumState()}, prec, "after the queries")
    got, want = _extra_rows(regs_d[0]), _extra_rows(regs_o[0])
    for i, (a, b) in enumerate(zip(got, want)):
        assert abs(a - b) <= tcpu.REF_REL_TOL[prec] * max(1.0, abs(b)) * 100, (i, a, b)


@pytest.mark.parametrize("n,prec", [(30, 32), (29, 64)])
def test_full_size_analytic(n, prec):
    """the product state (x)_q (cos t_q |0> + e^{i f_q} sin t_q |1>) prepared with U gates"""
    rng = random.Random(n)
    th = [rng.uniform(0.05, 0.3) if q % 3 else rng.uniform(0.7, 0.85) for q in range(n)]
    ph = [rng.uniform(-0.3, 0.3) if q % 2 else rng.uniform(1.3, 1.8) for q in range(n)]
    q = engine(n, prec)
    for b in range(n):
        q.U(b, 2 * th[b], ph[b], 0.0)
    c2, s2 = [math.cos(t) ** 2 for t in th], [math.sin(t) ** 2 for t in th]
    bits = list(range(n))[::-1]
    # Pauli: X / Y on the strongly rotated qubits (q % 3 == 0), Z elsewhere, and one I
    paulis = [(1 if ph[b] < 1 else 3) if b % 3 == 0 else 2 for b in bits]
    paulis[5] = 0
    want = 1.0
    for b, p in zip(bits, paulis):
        want *= {0: 1.0, 1: math.sin(2 * th[b]) * math.cos(ph[b]), 3: math.sin(2 * th[b]) * math.sin(ph[b]),
                 2: math.cos(2 * th[b])}[p]
    got = q.ExpectationPauliAll(bits, paulis)
    assert abs(got - want) <= 20 * TOL[prec], (got, want)
    weights = [v for b in bits for v in (rng.uniform(0.8, 1.2), rng.uniform(-1.2, 1.2))]
    want = scale = 1.0
    for p, b in enumerate(bits):
        want *= weights[2 * p] * c2[b] + weights[2 * p + 1] * s2[b]
        scale *= abs(weights[2 * p]) * c2[b] + abs(weights[2 * p + 1]) * s2[b]
    assert abs(q.ExpectationFloatsFactorized(bits, weights) - want) <= 20 * TOL[prec] * scale
    perms = [rng.randrange(1 << 58) for _ in range(2 * n)]
    offset = 123456789
    want = offset + sum(perms[2 * p] * c2[b] + perms[2 * p + 1] * s2[b] for p, b in enumerate(bits))
    assert abs(q.ExpectationBitsFactorized(bits, perms, offset) - want) <= 20 * TOL[prec] * want


# ---- the C++ drop-in (dropin/_build, built when the reference sources are present) -------------------------------------
B = os.path.join(util.ROOT, "dropin", "_build")


def _env():
    e = dict(os.environ)
    e["LD_LIBRARY_PATH"] = os.path.join(util.ROOT, "qrack_b200") + ":" + e.get("LD_LIBRARY_PATH", "")
    return e


def test_reference_expectation_unit_test_on_the_dropin():
    unit = os.path.join(B, "f32", "unittest_b200")
    if not os.path.exists(unit):
        pytest.skip("dropin/_build not built (needs the reference sources: QRACK_REFERENCE)")
    r = subprocess.run([unit, "--layer-qengine", "--proc-cuda", "--disable-hardware-rng", "test_expectationbitsall"],
                       capture_output=True, text=True, timeout=600, env=_env())
    out = r.stdout + r.stderr
    assert r.returncode == 0 and re.search(r"All tests passed \(\d+ assertions? in 1 test case", out), out[-3000:]


def test_dropin_observables_match_the_compiled_reference(tmp_path):
    exe = os.path.join(B, "observables_b200_f32")
    if not os.path.exists(exe):
        pytest.skip("dropin/_build not built (needs the reference sources: QRACK_REFERENCE)")
    sp = tmp_path / "obs.qs"
    sp.write_text(oo.observables_text())
    out = subprocess.run([exe, str(sp), "--engine", "cuda"], check=True, capture_output=True, text=True, timeout=600,
                         env=_env()).stdout
    ref = util.load_reference("observables_12q", 32)
    got = qscript.parse_results(out)
    psi = ref["state"]
    assert len(got) == len(ref["results"]) == 48
    for (gop, (g,)), (wop, (w,)), t in zip(got, ref["results"], tcpu._queries()):
        assert gop == wop == t[0]
        _, scale, psi = no.query_value(psi, t[0], t[1:])
        assert abs(g - w) <= tcpu.REF_REL_TOL[32] * scale, (t, g, w, scale)
