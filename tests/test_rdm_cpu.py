"""The reduced density matrix on the CPU: the float64 reference (tests/npref_rdm.py) and the literal QInterface loop
of the oracle (tests/oracle_rdm.py) against what the compiled reference returned (tests/golden/ref_rdm_12q.*), the
script op, and the sharded backend's refusal."""
import os
import re

import numpy as np
import pytest

from qrack_b200 import qscript
from qrack_b200.sharded import _ShardedBackend

import npref_rdm as no
import oracle_rdm as oo
import util

N = 12
# Error model of the reference (qinterface.cpp:933): entry (i, j) is a sum of N_e = 2^(12 - k) products a_ie conj(a_je), each
# formed in complex<real1> (two products and one add per part: at most 2u |a_ie| |a_je| off) and added one by one to a running
# sum whose size never exceeds s_ij = sum_e |a_ie| |a_je| (each add at most u s_ij off).  So |error| <= (N_e + 2) u s_ij with
# u = 2^-24 (fp32) / 2^-53 (fp64): the bar below.  NumPy is fed the reference's own state and sums in float64.
UNIT = {32: 2.0 ** -24, 64: 2.0 ** -53}


def bar(prec, k):
    return ((1 << (N - k)) + 2) * UNIT[prec]


def _sets():
    return [[int(b) for b in t[2:]] for _, t in qscript.parse(oo.rdm_queries())]


def _fixture(prec):
    z = np.load(os.path.join(util.GOLDEN, "ref_rdm_12q.f%d.npz" % prec))
    return z["state"], [z["rho%d" % i] for i in range(len(_sets()))]


def test_query_list_covers_the_code_paths():
    sets = _sets()
    assert sorted({len(s) for s in sets}) == [0, 1, 2, 3, 5, 7]
    assert any(0 in s for s in sets) and any(s and 0 not in s for s in sets)
    assert any(N - 1 in s for s in sets) and any(s != sorted(s) for s in sets)
    assert any(7 in s and 8 in s for s in sets)


@pytest.mark.parametrize("prec", [32, 64])
def test_npref_matches_the_compiled_reference(prec):
    psi, rhos = _fixture(prec)
    for qs, got in zip(_sets(), rhos):
        want, scale = no.rdm(psi, qs)
        assert got.shape == want.shape == (1 << len(qs),) * 2
        err = np.abs(got.astype(np.complex128) - want)
        assert (err <= bar(prec, len(qs)) * scale).all(), (qs, float((err / scale).max()))
        # both sums of an (i, j) / (j, i) pair run over the environment in the same order: the reference's rho is Hermitian
        assert np.array_equal(got, got.conj().T), qs


@pytest.mark.parametrize("prec", [32, 64])
def test_oracle_loop_matches_the_compiled_reference(prec):
    psi, rhos = _fixture(prec)
    states, results = util.run_engine(oo.rdm_text(), oo.QEngineRestateRdm, prec)
    mine = states[0]
    util.assert_states_close({0: mine}, {0: psi}, prec, "oracle circuit vs the reference's")
    # the oracle's state differs from the reference's by d = |mine - psi| per amplitude, which moves entry (i, j) by at most
    # sum_e (|a_ie| + d_ie) (|a_je| + d_je) - |a_ie| |a_je|
    m, d = np.abs(mine.astype(np.complex128)), np.abs(mine.astype(np.complex128) - psi)
    assert len(results) == len(rhos)
    for (op, vals), qs, ref in zip(results, _sets(), rhos):
        assert op == "GetReducedDensityMatrix"
        got = np.array(vals).view(np.complex128).reshape(ref.shape)
        want, scale = no.rdm(mine, qs)
        assert (np.abs(got - want) <= bar(prec, len(qs)) * scale).all(), qs
        moved = no.rdm(m + d, qs)[1] - no.rdm(m, qs)[1]
        assert (np.abs(got - ref) <= 2 * bar(prec, len(qs)) * scale + moved).all(), qs


def test_npref_rdm_definition():
    """bit p of the row index is qubits[p]: on a product state rho is the Kronecker product of the single-qubit matrices, the
    LAST listed qubit outermost"""
    rng = np.random.default_rng(3)
    vs = [rng.standard_normal(2) + 1j * rng.standard_normal(2) for _ in range(4)]
    psi = np.kron(np.kron(vs[3], vs[2]), np.kron(vs[1], vs[0]))  # qubit 0 = vs[0]
    one = [np.outer(v, v.conj()) for v in vs]
    rho, scale = no.rdm(psi, [2, 0])
    env = np.vdot(vs[1], vs[1]) * np.vdot(vs[3], vs[3])
    assert np.allclose(rho, env * np.kron(one[0], one[2]))
    assert np.allclose(np.trace(no.rdm(psi, [])[0]), np.vdot(psi, psi))
    assert (scale >= np.abs(rho) - 1e-12).all()


def test_query_op_round_trip():
    """the op parses, is a query of the script format, dispatches to GetReducedDensityMatrix with the listed qubits in order,
    and its result line (2 4^k values, row-major, re / im interleaved) is read back; the C++ harness handles the op"""
    text = oo.rdm_text()
    calls = []

    class Rec:
        def GetReducedDensityMatrix(self, qs):
            calls.append(list(qs))
            d = 1 << len(qs)
            return (np.arange(d * d) + 0.5j * np.arange(d * d)).reshape(d, d)

        def __getattr__(self, name):
            return lambda *a: None

    _, results = qscript.run(text, lambda n, p: Rec())
    assert "GetReducedDensityMatrix" in qscript.QUERY_OPS
    assert calls == _sets() and [r[0] for r in results] == ["GetReducedDensityMatrix"] * len(calls)
    for (_, vals), qs in zip(results, calls):
        d = 1 << len(qs)
        assert np.array_equal(np.array(vals).view(np.complex128), np.arange(d * d) + 0.5j * np.arange(d * d))
    line = "".join("%s %s\n" % (op, " ".join("%.17g" % v for v in vals)) for op, vals in results)
    assert qscript.parse_results(line) == results
    assert qscript.count_gate_ops(text) == qscript.count_gate_ops(oo.rdm_circuit())
    src = open(os.path.join(util.ROOT, "dropin", "observables_harness.cpp")).read()
    assert "GetReducedDensityMatrix" in re.findall(r'op == "(\w+)"', src)


def test_sharded_backend_refuses_the_primitive():
    be = _ShardedBackend.__new__(_ShardedBackend)
    with pytest.raises(NotImplementedError):
        be.reduced_density_matrix([0, 1])
