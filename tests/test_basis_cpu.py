"""Observables in a per-qubit basis on the CPU: the float64 reference (tests/npref_basis.py) against what the compiled
reference returned (tests/golden/ref_basis_12q.*), and the edge rules and errors of the mirror's ExpVarUnitaryAll over a
CPU stand-in backend whose moments_basis is the NumPy reference."""
import os
import random
import re

import numpy as np
import pytest

from oracle.restate_engine import QEngineRestate, _RestateBackend
from qrack_b200 import qscript
from qrack_b200.sharded import _ShardedBackend

import npref_basis as nb
import util

N = 12
# Relative to each result's scale (npref_basis).  The reference adds the 2^12 terms one by one in real1_f and, in fp32, also
# rounds the basis gates it applies before the query; the bars sit above what the stored fixtures show.
REF_REL_TOL = {32: 2e-5, 64: 1e-13}


def _fixture(prec):
    z = np.load(os.path.join(util.GOLDEN, "ref_basis_12q.f%d.npz" % prec))
    queries = [t for _, t in qscript.parse(str(z["queries"]))]
    posts = {int(k[4:]): z[k] for k in z.files if k.startswith("post")}
    return z["state"], queries, qscript.parse_results(str(z["results"])), posts


def parse_query(t):
    """(isExp, bits, form, ops, eigenvalues) of a query line's tokens; ops = angles or a list of 2x2 complex matrices"""
    k = int(t[1])
    bits = [int(b) for b in t[2:2 + k]]
    v = [float(x) for x in t[2 + k:]]
    if "Matrix" in t[0]:
        mats = [np.array([complex(v[8 * i + 2 * e], v[8 * i + 2 * e + 1]) for e in range(4)]).reshape(2, 2) for i in range(k)]
        return t[0][0] == "E", bits, "matrix", mats, v[8 * k:]
    return t[0][0] == "E", bits, "u3", v[:3 * k], v[3 * k:]


def test_queries_cover_the_code_paths():
    _, queries, results, posts = _fixture(32)
    assert len(queries) == len(results) == 56
    sets = [parse_query(t)[1] for t in queries]
    assert sorted({len(s) for s in sets}) == [1, 2, 3, 5, 12]
    assert any(0 in s for s in sets) and any(0 not in s for s in sets)
    assert any(N - 1 in s for s in sets) and any(s != sorted(s) for s in sets)
    forms = {(parse_query(t)[2], t[0][0], bool(parse_query(t)[4])) for t in queries}
    assert len(forms) == 8  # both forms, expectation and variance, with and without eigenvalues
    assert len(posts) == 7 and all(queries[q][0] == "ExpectationUnitaryAll" for q in posts)


@pytest.mark.parametrize("prec", [32, 64])
def test_npref_matches_the_compiled_reference(prec):
    psi, queries, results, posts = _fixture(prec)
    for t, (op, (got,)) in zip(queries, results):
        assert op == t[0]
        isExp, bits, form, ops, eig = parse_query(t)
        want, scale = nb.exp_var_unitary(psi, isExp, bits, nb.basis_mats(form, bits, ops), eig)
        assert abs(got - want) <= REF_REL_TOL[prec] * scale, (t[:2 + len(bits)], got, want, scale)


@pytest.mark.parametrize("prec", [32, 64])
def test_npref_post_state_matches_the_compiled_reference(prec):
    psi, queries, _, posts = _fixture(prec)
    for q, post in posts.items():
        _, bits, _, angles, _ = parse_query(queries[q])
        want = nb.u3_post_state(psi, bits, angles)
        assert np.abs(post - want).max() <= 4 * util.AMP_TOL[prec], queries[q][:2 + len(bits)]
        # the reference's undo is not the inverse of its first gate: the state does change
        assert np.abs(want - psi).max() > 1e-3


def test_npref_definition():
    """on a product state the transformed moments factorise: S1 = prod_p <v_p| A_p^H diag(w_p) A_p |v_p>"""
    rng = np.random.default_rng(5)
    vs = [rng.standard_normal(2) + 1j * rng.standard_normal(2) for _ in range(3)]
    psi = np.kron(vs[2], np.kron(vs[1], vs[0]))
    mats = [rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2)) for _ in range(2)]
    w = [0.5, -2.0, 1.5, 3.0]
    (s0, s1, _), _ = nb.moments_basis(psi, [2, 0], mats, w)
    f2, f0 = mats[0] @ vs[2], mats[1] @ vs[0]
    env = np.vdot(vs[1], vs[1]).real
    assert np.isclose(s0, env * np.vdot(f2, f2).real * np.vdot(f0, f0).real)
    assert np.isclose(s1, env * (np.abs(f2) ** 2 @ w[:2]) * (np.abs(f0) ** 2 @ w[2:]))


class _StandInBackend(_RestateBackend):
    """the restatement backend with the two moments sweeps the mirror's observables need, computed by the NumPy reference"""

    def __init__(self, n_qubits, precision):
        super().__init__(n_qubits, precision)
        self.sweeps = 0

    def moments_basis(self, bits, mats, weights, center):
        self.sweeps += 1
        return nb.moments_basis(self.get_state(), bits, [np.reshape(m, (2, 2)) for m in mats], weights, center)[0]

    def moments_floats(self, bits, weights, center):
        return nb.moments_basis(self.get_state(), bits, [np.eye(2)] * len(bits), weights, center)[0]


class _StandIn(QEngineRestate):
    def _make_backend(self, n_qubits):
        return _StandInBackend(n_qubits, self.precision)


def _engine(psi, prec, doNorm=False):
    q = _StandIn(int(np.log2(len(psi))), 0, random.Random(1), 1.0 + 0j, doNorm, False, precision=prec)
    q.SetQuantumState(psi)
    return q


def _call(q, t):
    isExp, bits, form, ops, eig = parse_query(t)
    fn = q.ExpectationUnitaryAll if isExp else q.VarianceUnitaryAll
    return fn(bits, [m.reshape(-1).tolist() for m in ops] if form == "matrix" else ops, eig)


@pytest.mark.parametrize("prec", [32, 64])
def test_mirror_matches_the_compiled_reference(prec):
    psi, queries, results, posts = _fixture(prec)
    for i, (t, (_, (want,))) in enumerate(zip(queries, results)):
        q = _engine(psi, prec)
        got = _call(q, t)
        isExp, bits, form, ops, eig = parse_query(t)
        _, scale = nb.exp_var_unitary(psi, isExp, bits, nb.basis_mats(form, bits, ops), eig)
        assert abs(got - want) <= REF_REL_TOL[prec] * scale, (t[:2], got, want)
        assert q.be.sweeps == 1
        after = q.GetQuantumState()
        if "Matrix" in t[0]:
            assert np.array_equal(after, psi)  # read-only
        elif i in posts:
            assert np.abs(after - posts[i]).max() <= 4 * util.AMP_TOL[prec]


def test_mirror_edge_rules():
    psi = _fixture(64)[0]
    q = _engine(psi, 64)
    assert q.ExpectationUnitaryAll([], []) == 1.0 and q.VarianceUnitaryAll([], [[1, 0, 0, 1]]) == 1.0
    assert q.be.sweeps == 0
    angles = [0.3, -1.1, 2.0, 0.7, 0.2, -0.4]
    assert q.ExpectationUnitaryAll([4, 1], angles) == _engine(psi, 64).ExpectationUnitaryAll([4, 1], angles, [1, -1, 1, -1])
    m = [[1.2, 0.3j, -0.2, 0.9 + 0.1j]]
    assert q.VarianceUnitaryAll([6], m) == _engine(psi, 64).VarianceUnitaryAll([6], m, [1.0, -1.0])
    # doNormalize: the state is normalised before the sweep
    scaled = _engine(psi * 1.7, 64, doNorm=True)
    assert np.isclose(scaled.ExpectationUnitaryAll([2, 9, 5], angles + [0.1, 0.2, 0.3]),
                      _engine(psi, 64).ExpectationUnitaryAll([2, 9, 5], angles + [0.1, 0.2, 0.3]), rtol=0, atol=1e-12)
    assert np.isclose(np.vdot(scaled.GetQuantumState(), scaled.GetQuantumState()).real, 1.0)


def test_mirror_errors():
    q = _engine(_fixture(64)[0], 64)
    with pytest.raises(ValueError, match="duplicate"):
        q.ExpectationUnitaryAll([3, 3], [0.1] * 6)
    with pytest.raises(ValueError, match="within allocated qubit bounds"):
        q.VarianceUnitaryAll([12], [[1, 0, 0, 1]])
    with pytest.raises(ValueError, match="at least twice as many weights"):
        q.ExpectationUnitaryAll([1, 2], [0.1] * 6, [1.0, 2.0, 3.0])
    assert q.be.sweeps == 0


def test_mirror_takes_the_gate_route_past_twelve_qubits():
    rng = np.random.default_rng(9)
    psi = rng.standard_normal(1 << 13) + 1j * rng.standard_normal(1 << 13)
    psi /= np.linalg.norm(psi)
    q = _engine(psi, 64)
    angles = rng.uniform(-3, 3, 39).tolist()
    got = q.ExpectationUnitaryAll(list(range(13)), angles)
    assert q.be.sweeps == 0
    mats = nb.basis_mats("u3", list(range(13)), angles)
    assert abs(got - nb.exp_var_unitary(psi, True, list(range(13)), mats)[0]) < 1e-12
    assert np.abs(q.GetQuantumState() - nb.u3_post_state(psi, list(range(13)), angles)).max() < 1e-12


def test_query_ops_round_trip():
    """the matrix ops and the U3 ops with eigenvalues parse, are queries, dispatch to ExpectationUnitaryAll /
    VarianceUnitaryAll with the right arguments, and the C++ harness handles them"""
    _, queries, _, _ = _fixture(64)
    text = "qubits 12\n" + "".join(" ".join(t) + "\n" for t in queries)
    calls = []

    class Rec:
        def __getattr__(self, name):
            def f(*args):
                calls.append((name, args))
                return 0.5
            return f

    _, results = qscript.run(text, lambda n, p: Rec())
    assert {"ExpectationMatrixAll", "VarianceMatrixAll"} <= qscript.QUERY_OPS
    assert [r[0] for r in results] == [t[0] for t in queries]
    for t, (name, args) in zip(queries, calls):
        isExp, bits, form, ops, eig = parse_query(t)
        assert name == ("ExpectationUnitaryAll" if isExp else "VarianceUnitaryAll")
        assert args[0] == bits
        if form == "matrix":
            assert np.array_equal(np.array(args[1]).reshape(-1, 2, 2), np.array(ops))
        else:
            assert args[1] == ops
        assert list(args[2] if len(args) > 2 else []) == eig
    src = open(os.path.join(util.ROOT, "dropin", "observables_harness.cpp")).read()
    assert {"ExpectationMatrixAll", "VarianceMatrixAll"} <= set(re.findall(r'op == "(\w+)"', src))


def test_sharded_backend_refuses_the_primitive():
    be = _ShardedBackend.__new__(_ShardedBackend)
    with pytest.raises(NotImplementedError):
        be.moments_basis([0, 1], [[1, 0, 0, 1]] * 2, [1.0, -1.0] * 2, 0.0)
