"""The n most probable basis states on the CPU: the float64 reference (tests/npref_topn.py) and the literal QInterface loop of
the oracle (tests/oracle_topn.py) against what the compiled reference returned (tests/golden/ref_topn_12q.*), the early-exit
divergence, the script op, and the sharded backend's refusal."""
import os
import re

import numpy as np
import pytest

from qrack_b200 import qscript
from qrack_b200.sharded import _ShardedBackend

import npref_topn as no
import oracle_topn as ot
import util

# two entries whose reference probabilities agree this closely may come out swapped when the state they are read from differs
# from the reference's by rounding (the oracle's circuit); exactly equal probabilities never may
NEAR = {32: 2.0 ** -22, 64: 1e-15}


def _fixture(prec):
    return np.load(os.path.join(util.GOLDEN, "ref_topn_12q.f%d.npz" % prec))


def assert_same_up_to_near_ties(got, ref, p_ref, p_got, prec, what, slack=0.0):
    """got is ref up to swaps of near-ties: at every position the two entries' reference probabilities p_ref agree within NEAR
    relative (plus `slack`, absolute, for a state that differs from the reference's by more than rounding in one engine); and
    in the probabilities p_got of the state got was computed from, got never lists an exactly equal pair out of index order"""
    listed = got[:int((p_got > 0).sum())]  # what follows is the zero fill
    assert len(got) == len(ref) and len(set(listed)) == len(listed), what
    for t, (g, r) in enumerate(zip(got, ref)):
        a, b = p_ref[g], p_ref[r]
        assert abs(a - b) <= NEAR[prec] * max(a, b) + slack, (what, t, g, r, a, b)
    for t in range(1, len(listed)):
        if p_got[listed[t]] == p_got[listed[t - 1]]:
            assert listed[t] > listed[t - 1], (what, t, listed[t - 1], listed[t])


def test_cases_cover_the_code_paths():
    cases = {name: (circ, sizes) for name, circ, sizes in ot.topn_cases()}
    assert cases["u3cnot"][1] == [2, 3, 17, 100, 4096]
    assert cases["basis5"][1] == [3] and cases["ghz"][1] == [4]
    for prec in (32, 64):
        z = _fixture(prec)
        p = no.probs(z["state_ties"])
        _, counts = np.unique(p, return_counts=True)
        # fp32: cos(pi / 4) and sin(pi / 4) round to the same float, so the six H qubits give 64 blocks of 64 equal
        # probabilities; in double they differ by one ulp and the blocks split into smaller groups of exactly equal ones
        assert counts.max() == (64 if prec == 32 else 29) and (counts > 1).sum() >= 64
        assert list(z["top_basis5_3"]) == [5, 0, 0]
        assert list(z["top_ghz_4"]) == [0, 4095, 0, 0]


@pytest.mark.parametrize("prec", [32, 64])
def test_npref_matches_the_compiled_reference(prec):
    """on the reference's own states the float64 reference gives the reference's lists exactly, ties and zero fill included"""
    z = _fixture(prec)
    for name, _, sizes in ot.topn_cases():
        for k in sizes:
            assert no.top_n(z["state_" + name], k) == list(z["top_%s_%d" % (name, k)]), (name, k)


@pytest.mark.parametrize("prec", [32, 64])
def test_oracle_loop_matches_the_compiled_reference(prec):
    z = _fixture(prec)
    for name, circ, sizes in ot.topn_cases():
        states, results = util.run_engine(ot.topn_text(circ, sizes), ot.QEngineRestateTopn, prec)
        util.assert_states_close({0: states[0]}, {0: z["state_" + name]}, prec, "oracle circuit vs the reference's: " + name)
        p_ref, p_mine = no.probs(z["state_" + name]), no.probs(states[0])
        assert len(results) == len(sizes)
        for k, (op, vals) in zip(sizes, results):
            assert op == "HighestProbAllN"
            assert_same_up_to_near_ties([int(v) for v in vals], list(z["top_%s_%d" % (name, k)]), p_ref, p_mine, prec, (name, k))


def _unnormalised(prec):
    q = util.make_factory(ot.QEngineRestateTopn, prec)(2, 0)
    psi = np.sqrt(np.array([0.7, 0.6, 0.1, 0.8]))
    q.SetQuantumState(psi)
    return q, psi


@pytest.mark.parametrize("prec", [32, 64])
def test_early_exit_divergence(prec):
    """probabilities (0.7, 0.6, 0.1, 0.8), n = 2: the reference's loop has 0.6 > 1 - 1.3 after index 1 and stops with [0, 1];
    the exact top two are [3, 0]"""
    q, psi = _unnormalised(prec)
    assert q.HighestProbAllN(2) == [0, 1]
    assert no.top_n(psi.astype(q.cplx), 2) == [3, 0]


def test_npref_definition():
    """P = min(|psi|^2, 1): a clamped tie goes to the smaller index; P = 0 never listed, zero fill; fp32 squares in double"""
    psi = np.array([0.5, 1.2, 0.0, -1.1j, 0.5, 0.0], dtype=np.complex128)
    assert no.top_n(psi, 6) == [1, 3, 0, 4, 0, 0]
    f = np.array([np.float32(0.1) + 1j * np.float32(0.3)], dtype=np.complex64)
    assert no.probs(f)[0] == float(np.float32(0.1)) ** 2 + float(np.float32(0.3)) ** 2


def test_query_op_round_trip():
    """the op parses, is a query of the script format, dispatches to HighestProbAllN, and its result line (the n indices) is
    read back; the C++ harness handles the op"""
    calls = []

    class Rec:
        def HighestProbAllN(self, n):
            calls.append(n)
            return list(range(n, 0, -1))

        def __getattr__(self, name):
            return lambda *a: None

    text = ot.topn_text("qubits 3\nH 0\n", [2, 5])
    _, results = qscript.run(text, lambda n, p: Rec())
    assert "HighestProbAllN" in qscript.QUERY_OPS
    assert calls == [2, 5] and results == [("HighestProbAllN", (2.0, 1.0)), ("HighestProbAllN", (5.0, 4.0, 3.0, 2.0, 1.0))]
    line = "".join("%s %s\n" % (op, " ".join("%d" % v for v in vals)) for op, vals in results)
    assert qscript.parse_results(line) == results
    src = open(os.path.join(util.ROOT, "dropin", "observables_harness.cpp")).read()
    assert "HighestProbAllN" in re.findall(r'op == "(\w+)"', src)


def test_sharded_backend_refuses_the_primitive():
    be = _ShardedBackend.__new__(_ShardedBackend)
    with pytest.raises(NotImplementedError):
        be.highest_probs(3)
