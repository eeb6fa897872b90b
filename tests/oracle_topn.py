"""The oracle of the n most probable basis states and the scripts it is pinned on (test infrastructure).

`QEngineRestateTopn` is oracle.restate_engine.QEngineRestate with QInterface::HighestProbAll(n) restated literally as the
reference's loop over ProbAll (src/qinterface/qinterface.cpp:962-1003), early exit included, in the engine's real type.
`topn_cases` lists the circuits and queries of tests/golden/ref_topn_12q.*.npz."""
import math

from oracle.restate_engine import QEngineRestate

import oracle_observables

N = 12
# H and X as U angles (the harness has only U and CNOT).  For H the angle is pi / 2, at which cos(theta / 2) and sin(theta / 2)
# round to the same float; in double they differ by one ulp (tests/test_topn_cpu.py counts the ties either way).
H_U = (math.pi / 2, 0.0, math.pi)
X_U = (math.pi, 0.0, math.pi)


class QEngineRestateTopn(QEngineRestate):
    def HighestProbAllN(self, n):  # qinterface.cpp:962-1003
        """the reference's loop as written: insertion into n default slots (perm 0, prob 0) where a probability never displaces
        an equal one, and the exit once the last slot's probability exceeds 1 - (the running sum)"""
        n = int(n)
        if not n:
            return []
        if n == 1:
            return [self.HighestProbAll()]
        if n > self.maxQPower:
            raise ValueError("QInterface::HighestProbAll(n) requested more !")
        totProb = self.real(0)
        highest = [(0, self.real(0))] * n
        for p in range(self.maxQPower):
            prob = self.real(self.ProbAll(p))
            totProb = self.real(totProb + prob)
            for t in range(n):
                if prob <= highest[t][1]:
                    continue
                highest[t + 1:] = highest[t:n - 1]
                highest[t] = (p, prob)
                break
            if highest[-1][1] > self.real(self.real(1) - totProb):
                break
        return [perm for perm, _ in highest]


def _u(q, a):
    return "U %d %.17g %.17g %.17g\n" % ((q,) + a)


def topn_cases(n=N):
    """(name, circuit, [query sizes]) of the fixture: the observables fixture's U3 + CNOT state; H on six qubits and U3 on the
    rest, no entangling gate (blocks of equal probability: the tie order); the basis state |5> (zero fill); GHZ (two states)"""
    circ = oracle_observables.observables_circuit(n)
    ties = "qubits %d\n" % n
    for q in range(n):
        ties += _u(q, H_U) if q in (0, 2, 3, 7, 8, 11) else _u(q, (0.3 + 0.21 * q, 0.1 * q, -0.2 * q))
    basis = "qubits %d\n" % n + _u(0, X_U) + _u(2, X_U)
    ghz = "qubits %d\n" % n + _u(0, H_U) + "".join("CNOT 0 %d\n" % q for q in range(1, n))
    return [("u3cnot", circ, [2, 3, 17, 100, 1 << n]), ("ties", ties, [2, 3, 64, 100]), ("basis5", basis, [3]),
            ("ghz", ghz, [4])]


def topn_text(circuit, sizes):
    """a circuit, then one HighestProbAllN per size"""
    return circuit + "".join("HighestProbAllN %d\n" % k for k in sizes)
