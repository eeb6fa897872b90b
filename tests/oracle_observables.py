"""The oracle of the observable queries and the script they are pinned on (test infrastructure).

`QEngineRestateObs` is oracle.restate_engine.QEngineRestate with the QInterface observable methods restated literally as the
reference's loops over ProbAll (src/qinterface/qinterface.cpp:478-806), in the engine's real type where the reference rounds
to real1_f.  `observables_text` is the 12-qubit U3 + CNOT circuit and query list of tests/golden/ref_observables_12q.*.npz."""
import math
import random

import numpy as np

from oracle.restate_engine import QEngineRestate
from qrack_b200 import qscript


class QEngineRestateObs(QEngineRestate):
    def _check(self, bits, table, what, tname):
        if len(table) < 2 * len(bits):
            raise ValueError("QInterface::%s() must supply at least twice as many %s as bits!" % (what, tname))
        msg = "QInterface::%s() parameter qubits vector values must be within allocated qubit bounds!" % what
        if any(b < 0 or b >= self.qubitCount for b in bits):
            raise ValueError(msg)
        if len(set(bits)) != len(bits):
            raise ValueError(msg + " (Found duplicate qubit indices!)")

    def ExpectationBitsFactorized(self, bits, perms, offset=0):  # qinterface.cpp:542-577
        bits, perms = list(bits), [int(v) for v in perms]
        self._check(bits, perms, "ExpectationBitsFactorized", "'perms'")
        if not bits:
            return 1.0
        if len(bits) == 1:
            prob = self.Prob(bits[0])
            return self._r(float(perms[0] + offset) * (1.0 - prob) + float(perms[1] + offset) * prob)
        r = self.real(0)
        for lcv in range(self.maxQPower):
            ret = offset
            for p, b in enumerate(bits):
                ret += perms[2 * p + 1] if (lcv >> b) & 1 else perms[2 * p]
            r += self.real(float(ret) * self.ProbAll(lcv))
        return float(r)

    def VarianceBitsFactorized(self, bits, perms, offset=0):  # :579-618
        bits, perms = list(bits), [int(v) for v in perms]
        self._check(bits, perms, "VarianceBitsFactorized", "'perms'")
        if not bits:
            return 1.0
        mean = self.ExpectationBitsFactorized(bits, perms, offset)
        if len(bits) == 1:
            prob = self.Prob(bits[0])
            d0, d1 = self._r(float(perms[0] + offset) - mean), self._r(float(perms[1] + offset) - mean)
            return self._r(d0 * d0 * (1.0 - prob) + d1 * d1 * prob)
        r = self.real(0)
        for lcv in range(self.maxQPower):
            ret = offset
            for p, b in enumerate(bits):
                ret += perms[2 * p + 1] if (lcv >> b) & 1 else perms[2 * p]
            d = self.real(self.real(float(ret)) - self.real(mean))
            r += self.real(d * d * self.real(self.ProbAll(lcv)))
        return float(r)

    def ExpectationBitsAll(self, bits, offset=0):  # qinterface.hpp:210-219
        perms = []
        for i in range(len(bits)):
            perms += [0, 1 << i]
        return self.ExpectationBitsFactorized(bits, perms, offset)

    def VarianceBitsAll(self, bits, offset=0):
        perms = []
        for i in range(len(bits)):
            perms += [0, 1 << i]
        return self.VarianceBitsFactorized(bits, perms, offset)

    def _weight(self, lcv, bits, weights):
        w = self.real(1)
        for p, b in enumerate(bits):
            w = self.real(w * self.real(weights[2 * p + 1] if (lcv >> b) & 1 else weights[2 * p]))
        return w

    def ExpectationFloatsFactorized(self, bits, weights):  # :771-806
        bits, weights = list(bits), [self._r(w) for w in weights]
        self._check(bits, weights, "ExpectationFloatsFactorized", "weights")
        if not bits:
            return 1.0
        if len(bits) == 1:
            prob = self.Prob(bits[0])
            return self._r(weights[0] * (1.0 - prob) + weights[1] * prob)
        r = self.real(0)
        for lcv in range(self.maxQPower):
            r += self.real(self._weight(lcv, bits, weights) * self.real(self.ProbAll(lcv)))
        return float(r)

    def VarianceFloatsFactorized(self, bits, weights):  # :620-657 (the k >= 2 sum is unsquared there, :653)
        bits, weights = list(bits), [self._r(w) for w in weights]
        self._check(bits, weights, "VarianceFloatsFactorized", "weights")
        if not bits:
            return 1.0
        mean = self.ExpectationFloatsFactorized(bits, weights)
        if len(bits) == 1:
            prob = self.Prob(bits[0])
            v0, v1 = self._r(weights[0] - mean), self._r(weights[1] - mean)
            return self._r(v0 * v0 * (1.0 - prob) + v1 * v1 * prob)
        r = self.real(0)
        for lcv in range(self.maxQPower):
            r += self.real((self._weight(lcv, bits, weights) - self.real(mean)) * self.real(self.ProbAll(lcv)))
        return float(r)

    def _pauli_all(self, isExp, bits, paulis):  # :659-769
        bits, paulis = [int(b) for b in bits], [int(p) for p in paulis]
        i = 0
        while i < len(bits):  # erases while re-reading bits.size(): some PauliI survive (and weigh like PauliZ)
            j = len(bits) - (i + 1)
            if paulis[j] == 0:
                del bits[j]
                del paulis[j]
            i += 1
        kept = list(zip(bits, paulis))
        if not kept:
            return 1.0
        for b, p in kept:
            if p == 1:
                self.H(b)
            elif p == 3:
                self.IS(b)
                self.H(b)
        qs = [b for b, _ in kept]
        ev = [1.0, -1.0] * len(qs)
        r = self.ExpectationFloatsFactorized(qs, ev) if isExp else self.VarianceFloatsFactorized(qs, ev)
        for b, p in kept:
            if p == 1:
                self.H(b)
            elif p == 3:
                self.H(b)
                self.S(b)
        return r

    def ExpectationPauliAll(self, bits, paulis):
        return self._pauli_all(True, bits, paulis)

    def VariancePauliAll(self, bits, paulis):
        return self._pauli_all(False, bits, paulis)

    def _unitary_all(self, isExp, bits, basisOps, eigenVals=()):  # :478-540
        bits = list(bits)
        if not bits:
            return 1.0
        ev = list(eigenVals) if eigenVals else [1.0, -1.0] * len(bits)
        mtrx = hasattr(basisOps[0], "__len__")
        for i, b in enumerate(bits):
            if mtrx:
                m = [complex(v) for v in basisOps[i]]
                det = 1.0 / (m[0] * m[3] - m[1] * m[2])
                self.Mtrx([det * m[3], det * -m[1], det * -m[2], det * m[0]], b)
            else:
                self.U(b, -basisOps[3 * i], -basisOps[3 * i + 1], -basisOps[3 * i + 2])
        r = self.ExpectationFloatsFactorized(bits, ev) if isExp else self.VarianceFloatsFactorized(bits, ev)
        for i, b in enumerate(bits):
            if mtrx:
                self.Mtrx([complex(v) for v in basisOps[i]], b)
            else:
                self.U(b, basisOps[3 * i], basisOps[3 * i + 1], basisOps[3 * i + 2])
        return r

    def ExpectationUnitaryAll(self, bits, basisOps, eigenVals=()):
        return self._unitary_all(True, bits, basisOps, eigenVals)

    def VarianceUnitaryAll(self, bits, basisOps, eigenVals=()):
        return self._unitary_all(False, bits, basisOps, eigenVals)


def _cs(bits):
    return "%d %s" % (len(bits), " ".join(str(b) for b in bits))


def observables_queries(n=12, seed=4242):
    """One line per query op: k in {1, 2, 5, n}, qubits on both sides of the byte boundary (7 | 8), nonzero offsets, mixed
    weights, Pauli strings with I / X / Y / Z and pure-Z strings, the U3 form of the Unitary queries."""
    rng = random.Random(seed)
    sets = [[3], [7, 8], [0, 7, 8, 11, 5], list(range(n))[::-1]]
    lines = []
    for bits in sets:
        cs = _cs(bits)
        for op in ("ExpectationBitsAll", "VarianceBitsAll"):
            lines.append("%s %s %d" % (op, cs, 5 if len(bits) > 1 else 0))
        perms = [rng.randrange(1 << 20) for _ in range(2 * len(bits))]
        for op in ("ExpectationBitsFactorized", "VarianceBitsFactorized"):
            lines.append("%s %s %d %s" % (op, cs, 1000 + len(bits), " ".join(map(str, perms))))
        ws = ["%.9g" % rng.uniform(-1.5, 1.5) for _ in range(2 * len(bits))]
        for op in ("ExpectationFloatsFactorized", "VarianceFloatsFactorized"):
            lines.append("%s %s %s" % (op, cs, " ".join(ws)))
        paulis = [rng.choice([0, 1, 2, 3]) for _ in bits]
        if len(bits) > 1:
            paulis[0], paulis[1] = 3, 1   # at least one Y and one X
        zs = [2] * len(bits)
        for op in ("ExpectationPauliAll", "VariancePauliAll"):
            lines.append("%s %s %s" % (op, cs, " ".join(map(str, paulis))))
            lines.append("%s %s %s" % (op, cs, " ".join(map(str, zs))))
        angles = ["%.9g" % rng.uniform(-math.pi, math.pi) for _ in range(3 * len(bits))]
        for op in ("ExpectationUnitaryAll", "VarianceUnitaryAll"):
            lines.append("%s %s %s" % (op, cs, " ".join(angles)))
    return "\n".join(lines) + "\n"


def observables_circuit(n=12):
    return qscript.random_u3_cnot(n, 6, seed=91)


def observables_text(n=12):
    """the circuit, then every query"""
    return observables_circuit(n) + observables_queries(n)


def results_values(results):
    return np.array([v[0] for _, v in results])
