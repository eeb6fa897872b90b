"""The oracle of the reduced density matrix and the script it is pinned on (test infrastructure).

`QEngineRestateRdm` is oracle.restate_engine.QEngineRestate with QInterface::GetReducedDensityMatrix restated literally as the
reference's loop over GetAmplitude (src/qinterface/qinterface.cpp:886-944), accumulated in the engine's complex type.
`rdm_text` is the 12-qubit U3 + CNOT circuit of the observables fixture followed by the queries of
tests/golden/ref_rdm_12q.*.npz."""
import numpy as np

from oracle.restate_engine import QEngineRestate

import oracle_observables


class QEngineRestateRdm(QEngineRestate):
    def GetReducedDensityMatrix(self, qubits):  # qinterface.cpp:886-944
        """the reference's loop as written: for every environment state and every pair of kept states one GetAmplitude each,
        accumulated into a complex matrix of the engine's type in environment order"""
        nQubits, kept = self.qubitCount, [int(q) for q in qubits]
        dimKept = 1 << len(kept)
        envBitPos = [q for q in range(nQubits) if q not in kept]
        out = np.zeros((dimKept, dimKept), dtype=self.cplx)
        for envState in range(1 << len(envBitPos)):
            envBaseIndex = 0
            for e, b in enumerate(envBitPos):
                if (envState >> e) & 1:
                    envBaseIndex |= 1 << b
            full = []
            for kept_i in range(dimKept):
                idx = envBaseIndex
                for k, b in enumerate(kept):
                    if (kept_i >> k) & 1:
                        idx |= 1 << b
                full.append(idx)
            for kept_i in range(dimKept):
                amp_i = self.cplx(self.GetAmplitude(full[kept_i]))
                for kept_j in range(dimKept):
                    out[kept_i, kept_j] += amp_i * np.conj(self.cplx(self.GetAmplitude(full[kept_j])))
        return out


def rdm_queries():
    """the kept sets of tests/golden/ref_rdm_12q.*.npz: k in {0, 1, 2, 3, 5, 7}; qubit 0 kept (the two amplitudes of an fp32
    16-byte chunk are two rows) and not kept (two columns); the top qubit; both sides of the byte boundary; unsorted lists"""
    sets = [[], [0], [11], [7, 8], [9, 0, 4], [3, 11, 1], [5, 0, 11, 7, 2], [10, 3, 8, 0, 6, 11, 1]]
    return "".join("GetReducedDensityMatrix %d %s\n" % (len(b), " ".join(str(q) for q in b)) for b in sets)


def rdm_circuit(n=12):
    """the circuit of tests/golden/ref_observables_12q.*.npz"""
    return oracle_observables.observables_circuit(n)


def rdm_text(n=12):
    """the circuit, then every reduced density matrix query"""
    return rdm_circuit(n) + rdm_queries()
