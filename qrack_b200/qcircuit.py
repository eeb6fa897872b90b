"""QCircuit — a recorded gate list that an engine runs in ONE call (SURVEY 8f N4).

The reference's ``QCircuit`` (``include/qcircuit.hpp:121-324``) holds a list of (target, controls, matrices) gates and
``QCircuit::Run(QInterfacePtr)`` (``src/qcircuit.cpp:173-281``) replays it on an engine gate by gate through the virtual
``MCMtrx/MACMtrx/Mtrx`` calls.  Here the gate list is recorded through the SAME host dispatch mirror the engines use
(``QEngineHost``: every ``QInterface``-named gate method — H, T, CNOT, U, MCMtrx, QFT, gate-level INC/DEC, ... — lowers to
``Apply2x2(offset1, offset2, mtrx, powers)`` exactly as ``src/qengine/qengine.cpp:19-75,212-460`` does) and handed to the engine
as arrays: ``QEngineCUDA.RunCircuit`` submits them through ``b200sv_apply_gates`` — one ABI call per circuit, so the fused
planner sees the whole window and the per-gate host round trip (7-11 us in this mirror) disappears.

    c = QCircuit(n)                 # records; has every gate method of QEngineHost
    c.H(0); c.CNOT(0, 1); c.QFT(0, n)
    c.Run(q)                        # q: QEngineCUDA (batched), or any QEngineHost (gate by gate, like the reference)
"""
from __future__ import annotations

import ctypes
import random
from typing import List, Tuple

from .qengine import QEngineHost, lower_two_target


class _RecordBackend:
    """Backend that records the single-target Apply2x2 forms the dispatch mirror produces; a two-target form (ISwap, SqrtSwap,
    FSim, CSwap, ...) is recorded as the three single-target gates of qengine.lower_two_target."""

    def __init__(self, n_qubits: int, precision: int):
        self.nq = n_qubits
        self.precision = precision
        self.gates: List[Tuple[int, int, int, tuple]] = []

    def is_zero(self) -> bool:
        return False

    def finish(self):
        pass

    def set_permutation(self, perm, phase):  # the constructor's initial state
        if self.gates:
            raise NotImplementedError("QCircuit: SetPermutation is not a gate")

    def apply2x2(self, off1, off2, mtrx, pows, nrm, thresh, calc_norm):
        diff = off1 ^ off2
        if calc_norm or nrm != 1.0:
            raise NotImplementedError("QCircuit: doNormalize bookkeeping cannot be recorded")
        pmask = 0
        for p in pows:
            pmask |= p
        if bin(diff).count("1") == 2:
            self.gates += [(o1, o2, pm, tuple(complex(z) for z in m)) for o1, o2, pm, m in lower_two_target(off1, off2, pmask, mtrx)]
            return None
        if not diff or (diff & (diff - 1)):
            raise NotImplementedError("QCircuit: only one- and two-target gate forms can be recorded")
        self.gates.append((off1, off2, pmask, tuple(complex(z) for z in mtrx)))
        return None

    def xmask(self, mask):
        # XMask = X on every masked qubit (QInterface::XMask, src/qinterface/gates.cpp); the engine's scheduler turns the
        # XMask ... XMask wrappers of anti-controlled gates into control polarities
        b = 0
        while mask >> b:
            if (mask >> b) & 1:
                self.gates.append((0, 1 << b, 1 << b, (0j, 1 + 0j, 1 + 0j, 0j)))
            b += 1

    def __getattr__(self, name):
        raise NotImplementedError("QCircuit: %r is not a gate that lowers to Apply2x2 (state access, measurement and the "
                                  "native sweeps are engine calls, not circuit elements)" % name)


class QCircuit(QEngineHost):
    """Records gates; ``Run(engine)`` replays them.  Construct with the qubit count (and the precision of the engines it
    will run on, because matrices are rounded to the engine's real type when lowered)."""

    def __init__(self, qBitCount: int, precision: int = 32):
        super().__init__(qBitCount, 0, random.Random(0), 1.0 + 0j, False, False, precision=precision)
        self._packed = None

    def _make_backend(self, n_qubits: int):
        return _RecordBackend(n_qubits, self.precision)

    def _has_alu(self) -> bool:
        return False  # INC/DEC in their gate-level QInterface form

    def GetGateCount(self) -> int:
        return len(self.be.gates)

    def packed(self):
        """(n, off1[], off2[], pmask[], mats8[]) as ctypes arrays, cached."""
        g = self.be.gates
        if self._packed is None or self._packed[0] != len(g):
            n = len(g)
            o1 = (ctypes.c_uint64 * max(n, 1))(*[x[0] for x in g])
            o2 = (ctypes.c_uint64 * max(n, 1))(*[x[1] for x in g])
            pm = (ctypes.c_uint64 * max(n, 1))(*[x[2] for x in g])
            m8 = (ctypes.c_double * max(8 * n, 1))()
            for i, x in enumerate(g):
                for k in range(4):
                    m8[8 * i + 2 * k] = x[3][k].real
                    m8[8 * i + 2 * k + 1] = x[3][k].imag
            self._packed = (n, o1, o2, pm, m8)
        return self._packed

    def Run(self, qsim):
        """QCircuit::Run: batched when the engine offers it, else one Apply2x2 per gate (what the reference does)."""
        if qsim.GetQubitCount() != self.qubitCount:
            raise ValueError("QCircuit::Run: qubit count differs from the engine's")
        if hasattr(qsim, "RunCircuit"):
            return qsim.RunCircuit(self)
        for off1, off2, pmask, m in self.be.gates:
            pows = [1 << b for b in range(pmask.bit_length()) if (pmask >> b) & 1]
            qsim.Apply2x2(off1, off2, list(m), len(pows), pows, False)
