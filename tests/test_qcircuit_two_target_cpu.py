"""QCircuit records the two-target gate forms (ISwap, IISwap, SqrtSwap, ISqrtSwap, FSim, CSwap, AntiCSwap) as three single-target
gates each, replays them like the gates themselves, and QEngineCUDA.RunCircuit still submits the whole circuit in one
b200sv_apply_gates call (checked against a stand-in library whose batch is run through the fused-sweep emulation)."""
import ctypes
import random

import numpy as np

from oracle.restate_engine import QEngineRestate
from qrack_b200 import QCircuit, _abi
from qrack_b200.qengine import QEngineCUDA

N = 8


def _gates(q):
    """the two-target forms on local pairs, with controls, in both orders; returns how many single-target gates each adds"""
    q.H(0)
    q.H(3)
    q.U(5, 0.4, 0.3, -0.2)
    q.ISwap(0, 5)
    q.IISwap(6, 1)
    q.SqrtSwap(3, 7)
    q.ISqrtSwap(2, 0)
    q.FSim(0.8, -0.6, 4, 1)
    q.FSim(1.2, 0.0, 2, 7)
    q.CSwap([1, 6], 0, 3)
    q.AntiCSwap([2], 7, 5)
    q.Swap(4, 6)
    return 3 + 3 * 4 + (3 + 1) + 3 + 3 + 3 + 3


def test_qcircuit_records_two_target_forms_as_three_gates():
    for prec in (32, 64):
        c = QCircuit(N, prec)
        want_count = _gates(c)
        assert c.GetGateCount() == want_count
        for off1, off2, pmask, m in c.be.gates:
            d = off1 ^ off2
            assert d and not (d & (d - 1)) and (off1 | off2) & ~pmask == 0
        q = QEngineRestate(N, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
        c.Run(q)
        ref = QEngineRestate(N, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
        _gates(ref)
        d = float(np.abs(q.GetQuantumState().astype(np.complex128) - ref.GetQuantumState().astype(np.complex128)).max())
        assert d <= (1e-6 if prec == 32 else 1e-12), (prec, d)


def test_run_circuit_submits_two_target_forms_in_one_call():
    """RunCircuit hands the recorded gates to the backend in one apply_gates call; that batch, run through the real fused
    planner and the host interpreter of its sweep programs, gives the state of the gates run one by one"""
    c = QCircuit(N, 64)
    _gates(c)
    calls = []

    class Be:
        def is_zero(self):
            return False

        def apply_gates(self, n, o1, o2, pm, m8):
            calls.append((n, o1, o2, pm, m8))
    q = object.__new__(QEngineCUDA)
    q.doNormalize, q.qubitCount, q.precision, q.be = False, N, 64, Be()
    q.RunCircuit(c)
    assert len(calls) == 1 and calls[0][0] == c.GetGateCount()
    st = np.zeros(1 << N, dtype=np.complex128)
    st[0] = 1
    rc = _abi.load().b200sv_emulate_fused(N, 64, *calls[0], st.ctypes.data_as(ctypes.c_void_p))
    assert rc == _abi.B200SV_OK
    ref = QEngineRestate(N, 0, random.Random(1), 1.0 + 0j, False, False, precision=64)
    _gates(ref)
    assert np.abs(st - ref.GetQuantumState()).max() <= 1e-12
