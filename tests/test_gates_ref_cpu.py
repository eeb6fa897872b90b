"""The gate families the sharded engine gained, on one engine, against the reference's own QEngineCPU
(tests/golden/ref_gates_9q.f{32,64}.npz, written by tests/golden/make_gates.py): the oracle restatement behind the dispatch
mirror returns the reference's state, including CUniformParityRZ with controls inside its mask, whose parity the reference
takes over the non-control bits only."""
import pytest

from qrack_b200 import qscript

import oracle_gates
import test_sharded_gates_cpu as tgc
import util


@pytest.mark.parametrize("prec", [32, 64])
def test_oracle_matches_the_reference_gate_fixture(prec):
    ref = tgc.ref_gates(prec)
    scripts = oracle_gates.ref_scripts()
    assert sorted(ref) == sorted(scripts)
    for name, text in scripts.items():
        regs, _ = qscript.run(text, util.make_factory(oracle_gates.QEngineRestateGates, prec))
        util.assert_states_close({0: regs[0].GetQuantumState()}, {0: ref[name]}, prec, name)


def test_cuniform_parity_rz_leaves_controls_out_of_the_parity():
    """the mask handed to the backend excludes the controls (state.cpp:1239-1261)"""
    calls = []
    q = oracle_gates.QEngineRestateGates(4, 0, None, 1.0 + 0j, False, False, precision=64)
    q.be.uniform_parity_rz = lambda cm, mask, angle: calls.append((cm, mask, angle))
    q.CUniformParityRZ([0, 2], 0b1101, 0.5)
    q.UniformParityRZ(0b1101, 0.25)
    assert calls == [(0b101, 0b1000, 0.5), (0, 0b1101, 0.25)]
