"""The gate scripts of tests/test_sharded_gates_cpu.py (two-target gates, (C)UniformParityRZ, UniformlyControlledSingleBit / RY /
RZ, the misc_8q fixture) on the sharded engine over real CUDA pages, W ranks on ONE device (tests/one_device.py), in the push,
pull and staged exchange modes, both precisions, against the float64 oracle; and QEngineCUDA.RunCircuit of an FSim circuit."""
import random

import numpy as np
import pytest

from qrack_b200 import QCircuit, qscript

import one_device
import oracle_gates
import test_sharded_gates_cpu as tgc
import util

pytestmark = pytest.mark.gpu

CASES = [(w, p, m) for w in (2, 4, 8) for m in ("push", "pull", "staged") for p in (32, 64)]


@pytest.mark.parametrize("world,prec,mode", CASES, ids=["w%d-fp%d-%s" % c for c in CASES])
def test_sharded_gates_on_one_device_match_the_oracle(world, prec, mode, tmp_path):
    one_device.spawn(tgc.run_ranks, world, prec, "cuda", mode, str(tmp_path))
    z = [dict(np.load(str(tmp_path / ("gates.%d.npz" % r)))) for r in range(world)]
    d = tgc.check_ranks(z, world, prec)
    print("\n[sharded gates] w%d fp%d %s: max |delta amp| %.2e (tol %.0e)" % (world, prec, mode, d, util.AMP_TOL[prec]))


def fsim_circuit(n, layers, seed):
    """FSim on a random matching per layer, U3 on every qubit between layers"""
    rng = random.Random(seed)
    text = "qubits %d\n" % n
    for _ in range(layers):
        for q in range(n):
            text += "U %d %.17g %.17g %.17g\n" % (q, rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3))
        for a, b in qscript.random_matching(rng, n):
            text += "FSim %.17g %.17g %d %d\n" % (rng.uniform(-3, 3), rng.uniform(-3, 3), a, b)
    return text


@pytest.mark.parametrize("prec", [32, 64])
def test_run_circuit_of_fsim_layers_matches_the_oracle(prec):
    """a 20-qubit FSim circuit recorded in a QCircuit runs in one b200sv_apply_gates submission on QEngineCUDA and matches
    the float64 oracle"""
    from qrack_b200 import QEngineCUDA
    n = 20
    text = fsim_circuit(n, 6, seed=4)
    c = QCircuit(n, prec)
    qscript.run(text, lambda nq, p: c)
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    q.be.reset_stats()
    calls = []
    submit = q.be.apply_gates
    q.be.apply_gates = lambda *a: (calls.append(a[0]), submit(*a))
    q.RunCircuit(c)
    got = q.GetQuantumState()
    st = q.be.stats()
    assert calls == [c.GetGateCount()] and st["gates_submitted"] == c.GetGateCount(), (calls, st)
    regs, _ = qscript.run(text, util.make_factory(oracle_gates.QEngineRestateGates, 64))
    d = float(np.abs(got.astype(np.complex128) - regs[0].GetQuantumState()).max())
    assert d <= util.AMP_TOL[prec], d


@pytest.mark.parametrize("prec", [32, 64])
def test_single_engine_matches_the_reference_gate_fixture(prec):
    """QEngineCUDA runs the scripts of tests/golden/ref_gates_9q.*.npz to the reference's states"""
    from qrack_b200 import QEngineCUDA
    for name, st in tgc.ref_gates(prec).items():
        regs, _ = qscript.run(oracle_gates.ref_scripts()[name], util.make_factory(QEngineCUDA, prec))
        util.assert_states_close({0: regs[0].GetQuantumState()}, {0: st}, prec, name)
