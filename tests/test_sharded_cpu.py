"""World-size-2/4 `gloo` tests (CPU) of the one-process-per-GPU sharding logic (qrack_b200/sharded.py): the sharded
engine over oracle local engines must reproduce the single-engine oracle state on circuits that exercise local gates,
rank-bit diagonals, rank-bit controls and the all-to-all qubit exchange."""
import os
import random
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.restate_engine import QEngineRestate
from qrack_b200 import qscript

import util


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, text, prec, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle.sharded_cpu import restate_engine_factory
        from qrack_b200.sharded import QEngineSharded

        def make(n, perm):
            return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                                  device="cpu", make_engine=restate_engine_factory(prec))
        regs, results = qscript.run(text, make)
        st = regs[0].GetQuantumState()
        if rank == 0:
            np.savez(out_path, state=st, results=np.array([v for _, vals in results for v in vals], dtype=np.float64),
                     exchanges=regs[0].be.exchanges)
    finally:
        dist.destroy_process_group()


def run_sharded(text, world, prec, tmp_path):
    out = str(tmp_path / ("out_%d.npz" % world))
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), text, prec, out), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    z = np.load(out)
    return z["state"], z["results"], int(z["exchanges"])


CIRCUITS = {
    "htcnot": qscript.random_htcnot(9, 8, seed=4, timed=False) + "".join("Prob %d\n" % q for q in range(9)) + "ProbAll 5\nNorm\n",
    "u3": qscript.random_u3_cnot(8, 5, seed=2) + "ProbMask 195 129\nProbParity 77\nGetAmplitude 9\n",
    "qft": qscript.qft(8, seed=3, timed=False) + "IQFT 1 6\nProb 7\nProb 0\n",
    "misc": "qubits 8\n" + "".join("H %d\n" % q for q in range(8)) + "T 7\nCZ 7 0\nCNOT 7 1\nCNOT 1 7\nAntiCNOT 6 7\nCCNOT 0 7 6\n"
            "Swap 7 2\nZMask 200\nPhaseParity 0.7 193\nPhaseRootNMask 3 224\nXMask 192\nMCMtrx 2 7 3 6 0.6 0 0 0.8 0 -0.8 0.6 0\n"
            "ForceM 7 1\nH 7\nProb 7\nProbReg 5 3 5\nNorm\n",
}


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("name", sorted(CIRCUITS))
def test_sharded_matches_single_engine(name, world, tmp_path):
    prec = 32
    text = CIRCUITS[name]
    want, wres = util.run_engine(text, QEngineRestate, prec)
    got, gres, exchanges = run_sharded(text, world, prec, tmp_path)
    d = float(np.abs(got.astype(np.complex128) - want[0].astype(np.complex128)).max())
    assert d <= util.AMP_TOL[prec], "%s world=%d: max |delta amp| = %.3e" % (name, world, d)
    flat = np.array([v for _, vals in wres for v in vals], dtype=np.float64)
    # scalar queries are fp32 reductions with a different summation tree (per-rank partials + all_reduce)
    assert (np.abs(gres - flat).max() <= 5e-6) if flat.size else True
    if name in ("htcnot", "u3"):
        assert exchanges >= 1   # these circuits put non-diagonal gates on rank-bit qubits


def _worker_sampling(rank, world, port, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle.sharded_cpu import restate_engine_factory
        from qrack_b200.sharded import QEngineSharded
        # rgp=None: the unseeded default must still draw the same numbers on every rank (seed broadcast from rank 0)
        q = QEngineSharded(7, 0, None, 1.0 + 0j, precision=32, dist=dist, world=world, rank=rank, device="cpu",
                           make_engine=restate_engine_factory(32))
        for b in range(7):
            q.H(b)
        q.CNOT(6, 0)                      # exchange: the qubit map is permuted afterwards
        q.T(5)
        pma = q.ProbMaskAll(0b1100001)
        hp_state = None
        outcomes = [int(q.M(b)) for b in (6, 5, 0)]       # rank-bit and local qubits, unforced
        perm = q.MAll()
        amp = q.GetAmplitude(perm)
        q.SetPermutation(0b1010101)
        hp = q.HighestProbAll()
        unsupported = 0
        for call in (lambda: q.ForceMParity(3, True), lambda: q.INCC(1, 0, 3, 4)):
            try:
                call()
            except NotImplementedError:
                unsupported += 1
        np.savez(out_path + ".%d.npz" % rank, pma=pma, outcomes=np.array(outcomes), perm=perm, amp=np.array([amp.real, amp.imag]),
                 hp=hp, unsupported=unsupported)
    finally:
        dist.destroy_process_group()


def test_sampling_and_unseeded_rng_are_rank_consistent(tmp_path):
    world = 4
    out = str(tmp_path / "samp")
    mp.spawn(_worker_sampling, args=(world, _free_port(), out), nprocs=world, join=True)
    z = [np.load(out + ".%d.npz" % r) for r in range(world)]
    for r in range(1, world):
        assert (z[r]["outcomes"] == z[0]["outcomes"]).all() and int(z[r]["perm"]) == int(z[0]["perm"])
    # uniform superposition (CNOT permutes it, T is a phase): every 3-qubit marginal entry is 1/8
    assert np.allclose(z[0]["pma"], 1.0 / 8, atol=1e-6)
    perm = int(z[0]["perm"])
    o = z[0]["outcomes"]
    assert ((perm >> 6) & 1, (perm >> 5) & 1, perm & 1) == (int(o[0]), int(o[1]), int(o[2]))   # MAll respects the collapsed qubits
    assert abs(complex(*z[0]["amp"])) > 0.99                                                   # and leaves |perm>
    assert int(z[0]["hp"]) == 0b1010101
    assert int(z[0]["unsupported"]) == 2


def test_grover_on_sharded_engine_follows_success_law(tmp_path):
    """BASELINE configs[4] at test size: gate-level INC/DEC + ZeroPhaseFlip across rank bits (8 qubits over 4 ranks)."""
    import math
    n, it = 8, 3
    text = qscript.grover(n, it, target=3, timed=False)
    want, wres = util.run_engine(text, QEngineRestate, 32)
    got, gres, exchanges = run_sharded(text, 4, 32, tmp_path)
    d = float(np.abs(got.astype(np.complex128) - want[0].astype(np.complex128)).max())
    assert d <= util.AMP_TOL[32], d
    law = math.sin((2 * it + 1) * math.asin(2.0 ** (-n / 2.0))) ** 2
    assert abs(float(gres[0]) - law) < 1e-5


# 40 gate layers on 10 qubits, then controls and phases across the rank bits: many exchanges at 4 ranks
DEEP = qscript.random_htcnot(10, 24, seed=9, timed=False) + qscript.random_u3_cnot(10, 8, seed=5).split("\n", 1)[1]
DEEP += "CCNOT 9 8 0\nMCPhase 2 9 1 8 0.6 0.8 1 0\nAntiCNOT 8 9\n" + "".join("Prob %d\n" % q for q in range(10))


@pytest.mark.parametrize("defer", ["0", "1"])
def test_deep_circuit_in_order_and_deferred_exchanges(defer, tmp_path, monkeypatch):
    """40 gate layers on 10 qubits over 4 ranks: both exchange policies (in-order, and deferral of the gates blocked by a
    rank-bit target with commutation-aware look-ahead) must reproduce the single-engine oracle."""
    monkeypatch.setenv("B200SV_SHARD_DEFER", defer)
    text = DEEP
    want, wres = util.run_engine(text, QEngineRestate, 32)
    got, gres, exchanges = run_sharded(text, 4, 32, tmp_path)
    d = float(np.abs(got.astype(np.complex128) - want[0].astype(np.complex128)).max())
    assert d <= util.AMP_TOL[32], "defer=%s: max |delta amp| = %.3e" % (defer, d)
    flat = np.array([v for _, vals in wres for v in vals], dtype=np.float64)
    assert np.abs(gres - flat).max() <= 5e-6
    assert exchanges >= 2


def test_deferral_cuts_exchanges_on_the_benchmark_circuit():
    """Host-only dry run of the planner (scripts/shard_plan_count.py) on BASELINE's random circuit at 8 ranks (33
    qubits, 1960 gates): deferral must need far fewer exchanges than in-order execution (24 -> 7 when written)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("shard_plan_count", os.path.join(util.ROOT, "scripts", "shard_plan_count.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    text = qscript.random_htcnot(33, 40, seed=20250921, timed=False)
    before = os.environ.get("B200SV_SHARD_DEFER")
    try:
        in_order = m.count(30, 8, text, False)
        deferred = m.count(30, 8, text, True)
    finally:
        if before is None:
            os.environ.pop("B200SV_SHARD_DEFER", None)
        else:
            os.environ["B200SV_SHARD_DEFER"] = before
    # (local gate CALLS differ between the policies: a gate controlled by a rank-bit qubit is skipped on the ranks where
    # the control is not satisfied, and which qubits are rank bits at that moment depends on the exchange schedule)
    assert deferred[0] * 2 <= in_order[0], (in_order, deferred)
    assert deferred[1] < in_order[1]           # fewer, longer local fused windows


# ---- the sharded scheduler over a local engine running the real fused planner + host interpreter -------------------------------
def _worker_emu(rank, world, port, text, prec, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import math
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from emu_shard import EmuP2PShard
        from qrack_b200 import sharded

        class Eng(sharded.QEngineSharded):
            def _make_backend(self, n_qubits):
                k = int(round(math.log2(world)))
                return sharded._ShardedBackend(n_qubits, prec, EmuP2PShard(n_qubits - k, prec, dist, world, rank), dist, world, rank)

        def make(n, perm):
            return Eng(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank, device="cpu")
        regs, results = qscript.run(text, make)
        st = regs[0].GetQuantumState()
        if rank == 0:
            np.savez(out_path, state=st, results=np.array([v for _, vals in results for v in vals], dtype=np.float64),
                     exchanges=regs[0].be.exchanges, flushes=regs[0].be.shard.stats()["flushes"])
    finally:
        dist.destroy_process_group()


def _run_emu(text, world, prec, tmp_path):
    out = str(tmp_path / ("emu_%d.npz" % world))
    for attempt in range(3):
        try:
            mp.spawn(_worker_emu, args=(world, _free_port(), text, prec, out), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    return np.load(out)


@pytest.mark.parametrize("world,prec,kind", [(2, 32, "htcnot"), (4, 32, "htcnot"), (2, 64, "qv"), (4, 32, "qv"), (2, 32, "grover"), (2, 32, "u3")])
def test_sharded_scheduler_on_fused_planner_matches_single_engine(world, prec, kind, tmp_path):
    """The sharded scheduler over gloo with P2P exchange semantics, its local engine running the real fused planner, encoder and
    host interpreter of the sweep programs: the rank-specialised gates it submits (rank-bit controls resolved per rank, diagonal
    gates on a rank-bit qubit folded into a phase or a scalar) go through the planner the CUDA engine runs.  16 local qubits =
    8 tiles per sweep, several sweeps per window.  Same result as one engine."""
    k = world.bit_length() - 1
    n = 16 + k
    text = {"htcnot": lambda: qscript.random_htcnot(n, 14, seed=21, timed=False),
            "qv": lambda: qscript.quantum_volume(n, depth=5, seed=9, timed=False),
            "u3": lambda: qscript.random_u3_cnot(n, 6, seed=4),
            "grover": lambda: "\n".join(l for l in qscript.grover(n, 1, target=5, timed=False).splitlines() if not l.startswith("ProbAll")) + "\n"}[kind]()
    text += "".join("Prob %d\n" % q for q in (0, 3, n - 2, n - 1)) + "Norm\n"
    want, wres = util.run_engine(text, QEngineRestate, prec)
    flat = np.array([v for _, vals in wres for v in vals], dtype=np.float64)
    z = _run_emu(text, world, prec, tmp_path)
    d = float(np.abs(z["state"].astype(np.complex128) - want[0].astype(np.complex128)).max())
    assert d <= util.AMP_TOL[prec], "%s world=%d: max |delta amp| = %.3e" % (kind, world, d)
    # scalar queries: fp32 engines round differently gate by gate (the oracle applies 2x2s one at a time, the sweeps fuse them): the
    # norm of a deep fp32 circuit drifts by ~2e-5 either way; the amplitude bound above is the parity criterion
    assert np.abs(z["results"] - flat).max() <= (5e-5 if prec == 32 else 1e-10)
    assert int(z["exchanges"]) >= 1
