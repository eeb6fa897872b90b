"""The sharded engine over real CUDA pages with W ranks on ONE device (tests/one_device.py: W processes on cuda:0, a loopback
gloo group, collectives staged through host copies, a barrier that synchronises the device).  Runs on a single H100, where
the multi-GPU tests skip; it puts together what no single-kernel test does: QEngineSharded on P2PShardBuffers (CUDA IPC
export/import of the pages, the push scatter, the pull gather that rides on the next fused sweep, partner pages read
through peer mappings) and on ShardBuffers over torch pages (the host-staged exchange, the engine rebound after each swap),
the keyed top-n and sampling searches with the logical-qubit key and the pending-inversion XOR the scheduler computes.

Every case (W ranks, precision, exchange mode) runs, in one spawn:
  * gate parity: tests/test_sharded_cpu.py's circuits, its deep deferral circuit, a 9-qubit circuit whose Belady victim
    is qubit 0 (inside an fp32 16-byte chunk), and a 20-qubit H/T/CNOT and quantum-volume circuit (>= 16 local qubits:
    multi-tile sweeps, several exchanges), then read-only queries; against the float64 oracle;
  * sampling, top-n and observables: the scripts and checkers of the CPU tests (and of the multi-GPU observables test);
  * at W = 8 in fp32: the 26-qubit circuits against what the compiled reference returned.
Pages are small on purpose: 9 qubits over 2, 4, 8 and 16 ranks leave 8 down to 5 local qubits.  Stream-ordering races
between ranks and the NCCL exchange are out of reach here (the barrier synchronises the device); the multi-GPU tests keep
those."""
import functools
import os
import random
import time

import numpy as np
import pytest

from oracle.restate_engine import QEngineRestate
from qrack_b200 import qscript

import one_device
import test_sharded_cpu as tsc
import test_sharded_gpu as tsg
import test_sharded_observables_cpu as tocpu
import test_sharded_observables_gpu as tog
import test_sharded_sample_cpu as tss
import test_sharded_topn_cpu as tst
import util

pytestmark = pytest.mark.gpu

# Belady's rule ranks qubit 0 (never used again) as the farthest victim of the exchange H 8 needs
VICTIM = "qubits 9\nH 8\n" + "".join("CNOT 8 %d\n" % q for q in range(1, 8))
BIG_N = 20
PARITY = dict(tsc.CIRCUITS, deep=tsc.DEEP, victim=VICTIM,
              htcnot20=qscript.random_htcnot(BIG_N, 10, seed=21, timed=False),
              qv20=qscript.quantum_volume(BIG_N, depth=4, seed=9, timed=False))
KINDS_26Q = ("htcnot", "qv", "grover")
FLOOR = {32: 1, 64: 0}  # lowest physical bit an exchange may take (P2PShardBuffers.CHUNK_FLOOR; ShardBuffers: 0)

CASES = ([(w, p, m) for w in (2, 4) for m in ("push", "pull", "staged") for p in (32, 64)]
         + [(8, p, m) for m in ("push", "pull") for p in (32, 64)] + [(16, 32, "push")])


def n_qubits(text):
    return int(text.split("\n", 1)[0].split()[1])


def probes(n):
    """read-only queries after a parity script: every per-qubit Prob, a mask, a parity, three amplitudes and the norm"""
    rng = random.Random(n)
    mask = rng.getrandbits(n) | 1 | (1 << (n - 1))
    return ("".join("Prob %d\n" % q for q in range(n)) + "ProbMask %d %d\n" % (mask, mask & rng.getrandbits(n))
            + "ProbParity %d\n" % (mask ^ (1 << (n // 2))) + "".join("GetAmplitude %d\n" % rng.getrandbits(n) for _ in range(3))
            + "Norm\n")


def probe_values(psi, text):
    """the values of the probes on the state psi, in float64"""
    psi = psi.astype(np.complex128)
    p = np.abs(psi) ** 2
    i = np.arange(p.size, dtype=np.int64)
    out = []
    for _, t in qscript.parse(text):
        op, a = t[0], [int(v) for v in t[1:]]
        if op == "Prob":
            out.append(p[(i >> a[0]) & 1 == 1].sum())
        elif op == "ProbMask":
            out.append(p[(i & a[0]) == a[1]].sum())
        elif op == "ProbParity":
            out.append(p[np.bitwise_count(i & a[0]) & 1 == 1].sum())
        elif op == "GetAmplitude":
            out += [psi[a[0]].real, psi[a[0]].imag]
        else:
            assert op == "Norm", op
            out.append(p.sum())
    return np.array(out)


def refused(n, world, prec, mode):
    """QEngineSharded refuses pages with fewer than k local qubits at or above the exchange's floor"""
    k = world.bit_length() - 1
    return n - k - (0 if mode == "staged" else FLOOR[prec]) < k


def _ranks(rank, world, dist, prec, mode, out):
    import torch
    from qrack_b200.sharded import QEngineSharded, cuda_engine_factory
    os.environ["B200SV_SHARD_PULL"] = "0" if mode == "push" else "1"
    dev = torch.device("cuda", 0)
    peak = [0]

    def sample_memory():
        free, total = torch.cuda.mem_get_info(dev)   # device-wide: every rank's context and pages
        peak[0] = max(peak[0], total - free)

    def make(n, perm):
        return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                              device=dev, make_engine=cuda_engine_factory(0, prec), p2p=mode != "staged")
    save = {}
    for name, text in PARITY.items():
        try:
            regs, results = qscript.run(text, make)
        except ValueError as e:
            save[name + "_refused"] = str(e)
            continue
        q = regs[0]
        before = q.GetQuantumState()
        _, more = qscript.run("qubits %d\n" % q.qubitCount + probes(q.qubitCount), lambda n, p: q)
        after = q.GetQuantumState()
        sample_memory()
        save.update({name + "_results": np.array([v for _, vals in results + more for v in vals], dtype=np.float64),
                     name + "_same": np.array_equal(before, after), name + "_exchanges": q.be.exchanges,
                     name + "_pull_sweeps": q.be.shard.stats().get("pull_sweeps", 0)})
        if rank == 0:
            save[name + "_state"] = after
        del q, regs
    np.savez(os.path.join(out, "parity.%d.npz" % rank), **save)
    tss.run_cases(make, os.path.join(out, "sample.%d.npz" % rank))
    sample_memory()
    tst.run_cases(make, os.path.join(out, "topn.%d.npz" % rank))
    sample_memory()
    if tocpu.N_QUBITS - (world.bit_length() - 1) >= 6:   # the query set lists six local qubits
        tog.run_observables(make, os.path.join(out, "obs.%d.npz" % rank))
        sample_memory()
    if world == 8 and prec == 32:
        for kind in KINDS_26Q:
            np.savez(os.path.join(out, "ref26_%s.%d.npz" % (kind, rank)), **tsg.queries_26q(make, util.sharded_26q_text(kind)))
            sample_memory()
    torch.cuda.synchronize(dev)
    np.savez(os.path.join(out, "peak.%d.npz" % rank), peak=peak[0])


@functools.lru_cache(maxsize=None)
def oracle64(text):
    regs, results = util.run_engine(text, QEngineRestate, 64)
    return regs[0], np.array([v for _, vals in results for v in vals], dtype=np.float64)


def check_parity(z, world, prec, mode):
    """every rank's query results identical, the probes left the state bit-identical, at least one exchange, pull sweeps
    in pull mode only, the state on the float64 oracle's, the probes on the float64 values of that state and every query
    on the oracle's; returns the largest |delta amp|, probe deviation and query deviation from the oracle"""
    d_amp = d_res = d_q64 = 0.0
    for name, text in PARITY.items():
        n = n_qubits(text)
        if refused(n, world, prec, mode):
            assert all(name + "_refused" in zr for zr in z), "%s: %d qubits over %d ranks must be refused" % (name, n, world)
            continue
        for r, zr in enumerate(z):
            assert name + "_refused" not in zr, (name, r, str(zr.get(name + "_refused")))
            assert np.array_equal(zr[name + "_results"], z[0][name + "_results"]), "%s: rank %d returned other values" % (name, r)
            assert bool(zr[name + "_same"]), "%s, rank %d: read-only queries changed the state" % (name, r)
            assert int(zr[name + "_exchanges"]) >= 1, (name, r)
            if mode == "pull" and world <= 8:
                assert int(zr[name + "_pull_sweeps"]) >= 1, (name, r)   # the re-page rode on a fused sweep
            else:
                assert int(zr[name + "_pull_sweeps"]) == 0, (name, r)
        want, wres = oracle64(text + probes(n))
        st = z[0][name + "_state"]
        delta = st.astype(np.complex128) - want
        d = float(np.abs(delta).max())
        assert d <= util.AMP_TOL[prec], "%s: max |delta amp| = %.3e" % (name, d)
        got = z[0][name + "_results"]
        assert got.shape == wres.shape, name
        # the probes' reductions on the engine's own state: float64 NumPy on the gathered pages
        own = probe_values(st, probes(n))
        e = float(np.abs(got[-own.size:] - own).max())
        assert e <= util.PROB_TOL[prec], "%s: max |delta probe| = %.3e against the engine's own state" % (name, e)
        # every query against the float64 oracle: a probability of the engine's state lies within 2 ||delta psi||_2 of
        # the oracle's, which in fp32 exceeds PROB_TOL on deep circuits (the state's own rounding, ~1e-5 after 400 gates)
        bound = util.PROB_TOL[prec] + 2 * float(np.linalg.norm(delta))
        e64 = float(np.abs(got - wres).max())
        assert e64 <= bound, "%s: max |delta query| = %.3e > %.3e" % (name, e64, bound)
        d_amp, d_res, d_q64 = max(d_amp, d), max(d_res, e), max(d_q64, e64)
    return d_amp, d_res, d_q64


@pytest.mark.parametrize("world,prec,mode", CASES, ids=["w%d-fp%d-%s" % c for c in CASES])
def test_sharded_ranks_on_one_device_match_the_oracle(world, prec, mode, tmp_path):
    t0 = time.time()
    one_device.spawn(_ranks, world, prec, mode, str(tmp_path))
    wall = time.time() - t0

    def load(what):
        return [dict(np.load(str(tmp_path / ("%s.%d.npz" % (what, r))))) for r in range(world)]
    d_amp, d_res, d_q64 = check_parity(load("parity"), world, prec, mode)
    s_amp, s_hist = tss.check_ranks_against_oracle(load("sample"), prec, exact=False)
    tst.check_ranks_against_oracle(load("topn"), prec, exact=False)
    obs = "-"
    if tocpu.N_QUBITS - (world.bit_length() - 1) >= 6:
        obs = "%.2e" % tog.check_observables(load("obs"), prec, "w%d %s" % (world, mode))
    ref = ""
    if world == 8 and prec == 32:
        for kind in KINDS_26Q:
            z = load("ref26_" + kind)
            for r in range(1, world):
                assert np.array_equal(z[r]["results"], z[0]["results"]) and int(z[r]["perm"]) == int(z[0]["perm"]), (kind, r)
            ref += " 26q %s |damp| %.2e dP %.2e;" % ((kind,) + tsg.check_26q(z[0], kind))
    peak = max(int(z["peak"]) for z in load("peak"))
    print("\n[one device] w%d fp%d %s: %.1f s, peak device memory %.2f GiB" % (world, prec, mode, wall, peak / 2 ** 30))
    print("  parity |damp| %.2e (tol %.0e), probes %.2e (tol %.0e), queries vs oracle %.2e; sampling |damp| %.2e, "
          "histogram %.3f (tol 0.06); observables dev/scale %s (tol %.0e);%s"
          % (d_amp, util.AMP_TOL[prec], d_res, util.PROB_TOL[prec], d_q64, s_amp, s_hist, obs, tocpu.TOL[prec], ref))
