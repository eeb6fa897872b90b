"""The cross-page Pauli sweep (b200sv_expectation_pauli_pair) on ONE device, against float64 NumPy: the partner is another
QEngineCUDA on the same GPU (a peer mapping of another process's page is a plain device pointer there too), or the state's
own buffer, where it must agree with b200sv_expectation_pauli.  Then what it leaves alone (both buffers), its launch count,
the queued gates it flushes, the zero state and every argument error.  With >= 2 GPUs (skipped otherwise) the sharded engine
runs the script of tests/test_sharded_observables_cpu.py over NCCL in all three exchange modes against the oracle."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle.restate_engine import QEngineRestate
from qrack_b200 import QEngineCUDA, _abi, qscript

import npref_observables as no
import test_sharded_observables_cpu as tcpu
import util
from test_sharded_cpu import _free_port
from test_sharded_gpu import _ngpu

pytestmark = pytest.mark.gpu

TOL = {32: 1e-6, 64: 1e-12}
SIZES = [1, 2, 3, 8, 9, 16, 17, 22, 26]


def engine(n, prec, seed):
    rng = np.random.default_rng(1000 * n + seed)
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    q.SetQuantumState((psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128))
    q.Finish()
    return q


def dptr(q) -> int:
    p = ctypes.c_void_p()
    _abi.check(q.be.lib, q.be.lib.b200sv_device_ptr(q.be.h, ctypes.byref(p)))
    return p.value


def pair_ref(psi, phi, x, z):
    """(sum_j conj(phi[j ^ x]) (-1)^popcount(j & z) psi[j], sum |psi|^2) in float64, 2^22 indices at a time"""
    psi, phi = psi.astype(np.complex128), phi.astype(np.complex128)
    t, s0 = 0j, 0.0
    for lo in range(0, psi.size, 1 << 22):
        j = np.arange(lo, min(psi.size, lo + (1 << 22)), dtype=np.uint64)
        sgn = 1.0 - 2.0 * (np.bitwise_count(j & np.uint64(z)) & 1)
        a = psi[lo:lo + j.size]
        t += complex(np.sum(np.conj(phi[j ^ np.uint64(x)]) * sgn * a))
        s0 += float(np.sum(np.abs(a) ** 2))
    return t, s0


def mask_cases(n, rng):
    """x = 0, bit 0 set, bit 0 clear, with the top qubit; random z for each"""
    top = n - 1
    xs = [0, 1 | (rng.getrandbits(n) & ~1 & ((1 << n) - 1)), (rng.getrandbits(n) & ~1) & ((1 << n) - 1), 1 << top,
          (1 << top) | 1]
    return [(x, rng.getrandbits(n)) for x in dict.fromkeys(xs)]


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_pauli_pair_vs_numpy(n, prec):
    rng = random.Random(13 * n + prec)
    q, p = engine(n, prec, 1), engine(n, prec, 2)
    psi, phi = q.GetQuantumState(), p.GetQuantumState()
    for x, z in mask_cases(n, rng):
        t, s0 = q.be.expectation_pauli_pair(dptr(p), x, z)
        wt, ws0 = pair_ref(psi, phi, x, z)
        assert abs(t - wt) <= TOL[prec] and abs(s0 - ws0) <= TOL[prec], (n, x, z, t, wt)
        if n <= 12:
            assert abs(wt - tcpu.pair_term(psi, phi, x, z)) <= 1e-12
        # partner = the state's own buffer: the local Pauli term
        t, s0 = q.be.expectation_pauli_pair(dptr(q), x, z)
        e0, e = q.be.expectation_pauli(x, z)
        ph = (1, 1j, -1, -1j)[bin(x & z).count("1") & 3]
        assert abs((ph * t).real - e) <= TOL[prec] and abs(s0 - e0) <= TOL[prec], (n, x, z, t, e)
    assert np.array_equal(q.GetQuantumState(), psi) and np.array_equal(p.GetQuantumState(), phi)


@pytest.mark.parametrize("prec", [32, 64])
def test_pauli_pair_read_only_launches_flush_zero_and_einval(prec):
    n = 12
    q, p = engine(n, prec, 3), engine(n, prec, 4)
    psi, phi = q.GetQuantumState(), p.GetQuantumState()
    pp = dptr(p)
    q.be.reset_stats()
    q.be.expectation_pauli_pair(pp, 0b100000000101, 0b010000000110)
    assert q.be.stats()["kernel_launches"] == 1
    assert np.array_equal(q.GetQuantumState(), psi) and np.array_equal(p.GetQuantumState(), phi)
    # queued gates of the state are part of what the sweep reads
    for b in range(n):
        q.H(b)
        q.T(b)
    t, s0 = q.be.expectation_pauli_pair(pp, 0b11, 0b1010)
    wt, ws0 = pair_ref(q.GetQuantumState(), phi, 0b11, 0b1010)
    assert abs(t - wt) <= TOL[prec] and abs(s0 - ws0) <= TOL[prec]
    # the zero state: zeros, no launch
    z = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    z.ZeroAmplitudes()
    z.be.reset_stats()
    assert z.be.expectation_pauli_pair(pp, 3, 1) == (0j, 0.0)
    assert z.be.stats()["kernel_launches"] == 0
    lib, h, E = q.be.lib, q.be.h, _abi.B200SV_EINVAL
    O3 = (ctypes.c_double * 3)()
    fn = lib.b200sv_expectation_pauli_pair
    assert fn(None, ctypes.c_void_p(pp), 0, 0, O3) == E
    assert fn(h, None, 0, 0, O3) == E
    assert fn(h, ctypes.c_void_p(pp), 0, 0, None) == E
    assert fn(h, ctypes.c_void_p(pp), 1 << n, 0, O3) == E and fn(h, ctypes.c_void_p(pp), 0, 1 << n, O3) == E
    assert fn(h, ctypes.c_void_p(pp), (1 << n) - 1, (1 << n) - 1, O3) == 0
    assert np.array_equal(p.GetQuantumState(), phi)


def run_observables(make, out_file):
    """the script of tests/test_sharded_observables_cpu.py on a sharded engine from make(n, perm): the pending X gates and
    the queries, then a non-diagonal gate on a rank-bit qubit, its exchange, and at once a Pauli string with X on a rank
    bit (in pull mode the partner's page exists only after the partner's pull sweep, which the query's flush and barrier
    must wait for).  Saves what check_observables reads."""
    regs, _ = qscript.run(tcpu.CIRCUIT, make)
    q = regs[0]
    q.Finish()
    text = tcpu.query_text(q.be.perm, q.be.nl)
    gates = "".join(l + "\n" for l in text.splitlines() if l.startswith("X "))
    queries = "".join(l + "\n" for l in text.splitlines() if not l.startswith("X "))
    qscript.run("qubits %d\n" % tcpu.N_QUBITS + gates, lambda n, p: q)
    before, ex0 = q.GetQuantumState(), q.be.exchanges
    _, results = qscript.run("qubits %d\n" % tcpu.N_QUBITS + queries, lambda n, p: q)
    same, ex1 = np.array_equal(before, q.GetQuantumState()), q.be.exchanges
    nl = q.be.nl
    r0 = [b for b in range(tcpu.N_QUBITS) if q.be.perm[b] >= nl][0]
    q.H(r0)
    q.be.flush()
    rq = [b for b in range(tcpu.N_QUBITS) if q.be.perm[b] >= nl][0]
    lq = [b for b in range(tcpu.N_QUBITS) if q.be.perm[b] < nl][1]
    last = q.ExpectationPauliAll([rq, lq], [1, 3])
    np.savez(out_file, results=np.array([v for _, vals in results for v in vals], dtype=np.float64), same=same,
             last=last, ex0=ex0, ex1=ex1, ex2=q.be.exchanges, gates=gates, queries=queries,
             tail="H %d\n" % r0, tailq="ExpectationPauliAll 2 %d %d 1 3\n" % (rq, lq))


def check_observables(z, prec, what=""):
    """every rank returned the same values, left the state alone and exchanged pages only for the tail's gate; the values
    are the float64 NumPy reference's on the float64 oracle state, within the engine precision's tolerance relative to each
    query's scale.  Returns the largest |deviation| / scale."""
    for r in range(len(z)):
        assert np.array_equal(z[r]["results"], z[0]["results"]) and float(z[r]["last"]) == float(z[0]["last"]), (what, r)
        assert bool(z[r]["same"]), "%s, rank %d: the queries changed the state" % (what, r)
        assert int(z[r]["ex1"]) == int(z[r]["ex0"]) and int(z[r]["ex2"]) == int(z[r]["ex1"]) + 1, (what, r)
    gates = str(z[0]["gates"])
    want, _ = util.run_engine(tcpu.CIRCUIT + gates, QEngineRestate, 64)
    ops = [t for _, t in qscript.parse(str(z[0]["queries"]))]
    assert z[0]["results"].size == len(ops)
    worst = 0.0
    for g, t in zip(z[0]["results"], ops):
        v, scale, _ = no.query_value(want[0], t[0], t[1:])
        assert abs(g - v) <= tcpu.TOL[prec] * max(scale, 1e-30), (what, t, g, v)
        worst = max(worst, abs(g - v) / max(scale, 1e-30))
    want, _ = util.run_engine(tcpu.CIRCUIT + gates + str(z[0]["tail"]), QEngineRestate, 64)
    t = qscript.parse(str(z[0]["tailq"]))[0][1]
    v, scale, _ = no.query_value(want[0], t[0], t[1:])
    assert abs(float(z[0]["last"]) - v) <= tcpu.TOL[prec] * scale, (what, float(z[0]["last"]), v)
    return max(worst, abs(float(z[0]["last"]) - v) / scale)


def _worker(rank, world, port, prec, out_path, mode):
    import torch
    import torch.distributed as dist
    os.environ["B200SV_SHARD_PULL"] = "1" if mode == "pull" else "0"
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from qrack_b200.sharded import QEngineSharded, cuda_engine_factory

        def make(n, perm):
            return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                                  device=torch.device("cuda", rank), make_engine=cuda_engine_factory(rank, prec),
                                  p2p=mode != "nccl")
        run_observables(make, out_path + ".%d.npz" % rank)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["nccl", "push", "pull"])
@pytest.mark.parametrize("prec", [32, 64])
def test_sharded_observables_on_gpus_match_the_oracle(prec, mode, tmp_path):
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    world = 2 if _ngpu() < 4 else 4
    out = str(tmp_path / "o")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out, mode), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    check_observables([np.load(out + ".%d.npz" % r) for r in range(world)], prec, mode)
