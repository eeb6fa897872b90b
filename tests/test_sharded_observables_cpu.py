"""World-size-2/4 `gloo` tests (CPU) of the observable queries on the sharded engine (qrack_b200/sharded.py): the weighted
moments (Expectation/Variance BitsAll, BitsFactorized, FloatsFactorized) and the Pauli strings (Expectation/VariancePauliAll),
with listed qubits on local and rank bits, pending X inversions and a qubit map scrambled by exchanges, against the float64
NumPy reference (tests/npref_observables.py) on the single-engine oracle state.  The local engine is the oracle restatement
over the torch CPU page with NumPy observable sweeps, so a Pauli string with X or Y on a rank-bit qubit takes the pairwise
gloo send/recv of the page into `scratch` and the pair sweep on it."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.restate_engine import QEngineRestate, _RestateBackend
from qrack_b200 import qscript

import npref_observables as no
import util
from test_sharded_cpu import _free_port

N_QUBITS = 9
# U3 layers put non-diagonal gates on the rank-bit qubits (exchanges scramble the qubit map); the XMask stays pending
CIRCUIT = qscript.random_u3_cnot(N_QUBITS, 3, seed=17) + "XMask 130\n"
TOL = {32: 1e-5, 64: 1e-10}


def pair_term(psi, phi, x, z):
    """sum_j conj(phi[j ^ x]) (-1)^popcount(j & z) psi[j] = <phi| X^x Z^z |psi>, with the single-qubit matrices of
    npref_observables applied qubit by qubit"""
    v = np.asarray(psi, dtype=np.complex128)
    n = int(np.log2(len(v)))
    for q in range(n):
        if (z >> q) & 1:
            v = no.apply_1q(v, no.PAULI[2], q)
    for q in range(n):
        if (x >> q) & 1:
            v = no.apply_1q(v, no.PAULI[1], q)
    return complex(np.vdot(np.asarray(phi, dtype=np.complex128), v))


class _ObsBackend(_RestateBackend):
    """the oracle restatement plus the observable sweeps of the CUDA backend, computed in NumPy"""

    def moments_bits(self, bits, perms, offset, center):
        return no.moments_bits(self.get_state(), bits, perms, offset, center)

    def moments_floats(self, bits, weights, center):
        return no.moments_floats(self.get_state(), bits, weights, center)

    def expectation_pauli(self, x, z):
        return no.pauli_expectation(self.get_state(), x, z)

    def expectation_pauli_pair(self, partner, x, z):
        nbytes = (1 << self.nq) * np.dtype(self.cplx).itemsize
        phi = np.frombuffer((ctypes.c_char * nbytes).from_address(partner), dtype=self.cplx).copy()
        psi = self.get_state()
        return pair_term(psi, phi, x, z), float(np.sum(np.abs(psi.astype(np.complex128)) ** 2))


class _ObsEngine(QEngineRestate):
    def _make_backend(self, n_qubits: int):
        return _ObsBackend(n_qubits, self.precision)


def obs_engine_factory(precision):
    cplx = np.complex64 if precision == 32 else np.complex128

    def make(buf, n_local):
        q = _ObsEngine(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        q.be.amps = buf.numpy().view(cplx)  # shares memory with the torch page
        return q
    return make


def query_text(perm, nl):
    """X gates (left pending) and the queries, chosen from the qubit map the circuit left: R = the rank-bit qubits, L the
    local ones.  R[0], L[0] and L[2] get an extra X, so inverted qubits are listed on both sides."""
    R = [q for q in range(len(perm)) if perm[q] >= nl]
    L = [q for q in range(len(perm)) if perm[q] < nl]
    lines = ["X %d" % R[0], "X %d" % L[0], "X %d" % L[2]]

    def cs(qs):
        return "%d %s" % (len(qs), " ".join(map(str, qs)))
    local, mixed, rank = [L[0], L[1], L[2]], [L[1], R[0], L[0]], list(R)
    for op in ("Expectation", "Variance"):
        for qs in (local, mixed, rank):
            lines.append("%sBitsAll %s 5" % (op, cs(qs)))
            w = [0.5, -1.25, 2.0, 0.75, -0.375, 1.125][:2 * len(qs)]
            lines.append("%sFloatsFactorized %s %s" % (op, cs(qs), " ".join(map(str, w))))
        lines.append("%sBitsFactorized %s 4 3 11 7 2 100 5 9 1" % (op, cs([L[3], R[-1], L[0], L[4]])))
        lines.append("%sFloatsFactorized %s -0.5 1.5 2.0 0.25 0.75 -1.0 1.25 0.5" % (op, cs((list(reversed(R)) + [L[2], L[1]])[:3] + [L[5]])))
        pauli = [
            ([L[0], L[1], R[0], L[2]], [1, 3, 2, 2]),      # X / Y on local qubits only, Z on a rank bit
            ([R[0], L[0], L[3]], [1, 2, 3]),               # X on a rank bit: the pair path
            ([R[0], L[0]], [2, 2]),                        # Z on an inverted rank bit and an inverted local qubit
            (list(R) + [L[1]], [3] * len(R) + [1]),        # Y on every rank bit
            ([L[3], L[4], R[0], L[1]], [0, 0, 3, 1]),      # the first I survives the reference's I-dropping loop: as Z
            ([R[-1]], [1]),                                # one qubit, X on a rank bit
            ([L[2]], [3]),                                 # one qubit, Y local
        ]
        for qs, ps in pauli:
            lines.append("%sPauliAll %s %s" % (op, cs(qs), " ".join(map(str, ps))))
    return "\n".join(lines) + "\n"


def _worker(rank, world, port, prec, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from qrack_b200.sharded import QEngineSharded

        def make(n, perm):
            return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                                  device="cpu", make_engine=obs_engine_factory(prec))
        regs, _ = qscript.run(CIRCUIT, make)
        q = regs[0]
        q.Finish()
        text = query_text(q.be.perm, q.be.nl)
        gates = "".join(l + "\n" for l in text.splitlines() if l.startswith("X "))
        queries = "".join(l + "\n" for l in text.splitlines() if not l.startswith("X "))
        qscript.run("qubits %d\n" % N_QUBITS + gates, lambda n, p: q)
        before, ex0, xinv = q.GetQuantumState(), q.be.exchanges, q.be.xinv
        _, results = qscript.run("qubits %d\n" % N_QUBITS + queries, lambda n, p: q)
        after, ex1 = q.GetQuantumState(), q.be.exchanges
        refused = 0
        for call in (lambda: q.ExpectationUnitaryAll([0, 1], [0.1, 0.2, 0.3, 0.4, 0.5, 0.6]),
                     lambda: q.GetReducedDensityMatrix([0, 1])):
            try:
                call()
            except NotImplementedError:
                refused += 1
        np.savez(out_path + ".%d.npz" % rank, results=np.array([v for _, vals in results for v in vals], dtype=np.float64),
                 same=np.array_equal(before, after), ex0=ex0, ex1=ex1, xinv=xinv, refused=refused, gates=gates, queries=queries)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_observables_match_single_engine(world, prec, tmp_path):
    out = str(tmp_path / "obs")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    z = [np.load(out + ".%d.npz" % r) for r in range(world)]
    gates, queries = str(z[0]["gates"]), str(z[0]["queries"])
    for r in range(world):
        assert np.array_equal(z[r]["results"], z[0]["results"]), "rank %d returned other values" % r
        assert bool(z[r]["same"]), "rank %d: the queries changed the state" % r
        assert int(z[r]["ex1"]) == int(z[r]["ex0"]), "rank %d: the queries exchanged pages" % r
        assert int(z[r]["refused"]) == 2
    assert int(z[0]["ex0"]) >= 1       # the circuit scrambled the qubit map
    xinv = int(z[0]["xinv"])
    assert xinv and bin(xinv).count("1") >= 3
    want, _ = util.run_engine(CIRCUIT + gates, QEngineRestate, prec)
    psi = want[0]
    ops = [t for _, t in qscript.parse(queries)]
    got = z[0]["results"]
    assert got.size == len(ops)
    for g, t in zip(got, ops):
        v, scale, _ = no.query_value(psi, t[0], t[1:])
        assert abs(g - v) <= TOL[prec] * max(scale, 1e-30), (t, g, v, scale)


def test_rank_split_pauli_identity():
    """E = sum_r Re(i^|X&Z| (-1)^popcount(r & Z_r) T_r) with T_r the pair term of page r against page r ^ X_r (the
    decomposition behind the sharded ExpectationPauliAll), for every split of a 7-qubit state into 2, 4 and 8 pages"""
    rng = np.random.default_rng(3)
    n = 7
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    psi /= np.linalg.norm(psi)
    for k in (1, 2, 3):
        nl = n - k
        pages = psi.reshape(1 << k, 1 << nl)
        for _ in range(20):
            x, z = int(rng.integers(0, 1 << n)), int(rng.integers(0, 1 << n))
            want = no.pauli_expectation(psi, x, z)[1]
            xl, xr, zl, zr = x & ((1 << nl) - 1), x >> nl, z & ((1 << nl) - 1), z >> nl
            ph = (1, 1j, -1, -1j)[bin(x & z).count("1") & 3]
            got = sum((ph * (-1) ** bin(r & zr).count("1") * pair_term(pages[r], pages[r ^ xr], xl, zl)).real
                      for r in range(1 << k))
            assert abs(got - want) <= 1e-12, (k, x, z, got, want)
