"""World-size-2/4 `gloo` tests (CPU) of HighestProbAll(n) on the sharded engine (qrack_b200/sharded.py): a keyed select per
rank, ties to the smaller logical index, and one all_gather and merge.  The qubit map is scrambled by exchanges and X gates
are left pending on rank-bit and local qubits; the lists must equal the float64 NumPy reference (tests/npref_topn.py) on the
single-engine oracle state exactly, on a random state, a uniform superposition (P ties everywhere) and a GHZ-like state.
The local engine is the oracle restatement over the torch CPU page with a NumPy `highest_probs_keyed`."""
import os
import random

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.restate_engine import QEngineRestate, _RestateBackend
from qrack_b200 import qscript
from qrack_b200.sharded import merge_top_n

import npref_topn as no
import test_topn_cpu as tcpu
import util
from test_sharded_cpu import _free_port

N_QUBITS = 9
TOP = N_QUBITS - 1  # a rank bit at the start in every world size
CIRCUITS = {
    # U3 layers put non-diagonal gates on the rank-bit qubits; the XMask stays pending
    "random": qscript.random_u3_cnot(N_QUBITS, 3, seed=17) + "XMask 130\n",
    # H on every qubit (the rank bits take exchanges) and CNOTs that keep it uniform: P ties everywhere
    "uniform": "qubits %d\n" % N_QUBITS + "".join("H %d\n" % b for b in range(N_QUBITS)) + "CNOT %d 0\nCNOT 1 %d\nSwap 2 %d\n"
    % (TOP, TOP - 1, TOP),
    # |0..0> + |1..1> with its CNOT targets on the rank bits: two entries of P = 1/2, the rest zero
    "ghz": "qubits %d\nH 0\n" % N_QUBITS + "".join("CNOT 0 %d\n" % b for b in range(N_QUBITS - 1, 0, -1)),
}


def keys_of(nq, key_pos, key_xor):
    """t(i) = key_xor ^ (OR over the bits b set in i of 2^key_pos[b]) for every index (key_pos None: b -> b)"""
    i = np.arange(1 << nq, dtype=np.uint64)
    t = np.full(i.size, key_xor, dtype=np.uint64)
    for b in range(nq):
        t ^= ((i >> np.uint64(b)) & np.uint64(1)) << np.uint64(b if key_pos is None else key_pos[b])
    return t


def top_n_keyed(psi, n, key_pos=None, key_xor=0):
    """(keys, probs) of b200sv_highest_probs_keyed, from its definition in include/b200sv.h"""
    p = no.probs(psi)
    t = keys_of(int(np.log2(len(p))), key_pos, key_xor)
    o = np.lexsort((t, -p))
    o = o[p[o] > 0][:n]
    keys, probs = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.float64)
    keys[:o.size], probs[:o.size] = t[o], p[o]
    return keys, probs


class _TopnBackend(_RestateBackend):
    """the oracle restatement plus the keyed select of the CUDA backend, computed in NumPy"""

    def highest_probs_keyed(self, n, key_bits, key_pos, key_xor):
        assert self.nq <= key_bits <= 64 and len(set(key_pos)) == self.nq and max(key_pos) < key_bits
        assert key_xor < (1 << key_bits)
        return top_n_keyed(self.get_state(), n, key_pos, key_xor)


class _TopnEngine(QEngineRestate):
    def _make_backend(self, n_qubits: int):
        return _TopnBackend(n_qubits, self.precision)


def topn_engine_factory(precision):
    cplx = np.complex64 if precision == 32 else np.complex128

    def make(buf, n_local):
        q = _TopnEngine(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        q.be.amps = buf.numpy().view(cplx)  # shares memory with the torch page
        return q
    return make


def pending_x(perm, nl):
    """X gates left pending on the first rank-bit qubit and on two local ones of the map the circuit left"""
    R = [q for q in range(len(perm)) if perm[q] >= nl]
    L = [q for q in range(len(perm)) if perm[q] < nl]
    return "X %d\nX %d\nX %d\n" % (R[0], L[0], L[2])


def sizes(nl):
    """2, more than one page, every state, and one past a GHZ's two nonzero entries"""
    return [2, 5, (1 << nl) + 3, 1 << N_QUBITS]


def run_script(q, nl):
    """the pending X gates, then the queries and the edge rules; returns (gates, lists, state before and after the queries,
    exchanges before and after, whether the edge rules held)"""
    gates = pending_x(q.be.perm, nl)
    qscript.run("qubits %d\n" % N_QUBITS + gates, lambda n, p: q)
    before, ex0 = q.GetQuantumState(), q.be.exchanges
    queries = "".join("HighestProbAllN %d\n" % k for k in sizes(nl))
    _, results = qscript.run("qubits %d\n" % N_QUBITS + queries, lambda n, p: q)
    lists = [[int(v) for v in vals] for _, vals in results]
    edge = [q.HighestProbAllN(0) == [], q.HighestProbAllN(1) == [q.HighestProbAll()]]
    try:
        q.HighestProbAllN((1 << N_QUBITS) + 1)
    except ValueError:
        edge.append(True)
    return gates, lists, before, q.GetQuantumState(), ex0, q.be.exchanges, all(edge) and len(edge) == 3


def run_cases(make, out_file):
    """every circuit on a sharded engine from make(n, perm), then run_script; what check_ranks_against_oracle reads"""
    save = {}
    for name, circ in CIRCUITS.items():
        regs, _ = qscript.run(circ, make)
        q = regs[0]
        q.Finish()
        gates, lists, before, after, ex0, ex1, edge = run_script(q, q.be.nl)
        save.update({name + "_gates": gates, name + "_lists": np.array(sum(lists, []), dtype=np.int64),
                     name + "_same": np.array_equal(before, after), name + "_state": before, name + "_ex0": ex0,
                     name + "_ex1": ex1, name + "_edge": edge, name + "_xinv": q.be.xinv, name + "_nl": q.be.nl})
        del q, regs
    np.savez(out_file, **save)


def _worker(rank, world, port, prec, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from qrack_b200.sharded import QEngineSharded

        def make(n, perm):
            return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                                  device="cpu", make_engine=topn_engine_factory(prec))
        run_cases(make, out_path + ".%d.npz" % rank)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_highest_prob_all_n_matches_single_engine(world, prec, tmp_path):
    out = str(tmp_path / "topn")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    z = [np.load(out + ".%d.npz" % r) for r in range(world)]
    check_ranks_against_oracle(z, prec)


def check_ranks_against_oracle(z, prec, exact=True):
    """every rank returned the same lists and left the state and the qubit map alone; the lists are NumPy's on the state the
    pages hold, and the oracle's: exactly (the restatement's pages round every gate as the single engine does) or, for pages
    that round differently (the fused sweeps on the device), up to swaps of near-ties"""
    for name, circ in CIRCUITS.items():
        for r in range(len(z)):
            assert np.array_equal(z[r][name + "_lists"], z[0][name + "_lists"]), (name, r)
            assert bool(z[r][name + "_same"]), "%s, rank %d: the query changed the state" % (name, r)
            assert int(z[r][name + "_ex1"]) == int(z[r][name + "_ex0"]), "%s, rank %d: the query exchanged pages" % (name, r)
            assert bool(z[r][name + "_edge"]), (name, r)
        assert int(z[0][name + "_ex0"]) >= 1  # the circuit scrambled the qubit map
        xinv = int(z[0][name + "_xinv"])
        assert bin(xinv).count("1") >= 3
        want, _ = util.run_engine(circ + str(z[0][name + "_gates"]), QEngineRestate, prec)
        psi, mine = want[0], z[0][name + "_state"]
        util.assert_states_close({0: mine}, {0: psi}, prec, name)
        got = z[0][name + "_lists"]
        nl = int(z[0][name + "_nl"])
        at = 0
        for k in sizes(nl):
            assert list(got[at:at + k]) == no.top_n(mine, k), (name, k)
            if exact:
                assert list(got[at:at + k]) == no.top_n(psi, k), (name, k)
            else:
                tcpu.assert_same_up_to_near_ties(list(got[at:at + k]), no.top_n(psi, k), no.probs(psi), no.probs(mine), prec,
                                                 (name, k), 2 * float(np.abs(no.probs(psi) - no.probs(mine)).max()))
            at += k
        assert at == got.size
        if not exact:
            continue
        # got[:2] is the n = 2 list, got[2:7] the n = 5 one
        if name == "uniform":
            assert np.unique(no.probs(psi)).size == 1  # P ties everywhere: the smallest logical indices
            assert list(got[:7]) == [0, 1, 0, 1, 2, 3, 4]
        if name == "ghz":
            pair = sorted([xinv, xinv ^ ((1 << N_QUBITS) - 1)])
            assert list(got[:7]) == pair + pair + [0, 0, 0]


def test_merged_page_tops_equal_the_global_top():
    """For random pages (a logical state scattered by a qubit map and pending inversions, with many exact P ties), the merge of
    every page's keyed top min(n, 2^nl) equals the global top n: the decomposition behind highest_probs_merged"""
    rng = np.random.default_rng(5)
    n = 8
    for trial in range(40):
        k = 1 + trial % 3
        nl = n - k
        levels = rng.integers(0, 4, size=1 << n)  # four values of |psi|: ties and zeros everywhere
        psi = (levels * (0.5 + 0.25j)).astype(np.complex128)
        perm = list(rng.permutation(n))            # logical qubit -> physical bit
        xinv = int(rng.integers(0, 1 << n))
        inv = {p: q for q, p in enumerate(perm)}
        # stored physical vector: physical index J holds logical index L(J) ^ xinv
        J = np.arange(1 << n)
        L = np.zeros_like(J)
        for q in range(n):
            L |= ((J >> perm[q]) & 1) << q
        phys = psi[L ^ xinv]
        for m in (1, 2, 7, (1 << nl) + 1, 1 << n):
            keys, probs = [], []
            for r in range(1 << k):
                xr = xinv
                for g in range(k):
                    if (r >> g) & 1:
                        xr ^= 1 << inv[nl + g]
                kk, pp = top_n_keyed(phys[r << nl:(r + 1) << nl], min(m, 1 << nl), [inv[b] for b in range(nl)], xr)
                keys.append(kk)
                probs.append(pp)
            got = merge_top_n(np.concatenate(keys), np.concatenate(probs), m)
            assert got == no.top_n(psi, m), (trial, k, m)

