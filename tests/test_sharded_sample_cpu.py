"""World-size-2/4 `gloo` tests (CPU) of sampling on the sharded engine (qrack_b200/sharded.py): `sample_many` walks the page
totals for every shot at once, each rank searches its page for its own shots with the keyed search (logical indices), and one
all_reduce gathers them.  Every shot must be exactly what `sample` gives for its rnd, on every rank, and MultiShotMeasureMask
over more than 16 qubits (18 here) takes that route.  The qubit map is scrambled by exchanges and X gates are left pending on
rank-bit and local qubits.  The local engine is the oracle restatement over the torch CPU page; its `sample_keyed` applies the
key to the restatement's own `sample` for each rnd, so the walk, the keys and the gather are checked exactly whatever order
the restatement sums in."""
import math
import os
import random

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.restate_engine import QEngineRestate, _RestateBackend
from qrack_b200 import qscript
from qrack_b200.sharded import rank_walk

import npref
import util
from test_sharded_cpu import _free_port
from test_sharded_topn_cpu import pending_x

N_QUBITS = 18  # more than 16 measured qubits: MultiShotMeasureMask samples basis states
CIRCUITS = {
    # U3 layers put non-diagonal gates on the rank-bit qubits; the XMask stays pending
    "random": qscript.random_u3_cnot(N_QUBITS, 2, seed=23) + "XMask %d\n" % ((1 << 17) | (1 << 4) | 1),
    # |0..0> + |1..1> with its CNOT targets on the rank bits: two nonzero entries, so with 4 ranks two pages are zero
    "ghz": "qubits %d\nH 0\n" % N_QUBITS + "".join("CNOT 0 %d\n" % b for b in range(N_QUBITS - 1, 0, -1)),
    # H on rank-bit and local qubits: 2^5 entries of equal P, page totals that are sums of them
    "dyadic": "qubits %d\n" % N_QUBITS + "H 17\nH 16\nH 3\nH 9\nCNOT 17 5\nH 12\nSwap 2 16\n",
}
SHOTS_REPLAY = 64      # each replayed shot is one sharded `sample` call
SHOTS_HISTOGRAM = 1000


def key_of(j, key_pos, key_xor):
    t = key_xor
    for b, p in enumerate(key_pos):
        if (j >> b) & 1:
            t ^= 1 << p
    return t


class _SampleBackend(_RestateBackend):
    """the oracle restatement plus the keyed search of the CUDA backend: the key of the restatement's own search"""

    def sample_keyed(self, rnds, key_bits, key_pos, key_xor):
        assert self.nq <= key_bits <= 64 and len(set(key_pos)) == self.nq and max(key_pos) < key_bits
        assert key_xor < (1 << key_bits)
        return np.array([key_of(self.sample(float(r)), key_pos, key_xor) for r in rnds], dtype=np.uint64)


class _SampleEngine(QEngineRestate):
    def _make_backend(self, n_qubits: int):
        return _SampleBackend(n_qubits, self.precision)


def sample_engine_factory(precision):
    cplx = np.complex64 if precision == 32 else np.complex128

    def make(buf, n_local):
        q = _SampleEngine(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        q.be.amps = buf.numpy().view(cplx)  # shares memory with the torch page
        return q
    return make


def read_off(perms, bits):
    """{outcome: count} in order of first appearance, outcome bit p = bit bits[p] of the sampled index"""
    out = {}
    for perm in perms:
        k = 0
        for p, b in enumerate(bits):
            k |= ((perm >> b) & 1) << p
        out[k] = out.get(k, 0) + 1
    return out


def probe_rnds(tots):
    """0, interior values, values near 1, above the total and below 0; every page boundary and the double below it"""
    cum = [float(c) for c in np.cumsum(np.asarray(tots, dtype=np.float64))]
    rnds = [0.0, 0.1, 0.37, 0.5, 0.9, 0.9999999, 1 - 2.0 ** -26, 1 - 2.0 ** -40, 1.0, 1.5, -0.25]
    return rnds + cum + [math.nextafter(c, 0) for c in cum]


def run_script(q):
    """the pending X gates, then the checks on the sharded engine; returns what check_ranks_against_oracle reads"""
    # H H on a rank-bit qubit: the first query's flush exchanges pages (in pull mode the re-page is still pending when the
    # query starts)
    top = [b for b in range(N_QUBITS) if q.be.perm[b] >= q.be.nl][0]
    gates = pending_x(q.be.perm, q.be.nl) + "H %d\nH %d\n" % (top, top)
    qscript.run("qubits %d\n" % N_QUBITS + gates, lambda n, p: q)
    ex_queued = q.be.exchanges
    first_rnds = [0.2, 0.55, 0.8]
    first = q.be.sample_many(first_rnds)
    before, ex0 = q.GetQuantumState(), q.be.exchanges
    tots = [t[0] for t in q.be._gather_scalars([q.be.loc.be.norm(0.0)])]
    rnds = probe_rnds(tots) + first_rnds
    many = q.be.sample_many(rnds)
    one = [q.be.sample(r) for r in rnds]
    assert first == one[-len(first_rnds):]
    rng = random.Random(5)
    bits17 = rng.sample(range(N_QUBITS), 17)
    bits18 = rng.sample(range(N_QUBITS), 18)
    replay_ok = []
    for bits in (bits17, bits18):
        st = q.rng.getstate()
        got = q.MultiShotMeasureMask([1 << b for b in bits], SHOTS_REPLAY)
        q.rng.setstate(st)
        want = read_off([q.be.sample(q.Rand()) for _ in range(SHOTS_REPLAY)], bits)
        replay_ok.append(list(got.items()) == list(want.items()))
    hist = q.MultiShotMeasureMask([1 << b for b in bits18], SHOTS_HISTOGRAM)
    return {"gates": gates, "rnds": np.array(rnds), "many": np.array(many, dtype=np.int64),
            "one": np.array(one, dtype=np.int64), "replay_ok": np.array(replay_ok), "bits18": np.array(bits18),
            "hist_keys": np.array(list(hist.keys()), dtype=np.int64), "hist_counts": np.array(list(hist.values())),
            "same": np.array_equal(before, q.GetQuantumState()), "state": before, "ex0": ex0, "ex1": q.be.exchanges,
            "xinv": q.be.xinv, "tots": np.array(tots), "exchanged_first": ex0 > ex_queued}


def run_cases(make, out_file):
    save = {}
    for name, circ in CIRCUITS.items():
        regs, _ = qscript.run(circ, make)
        q = regs[0]
        q.Finish()
        save.update({name + "_" + k: v for k, v in run_script(q).items()})
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
                                  device="cpu", make_engine=sample_engine_factory(prec))
        run_cases(make, out_path + ".%d.npz" % rank)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_sampling_matches_sample(world, prec, tmp_path):
    out = str(tmp_path / "sample")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    check_ranks_against_oracle([np.load(out + ".%d.npz" % r) for r in range(world)], prec)


def coarse(keys, weights, top=4):
    """the weights summed by the top `top` of the 18 outcome bits"""
    out = np.zeros(1 << top)
    np.add.at(out, np.asarray(keys, dtype=np.int64) >> (N_QUBITS - top), weights)
    return out


def check_ranks_against_oracle(z, prec, exact=True):
    """every rank returned the same samples and left the state and the qubit map alone; sample_many is sample shot for shot
    (exact), or (pages whose totals come from a reduction that may round differently from one call to the next, as the
    device's atomic-add norm does) for every rnd but those within 1e-12 of a page boundary; MultiShotMeasureMask is the
    read-off of sample for the replayed rnds; the state is the float64 oracle's and the histogram follows its |psi|^2.
    Returns the largest |delta amp| and histogram deviation."""
    d_amp = d_hist = 0.0
    for name, circ in CIRCUITS.items():
        for r in range(len(z)):
            for k in ("many", "one", "hist_keys", "hist_counts"):
                assert np.array_equal(z[r][name + "_" + k], z[0][name + "_" + k]), (name, k, r)
            many, one, rnds = z[r][name + "_many"], z[r][name + "_one"], z[r][name + "_rnds"]
            off = np.flatnonzero(many != one)
            if not exact and off.size:
                cum = np.cumsum(z[r][name + "_tots"])
                assert (np.abs(rnds[off, None] - cum[None, :]).min(axis=1) <= 1e-12).all(), (name, r, rnds[off], cum)
            else:
                assert not off.size, (name, r, rnds[off])
            assert bool(z[r][name + "_replay_ok"].all()), (name, r)
            assert bool(z[r][name + "_same"]), "%s, rank %d: sampling changed the state" % (name, r)
            assert int(z[r][name + "_ex1"]) == int(z[r][name + "_ex0"]), "%s, rank %d: sampling exchanged pages" % (name, r)
        assert int(z[0][name + "_ex0"]) >= 1  # the circuit scrambled the qubit map
        assert bool(z[0][name + "_exchanged_first"])  # the first query ran right after an exchange
        assert bin(int(z[0][name + "_xinv"])).count("1") >= 3
        want, _ = util.run_engine(circ + str(z[0][name + "_gates"]), QEngineRestate, 64)
        psi, mine = want[0], z[0][name + "_state"]
        util.assert_states_close({0: mine}, {0: psi}, prec, name)
        d_amp = max(d_amp, float(np.abs(mine.astype(np.complex128) - psi).max()))
        # every sample has P > 0, and outside the fallback rules of an all-zero page it lies in [0, 2^n)
        p = npref.probs(psi)
        got = z[0][name + "_many"]
        assert (got >= 0).all() and (got < (1 << N_QUBITS)).all() and (p[got] > 0).all(), name
        if len(z) == 4 and name == "ghz":
            assert (z[0][name + "_tots"] == 0).sum() == 2  # the walk skipped zero pages
        # outcome bit m of the histogram is qubit bits18[m]
        bits = [int(b) for b in z[0][name + "_bits18"]]
        idx = np.arange(p.size, dtype=np.int64)
        key = np.zeros(p.size, dtype=np.int64)
        for m, b in enumerate(bits):
            key |= ((idx >> b) & 1) << m
        counts = z[0][name + "_hist_counts"]
        assert counts.sum() == SHOTS_HISTOGRAM
        emp = coarse(z[0][name + "_hist_keys"], counts / SHOTS_HISTOGRAM)
        assert np.abs(emp - coarse(key, p)).max() < 0.06, (name, emp, coarse(key, p))
        d_hist = max(d_hist, float(np.abs(emp - coarse(key, p)).max()))
    return d_amp, d_hist


def walk_loop(tots, rnd):
    """_ShardedBackend.sample's rank walk as written there: (rank, rnd passed to its page), rank -1 when every page is zero"""
    cum, pick, last_nz = 0.0, None, None
    for r in range(len(tots)):
        if tots[r] > 0:
            last_nz = r
            if cum + tots[r] > rnd:
                pick = r
                break
            cum += tots[r]
    if pick is None:
        if last_nz is None:
            return -1, rnd
        pick, cum = last_nz, cum - tots[last_nz]
    return pick, rnd - cum


def test_vectorised_rank_walk_equals_the_loop():
    """rank_walk (every rnd at once) equals sample's loop bit for bit, on random and zero-containing page totals, including
    rnds at every boundary, just below it, above the total and below 0"""
    rng = np.random.default_rng(9)
    for trial in range(200):
        w = [1, 2, 4, 8][trial % 4]
        tots = rng.random(w) * rng.choice([1.0, 1e-3, 0.3])
        tots[rng.random(w) < 0.35] = 0.0
        if trial % 7 == 0:
            tots[:] = 0.0
        tots = [float(t) for t in tots]
        cum = [float(c) for c in np.cumsum(tots)]
        rnds = list(rng.random(20) * (sum(tots) * 1.2 + 1e-9)) + cum + [math.nextafter(c, 0) for c in cum]
        rnds += [0.0, -0.5, 1.0, 2.0]
        pick, res = rank_walk(tots, rnds)
        for i, r in enumerate(rnds):
            wp, wr = walk_loop(tots, r)
            assert int(pick[i]) == wp and float(res[i]).hex() == float(wr).hex(), (trial, tots, r)
