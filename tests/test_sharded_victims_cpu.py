"""Victim choice of the sharded engine's exchange (qrack_b200/sharded.py, _ShardedBackend._exchange), host logic only: the
scheduler runs over a stub shard that records the physical bits it hands to the exchange.  The P2P re-page kernels move
whole 16-byte chunks, so an fp32 victim on physical bit 0 (inside the chunk) is refused with EINVAL mid-circuit.  Small
pages (fewer than min_victim_bit + k local qubits) used to fall back to every local qubit, bit 0 included."""
import random

import pytest

from qrack_b200 import sharded

H = [2 ** -0.5 + 0j, 2 ** -0.5 + 0j, 2 ** -0.5 + 0j, -(2 ** -0.5) + 0j]
X = [0j, 1 + 0j, 1 + 0j, 0j]


class _Engine:
    """accepts the local gates the scheduler submits (no `be`: one UCMtrx call per gate) and does nothing"""

    def UCMtrx(self, ctrls, m, pt, cperm):
        pass


class _StubShard:
    """P2PShardBuffers' victim rules (any k local bits, preferred from min_victim_bit, never below its chunk floor), no data"""
    needs_top = False
    min_victim_bit = sharded.P2PShardBuffers.min_victim_bit

    def __init__(self, prec):
        self.chunk_floor = sharded.P2PShardBuffers.CHUNK_FLOOR[prec]
        self.engine = _Engine()
        self.victims = []

    def exchange(self, dist, world, rank, k, victim_bits):
        self.victims.append(list(victim_bits))
        return 0


def victims_of(n, world, prec):
    """the victims of `H t; CNOT t 1; ...; CNOT t 7` (t = n - 1, a rank bit) on rank 0: qubit 0 is never used again, so
    Belady's rule ranks it farthest; qubit 7 is the farthest of the rest"""
    shard = _StubShard(prec)
    be = sharded._ShardedBackend(n, prec, shard, None, world, 0)
    t = n - 1
    be.pending.append(sharded._Gate(t, 0, 0, H))
    for q in range(1, 8):
        be.pending.append(sharded._Gate(q, 1 << t, 1 << t, X))
    be.flush()
    return shard, be


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n,world", [(9, 2), (9, 4), (18, 8)])
def test_victims_never_fall_below_the_chunk_floor(n, world, prec):
    shard, be = victims_of(n, world, prec)
    k, nl = be.k, be.nl
    assert shard.victims and be.exchanges == len(shard.victims)
    for vb in shard.victims:
        assert len(vb) == k and len(set(vb)) == k and all(b < nl for b in vb), vb
        assert min(vb) >= shard.chunk_floor, "fp%d, %d qubits over %d ranks: victim bits %s" % (prec, n, world, vb)
        if nl - shard.min_victim_bit >= k:
            assert min(vb) >= shard.min_victim_bit, vb   # the page has k bits >= 8: the preference still holds
    if nl - shard.min_victim_bit < k:
        # the fallback still follows Belady's rule above the floor: the first exchange takes qubit 0 in fp64 (never used
        # again), and in fp32 the local qubits of the CNOT targets used last
        last = min(7, nl - 1)
        want = list(range(last - k + 1, last + 1)) if prec == 32 else [0] + list(range(last - k + 2, last + 1))
        assert shard.victims[0] == want, shard.victims


@pytest.mark.parametrize("p2p,prec,n,world", [(True, 32, 8, 16), (True, 32, 4, 4), (True, 64, 5, 8), (False, 32, 3, 4)])
def test_too_few_local_qubits_for_an_exchange_is_refused_at_construction(p2p, prec, n, world):
    """nl - floor < k: no exchange could run, so the engine refuses to exist instead of failing with EINVAL mid-circuit
    (checked before any page is allocated or any collective runs)"""
    with pytest.raises(ValueError, match="local qubits"):
        sharded.QEngineSharded(n, 0, random.Random(1), precision=prec, dist=None, world=world, rank=0, p2p=p2p)
