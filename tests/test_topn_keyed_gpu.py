"""The top-n radix select under a tie key (b200sv_highest_probs_keyed) on ONE device, against the float64 NumPy select of
tests/test_sharded_topn_cpu.py, exactly: keys and P.  The identity map must give b200sv_highest_probs's list entry for entry;
permutation maps with an XOR and key_bits > qubits are what a page of the sharded engine passes.  Also P-tie states, n on both
sides of the 1 MiB scratch, a prefix class above and below the 2^20 candidate cap, the flush, what the call leaves alone, the
zero state and every argument error.  With >= 2 GPUs (skipped otherwise) the sharded engine runs the script of
tests/test_sharded_topn_cpu.py over NCCL in all three exchange modes against the oracle."""
import ctypes
import os
import random

import numpy as np
import pytest

from qrack_b200 import _abi

import test_sharded_topn_cpu as tcpu
import test_topn_gpu as tg
from test_sharded_cpu import _free_port
from test_sharded_gpu import _ngpu

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 5, 12, 17, 22]


def random_map(rng, nq, extra):
    """a rank's kind of map: the nq positions scattered over key_bits = nq + extra bits, and an XOR below 2^key_bits"""
    bits = nq + extra
    pos = [int(v) for v in rng.permutation(bits)[:nq]]
    return bits, pos, int.from_bytes(rng.bytes(8), "little") & ((1 << bits) - 1)


def check(q, ks, bits, pos, xr, what):
    """every n of ks against the first n entries of the NumPy order of all states (zero-filled alike)"""
    psi = q.be.get_state()
    wk, wp = tcpu.top_n_keyed(psi, psi.size, pos, xr)
    for k in ks:
        keys, probs = q.be.highest_probs_keyed(k, bits, pos, xr)
        assert np.array_equal(keys, wk[:k]), (what, k, np.flatnonzero(keys != wk[:k])[:5])
        assert np.array_equal(probs, wp[:k]), (what, k, np.flatnonzero(probs != wp[:k])[:5])
    return wk


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_identity_map_is_the_plain_select(n, prec):
    for kind in ("dense", "uniform", "blocks", "zeros"):
        q = tg.engine(n, prec, tg.make_state(kind, n, prec))
        ks = tg.sizes_for(n, q.be.get_state())
        for pos in (None, list(range(n))):
            keys = check(q, ks, n, pos, 0, (kind, pos is None))
        for k in ks:
            assert [int(v) for v in keys[:k]] == q.be.highest_probs(k), (kind, n, k)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_keyed_maps_vs_numpy(n, prec):
    rng = np.random.default_rng(17 * n + prec)
    for kind in tg.STATES if n <= 17 else ["dense", "uniform", "blocks"]:
        q = tg.engine(n, prec, tg.make_state(kind, n, prec, 1))
        psi = q.be.get_state()
        for extra in (0, 1, 3, 64 - n):
            bits, pos, xr = random_map(rng, n, extra)
            check(q, tg.sizes_for(n, psi), bits, pos, xr, (kind, extra))
        assert np.array_equal(q.be.get_state(), psi), kind


@pytest.mark.parametrize("prec", [32, 64])
def test_scratch_limit_and_candidate_cap(prec):
    """n past 65536 entries (16 B each) never fits the 1 MiB scratch; a fresh state's first keyed call grows its scratch after
    staging the key tables (n = 1000 at 14 qubits: 17384 entries; all 2^14: the output alone); a uniform state at 20 qubits is one class of exactly the
    2^20 candidate cap, at 22 qubits a class above it, so the index digits are resolved on the state by the keyed kernels"""
    rng = np.random.default_rng(prec)
    for nq, kind, ks in ((14, "dense", [1000, 1 << 14]), (17, "dense", [30000, 70000]),
                         (22, "dense", [60000, 70000]), (20, "uniform", [2, 70000]), (22, "uniform", [3, 4097]),
                         (22, "blocks", [5, 66000])):
        q = tg.engine(nq, prec, tg.make_state(kind, nq, prec, 2))
        bits, pos, xr = random_map(rng, nq, 2)
        check(q, ks, bits, pos, xr, (nq, kind))


@pytest.mark.parametrize("prec", [32, 64])
def test_read_only_flush_and_zero_state(prec):
    n = 11
    q = tg.engine(n, prec, tg.make_state("dense", n, prec, 2))
    for b in range(n):
        q.H(b)
        q.T(b)
    # queued, unflushed gates are part of the state the query sees
    pos = list(reversed(range(n)))
    keys, probs = q.be.highest_probs_keyed(50, n + 1, pos, 1 << n)
    psi = q.GetQuantumState()
    wk, wp = tcpu.top_n_keyed(psi, 50, pos, 1 << n)
    assert np.array_equal(keys, wk) and np.array_equal(probs, wp)
    # bit-identical state; memoised marginals survive without a new launch
    p3 = q.Prob(3)
    before = q.be.stats()["kernel_launches"]
    q.be.highest_probs_keyed(200, n, pos, 5)
    mid = q.be.stats()["kernel_launches"]
    assert mid > before
    assert q.Prob(3) == p3 and q.be.stats()["kernel_launches"] == mid
    assert np.array_equal(q.GetQuantumState(), psi)
    # the zero state: zeros without a launch
    q.ZeroAmplitudes()
    q.be.reset_stats()
    keys, probs = q.be.highest_probs_keyed(5, n, pos, 3)
    assert not keys.any() and not probs.any() and q.be.stats()["kernel_launches"] == 0


@pytest.mark.parametrize("prec", [32, 64])
def test_every_einval(prec):
    n = 6
    q = tg.engine(n, prec, tg.make_state("dense", n, prec, 3))
    psi = q.GetQuantumState()
    lib, h, E = q.be.lib, q.be.h, _abi.B200SV_EINVAL
    fn = lib.b200sv_highest_probs_keyed
    K, P = (ctypes.c_uint64 * 64)(), (ctypes.c_double * 64)()

    def pos(*v):
        return (ctypes.c_int * n)(*v)
    ident = pos(*range(n))
    assert fn(None, 3, n, ident, 0, K, P) == E
    assert fn(h, 3, n, ident, 0, None, P) == E and fn(h, 3, n, ident, 0, K, None) == E
    assert fn(h, 65, n, ident, 0, K, P) == E
    assert fn(h, 3, n - 1, None, 0, K, P) == E and fn(h, 3, 65, None, 0, K, P) == E
    assert fn(h, 3, n, pos(0, 1, 2, 3, 4, 4), 0, K, P) == E     # repeated
    assert fn(h, 3, n, pos(0, 1, 2, 3, 4, 6), 0, K, P) == E     # >= key_bits
    assert fn(h, 3, 8, pos(0, 1, 2, -1, 4, 5), 0, K, P) == E    # negative
    assert fn(h, 3, n, ident, 1 << n, K, P) == E and fn(h, 3, 8, None, 1 << 8, K, P) == E
    # n = 0 checks the key and writes nothing
    assert fn(h, 0, n, ident, 0, None, None) == 0 and fn(h, 0, n - 1, ident, 0, None, None) == E
    # the widest key: 64 bits, position 63, every XOR bit
    assert fn(h, 64, 64, pos(63, 1, 2, 3, 4, 5), (1 << 64) - 1, K, P) == 0
    wk, wp = tcpu.top_n_keyed(psi, 64, [63, 1, 2, 3, 4, 5], (1 << 64) - 1)
    assert list(K) == [int(v) for v in wk] and list(P) == list(wp)
    with pytest.raises(ValueError):
        q.be.highest_probs_keyed(3, n, [0, 1], 0)
    assert np.array_equal(q.GetQuantumState(), psi)


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
        tcpu.run_cases(make, out_path + ".%d.npz" % rank)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["nccl", "push", "pull"])
@pytest.mark.parametrize("prec", [32, 64])
def test_sharded_highest_prob_all_n_on_gpus_matches_the_oracle(prec, mode, tmp_path):
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    world = 2 if _ngpu() < 4 else 4
    out = str(tmp_path / "t")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out, mode), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    tcpu.check_ranks_against_oracle([np.load(out + ".%d.npz" % r) for r in range(world)], prec, exact=False)
