"""MAll's search for many shots on the device (b200sv_sample_keyed; b200sv_sample and b200sv_sample_many are its identity
call) on ONE device: the dyadic exact-boundary states against the float64 NumPy search exactly, random states up to 26 qubits
(a mismatch only where rnd lies within rounding of a cumulative boundary), key maps up to 64 bits, 0 / 1 / 2^20 shots, the
unnormalised and zero states, the launch count, what the call leaves alone, and every argument error.  With >= 2 GPUs
(skipped otherwise) the sharded engine runs the script of tests/test_sharded_sample_cpu.py over NCCL in all three exchange
modes."""
import ctypes
import math
import os
import random

import numpy as np
import pytest

from qrack_b200 import _abi

import npref
import test_kernels_vs_numpy_gpu as tk
import test_sharded_sample_cpu as scpu
from test_sharded_cpu import _free_port
from test_sharded_gpu import _ngpu
from test_topn_keyed_gpu import random_map

pytestmark = pytest.mark.gpu

BOUNDARY_TOL = {32: 1e-6, 64: 1e-12}  # fp32 rounds each |psi|^2 in single precision


def keys_of(idx, nq, pos, xr):
    """t(i) = xr ^ (OR over the bits b set in i of 2^pos[b]) for an array of indices (pos None: b -> b)"""
    idx = np.asarray(idx, dtype=np.uint64)
    t = np.zeros(idx.size, dtype=np.uint64)
    for b in range(nq):
        t |= ((idx >> np.uint64(b)) & np.uint64(1)) << np.uint64(b if pos is None else pos[b])
    return t ^ np.uint64(xr)


def np_search(psi, rnds, prec):
    """npref.sample for every rnd at once, and each rnd's distance to the nearest cumulative sum"""
    p = npref.probs(psi)
    nz = np.flatnonzero(p > npref.REAL1_EPSILON[prec])
    rnds = np.asarray(rnds, dtype=np.float64)
    if not nz.size:
        return np.full(rnds.size, p.size - 1, dtype=np.int64), np.full(rnds.size, np.inf)
    cum = np.cumsum(p[nz])
    early = np.flatnonzero((1.0 - cum) <= npref.FP_NORM_EPSILON[prec])
    first = np.searchsorted(cum, rnds, side="right")
    if early.size:
        first = np.minimum(first, early[0])
    want = nz[np.minimum(first, nz.size - 1)]
    at = np.searchsorted(cum, rnds)
    lo, hi = cum[np.clip(at - 1, 0, cum.size - 1)], cum[np.clip(at, 0, cum.size - 1)]
    return want.astype(np.int64), np.minimum(np.abs(lo - rnds), np.abs(hi - rnds))


def launches(q):
    return q.be.stats()["kernel_launches"]


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [12, 13, 15, 17])
def test_identity_key_on_exact_boundaries(n, prec):
    """the dyadic states of test_sample_exact_boundaries: the identity key is sample_many and npref.sample exactly"""
    s, t = 1 << (n - 3), 1 << (n - 2)
    cases = [
        {s + 4: 2, s + 6: 3, 2 * s + 2: 3, 3 * s: 1},
        dict([(2 * i + (t if i > 12 else 0), i + 1) for i in range(25)] + [(3 * t + 2, 25)]),
        {s + 4: 2, 3 * s: 3, 3 * s + 2: 3},
    ]
    for probs_at in cases:
        q = tk.engine(n, prec, tk.dyadic_state(n, probs_at, prec))
        psi = q.GetQuantumState()
        cum = sorted({float(c) for c in np.cumsum(npref.probs(psi)[sorted(probs_at)])})
        rnds = [0.0, 0.1, 0.5, 0.6, 0.9999999, 1 - 2.0 ** -26, 1 - 2.0 ** -40]
        rnds += cum[:-1] + [math.nextafter(c, 0) for c in cum[:-1]]
        want = [npref.sample(psi, r, prec) for r in rnds]
        for pos in (None, list(range(n))):
            got = q.be.sample_keyed(rnds, n, pos, 0)
            assert [int(v) for v in got] == want == q.be.sample_many(rnds), (probs_at, pos)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [1, 2, 13, 14, 15, 22, 26])
def test_random_states_vs_numpy(n, prec):
    rng = np.random.default_rng(n * 7 + prec)
    q = tk.engine(n, prec, tk.dense(rng, n, prec))
    psi = q.GetQuantumState()
    rnds = np.concatenate([rng.random(4096), [0.0, 1 - 2.0 ** -30, 0.999999]])
    got = q.be.sample_keyed(rnds, n, None, 0).astype(np.int64)
    want, dist = np_search(psi, rnds, prec)
    bad = np.flatnonzero(got != want)
    assert (dist[bad] <= BOUNDARY_TOL[prec]).all(), (n, bad[:5], rnds[bad[:5]], got[bad[:5]], want[bad[:5]], dist[bad[:5]])
    print("n=%d fp%d: %d of %d shots within rounding of a boundary differ from float64 NumPy" % (n, prec, bad.size, rnds.size))
    # one shot at a time is the same search
    some = rnds[rng.choice(rnds.size, 64, replace=False)]
    assert [q.be.sample(float(r)) for r in some] == [int(v) for v in q.be.sample_keyed(some, n, None, 0)]


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [5, 17, 20])
def test_key_maps(n, prec):
    rng = np.random.default_rng(3 * n + prec)
    q = tk.engine(n, prec, tk.dense(rng, n, prec))
    rnds = rng.random(3000)
    plain = np.asarray(q.be.sample_many(list(rnds)), dtype=np.uint64)
    for extra in (0, 1, 7, 64 - n):
        bits, pos, xr = random_map(rng, n, extra)
        got = q.be.sample_keyed(rnds, bits, pos, xr)
        assert np.array_equal(got, keys_of(plain, n, pos, xr)), (n, extra)
    # the widest key: position 63 and every XOR bit
    pos = [63] + list(range(1, n))
    got = q.be.sample_keyed(rnds, 64, pos, (1 << 64) - 1)
    assert np.array_equal(got, keys_of(plain, n, pos, (1 << 64) - 1))
    # key_xor on the positions of set index bits clears them (a page's pending X on a local qubit): the identity map with
    # an XOR is the sample XOR key_xor, checked without keys_of
    for xr in (1, (1 << n) - 1, 0b101 & ((1 << n) - 1)):
        assert np.array_equal(q.be.sample_keyed(rnds, n, None, xr), plain ^ np.uint64(xr)), (n, xr)
    rev = list(reversed(range(n)))
    want = [sum(1 << rev[b] for b in range(n) if (int(j) >> b) & 1) ^ 1 for j in plain[:200]]
    assert [int(v) for v in q.be.sample_keyed(rnds[:200], n, rev, 1)] == want


@pytest.mark.parametrize("prec", [32, 64])
def test_shot_counts(prec):
    """0 shots (no launch), 1 shot, and 2^20 shots over the 64 chunks of a 20-qubit state (every chunk holds ~16k shots)"""
    n = 20
    rng = np.random.default_rng(prec)
    q = tk.engine(n, prec, tk.dense(rng, n, prec))
    q.Finish()
    q.be.reset_stats()
    assert q.be.sample_keyed([], n, None, 0).size == 0 and q.be.sample_many([]) == [] and launches(q) == 0
    assert [int(v) for v in q.be.sample_keyed([0.3], n, None, 0)] == [q.be.sample(0.3)]
    rnds = rng.random(1 << 20)
    q.be.reset_stats()
    got = q.be.sample_keyed(rnds, n, None, 0).astype(np.int64)
    assert launches(q) == 2
    psi = q.GetQuantumState()
    want, dist = np_search(psi, rnds, prec)
    bad = np.flatnonzero(got != want)
    assert (dist[bad] <= BOUNDARY_TOL[prec]).all()
    assert np.unique(got >> 14).size == 1 << (n - 14)
    some = rng.choice(rnds.size, 200, replace=False)
    assert [q.be.sample(float(rnds[i])) for i in some] == [int(got[i]) for i in some]


@pytest.mark.parametrize("prec", [32, 64])
def test_unnormalised_zero_and_read_only(prec):
    n = 16
    rng = np.random.default_rng(11 + prec)
    psi = tk.dense(rng, n, prec) * np.asarray(0.5, dtype=np.float32 if prec == 32 else np.float64)
    q = tk.engine(n, prec, psi)
    for b in range(n):  # queued, unflushed gates are part of the state the search sees
        q.H(b)
        q.T(b)
    rnds = list(rng.random(500)) + [0.26, 0.9, 1.5]   # the total is 1/4: most rnds take the last nonzero index
    got = q.be.sample_keyed(rnds, n, None, 0)
    st = q.GetQuantumState()
    want, dist = np_search(st, rnds, prec)
    bad = np.flatnonzero(got.astype(np.int64) != want)
    assert (dist[bad] <= BOUNDARY_TOL[prec]).all()
    assert int(got[-1]) == int(np.flatnonzero(npref.probs(st) > npref.REAL1_EPSILON[prec])[-1])
    # two launches; bit-identical state; the memoised marginals survive without a new launch
    p3 = q.Prob(3)
    q.be.reset_stats()
    q.be.sample_keyed(rnds, n + 2, list(reversed(range(n))), 3)
    assert launches(q) == 2
    assert q.Prob(3) == p3 and launches(q) == 2
    assert np.array_equal(q.GetQuantumState(), st)
    # an all-zero buffer: the chunk sums only; the zero state: no launch.  Both give t(2^n - 1).
    pos = list(reversed(range(n)))
    z = tk.engine(n, prec, np.zeros(1 << n, dtype=np.complex64 if prec == 32 else np.complex128))
    z.Finish()
    z.be.reset_stats()
    want = int(keys_of([(1 << n) - 1], n, pos, 1 << n)[0])
    assert [int(v) for v in z.be.sample_keyed([0.0, 0.5], n + 1, pos, 1 << n)] == [want] * 2 and launches(z) == 1
    z.ZeroAmplitudes()
    z.be.reset_stats()
    assert [int(v) for v in z.be.sample_keyed([0.3], n + 1, pos, 1 << n)] == [want] and launches(z) == 0


@pytest.mark.parametrize("prec", [32, 64])
def test_every_einval(prec):
    n = 6
    q = tk.engine(n, prec, tk.dense(np.random.default_rng(1), n, prec))
    psi = q.GetQuantumState()
    lib, h, E = q.be.lib, q.be.h, _abi.B200SV_EINVAL
    fn = lib.b200sv_sample_keyed
    R, K = (ctypes.c_double * 4)(0.1, 0.5, 0.7, 0.99), (ctypes.c_uint64 * 4)()

    def pos(*v):
        return (ctypes.c_int * n)(*v)
    ident = pos(*range(n))
    assert fn(None, 4, R, n, ident, 0, K) == E
    assert fn(h, -1, R, n, ident, 0, K) == E
    assert fn(h, 4, None, n, ident, 0, K) == E and fn(h, 4, R, n, ident, 0, None) == E
    assert fn(h, 4, R, n - 1, None, 0, K) == E and fn(h, 4, R, 65, None, 0, K) == E
    assert fn(h, 4, R, n, pos(0, 1, 2, 3, 4, 4), 0, K) == E     # repeated
    assert fn(h, 4, R, n, pos(0, 1, 2, 3, 4, 6), 0, K) == E     # >= key_bits
    assert fn(h, 4, R, 8, pos(0, 1, 2, -1, 4, 5), 0, K) == E    # negative
    assert fn(h, 4, R, n, ident, 1 << n, K) == E and fn(h, 4, R, 8, None, 1 << 8, K) == E
    # 0 shots checks the key and writes nothing
    assert fn(h, 0, None, n, ident, 0, None) == 0 and fn(h, 0, None, n - 1, ident, 0, None) == E
    assert fn(h, 4, R, 64, pos(63, 1, 2, 3, 4, 5), (1 << 64) - 1, K) == 0
    plain = q.be.sample_many(list(R))
    assert list(K) == [int(v) for v in keys_of(plain, n, [63, 1, 2, 3, 4, 5], (1 << 64) - 1)]
    with pytest.raises(ValueError):
        q.be.sample_keyed([0.5], n, [0, 1], 0)
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
        scpu.run_cases(make, out_path + ".%d.npz" % rank)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["nccl", "push", "pull"])
@pytest.mark.parametrize("prec", [32, 64])
def test_sharded_sampling_on_gpus(prec, mode, tmp_path):
    """in pull mode the first query after the script's pending exchange runs directly after it (the page totals flush it)"""
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    world = 2 if _ngpu() < 4 else 4
    out = str(tmp_path / "s")
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_worker, args=(world, _free_port(), prec, out, mode), nprocs=world, join=True)
            break
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
    scpu.check_ranks_against_oracle([np.load(out + ".%d.npz" % r) for r in range(world)], prec, exact=False)
