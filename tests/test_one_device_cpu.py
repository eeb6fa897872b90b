"""The one-device rank harness (tests/one_device.py) adds nothing but staging and synchronisation: the sharded engine over
the oracle restatement on CPU pages runs the deep deferral circuit of tests/test_sharded_cpu.py at 4 ranks, then a
ProbMaskAll and a MAll, once with torch.distributed itself and once through StagedDist, and both runs end in bit-identical
states, query results and exchange counts."""
import random

import numpy as np

from qrack_b200 import qscript

import one_device
import test_sharded_cpu as tsc


def _ranks(rank, world, dist, out):
    from oracle.sharded_cpu import restate_engine_factory
    from qrack_b200.sharded import QEngineSharded

    def make(n, perm):
        return QEngineSharded(n, perm, random.Random(1), 1.0 + 0j, precision=32, dist=dist, world=world, rank=rank,
                              device="cpu", make_engine=restate_engine_factory(32))
    regs, results = qscript.run(tsc.DEEP, make)
    q = regs[0]
    results = [v for _, vals in results for v in vals] + list(q.ProbMaskAll(0b1100001001)) + [q.MAll()]
    np.savez(out + ".%d.npz" % rank, state=q.GetQuantumState(), exchanges=q.be.exchanges,
             results=np.array(results, dtype=np.float64))


def test_staged_dist_changes_nothing_but_staging(tmp_path):
    world = 4
    runs = []
    for staged in (False, True):
        out = str(tmp_path / ("staged%d" % staged))
        one_device.spawn(_ranks, world, out, use_cuda=False, staged=staged)
        runs.append([np.load(out + ".%d.npz" % r) for r in range(world)])
    plain, proxied = runs
    assert int(plain[0]["exchanges"]) >= 2
    for r in range(world):
        for k in ("state", "results", "exchanges"):
            assert np.array_equal(plain[r][k], proxied[r][k]), (k, r)
            assert np.array_equal(proxied[r][k], proxied[0][k]), (k, r)
