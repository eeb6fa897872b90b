"""Host-only model of a sharded step: replays a circuit through QEngineSharded's dispatch with a shard that moves no data, captures the
gate batch of every window (what `_submit_batch` hands to b200sv_apply_gates between two exchanges) and asks the REAL fused planner
(b200sv_plan_gates, host only) how many sweeps / passes / device ops each window costs.  No GPU, no torch.distributed."""
import ctypes
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qrack_b200 import _abi, qscript, sharded  # noqa: E402


class _Be:
    """stands in for the local CUDA backend: keeps the queued gates, plans them with the real planner when flushed"""

    def __init__(self, owner):
        self.owner = owner
        self.q = []
        self.lib = _abi.load()

    def apply_gates(self, n, o1, o2, pm, m8):
        for i in range(n):
            self.q.append((o1[i], o2[i], pm[i], [m8[8 * i + j] for j in range(8)]))
            if len(self.q) >= 4096:   # b200sv_apply_gates flushes a queue this long
                self.flush()

    def flush(self):
        g, self.q = self.q, []
        n = len(g)
        if not n:
            return
        o1 = (ctypes.c_uint64 * n)(*[x[0] for x in g])
        o2 = (ctypes.c_uint64 * n)(*[x[1] for x in g])
        pm = (ctypes.c_uint64 * n)(*[x[2] for x in g])
        m8 = (ctypes.c_double * (8 * n))(*[v for x in g for v in x[3]])
        sweeps, passes, ops = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _abi.check(self.lib, self.lib.b200sv_plan_gates(self.owner.n_local, 32, n, o1, o2, pm, m8, ctypes.byref(sweeps),
                                                        ctypes.byref(passes), ctypes.byref(ops)))
        self.owner.windows.append((n, sweeps.value))


class _NullEngine:
    runningNorm = 1.0

    n_local = 30

    def __init__(self):
        self.windows = []   # (gates in, sweeps launched) per local flush
        self.be = _Be(self)

    def Finish(self):
        pass

    def SetAmplitude(self, *a):
        pass


class _NullShard:
    min_victim_bit = 8
    needs_top = False

    def __init__(self):
        self.engine = _NullEngine()
        self.cuts = []

    def zero_live(self):
        pass

    def exchange(self, dist, world, rank, k, vbits):
        self.engine.be.flush()   # what the real exchange does first
        self.cuts.append(len(self.engine.windows))
        return 0


def windows(n_local, world, rank, text):
    _NullEngine.n_local = n_local

    class Eng(sharded.QEngineSharded):
        def _make_backend(self, n_qubits):
            return sharded._ShardedBackend(n_qubits, 32, _NullShard(), None, world, rank)

    def make(n, perm):
        return Eng(n, perm, random.Random(1), 1.0 + 0j, precision=32, world=world, rank=rank)
    regs, _ = qscript.run(text, make)
    q = regs[0]
    q.be.flush()
    q.be.shard.engine.be.flush()
    return q.be.exchanges, q.be.shard.engine.windows


def report(name, n_local, world, text, ranks=(0,), verbose=True):
    out = []
    for rank in ranks:
        ex, rows = windows(n_local, world, rank, text)
        sweeps = sum(r[1] for r in rows)
        out.append((ex, sweeps))
        if verbose:
            print("%s world %d rank %d: %d exchanges, %d local flushes, %d sweeps" % (name, world, rank, ex, len(rows), sweeps))
            print("   per flush (gates in / sweeps): " + " ".join("%d/%d" % r for r in rows))
    return out


if __name__ == "__main__":
    worlds = [int(a) for a in sys.argv[1:]] or [2, 8]
    for world in worlds:
        k = world.bit_length() - 1
        n = 30 + k
        report("htcnot", 30, world, qscript.random_htcnot(n, 40, seed=20250921, timed=False), ranks=(0, world - 1) if world > 1 else (0,))
        report("qv", 30, world, qscript.quantum_volume(n, depth=n, seed=33, timed=False))
        report("grover", 31, world, "\n".join(l for l in qscript.grover(31 + k, 3, target=3, timed=False).splitlines() if not l.startswith("ProbAll")) + "\n")
