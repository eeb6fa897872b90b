"""Test-only shard for QEngineSharded over gloo with the semantics of P2PShardBuffers (the k rank bits are exchanged with ANY k
local qubits) and a local engine whose gates go through the real fused planner + the host interpreter of its programs
(emu_engine.QEngineEmu).  Lets `-m "not gpu"` tests run the sharded scheduler on the planner the CUDA engine runs."""
import random

import numpy as np
import torch

from emu_engine import QEngineEmu


class EmuP2PShard:
    needs_top = False
    min_victim_bit = 1

    def __init__(self, n_local, precision, dist, world, rank):
        self.nl, self.precision, self.dist, self.world, self.rank = n_local, precision, dist, world, rank
        self.cplx = np.complex64 if precision == 32 else np.complex128
        self.real = np.float32 if precision == 32 else np.float64
        self.engine = QEngineEmu(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        self.device = "cpu"
        self.torch = torch
        self.zero_live()

    def zero_live(self):
        be = self.engine.be
        be.queue.clear()
        be.amps = np.zeros(1 << self.nl, dtype=self.cplx)

    def local_host(self, cplx):
        self.engine.be.flush()
        return self.engine.be.amps.copy()

    def stats(self):
        return {"flushes": self.engine.be.flushes}

    def exchange(self, dist, world, rank, k, victim_bits):
        be = self.engine.be
        be.flush()
        nl = self.nl
        # S: bring victim bit vb[b] to position nl-k+b (any bijection elsewhere); E: top-k bits <-> rank bits; then S^-1
        order = [None] * nl
        for b in range(k):
            order[nl - k + b] = victim_bits[b]
        rest = [q for q in range(nl) if q not in victim_bits]
        for p in range(nl):
            if order[p] is None:
                order[p] = rest.pop(0)
        axes = [nl - 1 - order[nl - 1 - j] for j in range(nl)]
        t = np.ascontiguousarray(be.amps.reshape([2] * nl).transpose(axes)).reshape(-1)
        src = torch.from_numpy(t.view(self.real))
        dst = torch.empty_like(src)
        chunk = src.numel() // world
        reqs = []
        for peer in range(world):
            if peer == rank:
                dst[peer * chunk:(peer + 1) * chunk].copy_(src[peer * chunk:(peer + 1) * chunk])
            else:
                reqs.append(dist.isend(src[peer * chunk:(peer + 1) * chunk].clone(), peer))
                reqs.append(dist.irecv(dst[peer * chunk:(peer + 1) * chunk], peer))
        for r in reqs:
            r.wait()
        u = dst.numpy().view(self.cplx).reshape([2] * nl)
        be.amps = np.ascontiguousarray(u.transpose(np.argsort(axes))).reshape(-1)
        return src.numel() * src.element_size() * (world - 1) // world
