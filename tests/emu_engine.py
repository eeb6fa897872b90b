"""Test-only engine: the reference dispatch mirror over a backend whose single-target gates go through the REAL fused
planner + encoder of libb200sv.so and the host interpreter of the encoded sweep programs (b200sv_emulate_fused — no
device needed); every other operation runs on the oracle restatement.  Lets `-m "not gpu"` tests check the scheduler and
the program encoding (pass tables, swizzle, DIAG groups, staged/direct passes) against the oracle."""
import ctypes

import numpy as np

from oracle.restate_engine import _RestateBackend
from qrack_b200 import _abi
from qrack_b200.qengine import QEngineHost


class _EmuBackend(_RestateBackend):
    def __init__(self, n_qubits: int, precision: int):
        super().__init__(n_qubits, precision)
        self.abi_lib = _abi.load()
        self.queue = []
        self.flushes = 0
        for name in dir(_RestateBackend):
            if name.startswith("_") or name in ("apply2x2", "fn", "finish", "xmask", "apply_gates", "flush"):
                continue
            attr = getattr(self, name)
            if callable(attr):
                setattr(self, name, self._flushing(attr))

    def _flushing(self, fn):
        def call(*a, **k):
            self.flush()
            return fn(*a, **k)
        return call

    def finish(self):
        self.flush()

    def apply2x2(self, off1, off2, mtrx, pows, nrm, thresh, calc_norm):
        diff = off1 ^ off2
        if calc_norm or diff == 0 or (diff & (diff - 1)) or self.nq < 5 or self.amps is None:
            self.flush()
            return super().apply2x2(off1, off2, mtrx, pows, nrm, thresh, calc_norm)
        pmask = 0
        for p in pows:
            pmask |= p
        self.queue.append((off1, off2, pmask, [complex(z) * nrm for z in mtrx]))
        return None

    def xmask(self, mask):
        # like b200sv_xmask with fusion on: queued as X gates (the rewrite turns XMask..XMask wrappers into control polarities)
        if self.nq < 5 or self.amps is None:
            self.flush()
            return super().xmask(mask)
        b = 0
        while mask >> b:
            if (mask >> b) & 1:
                self.queue.append((0, 1 << b, 1 << b, [0j, 1 + 0j, 1 + 0j, 0j]))
            b += 1

    def _packed(self, q):
        n = len(q)
        o1 = (ctypes.c_uint64 * n)(*[g[0] for g in q])
        o2 = (ctypes.c_uint64 * n)(*[g[1] for g in q])
        pm = (ctypes.c_uint64 * n)(*[g[2] for g in q])
        mats = (ctypes.c_double * (8 * n))()
        for i, g in enumerate(q):
            for k in range(4):
                mats[8 * i + 2 * k] = g[3][k].real
                mats[8 * i + 2 * k + 1] = g[3][k].imag
        return n, o1, o2, pm, mats

    def flush(self):
        if not self.queue:
            return
        q, self.queue = self.queue, []
        n, o1, o2, pm, mats = self._packed(q)
        self._alloc()
        rc = self.abi_lib.b200sv_emulate_fused(self.nq, self.precision, n, o1, o2, pm, mats, self.amps.ctypes.data_as(ctypes.c_void_p))
        _abi.check(self.abi_lib, rc)
        self.flushes += 1

    # ---- the batch entry point of the CUDA backend the sharded engine uses (qengine._CudaBackend.apply_gates) ----
    def apply_gates(self, n, off1, off2, pmasks, mats8):
        for i in range(n):
            self.queue.append((off1[i], off2[i], pmasks[i], [complex(mats8[8 * i + 2 * j], mats8[8 * i + 2 * j + 1]) for j in range(4)]))


class QEngineEmu(QEngineHost):
    def _make_backend(self, n_qubits: int):
        return _EmuBackend(n_qubits, self.precision)
