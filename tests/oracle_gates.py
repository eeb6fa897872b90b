"""The oracle of the uniformly controlled gate and the local engines of the sharded gate tests (test infrastructure).

`QEngineRestateGates` is oracle.restate_engine.QEngineRestate with the backend primitive `uniformly_controlled` over the
restatement's orc_uniformly_controlled (state.cpp:1094-1198), so the float64 oracle runs every QInterface gate the sharded
engine does.  `restate_factory` and `EmuGatesShard` are the two local engines of the CPU tests with that primitive: the
oracle restatement over torch CPU pages, and tests/emu_shard.py's shard over the real fused planner.  `ref_scripts` are the
scripts of tests/golden/ref_gates_9q.f{32,64}.npz, the states the reference's QEngineCPU returns for them
(tests/golden/make_gates.py)."""
import math
import random
from ctypes import c_int, c_uint64, c_void_p

import numpy as np

from oracle.restate_engine import QEngineRestate, _RestateBackend
from qrack_b200.qengine import QEngineHost

import emu_engine
import emu_shard


def _uc(be, controls, target, mtrxs, skip_powers, skip_value_mask, nrm):
    if be.amps is None:
        return
    m = np.ascontiguousarray(np.asarray(mtrxs, dtype=be.cplx).reshape(-1))
    be.fn("orc_uniformly_controlled")(be._p(), c_int(be.nq), c_int(len(controls)), (c_int * max(1, len(controls)))(*controls),
                                      c_int(target), m.ctypes.data_as(c_void_p), c_int(len(skip_powers)),
                                      (c_uint64 * max(1, len(skip_powers)))(*skip_powers), c_uint64(skip_value_mask),
                                      be.creal(nrm))


class _GatesBackend(_RestateBackend):
    def uniformly_controlled(self, controls, target, mtrxs, skip_powers, skip_value_mask, nrm):
        _uc(self, controls, target, mtrxs, skip_powers, skip_value_mask, nrm)


class QEngineRestateGates(QEngineRestate):
    def _make_backend(self, n_qubits: int):
        return _GatesBackend(n_qubits, self.precision)


def restate_factory(precision: int = 32):
    """oracle/sharded_cpu.restate_engine_factory with the uniformly controlled primitive"""
    cplx = np.complex64 if precision == 32 else np.complex128

    def make(buf, n_local):
        q = QEngineRestateGates(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        q.be.amps = buf.numpy().view(cplx)  # shares memory with the torch page
        return q
    return make


class _EmuGatesBackend(emu_engine._EmuBackend):
    def uniformly_controlled(self, controls, target, mtrxs, skip_powers, skip_value_mask, nrm):
        self.flush()
        _uc(self, controls, target, mtrxs, skip_powers, skip_value_mask, nrm)


class _EmuGatesEngine(QEngineHost):
    def _make_backend(self, n_qubits: int):
        return _EmuGatesBackend(n_qubits, self.precision)


class EmuGatesShard(emu_shard.EmuP2PShard):
    def __init__(self, n_local, precision, dist, world, rank):
        super().__init__(n_local, precision, dist, world, rank)
        self.engine = _EmuGatesEngine(n_local, 0, random.Random(1), 1.0 + 0j, False, False, precision=precision)
        self.zero_live()


REF_N = 9


def _prep(n, seed):
    rng = random.Random(seed)
    text = "qubits %d\n" % n
    text += "".join("U %d %.17g %.17g %.17g\n" % (q, rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3)) for q in range(n))
    return text + "".join("CNOT %d %d\n" % (q, q + 1) for q in range(n - 1))


def _m8(rng):
    th, ph, la = (rng.uniform(-math.pi, math.pi) for _ in range(3))
    c, s = math.cos(th / 2), math.sin(th / 2)
    m = [complex(c), -complex(math.cos(la), math.sin(la)) * s, complex(math.cos(ph), math.sin(ph)) * s,
         complex(math.cos(ph + la), math.sin(ph + la)) * c]
    return " ".join("%.17g %.17g" % (z.real, z.imag) for z in m)


def _uc_line(rng, controls, target, skips=(), svm=0):
    words = ["UniformlyControlledSingleBit", str(len(controls))] + [str(c) for c in controls] + [str(target), str(len(skips))]
    words += [str(p) for p in skips] + [str(svm)] + [_m8(rng) for _ in range(1 << (len(controls) + len(skips)))]
    return " ".join(words) + "\n"


def ref_scripts(n=REF_N):
    """name -> script of the reference fixture: each family on the top qubits (rank bits of a sharded engine) and on low
    ones, CUniformParityRZ with controls inside its mask as well as outside, pending X gates (XMask) throughout"""
    rng = random.Random(29)
    t, u = n - 1, n - 2
    prz = (_prep(n, 1) + "XMask %d\n" % ((1 << t) | 0b10100)
           + "UniformParityRZ %d 0.37\nUniformParityRZ %d -1.1\n" % ((1 << t) | (1 << u) | 0b10110, (1 << t) | (1 << u))
           + "CUniformParityRZ 1 2 %d 0.9\n" % (0b1101 | (1 << t))             # local control inside the mask
           + "CUniformParityRZ 1 %d %d 0.55\n" % (t, (1 << t) | (1 << u) | 1)  # rank-bit control inside the mask
           + "CUniformParityRZ 2 4 %d %d -0.8\n" % (u, (1 << 4) | (1 << u))    # every mask bit is a control
           + "CUniformParityRZ 2 0 %d %d 1.3\n" % (t, 0b1000110)               # controls outside the mask
           + "".join("H %d\n" % q for q in range(n)) + "CUniformParityRZ 1 3 %d 0.21\n" % ((1 << n) - 1))
    uc = (_prep(n, 2) + "XMask %d\n" % ((1 << t) | (1 << u) | 0b110)
          + _uc_line(rng, [1, 3], 0) + _uc_line(rng, [2, t, 4], 5) + _uc_line(rng, [u, 1], 6, [2], 1)
          + _uc_line(rng, [3, t, 2], u, [8, 1], 5)
          + _uc_line(rng, [0], t, [2, 1], 3) + _uc_line(rng, [t, u], 3)
          + "UniformlyControlledRY 2 %d 1 0 0.3 -0.7 1.9 2.4\n" % t
          + "UniformlyControlledRZ 3 0 %d 5 2 %s\n" % (u, " ".join("%.3f" % (0.4 * k - 1.1) for k in range(8))))
    two = (_prep(n, 3) + "XMask %d\n" % ((1 << t) | 0b101000)
           + "ISwap 0 1\nSqrtSwap 2 %d\nISwap %d %d\nFSim 0.7 -1.3 %d 4\nFSim -2.1 0.4 %d %d\n" % (t, u, t, t, u, t)
           + "CSwap 2 3 %d 5 6\nCSwap 2 0 %d %d 1\nAntiCSwap 1 %d 2 4\nAntiCSwap 2 1 %d 6 %d\n" % (t, u, t, t, u, t))
    return {"prz": prz, "uc": uc, "two": two}
