"""Host-side mirror of the reference's ``QInterface``/``QEngine`` gate dispatch for the hot path.

``QEngineHost`` restates — with the reference's own method names, argument order and error behaviour — the
part of ``Qrack::QInterface`` / ``Qrack::QEngine`` that turns gates into ``Apply2x2`` / ``ApplyM`` / ``Prob``
calls (reference ``include/qinterface.hpp``, ``src/qengine/qengine.cpp``, ``src/qinterface/*.cpp``).  It owns the
QEngine-level bookkeeping (``runningNorm``, ``doNormalize``, ``randGlobalPhase``) and delegates every sweep over the
amplitudes to a *backend* through a small primitive interface.

``QEngineCUDA`` is that class over ``libb200sv.so`` (hand-written sm_90a kernels behind the C ABI in
``include/b200sv.h``).  It takes the reference's shared positional constructor signature
(``include/qengine_cuda.hpp:280-284``).  There is NO CPU fallback: if the CUDA library cannot be loaded the import of
the backend raises.

The C++ drop-in (``dropin/``) is the production adapter; this Python mirror exists so the parity tests and ``bench.py``
read like the reference's own tests (SURVEY.md §4) without needing the reference sources on the GPU box.
"""
from __future__ import annotations

import cmath
import math
import random
from typing import List, Optional, Sequence

import numpy as np

REAL1_DEFAULT_ARG = -999.0


class QEngineHost:
    """Gate dispatch + norm bookkeeping.  Subclasses provide ``self.be`` (backend primitives)."""

    # ---- construction -------------------------------------------------------------------------------------
    def __init__(self, qBitCount: int, initState: int = 0, rgp: Optional[random.Random] = None,
                 phaseFac: Optional[complex] = None, doNorm: bool = False, randomGlobalPhase: bool = True,
                 useHostMem: bool = False, deviceId: int = -1, useHardwareRNG: bool = True, useSparse: bool = False,
                 norm_thresh: Optional[float] = None, devList: Sequence[int] = (), qubitThreshold: int = 0,
                 sep_thresh: Optional[float] = None, precision: int = 32):
        if precision not in (32, 64):
            raise ValueError("precision must be 32 or 64")
        self.precision = precision
        self.real = np.float32 if precision == 32 else np.float64
        self.cplx = np.complex64 if precision == 32 else np.complex128
        # reference include/common/qrack_types.hpp:203-266
        self.REAL1_EPSILON = 1.7763568394002505e-15 if precision == 32 else 6.310887241768095e-30
        self.FP_NORM_EPSILON = float(np.finfo(self.real).eps) / 4
        self.qubitCount = int(qBitCount)
        self.doNormalize = bool(doNorm)
        self.randGlobalPhase = bool(randomGlobalPhase)
        self.amplitudeFloor = self.REAL1_EPSILON if norm_thresh is None else float(norm_thresh)
        self.runningNorm = 1.0
        self.rng = rgp if rgp is not None else random.Random()
        self.deviceId = deviceId
        self._ctor_args = dict(rgp=self.rng, doNorm=doNorm, randomGlobalPhase=randomGlobalPhase, useHostMem=useHostMem,
                               deviceId=deviceId, useHardwareRNG=useHardwareRNG, useSparse=useSparse,
                               norm_thresh=norm_thresh, devList=devList, qubitThreshold=qubitThreshold,
                               sep_thresh=sep_thresh, precision=precision)
        self.be = self._make_backend(self.qubitCount)
        if self.qubitCount:
            # reference QEngineCPU ctor, state.cpp:56-63
            ph = self.GetNonunitaryPhase() if phaseFac is None else complex(phaseFac)
            self.be.set_permutation(int(initState), ph)
        else:
            self.runningNorm = 0.0

    def _make_backend(self, n_qubits: int):  # pragma: no cover - abstract
        raise NotImplementedError

    # ---- small helpers ------------------------------------------------------------------------------------
    @property
    def maxQPower(self) -> int:
        return 1 << self.qubitCount

    def GetQubitCount(self) -> int:
        return self.qubitCount

    def GetMaxQPower(self) -> int:
        return self.maxQPower

    def Rand(self) -> float:
        return self.rng.random()

    def _c(self, z) -> complex:
        """round a python complex to the engine's complex type (what `complex(real1, real1)` does in the reference)"""
        try:
            return self._memo("c", z, lambda: complex(self.cplx(z)))
        except TypeError:
            return complex(self.cplx(z))

    def _r(self, x) -> float:
        try:
            return self._memo("r", x, lambda: float(self.real(x)))
        except TypeError:
            return float(self.real(x))

    def _norm(self, z) -> float:
        z = self.cplx(z)
        return float(self.real(z.real) * self.real(z.real) + self.real(z.imag) * self.real(z.imag))

    def _is_norm_0(self, z) -> bool:  # IS_NORM_0, qrack_types.hpp:28
        try:
            return self._memo("n", z, lambda: self._norm(z) <= self.FP_NORM_EPSILON)
        except TypeError:
            return self._norm(z) <= self.FP_NORM_EPSILON

    def GetNonunitaryPhase(self) -> complex:  # qinterface.hpp:169-177
        if self.randGlobalPhase:
            angle = self.Rand() * 2 * math.pi
            return self._c(complex(math.cos(angle), math.sin(angle)))
        return 1.0 + 0j

    @staticmethod
    def clampProb(p: float) -> float:  # qinterface.hpp:158-167
        return min(max(p, 0.0), 1.0)

    def _check_qubit(self, q: int, what: str):
        if q < 0 or q >= self.qubitCount:
            raise ValueError("%s qubit index parameter must be within allocated qubit bounds!" % what)

    # A circuit applies the same few matrices (H, T, X, ...) thousands of times; rounding them to the engine's complex type and
    # classifying them goes through numpy scalars (~1 us each), which is most of the per-gate cost of this mirror.  The results are
    # pure functions of the entries, so they are memoised per engine (the table is dropped when it grows: random-angle circuits).
    _MEMO_CAP = 4096

    def _memo(self, kind, key, fn):
        tab = self.__dict__.setdefault("_mtrx_memo", {})
        k = (kind, key)
        v = tab.get(k)
        if v is None:
            if len(tab) >= self._MEMO_CAP:
                tab.clear()
            v = tab[k] = fn()
        return v

    def _mtrx(self, m) -> List[complex]:
        try:
            key = tuple(m)
            return list(self._memo("m", key, lambda: tuple(self._c(x) for x in key)))
        except TypeError:  # unhashable entries: no memo
            return [self._c(x) for x in m]

    def IsPhase(self, m) -> bool:
        return self._memo("p", (m[1], m[2]), lambda: self._is_norm_0(m[1]) and self._is_norm_0(m[2]))

    def IsInvert(self, m) -> bool:
        return self._memo("i", (m[0], m[3]), lambda: self._is_norm_0(m[0]) and self._is_norm_0(m[3]))

    def _is_identity(self, m, isControlled: bool) -> bool:
        if not self._is_norm_0(self._c(m[0] - m[3])) or not self.IsPhase(m):
            return False
        if (isControlled or not self.randGlobalPhase) and not self._is_norm_0(self._c(1.0 - m[0])):
            return False
        return True

    def IsIdentity(self, m, isControlled: bool) -> bool:  # qengine.hpp:46-67
        return self._memo("d", (m[0], m[1], m[2], m[3], bool(isControlled), bool(self.randGlobalPhase)), lambda: self._is_identity(m, isControlled))

    # ---- the engine-level virtuals (reference qengine.hpp) ----------------------------------------------------------
    def Finish(self):
        self.be.finish()

    def Apply2x2(self, offset1: int, offset2: int, mtrx, bitCount: int, qPowersSorted: Sequence[int], doCalcNorm: bool,
                 norm_thresh: float = REAL1_DEFAULT_ARG):
        """QEngineCPU::Apply2x2 host part (state.cpp:392-431, 514-531): bounds checks and running-norm bookkeeping;
        the sweep itself is the backend's."""
        if self.be.is_zero():  # CHECK_ZERO_SKIP
            return
        maxq = self.maxQPower
        if offset1 >= maxq or offset2 >= maxq:
            raise ValueError("Apply2x2 offset1 and offset2 parameters must be within allocated qubit bounds!")
        for i in range(bitCount):
            if qPowersSorted[i] >= maxq:
                raise ValueError("Apply2x2 parameter qPowsSorted array values must be within allocated qubit bounds!")
            if i and qPowersSorted[i - 1] == qPowersSorted[i]:
                raise ValueError("Apply2x2 parameter qPowSorted array values cannot be duplicated!")
        doApplyNorm = self.doNormalize and bitCount == 1 and self.runningNorm > 0
        doCalcNorm = doCalcNorm and (doApplyNorm or self.runningNorm <= 0)
        nrm = self._r(1.0 / math.sqrt(self.runningNorm)) if doApplyNorm else 1.0
        if doCalcNorm:
            self.runningNorm = 1.0
        thresh = self.amplitudeFloor if norm_thresh < 0 else norm_thresh
        res = self.be.apply2x2(offset1, offset2, self._mtrx(mtrx), list(qPowersSorted[:bitCount]), nrm,
                               thresh if doCalcNorm else 0.0, doCalcNorm)
        if doApplyNorm:
            self.runningNorm = 1.0
        if doCalcNorm:
            self.runningNorm = self._r(res)
            if self.runningNorm <= self.FP_NORM_EPSILON:
                self.ZeroAmplitudes()

    def Mtrx(self, mtrx, qubit: int):  # qengine.cpp:19-27
        mtrx = self._mtrx(mtrx)
        if self.IsIdentity(mtrx, False):
            return
        p = 1 << qubit
        self._check_qubit(qubit, "Mtrx")
        self.Apply2x2(0, p, mtrx, 1, [p], self.doNormalize and not (self.IsPhase(mtrx) or self.IsInvert(mtrx)))

    def EitherMtrx(self, controls, mtrx, target: int, isAnti: bool):  # qengine.cpp:29-48
        if not controls:
            return self.Mtrx(mtrx, target)
        mtrx = self._mtrx(mtrx)
        if self.IsIdentity(mtrx, True):
            return
        if isAnti:
            self.ApplyAntiControlled2x2(controls, target, mtrx)
        else:
            self.ApplyControlled2x2(controls, target, mtrx)
        if self.doNormalize and not (self.IsPhase(mtrx) or self.IsInvert(mtrx)):
            self.UpdateRunningNorm()

    def MCMtrx(self, controls, mtrx, target: int):
        self.EitherMtrx(list(controls), mtrx, target, False)

    def MACMtrx(self, controls, mtrx, target: int):  # QEngine::MACMtrx, qengine.hpp:173-176
        self.EitherMtrx(list(controls), mtrx, target, True)

    def _powers(self, qubits) -> List[int]:
        for q in qubits:
            self._check_qubit(q, "control/target")
        p = sorted(1 << q for q in qubits)
        return p

    def ApplyControlled2x2(self, controls, target, mtrx):  # qengine.cpp:371-385
        pows = self._powers(list(controls) + [target])
        cmask = 0
        for c in controls:
            cmask |= 1 << c
        self.Apply2x2(cmask, cmask | (1 << target), mtrx, len(pows), pows, False)

    def ApplyAntiControlled2x2(self, controls, target, mtrx):  # qengine.cpp:387-397
        pows = self._powers(list(controls) + [target])
        self.Apply2x2(0, 1 << target, mtrx, len(pows), pows, False)

    def UCMtrx(self, controls, mtrx, target: int, controlPerm: int):  # qengine.cpp:50-75
        if not controls:
            return self.Mtrx(mtrx, target)
        mtrx = self._mtrx(mtrx)
        if self.IsIdentity(mtrx, True):
            return
        pows = self._powers(list(controls) + [target])
        cmask = 0
        for i, c in enumerate(controls):
            if (controlPerm >> i) & 1:
                cmask |= 1 << c
        self.Apply2x2(cmask, cmask | (1 << target), mtrx, len(pows), pows, False)

    # ---- QInterface gate sugar (qinterface.hpp:503-1350) --------------------------------------------------------
    def Phase(self, topLeft, bottomRight, qubit: int):  # :534-542
        tl, br = self._c(topLeft), self._c(bottomRight)
        if (self.randGlobalPhase or self._is_norm_0(self._c(1.0 - tl))) and self._is_norm_0(self._c(tl - br)):
            return
        self.Mtrx([tl, 0j, 0j, br], qubit)

    def Invert(self, topRight, bottomLeft, qubit: int):  # :547-551
        self.Mtrx([0j, self._c(topRight), self._c(bottomLeft), 0j], qubit)

    def MCPhase(self, controls, topLeft, bottomRight, target: int):  # :556-565
        tl, br = self._c(topLeft), self._c(bottomRight)
        if self._is_norm_0(self._c(1.0 - tl)) and self._is_norm_0(self._c(1.0 - br)):
            return
        self.MCMtrx(controls, [tl, 0j, 0j, br], target)

    def MCInvert(self, controls, topRight, bottomLeft, target: int):  # :571-576
        self.MCMtrx(controls, [0j, self._c(topRight), self._c(bottomLeft), 0j], target)

    def MACWrapper(self, controls, fn):  # :179-189
        xMask = 0
        for c in controls:
            xMask |= 1 << c
        self.XMask(xMask)
        fn(controls)
        self.XMask(xMask)

    def MACPhase(self, controls, topLeft, bottomRight, target: int):  # :581-592
        tl, br = self._c(topLeft), self._c(bottomRight)
        if self._is_norm_0(self._c(1.0 - tl)) and self._is_norm_0(self._c(1.0 - br)):
            return
        self.MACWrapper(list(controls), lambda lc: self.MCPhase(lc, tl, br, target))

    def MACInvert(self, controls, topRight, bottomLeft, target: int):  # :597-603
        self.MACWrapper(list(controls), lambda lc: self.MCInvert(lc, topRight, bottomLeft, target))

    def H(self, q: int):  # :931-937
        s = self._r(math.sqrt(0.5))
        self.Mtrx([s, s, s, -s], q)

    def X(self, q: int):
        self.Invert(1.0, 1.0, q)

    def Y(self, q: int):
        self.Invert(-1j, 1j, q)

    def Z(self, q: int):
        self.Phase(1.0, -1.0, q)

    def S(self, q: int):
        self.Phase(1.0, 1j, q)

    def IS(self, q: int):
        self.Phase(1.0, -1j, q)

    def T(self, q: int):  # :1059
        s = self._r(math.sqrt(0.5))
        self.Phase(1.0, complex(s, s), q)

    def IT(self, q: int):
        s = self._r(math.sqrt(0.5))
        self.Phase(1.0, complex(s, -s), q)

    def SqrtX(self, q: int):  # :1151-1157
        self.Mtrx([complex(0.5, 0.5), complex(0.5, -0.5), complex(0.5, -0.5), complex(0.5, 0.5)], q)

    def _root_phase(self, n: int, inverse: bool = False) -> complex:
        # pow(-ONE_CMPLX, (real1)(+-ONE_R1 / pow2Ocl(n - 1U))), qinterface.hpp:1079,1346,1378.  NOTE: -ONE_CMPLX is
        # (-1, -0), whose std::arg is -pi, so the reference's "root-N" phase is e^{-i pi / 2^(n-1)} (matching the
        # "-2*PI/2^N" of its doc comment and PhaseRootNMask, state.cpp:1072); the inverse gate conjugates it.
        x = self._r(1.0 / (1 << (n - 1)))
        theta = self._r((-x if inverse else x) * self._r(-math.pi))
        return self._c(complex(math.cos(theta), math.sin(theta)))

    def PhaseRootN(self, n: int, q: int):  # :1073-1080
        if n == 0:
            return
        self.Phase(1.0, self._root_phase(n), q)

    def CPhaseRootN(self, n: int, control: int, target: int):  # :1339-1347
        if n == 0:
            return
        self.MCPhase([control], 1.0, self._root_phase(n), target)

    def CNOT(self, c: int, t: int):  # :727-731
        self.MCInvert([c], 1.0, 1.0, t)

    def AntiCNOT(self, c: int, t: int):  # :738-742
        self.MACInvert([c], 1.0, 1.0, t)

    def CCNOT(self, c1: int, c2: int, t: int):  # :705-709
        self.MCInvert([c1, c2], 1.0, 1.0, t)

    def CY(self, c: int, t: int):
        self.MCInvert([c], -1j, 1j, t)

    def CZ(self, c: int, t: int):  # :796-800
        self.MCPhase([c], 1.0, -1.0, t)

    def U(self, target: int, theta: float, phi: float, lam: float):  # rotational.cpp:18-26
        cos0 = self._r(math.cos(theta / 2))
        sin0 = self._r(math.sin(theta / 2))
        m = [complex(cos0, 0.0),
             sin0 * self._c(complex(-math.cos(lam), -math.sin(lam))),
             sin0 * self._c(complex(math.cos(phi), math.sin(phi))),
             cos0 * self._c(complex(math.cos(phi + lam), math.sin(phi + lam)))]
        self.Mtrx(m, target)

    def AI(self, target: int, azimuth: float, inclination: float):  # rotational.cpp:53-61
        ca, sa = self._r(math.cos(azimuth)), self._r(math.sin(azimuth))
        ci, si = self._r(math.cos(inclination / 2)), self._r(math.sin(inclination / 2))
        self.Mtrx([ci, self._c(complex(-ca, sa)) * si, self._c(complex(ca, sa)) * si, ci], target)

    def IAI(self, target: int, azimuth: float, inclination: float):  # rotational.cpp:64-75 (inverse of AI)
        ca, sa = self._r(math.cos(azimuth)), self._r(math.sin(azimuth))
        ci, si = self._r(math.cos(inclination / 2)), self._r(math.sin(inclination / 2))
        m = [ci, self._c(complex(-ca, sa)) * si, self._c(complex(ca, sa)) * si, ci]
        # inv2x2 of a unitary = conjugate transpose
        inv = [m[0].conjugate(), m[2].conjugate(), m[1].conjugate(), m[3].conjugate()]
        self.Mtrx(inv, target)

    def QFT(self, start: int, length: int, trySeparate: bool = False):  # qinterface.cpp:114-133
        if not length:
            return
        end = start + (length - 1)
        for i in range(length):
            hBit = end - i
            for j in range(i):
                self.CPhaseRootN(j + 2, hBit, hBit + 1 + j)
            self.H(hBit)

    def IQFT(self, start: int, length: int, trySeparate: bool = False):  # qinterface.cpp:136-155
        if not length:
            return
        for i in range(length):
            for j in range(i):
                c = (start + i) - (j + 1)
                t = start + i
                self.CIPhaseRootN(j + 2, c, t)
            self.H(start + i)

    def CIPhaseRootN(self, n: int, control: int, target: int):  # qinterface.hpp:1369-1377
        if n == 0:
            return
        self.MCPhase([control], 1.0, self._root_phase(n, inverse=True), target)

    def ZeroPhaseFlip(self, start: int, length: int):  # gates.cpp:84-99
        if not length:
            return
        if length == 1:
            return self.Phase(-1.0, 1.0, start)
        controls = [start + i for i in range(length - 1)]
        self.MACPhase(controls, -1.0, 1.0, start + len(controls))

    def INC(self, toAdd: int, start: int, length: int):
        """QEngineCPU::INC (src/qengine/arithmetic.cpp:73-118) as one basis-map sweep when the backend has ALU kernels;
        otherwise the gate-level QInterface::INC (src/qinterface/arithmetic.cpp:20-51)."""
        if self._has_alu():
            self._check_range(start, length, "INC")
            return self.be.alu_inc(toAdd & self._U64, start, length, 0)
        if not length:
            return
        if length == 1:
            if toAdd & 1:
                self.X(start)
            return
        bits = [start + i for i in range(length)]
        lengthMin1 = length - 1
        for i in range(length):
            if not ((toAdd >> i) & 1):
                continue
            self.X(start + i)
            for j in range(lengthMin1 - i):
                self.MACInvert(bits[i:i + j + 1], 1.0, 1.0, start + ((i + j + 1) % length))

    def DEC(self, toSub: int, start: int, length: int):  # qinterface.hpp:2050-2054: INC(2^length - toSub)
        invToSub = (1 << length) - toSub
        self.INC(invToSub & ((1 << length) - 1), start, length)

    # ------------------------------------------------------------------------------------------------
    # QAlu (include/qalu.hpp, src/qalu.cpp, src/qengine/arithmetic.cpp).  Engines whose backend provides the basis-map
    # primitives (``alu_*``) run each member as ONE sweep; otherwise INC/DEC fall back to the gate-level QInterface form.
    # ------------------------------------------------------------------------------------------------
    _U64 = (1 << 64) - 1

    def _has_alu(self) -> bool:
        return hasattr(self.be, "alu_inc")

    def _need_alu(self, what: str):
        if not self._has_alu():
            raise NotImplementedError("%s needs an engine with native ALU kernels" % what)

    def _check_range(self, start: int, length: int, what: str):  # isBadBitRange
        if start < 0 or length < 0 or start + length > self.qubitCount:
            raise ValueError("%s range is out-of-bounds!" % what)

    def _ctrl_mask(self, controls, what: str) -> int:  # ThrowIfQbIdArrayIsBad
        m = 0
        for c in controls:
            self._check_qubit(c, what + " control")
            m |= 1 << c
        return m

    def SetBit(self, qubit: int, value: bool):  # qinterface.hpp: if (value != M(qubit)) X(qubit)
        if bool(value) != self.M(qubit):
            self.X(qubit)

    def MReg(self, start: int, length: int) -> int:
        return self.ForceMReg(start, length, 0, False, True)

    def SetReg(self, start: int, length: int, value: int):  # src/qinterface/qinterface.cpp:195-212
        if length == 1:
            return self.SetBit(start, bool(value & 1))
        if start == 0 and length == self.qubitCount:
            return self.SetPermutation(value)
        reg = self.MReg(start, length)
        for i in range(length):
            if ((reg >> i) & 1) != ((value >> i) & 1):
                self.X(start + i)

    def ROL(self, shift: int, start: int, length: int):  # arithmetic.cpp:23-70
        self._need_alu("ROL")
        self._check_range(start, length, "ROL")
        self.be.alu_rol(shift, start, length)

    def ROR(self, shift: int, start: int, length: int):  # qengine.hpp: ROL(length - shift)
        if not length:
            return
        self.ROL(length - (shift % length), start, length)

    def CINC(self, toAdd: int, start: int, length: int, controls):  # arithmetic.cpp:121-172
        self._need_alu("CINC")
        self._check_range(start, length, "CINC")
        self.be.alu_inc(toAdd & self._U64, start, length, self._ctrl_mask(controls, "CINC"))

    def CDEC(self, toSub: int, start: int, length: int, controls):  # qalu.cpp:30-34
        self.CINC(((1 << length) - toSub) & self._U64, start, length, controls)

    def INCDECC(self, toMod: int, start: int, length: int, carryIndex: int):  # arithmetic.cpp:175-224
        self._need_alu("INCDECC")
        self._check_range(start, length, "INCDECC")
        self._check_qubit(carryIndex, "INCDECC carryIndex")
        self.be.alu_incdecc(toMod & self._U64, start, length, carryIndex)

    def INCC(self, toAdd: int, start: int, length: int, carryIndex: int):  # qalu.cpp:48-61
        if not length:
            return
        if self.M(carryIndex):
            self.X(carryIndex)
            self.INCDECC((toAdd + 1) & self._U64, start, length, carryIndex)
        else:
            self.INCDECC(toAdd, start, length, carryIndex)

    def _inv_carry(self, toSub: int, length: int, carryIndex: int) -> int:  # qalu.cpp:64-77 (shared by DECC / DECSC)
        inv = (1 << length) - toSub
        if self.M(carryIndex):
            self.X(carryIndex)
        elif inv == 0:
            inv = self._U64
        else:
            inv -= 1
        return inv & self._U64

    def DECC(self, toSub: int, start: int, length: int, carryIndex: int):
        self.INCDECC(self._inv_carry(toSub, length, carryIndex), start, length, carryIndex)

    def INCS(self, toAdd: int, start: int, length: int, overflowIndex: int):  # arithmetic.cpp:227-309
        self._need_alu("INCS")
        self._check_range(start, length, "INCS")
        self._check_qubit(overflowIndex, "INCS overflowIndex")
        self.be.alu_incs(toAdd & self._U64, start, length, overflowIndex)

    def DECS(self, toSub: int, start: int, length: int, overflowIndex: int):  # qalu.cpp:41-45
        self.INCS(((1 << length) - toSub) & self._U64, start, length, overflowIndex)

    def INCDECSC(self, toMod: int, start: int, length: int, *idx):  # arithmetic.cpp:312-419; idx = (carry) | (overflow, carry)
        self._need_alu("INCDECSC")
        self._check_range(start, length, "INCDECSC")
        overflowIndex, carryIndex = (-1, idx[0]) if len(idx) == 1 else (idx[0], idx[1])
        self._check_qubit(carryIndex, "INCDECSC carryIndex")
        if overflowIndex >= 0:
            self._check_qubit(overflowIndex, "INCDECSC overflowIndex")
        self.be.alu_incdecsc(toMod & self._U64, start, length, overflowIndex, carryIndex)

    def INCSC(self, toAdd: int, start: int, length: int, *idx):  # qalu.cpp:85-96, 131-140
        carryIndex = idx[-1]
        if self.M(carryIndex):
            self.X(carryIndex)
            self.INCDECSC((toAdd + 1) & self._U64, start, length, *idx)
        else:
            self.INCDECSC(toAdd, start, length, *idx)

    def DECSC(self, toSub: int, start: int, length: int, *idx):  # qalu.cpp:103-117, 148-160
        self.INCDECSC(self._inv_carry(toSub, length, idx[-1]), start, length, *idx)

    def MUL(self, toMul: int, inOutStart: int, carryStart: int, length: int):  # arithmetic.cpp:458-471
        self._need_alu("MUL")
        self.SetReg(carryStart, length, 0)
        if toMul == 0:
            return self.SetReg(inOutStart, length, 0)
        if toMul == 1:
            return
        self._check_range(inOutStart, length, "MUL")
        self._check_range(carryStart, length, "MUL carry")
        self.be.alu_muldiv(0, toMul & self._U64, inOutStart, carryStart, length, 0)

    def DIV(self, toDiv: int, inOutStart: int, carryStart: int, length: int):  # :474-485
        self._need_alu("DIV")
        if toDiv == 0:
            raise ValueError("DIV by zero")
        if toDiv == 1:
            return
        self._check_range(inOutStart, length, "DIV")
        self._check_range(carryStart, length, "DIV carry")
        self.be.alu_muldiv(1, toDiv & self._U64, inOutStart, carryStart, length, 0)

    def CMUL(self, toMul: int, inOutStart: int, carryStart: int, length: int, controls):  # :553-573
        if not controls:
            return self.MUL(toMul, inOutStart, carryStart, length)
        self._need_alu("CMUL")
        self.SetReg(carryStart, length, 0)
        if toMul == 0:
            return self.SetReg(inOutStart, length, 0)
        if toMul == 1:
            return
        self._check_range(inOutStart, length, "CMUL")
        self._check_range(carryStart, length, "CMUL carry")
        self.be.alu_muldiv(0, toMul & self._U64, inOutStart, carryStart, length, self._ctrl_mask(controls, "CMUL"))

    def CDIV(self, toDiv: int, inOutStart: int, carryStart: int, length: int, controls):  # :575-593
        if not controls:
            return self.DIV(toDiv, inOutStart, carryStart, length)
        self._need_alu("CDIV")
        if toDiv == 0:
            raise ValueError("CDIV by zero")
        if toDiv == 1:
            return
        self._check_range(inOutStart, length, "CDIV")
        self._check_range(carryStart, length, "CDIV carry")
        self.be.alu_muldiv(1, toDiv & self._U64, inOutStart, carryStart, length, self._ctrl_mask(controls, "CDIV"))

    def _modnout(self, kind: int, toMod: int, modN: int, inStart: int, outStart: int, length: int, controls, what: str):
        self._need_alu(what)
        self._check_range(inStart, length, what + " inStart")
        self._check_range(outStart, length, what + " outStart")
        self.be.alu_modnout(kind, toMod & self._U64, modN & self._U64, inStart, outStart, length,
                             self._ctrl_mask(controls, what))

    def MULModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int):  # :634-644
        self.SetReg(outStart, length, 0)
        if toMod == 0:
            return
        self._modnout(0, toMod, modN, inStart, outStart, length, (), "MULModNOut")

    def IMULModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int):  # :647-655
        if toMod == 0:
            return
        self._modnout(1, toMod, modN, inStart, outStart, length, (), "IMULModNOut")

    def POWModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int):  # :658-667
        if toMod == 1:
            return self.SetReg(outStart, length, 1)
        self._modnout(2, toMod, modN, inStart, outStart, length, (), "POWModNOut")

    def CMULModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int, controls):  # :737-748
        if not controls:
            return self.MULModNOut(toMod, modN, inStart, outStart, length)
        self.SetReg(outStart, length, 0)
        self._modnout(0, toMod, modN, inStart, outStart, length, controls, "CMULModNOut")

    def CIMULModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int, controls):  # :751-760
        if not controls:
            return self.IMULModNOut(toMod, modN, inStart, outStart, length)
        self._modnout(1, toMod, modN, inStart, outStart, length, controls, "CIMULModNOut")

    def CPOWModNOut(self, toMod: int, modN: int, inStart: int, outStart: int, length: int, controls):  # :763-774
        if not controls:
            return self.POWModNOut(toMod, modN, inStart, outStart, length)
        self._modnout(2, toMod, modN, inStart, outStart, length, controls, "CPOWModNOut")

    def _table(self, values, entries: int, entryBytes: int) -> bytes:
        b = bytes(values)
        if len(b) < entries * entryBytes:
            raise ValueError("classical table is too short")
        return b

    def IndexedLDA(self, indexStart: int, indexLength: int, valueStart: int, valueLength: int, values,
                   resetValue: bool = True) -> int:  # :983-1083
        self._need_alu("IndexedLDA")
        self._check_range(indexStart, indexLength, "IndexedLDA index")
        self._check_range(valueStart, valueLength, "IndexedLDA value")
        if resetValue:
            self.SetReg(valueStart, valueLength, 0)
        tab = self._table(values, 1 << indexLength, (valueLength + 7) >> 3)
        self.be.alu_indexed(0, indexStart, indexLength, valueStart, valueLength, 0, 0, tab)
        return 0

    def IndexedADC(self, indexStart: int, indexLength: int, valueStart: int, valueLength: int, carryIndex: int,
                   values) -> int:  # :1086-1260
        self._need_alu("IndexedADC")
        self._check_range(indexStart, indexLength, "IndexedADC index")
        self._check_range(valueStart, valueLength, "IndexedADC value")
        self._check_qubit(carryIndex, "IndexedADC carryIndex")
        carryIn = 0
        if self.M(carryIndex):
            carryIn = 1
            self.X(carryIndex)
        tab = self._table(values, 1 << indexLength, (valueLength + 7) >> 3)
        self.be.alu_indexed(1, indexStart, indexLength, valueStart, valueLength, carryIndex, carryIn, tab)
        return 0

    def IndexedSBC(self, indexStart: int, indexLength: int, valueStart: int, valueLength: int, carryIndex: int,
                   values) -> int:  # :1263-1444
        self._need_alu("IndexedSBC")
        self._check_range(indexStart, indexLength, "IndexedSBC index")
        self._check_range(valueStart, valueLength, "IndexedSBC value")
        self._check_qubit(carryIndex, "IndexedSBC carryIndex")
        carryIn = 1
        if self.M(carryIndex):
            carryIn = 0
            self.X(carryIndex)
        tab = self._table(values, 1 << indexLength, (valueLength + 7) >> 3)
        self.be.alu_indexed(2, indexStart, indexLength, valueStart, valueLength, carryIndex, carryIn, tab)
        return 0

    def Hash(self, start: int, length: int, values):  # :1447-1506
        self._need_alu("Hash")
        self._check_range(start, length, "Hash")
        self.be.alu_hash(start, length, self._table(values, 1 << length, (length + 7) >> 3))

    def PhaseFlipIfLess(self, greaterPerm: int, start: int, length: int):  # :1703-1720
        self._need_alu("PhaseFlipIfLess")
        self._check_range(start, length, "PhaseFlipIfLess")
        self.be.alu_phase_flip_if_less(greaterPerm & self._U64, start, length, -1)

    def CPhaseFlipIfLess(self, greaterPerm: int, start: int, length: int, flagIndex: int):  # :1678-1701
        self._need_alu("CPhaseFlipIfLess")
        self._check_range(start, length, "CPhaseFlipIfLess")
        self._check_qubit(flagIndex, "CPhaseFlipIfLess flagIndex")
        self.be.alu_phase_flip_if_less(greaterPerm & self._U64, start, length, flagIndex)

    # swap family (qengine.cpp:407-460)
    def _swap2(self, q1: int, q2: int, m):
        if q1 == q2:
            return
        if q2 < q1:
            q1, q2 = q2, q1
        self._check_qubit(q2, "Swap")
        self._check_qubit(q1, "Swap")
        p = [1 << q1, 1 << q2]
        self.Apply2x2(p[0], p[1], m, 2, p, False)

    def Swap(self, q1: int, q2: int):
        self._swap2(q1, q2, [0j, 1.0, 1.0, 0j])

    def ISwap(self, q1: int, q2: int):
        self._swap2(q1, q2, [0j, 1j, 1j, 0j])

    def IISwap(self, q1: int, q2: int):
        self._swap2(q1, q2, [0j, -1j, -1j, 0j])

    def SqrtSwap(self, q1: int, q2: int):
        self._swap2(q1, q2, [complex(0.5, 0.5), complex(0.5, -0.5), complex(0.5, -0.5), complex(0.5, 0.5)])

    def ISqrtSwap(self, q1: int, q2: int):
        self._swap2(q1, q2, [complex(0.5, -0.5), complex(0.5, 0.5), complex(0.5, 0.5), complex(0.5, -0.5)])

    def FSim(self, theta: float, phi: float, q1: int, q2: int):  # qengine.cpp:443-460
        if q2 < q1:
            q1, q2 = q2, q1
        sinTheta = self._r(math.sin(theta))
        if sinTheta * sinTheta > self.FP_NORM_EPSILON:
            cosTheta = self._r(math.cos(theta))
            p = [1 << q1, 1 << q2]
            self.Apply2x2(p[0], p[1], [complex(cosTheta, 0), complex(0, -sinTheta), complex(0, -sinTheta),
                                       complex(cosTheta, 0)], 2, p, False)
        self.MCPhase([q1], 1.0, self._c(cmath.exp(complex(0, -self._r(phi)))), q2)

    def _cswap(self, controls, q1, q2, m, anti: bool):  # qengine.cpp:212-369
        if q1 == q2:
            return
        if q2 < q1:
            q1, q2 = q2, q1
        pows = self._powers(list(controls) + [q1, q2])
        skip = 0
        if not anti:
            for c in controls:
                skip |= 1 << c
        self.Apply2x2(skip | (1 << q1), skip | (1 << q2), m, len(pows), pows, False)

    def CSwap(self, controls, q1: int, q2: int):
        if not controls:
            return self.Swap(q1, q2)
        self._cswap(controls, q1, q2, [0j, 1.0, 1.0, 0j], False)

    def AntiCSwap(self, controls, q1: int, q2: int):
        if not controls:
            return self.Swap(q1, q2)
        self._cswap(controls, q1, q2, [0j, 1.0, 1.0, 0j], True)

    # masks (QEngineCPU overrides, state.cpp:965-1092)
    def XMask(self, mask: int):
        if mask >= self.maxQPower:
            raise ValueError("XMask mask out-of-bounds!")
        if self.be.is_zero() or not mask:
            return
        if mask & (mask - 1) == 0:
            return self.X(mask.bit_length() - 1)
        self.be.xmask(mask)

    def ZMask(self, mask: int):  # qengine.hpp:154
        self.PhaseParity(math.pi, mask)

    def PhaseParity(self, radians: float, mask: int):
        if mask >= self.maxQPower:
            raise ValueError("PhaseParity mask out-of-bounds!")
        if self.be.is_zero() or not mask:
            return
        if mask & (mask - 1) == 0:
            ph = self._c(cmath.rect(1.0, self._r(radians / 2)))
            return self.Phase(self._c(1.0 / ph), ph, mask.bit_length() - 1)
        self.be.phase_parity(radians, mask)

    def PhaseRootNMask(self, n: int, mask: int):
        if mask >= self.maxQPower:
            raise ValueError("PhaseRootNMask mask out-of-bounds!")
        if self.be.is_zero() or not n or not mask:
            return
        if n == 1:
            return self.ZMask(mask)
        radians = -math.pi / (1 << (n - 1))
        if mask & (mask - 1) == 0:
            return self.Phase(1.0, self._c(cmath.rect(1.0, self._r(radians))), mask.bit_length() - 1)
        self.be.phase_root_n_mask(n, mask)

    def UniformParityRZ(self, mask: int, angle: float):
        if mask >= self.maxQPower:
            raise ValueError("UniformParityRZ mask out-of-bounds!")
        if self.be.is_zero():
            return
        self.be.uniform_parity_rz(0, mask, angle)

    def CUniformParityRZ(self, controls, mask: int, angle: float):
        if not controls:
            return self.UniformParityRZ(mask, angle)
        if mask >= self.maxQPower:
            raise ValueError("CUniformParityRZ mask out-of-bounds!")
        cm = 0
        for c in controls:
            self._check_qubit(c, "CUniformParityRZ")
            cm |= 1 << c
        if self.be.is_zero():
            return
        self.be.uniform_parity_rz(cm, mask, angle)

    # ---- state management ----------------------------------------------------------------------------------
    def SetPermutation(self, perm: int, phaseFac: Optional[complex] = None):  # state.cpp:228-254
        if phaseFac is None:
            ph = self.GetNonunitaryPhase() if self.randGlobalPhase else 1.0 + 0j
        else:
            z = self._c(phaseFac)
            ph = self._c(z / abs(z))
        self.be.set_permutation(int(perm), ph)
        self.runningNorm = 1.0

    def ZeroAmplitudes(self):
        self.be.zero()
        self.runningNorm = 0.0

    def IsZeroAmplitude(self) -> bool:
        return self.be.is_zero()

    def SetQuantumState(self, state):
        self.be.set_state(np.ascontiguousarray(state, dtype=self.cplx))
        self.runningNorm = REAL1_DEFAULT_ARG

    def GetQuantumState(self) -> np.ndarray:
        if self.doNormalize:
            self.NormalizeState()
        return self.be.get_state()

    def GetProbs(self) -> np.ndarray:
        if self.doNormalize:
            self.NormalizeState()
        return self.be.get_probs()

    def GetAmplitude(self, perm: int) -> complex:
        if perm >= self.maxQPower:
            raise ValueError("GetAmplitude argument out-of-bounds!")
        return self.be.get_amplitude(int(perm))

    def SetAmplitude(self, perm: int, amp: complex):
        if perm >= self.maxQPower:
            raise ValueError("SetAmplitude argument out-of-bounds!")
        amp = self._c(amp)
        if self.be.is_zero() and not self._norm(amp):
            return
        if self.runningNorm != REAL1_DEFAULT_ARG:
            self.runningNorm += self._norm(amp) - self._norm(self.be.get_amplitude(int(perm)))
        self.be.set_amplitude(int(perm), amp)

    def GetAmplitudePage(self, offset: int, length: int) -> np.ndarray:
        if offset + length > self.maxQPower:
            raise ValueError("GetAmplitudePage range is out-of-bounds!")
        return self.be.get_page(offset, length)

    def SetAmplitudePage(self, page, offset: int, length: Optional[int] = None, dstOffset: Optional[int] = None,
                         _length: Optional[int] = None):
        """Two reference overloads (qengine.hpp:136-140): (hostArray, offset, length) and
        (engine, srcOffset, dstOffset, length)."""
        if isinstance(page, QEngineHost):
            src, srcOffset, dstOff, ln = page, offset, length, dstOffset
            if dstOff + ln > self.maxQPower or srcOffset + ln > src.maxQPower:
                raise ValueError("SetAmplitudePage source range is out-of-bounds!")
            self.be.copy_page(src.be, srcOffset, dstOff, ln)
            self.runningNorm = REAL1_DEFAULT_ARG
            return
        arr = np.ascontiguousarray(page, dtype=self.cplx)
        ln = arr.size if length is None else length
        if offset + ln > self.maxQPower:
            raise ValueError("SetAmplitudePage range is out-of-bounds!")
        self.be.set_page(arr[:ln], offset)
        if self.doNormalize:
            self.runningNorm = REAL1_DEFAULT_ARG

    def ShuffleBuffers(self, other: "QEngineHost"):  # state.cpp:134-163
        if self.qubitCount != other.qubitCount:
            raise ValueError("ShuffleBuffers argument size differs from this!")
        self.be.shuffle(other.be)
        self.runningNorm = REAL1_DEFAULT_ARG
        other.runningNorm = REAL1_DEFAULT_ARG

    def CopyStateVec(self, src: "QEngineHost"):  # state.cpp:165-185
        if self.qubitCount != src.qubitCount:
            raise ValueError("CopyStateVec argument size differs from this!")
        if src.IsZeroAmplitude():
            return self.ZeroAmplitudes()
        self.be.copy_state(src.be)
        self.runningNorm = src.GetRunningNorm()

    def GetRunningNorm(self) -> float:
        self.Finish()
        return self.runningNorm

    def CloneEmpty(self) -> "QEngineHost":
        c = type(self)(0, 0, **self._ctor_args)
        c.SetQubitCount(self.qubitCount)
        return c

    def Clone(self) -> "QEngineHost":
        c = self.CloneEmpty()
        c.be.copy_state(self.be)
        c.runningNorm = self.runningNorm
        return c

    def SetQubitCount(self, qb: int):
        self.qubitCount = qb
        self.be.resize_zero(qb)

    # ---- measurement / probability ----------------------------------------------------------------------------
    def Prob(self, qubit: int) -> float:  # state.cpp:1751-1810
        self._check_qubit(qubit, "Prob")
        if self.doNormalize:
            self.NormalizeState()
        if self.be.is_zero():
            return 0.0
        p = 1 << qubit
        return self.clampProb(self._r(self.be.prob_mask(p, p)))

    def ProbAll(self, perm: int) -> float:  # qengine.hpp:264-271
        if self.doNormalize:
            self.NormalizeState()
        return self.clampProb(self._norm(self.GetAmplitude(perm)))

    def ProbReg(self, start: int, length: int, permutation: int) -> float:  # state.cpp:1872-1907
        if self.doNormalize:
            self.NormalizeState()
        if self.be.is_zero():
            return 0.0
        mask = ((1 << length) - 1) << start
        return self.clampProb(self._r(self.be.prob_mask(mask, permutation << start)))

    def ProbMask(self, mask: int, permutation: int) -> float:  # state.cpp:1910-1947
        if mask >= self.maxQPower:
            raise ValueError("ProbMask mask out-of-bounds!")
        if self.doNormalize:
            self.NormalizeState()
        if self.be.is_zero():
            return 0.0
        return self.clampProb(self._r(self.be.prob_mask(mask, permutation)))

    def ProbParity(self, mask: int) -> float:  # state.cpp:1949-1993
        if mask >= self.maxQPower:
            raise ValueError("ProbParity mask out-of-bounds!")
        if self.doNormalize:
            self.NormalizeState()
        if self.be.is_zero() or not mask:
            return 0.0
        return self.clampProb(self._r(self.be.prob_parity(mask)))

    def ProbMaskAll(self, mask: int) -> np.ndarray:
        if self.doNormalize:
            self.NormalizeState()
        return self.be.prob_mask_all(mask)

    def ProbBitsAll(self, bits: Sequence[int]) -> np.ndarray:
        """QInterface::ProbBitsAll (src/qinterface/qinterface.cpp:446-476): histogram over the listed qubits, bits[p] -> output
        bit p.  The reference loops over all 2^n basis states on the host; here ONE device sweep builds the histogram
        (prob_mask_all, ascending qubit order) and the host only permutes its 2^k entries into the requested bit order."""
        bits = [int(b) for b in bits]
        for b in bits:
            self._check_qubit(b, "ProbBitsAll")
        if len(set(bits)) != len(bits):
            raise ValueError("ProbBitsAll: duplicate qubit")
        if self.doNormalize:
            self.NormalizeState()
        mask = 0
        for b in bits:
            mask |= 1 << b
        asc = self.be.prob_mask_all(mask)          # index bit j <-> j-th lowest qubit of the mask
        order = sorted(bits)
        if order == bits:
            return asc
        k = len(bits)
        idx = np.arange(1 << k, dtype=np.int64)
        src = np.zeros(1 << k, dtype=np.int64)     # ascending-order index of every requested-order index
        for p, b in enumerate(bits):
            src |= ((idx >> p) & 1) << order.index(b)
        return asc[src]

    # ---- observables ------------------------------------------------------------------------------------------
    # The QInterface defaults (src/qinterface/qinterface.cpp:478-800) loop over all 2^n basis states and ask ProbAll(i) for each.
    # Here every k >= 2 query is one read-only device sweep (b200sv_moments_bits / _floats / b200sv_expectation_pauli), a
    # sum-form variance two; the k = 0 and k = 1 branches are the reference's own (1, and the Prob(bits[0]) formula).
    _U64 = (1 << 64) - 1

    def _obs_check(self, bits, table, what: str, tname: str):  # the checks of :546-553 and their messages
        if len(table) < 2 * len(bits):
            raise ValueError("QInterface::%s() must supply at least twice as many %s as bits!" % (what, tname))
        msg = "QInterface::%s() parameter qubits vector values must be within allocated qubit bounds!" % what
        seen = set()
        for b in bits:
            if b < 0 or b >= self.qubitCount:
                raise ValueError(msg)
            if b in seen:
                raise ValueError(msg + " (Found duplicate qubit indices!)")
            seen.add(b)

    def _bits_weights(self, bits, perms, offset, mean: Optional[float]) -> float:
        """k >= 2 sum form with a perm, offset or largest weight beyond uint64: the reference's loop over ProbAll (:560-576,
        :600-616) in Python integers, so nothing changes there."""
        tot = 0.0
        for lcv in range(self.maxQPower):
            w = offset + sum(perms[2 * p + ((lcv >> b) & 1)] for p, b in enumerate(bits))
            pr = self.ProbAll(lcv)
            tot += float(w) * pr if mean is None else (float(w) - mean) ** 2 * pr
        return self._r(tot)

    def _bits_fit(self, perms, offset) -> bool:
        top = offset + sum(max(perms[2 * p], perms[2 * p + 1]) for p in range(len(perms) // 2))
        return 0 <= offset and all(0 <= v <= self._U64 for v in perms) and top <= self._U64

    def ExpectationBitsFactorized(self, bits, perms, offset: int = 0) -> float:  # qinterface.cpp:542-577
        bits, perms, offset = [int(b) for b in bits], [int(v) for v in perms], int(offset)
        self._obs_check(bits, perms, "ExpectationBitsFactorized", "'perms'")
        return self._expectation_bits(bits, perms, offset)

    def _expectation_bits(self, bits, perms, offset) -> float:
        if not bits:
            return 1.0
        if len(bits) == 1:
            pr = self.Prob(bits[0])
            return self._r(float(perms[0] + offset) * (1.0 - pr) + float(perms[1] + offset) * pr)
        perms = perms[:2 * len(bits)]
        if not self._bits_fit(perms, offset):
            return self._bits_weights(bits, perms, offset, None)
        if self.doNormalize:
            self.NormalizeState()
        return self._r(self.be.moments_bits(bits, perms, offset, 0.0)[1])

    def VarianceBitsFactorized(self, bits, perms, offset: int = 0) -> float:  # qinterface.cpp:579-618
        bits, perms, offset = [int(b) for b in bits], [int(v) for v in perms], int(offset)
        self._obs_check(bits, perms, "VarianceBitsFactorized", "'perms'")
        if not bits:
            return 1.0
        mean = self._expectation_bits(bits, perms, offset)
        if len(bits) == 1:
            pr = self.Prob(bits[0])
            d0, d1 = self._r(float(perms[0] + offset) - mean), self._r(float(perms[1] + offset) - mean)
            return self._r(d0 * d0 * (1.0 - pr) + d1 * d1 * pr)
        perms = perms[:2 * len(bits)]
        if not self._bits_fit(perms, offset):
            return self._bits_weights(bits, perms, offset, mean)
        # a second sweep centred on the mean: no cancellation of E[w^2] - E[w]^2
        return self._r(self.be.moments_bits(bits, perms, offset, mean)[2])

    def ExpectationBitsAll(self, bits, offset: int = 0) -> float:  # ExpVarBitsAll, qinterface.hpp:210-219
        return self.ExpectationBitsFactorized(bits, self._bits_all_perms(len(bits)), offset)

    def VarianceBitsAll(self, bits, offset: int = 0) -> float:
        return self.VarianceBitsFactorized(bits, self._bits_all_perms(len(bits)), offset)

    @staticmethod
    def _bits_all_perms(k: int) -> List[int]:
        perms = []
        for i in range(k):
            perms += [0, 1 << i]
        return perms

    def _floats_sweep(self, bits, weights):
        if self.doNormalize:
            self.NormalizeState()
        return self.be.moments_floats(bits, weights[:2 * len(bits)], 0.0)

    def ExpectationFloatsFactorized(self, bits, weights) -> float:  # qinterface.cpp:771-806
        bits, weights = [int(b) for b in bits], [self._r(w) for w in weights]
        self._obs_check(bits, weights, "ExpectationFloatsFactorized", "weights")
        if not bits:
            return 1.0
        if len(bits) == 1:
            pr = self.Prob(bits[0])
            return self._r(weights[0] * (1.0 - pr) + weights[1] * pr)
        return self._r(self._floats_sweep(bits, weights)[1])

    def VarianceFloatsFactorized(self, bits, weights) -> float:  # qinterface.cpp:620-657
        bits, weights = [int(b) for b in bits], [self._r(w) for w in weights]
        self._obs_check(bits, weights, "VarianceFloatsFactorized", "weights")
        if not bits:
            return 1.0
        if len(bits) == 1:
            pr = self.Prob(bits[0])
            mean = self._r(weights[0] * (1.0 - pr) + weights[1] * pr)
            v0, v1 = self._r(weights[0] - mean), self._r(weights[1] - mean)
            return self._r(v0 * v0 * (1.0 - pr) + v1 * v1 * pr)
        s0, s1, _ = self._floats_sweep(bits, weights)
        # the reference sums p_i (w_i - mean) UNSQUARED here (:653); parity with it, not the variance (that is s2 centred on
        # the mean)
        mean = self._r(s1)
        return self._r(s1 - mean * s0)

    @staticmethod
    def _drop_pauli_i(bits, paulis):
        """the PauliI-dropping loop of qinterface.cpp:663-670 / 719-726 as written: it re-reads bits.size() after each erase,
        so some PauliI entries survive it — and then weigh like PauliZ (weights (1, -1), no basis gate)"""
        bits, paulis = [int(b) for b in bits], [int(p) for p in paulis]
        i = 0
        while i < len(bits):
            j = len(bits) - (i + 1)
            if paulis[j] == 0:
                del bits[j]
                del paulis[j]
            i += 1
        return bits, paulis

    def _pauli(self, bits, paulis):
        """(kept bits, S0, E) for the string left by _drop_pauli_i, with X = 1, Z = 2, Y = 3 (include/pauli.hpp) and a
        surviving I as Z"""
        kept, x, z = [], 0, 0
        for b, p in zip(*self._drop_pauli_i(bits, paulis)):
            if p == 0:
                p = 2
            self._check_qubit(b, "ExpectationPauliAll")
            if b in kept:
                raise ValueError("ExpectationPauliAll: duplicate qubit")
            kept.append(b)
            x |= (p & 1) << b
            z |= ((p >> 1) & 1) << b
        if not kept:
            return kept, 0.0, 0.0
        if self.doNormalize:
            self.NormalizeState()
        s0, e = self.be.expectation_pauli(x, z)
        return kept, s0, e

    def ExpectationPauliAll(self, bits, paulis) -> float:  # qinterface.cpp:715-769
        kept, s0, e = self._pauli(bits, paulis)
        if not kept:
            return 1.0
        if len(kept) == 1:
            # Prob of the rotated qubit is (S0 - E) / 2; weights (1, -1)
            pr = self.clampProb(self._r((s0 - e) / 2.0))
            return self._r((1.0 - pr) - pr)
        return self._r(e)

    def VariancePauliAll(self, bits, paulis) -> float:  # qinterface.cpp:659-713
        kept, s0, e = self._pauli(bits, paulis)
        if not kept:
            return 1.0
        if len(kept) == 1:
            pr = self.clampProb(self._r((s0 - e) / 2.0))
            mean = self._r((1.0 - pr) - pr)
            v0, v1 = self._r(1.0 - mean), self._r(-1.0 - mean)
            return self._r(v0 * v0 * (1.0 - pr) + v1 * v1 * pr)
        # VarianceFloatsFactorized's unsquared sum with weights (1, -1): E - E * S0
        mean = self._r(e)
        return self._r(e - mean * s0)

    def _exp_var_unitary(self, isExp: bool, bits, basisOps, eigenVals) -> float:
        """QInterface::ExpVarUnitaryAll (qinterface.cpp:478-540): the inverse basis gates, the Floats query, the gates again.
        basisOps = 3 U angles per qubit (theta, phi, lambda) or one 2x2 matrix per qubit."""
        bits = [int(b) for b in bits]
        if not bits:
            return 1.0
        eigenVals = list(eigenVals) if eigenVals else [1.0, -1.0] * len(bits)
        mtrx = len(basisOps) > 0 and hasattr(basisOps[0], "__len__")
        for i, b in enumerate(bits):
            if mtrx:
                m = [complex(v) for v in basisOps[i]]
                det = 1.0 / (m[0] * m[3] - m[1] * m[2])  # inv2x2, src/common/functions.cpp:204-211
                self.Mtrx([det * m[3], det * -m[1], det * -m[2], det * m[0]], b)
            else:
                self.U(b, -basisOps[3 * i], -basisOps[3 * i + 1], -basisOps[3 * i + 2])
        r = self.ExpectationFloatsFactorized(bits, eigenVals) if isExp else self.VarianceFloatsFactorized(bits, eigenVals)
        for i, b in enumerate(bits):
            if mtrx:
                self.Mtrx([complex(v) for v in basisOps[i]], b)
            else:
                self.U(b, basisOps[3 * i], basisOps[3 * i + 1], basisOps[3 * i + 2])
        return r

    def ExpectationUnitaryAll(self, bits, basisOps, eigenVals=()) -> float:
        return self._exp_var_unitary(True, bits, basisOps, eigenVals)

    def VarianceUnitaryAll(self, bits, basisOps, eigenVals=()) -> float:
        return self._exp_var_unitary(False, bits, basisOps, eigenVals)

    # ---- reduced density matrix -------------------------------------------------------------------------------
    RDM_MAX_QUBITS = 14  # B200SV_RDM_MAX_QUBITS

    def GetReducedDensityMatrix(self, qubits) -> np.ndarray:
        """QInterface::GetReducedDensityMatrix (src/qinterface/qinterface.cpp:886-944) as one read-only device sweep
        (b200sv_reduced_density_matrix) instead of 2^n (1 + 2^k) GetAmplitude calls: rho[i, j] = sum_e psi[i, e] conj(psi[j, e]),
        bit p of i and j being qubit qubits[p] in the order given, e running over the other qubits.  Shape (2^k, 2^k), in the
        engine's complex type.  Like the reference (which reads through GetAmplitude, state.cpp:193) it does not normalise, so
        the trace is sum |psi|^2 whatever doNormalize says.  A qubit out of range or repeated, or more than 14 qubits, raise
        ValueError (the reference indexes out of bounds there)."""
        qubits = [int(q) for q in qubits]
        if len(qubits) > self.RDM_MAX_QUBITS:
            raise ValueError("GetReducedDensityMatrix: at most %d qubits" % self.RDM_MAX_QUBITS)
        for q in qubits:
            self._check_qubit(q, "GetReducedDensityMatrix")
        if len(set(qubits)) != len(qubits):
            raise ValueError("GetReducedDensityMatrix: repeated qubit")
        return self.be.reduced_density_matrix(qubits).astype(self.cplx)

    def MultiShotMeasureMask(self, qPowers: Sequence[int], shots: int) -> dict:
        """QEngine::MultiShotMeasureMask (src/qengine/qengine.cpp:542-576): `shots` samples of the listed qubits without
        collapse, as {outcome: count} with qPowers[p] -> outcome bit p.  Few measured qubits: one histogram sweep
        (ProbBitsAll) and host draws, like the reference.  Many measured qubits (where the reference builds a 2^k histogram by
        reading the whole state): basis states are sampled on the device (one chunk-sum sweep for all shots) and the measured
        bits are read off them — the same distribution.  Draws come from this engine's generator (the reference seeds
        std::mt19937 from std::random_device: outcomes are not reproducible there either)."""
        if not shots:
            return {}
        bits = []
        for p in qPowers:
            p = int(p)
            if p <= 0 or (p & (p - 1)) or p >= self.maxQPower:
                raise ValueError("QInterface::MultiShotMeasureMask parameter qPowers array values must be within allocated qubit bounds!")
            bits.append(p.bit_length() - 1)
        if len(set(bits)) != len(bits):
            raise ValueError("QInterface::MultiShotMeasureMask parameter qPowers array values must not repeat!")
        out = {}
        if len(bits) <= 16 or not hasattr(self.be, "sample_many"):
            probs = np.asarray(self.ProbBitsAll(bits), dtype=np.float64)
            tot = float(probs.sum())
            if tot <= 0:
                return {0: int(shots)}
            cum = np.cumsum(probs / tot)
            draws = np.searchsorted(cum, [self.Rand() for _ in range(shots)], side="right")
            for d in np.minimum(draws, probs.size - 1):
                out[int(d)] = out.get(int(d), 0) + 1
            return out
        if self.doNormalize:
            self.NormalizeState()
        perms = self.be.sample_many([self.Rand() for _ in range(shots)])
        for perm in perms:
            key = 0
            for p, b in enumerate(bits):
                key |= ((int(perm) >> b) & 1) << p
            out[key] = out.get(key, 0) + 1
        return out

    def CtrlOrAntiProb(self, controlState: bool, control: int, target: int) -> float:  # state.cpp:1814-1869
        if self.be.is_zero():
            return 0.0
        controlProb = self.Prob(control)
        if not controlState:
            controlProb = 1.0 - controlProb
        if controlProb <= self.FP_NORM_EPSILON:
            return 0.0
        if (1.0 - controlProb) <= self.FP_NORM_EPSILON:
            return self.Prob(target)
        self._check_qubit(target, "CtrlOrAntiProb")
        cp, tp = 1 << control, 1 << target
        one = self._r(self.be.prob_mask(cp | tp, (cp if controlState else 0) | tp))
        return self.clampProb(self._r(one / controlProb))

    def CProb(self, control: int, target: int) -> float:
        return self.CtrlOrAntiProb(True, control, target)

    def ACProb(self, control: int, target: int) -> float:
        return self.CtrlOrAntiProb(False, control, target)

    def ApplyM(self, regMask: int, result, nrm: complex):  # qengine.hpp:161-166, state.cpp:2167-2196
        if isinstance(result, bool):
            result = regMask if result else 0
        if self.be.is_zero():
            return
        self.be.apply_m(regMask, result, self._c(nrm))
        self.runningNorm = 1.0

    def ForceM(self, qubit: int, result: bool, doForce: bool = True, doApply: bool = True) -> bool:  # qengine.cpp:78-106
        if qubit >= self.qubitCount:
            raise ValueError("QEngine::ForceM qubit index parameter must be within allocated qubit bounds!")
        oneChance = self.Prob(qubit)
        if not doForce:
            if oneChance >= 1.0:
                result = True
            elif oneChance <= 0.0:
                result = False
            else:
                result = self.Rand() <= oneChance
        nrmlzr = oneChance if result else (1.0 - oneChance)
        if nrmlzr <= 0.0:
            raise ValueError("QEngine::ForceM() forced a measurement result with 0 probability!")
        if doApply and (1.0 - nrmlzr) > self.REAL1_EPSILON:
            qPower = 1 << qubit
            self.ApplyM(qPower, qPower if result else 0, self.GetNonunitaryPhase() / self._r(math.sqrt(nrmlzr)))
        return result

    def M(self, qubit: int) -> bool:
        return self.ForceM(qubit, False, False)

    def ForceMReg(self, start: int, length: int, result: int, doForce: bool = True, doApply: bool = True) -> int:
        # qengine.cpp:489-540
        if start + length > self.qubitCount:
            raise ValueError("QEngine::ForceMReg range is out-of-bounds!")
        if length == 1:
            return 1 if self.ForceM(start, bool(result & 1), doForce, doApply) else 0
        lengthPower = 1 << length
        regMask = (lengthPower - 1) << start
        nrmlzr = 1.0
        if doForce:
            nrmlzr = self.ProbMask(regMask, result << start)
        else:
            probs = self.ProbMaskAll(regMask)
            prob = self.Rand()
            lower = 0.0
            result = lengthPower - 1
            lcv = 0
            while lower < prob and lcv < lengthPower:
                lower += float(probs[lcv])
                if probs[lcv] > 0:
                    nrmlzr = float(probs[lcv])
                    result = lcv
                lcv += 1
        if doApply:
            nrm = self.GetNonunitaryPhase() / self._r(math.sqrt(nrmlzr))
            self.ApplyM(regMask, result << start, nrm)
        return result

    def MAll(self) -> int:  # state.cpp:2026-2050 (on-device sampling instead of a 2^n host loop)
        rnd = self.Rand()
        if self.doNormalize:
            self.NormalizeState()
        perm = self.be.sample(rnd)
        self.SetPermutation(perm)
        return perm

    def HighestProbAll(self) -> int:
        return self.be.highest_prob()

    def ForceMParity(self, mask: int, result: bool, doForce: bool = True) -> bool:  # state.cpp:2052-2107
        if mask >= self.maxQPower:
            raise ValueError("ForceMParity mask out-of-bounds!")
        if self.be.is_zero() or not mask:
            return False
        if not doForce:
            result = self.Rand() <= self.ProbParity(mask)
        self.runningNorm = self._r(self.be.collapse_parity(mask, bool(result)))
        if not self.doNormalize:
            self.NormalizeState()
        return result

    def SumSqrDiff(self, other: "QEngineHost") -> float:  # state.cpp:2109-2165
        if other is None:
            return 1.0
        if other is self:
            return 0.0
        if self.qubitCount != other.qubitCount:
            return 1.0
        if self.doNormalize:
            self.NormalizeState()
        if other.doNormalize:
            other.NormalizeState()
        if self.be.is_zero() and other.be.is_zero():
            return 0.0
        if self.be.is_zero():
            other.UpdateRunningNorm()
            return other.runningNorm
        if other.be.is_zero():
            self.UpdateRunningNorm()
            return self.runningNorm
        z = self._c(self.be.inner(other.be))
        return 1.0 - self.clampProb(self._norm(z))

    def NormalizeState(self, nrm: float = REAL1_DEFAULT_ARG, norm_thresh: float = REAL1_DEFAULT_ARG, phaseArg: float = 0.0):
        # state.cpp:2198-2248
        if self.be.is_zero():
            return
        if self.runningNorm == REAL1_DEFAULT_ARG and nrm == REAL1_DEFAULT_ARG:
            self.UpdateRunningNorm()
        if nrm < 0:
            nrm = self.runningNorm
        if nrm <= self.FP_NORM_EPSILON:
            return self.ZeroAmplitudes()
        if abs(1.0 - nrm) <= self.FP_NORM_EPSILON and (phaseArg * phaseArg) <= self.FP_NORM_EPSILON:
            return
        if norm_thresh < 0:
            norm_thresh = self.amplitudeFloor
        self.be.normalize(nrm, norm_thresh, phaseArg)
        self.runningNorm = 1.0

    def UpdateRunningNorm(self, norm_thresh: float = REAL1_DEFAULT_ARG):  # state.cpp:2250-2268
        if self.be.is_zero():
            self.runningNorm = 0.0
            return
        if norm_thresh < 0:
            norm_thresh = self.amplitudeFloor
        self.runningNorm = self._r(self.be.norm(norm_thresh))
        if self.runningNorm <= self.FP_NORM_EPSILON:
            self.ZeroAmplitudes()

    # ---- structure -------------------------------------------------------------------------------------------
    def Compose(self, toCopy: "QEngineHost", start: Optional[int] = None) -> int:  # state.cpp:1271-1459
        if start is None:
            start = self.qubitCount
        if start > self.qubitCount:
            raise ValueError("Compose start index is out-of-bounds!")
        if not toCopy.qubitCount:
            return start
        if not self.qubitCount:
            self.be.resize_zero(toCopy.qubitCount)
            self.qubitCount = toCopy.qubitCount
            self.be.copy_state(toCopy.be)
            self.runningNorm = toCopy.runningNorm
            return 0
        if self.doNormalize:
            self.NormalizeState()
        if toCopy.doNormalize:
            toCopy.NormalizeState()
        self.be.compose(toCopy.be, start)
        if self.be.is_zero():
            self.runningNorm = 0.0
        self.qubitCount += toCopy.qubitCount
        return start

    def Decompose(self, start: int, length_or_dest):  # qengine.hpp:287-293, state.cpp:1551-1701
        if isinstance(length_or_dest, QEngineHost):
            dest = length_or_dest
            length = dest.qubitCount
        else:
            length = int(length_or_dest)
            dest = self.CloneEmpty()
            dest.SetQubitCount(length)
        self._decompose_dispose(start, length, dest)
        return dest

    def Dispose(self, start: int, length: int, disposedPerm: Optional[int] = None):  # state.cpp:1703-1748
        if disposedPerm is None:
            return self._decompose_dispose(start, length, None)
        if start + length > self.qubitCount:
            raise ValueError("Dispose range is out-of-bounds!")
        if not length:
            return
        if self.doNormalize:
            self.NormalizeState()
        nl = self.qubitCount - length
        self.be.dispose_perm(start, length, int(disposedPerm))
        self.qubitCount = nl

    def _decompose_dispose(self, start: int, length: int, dest: Optional["QEngineHost"]):
        if start + length > self.qubitCount:
            raise ValueError("DecomposeDispose range is out-of-bounds!")
        if not length:
            return
        if self.doNormalize:
            self.NormalizeState()
        self.be.decompose(start, length, dest.be if dest is not None else None)
        self.qubitCount -= length
        if dest is not None:
            dest.runningNorm = 0.0 if dest.be.is_zero() else 1.0

    def Allocate(self, start: int, length: int) -> int:  # utility.cpp:54-68
        if not length:
            return start
        nq = type(self)(length, 0, phaseFac=1.0 + 0j, **{k: v for k, v in self._ctor_args.items()})
        return self.Compose(nq, start)


# ================================================================================================================
# CUDA backend over the C ABI
# ================================================================================================================

class _CudaBackend:
    """Backend primitives over libb200sv.so (include/b200sv.h).  One b200sv handle."""

    def __init__(self, n_qubits: int, precision: int, device: int, external_ptr: int = 0):
        from . import _abi
        self.abi = _abi
        self.lib = _abi.load()
        self.precision = precision
        self.cplx = np.complex64 if precision == 32 else np.complex128
        self.real = np.float32 if precision == 32 else np.float64
        self.device = max(device, 0)
        self.h = _abi.create(self.lib, self.device, n_qubits, precision, external_ptr)

    def rebind_external(self, device_ptr: int):
        import ctypes
        self._ck(self.lib.b200sv_rebind_external(self.h, ctypes.c_void_p(device_ptr)))

    def set_stream(self, cuda_stream, adopt: bool = True):
        """run on a caller-owned stream (e.g. torch.cuda.current_stream().cuda_stream, 0 = legacy default stream);
        adopt=False restores a private stream"""
        import ctypes
        self._ck(self.lib.b200sv_set_stream(self.h, ctypes.c_void_p(cuda_stream or 0), 1 if adopt else 0))

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.b200sv_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def _ck(self, rc):
        self.abi.check(self.lib, rc)

    def n_qubits(self) -> int:
        import ctypes
        n = ctypes.c_int()
        self._ck(self.lib.b200sv_qubit_count(self.h, ctypes.byref(n)))
        return n.value

    def dim(self) -> int:
        return 1 << self.n_qubits()

    def resize_zero(self, n_qubits: int):
        self.lib.b200sv_destroy(self.h)
        self.h = self.abi.create(self.lib, self.device, n_qubits, self.precision)

    def finish(self):
        self._ck(self.lib.b200sv_finish(self.h))

    def flush(self):
        self._ck(self.lib.b200sv_flush(self.h))

    def is_zero(self) -> bool:
        import ctypes
        z = ctypes.c_int()
        self._ck(self.lib.b200sv_is_zero(self.h, ctypes.byref(z)))
        return bool(z.value)

    def zero(self):
        self._ck(self.lib.b200sv_zero(self.h))

    def set_permutation(self, perm: int, phase: complex):
        self._ck(self.lib.b200sv_set_permutation(self.h, perm, phase.real, phase.imag))

    def set_state(self, arr: np.ndarray):
        assert arr.dtype == self.cplx and arr.size == self.dim()
        self._ck(self.lib.b200sv_set_state(self.h, arr.ctypes.data))

    def get_state(self) -> np.ndarray:
        out = np.empty(self.dim(), dtype=self.cplx)
        self._ck(self.lib.b200sv_get_state(self.h, out.ctypes.data))
        return out

    def get_probs(self) -> np.ndarray:
        out = np.empty(self.dim(), dtype=self.real)
        self._ck(self.lib.b200sv_get_probs(self.h, out.ctypes.data))
        return out

    def get_page(self, offset: int, length: int) -> np.ndarray:
        out = np.empty(length, dtype=self.cplx)
        self._ck(self.lib.b200sv_get_page(self.h, out.ctypes.data, offset, length))
        return out

    def set_page(self, arr: np.ndarray, offset: int):
        self._ck(self.lib.b200sv_set_page(self.h, arr.ctypes.data, offset, arr.size))

    def copy_page(self, src: "_CudaBackend", src_off: int, dst_off: int, length: int):
        self._ck(self.lib.b200sv_copy_page(self.h, src.h, src_off, dst_off, length))

    def shuffle(self, other: "_CudaBackend"):
        self._ck(self.lib.b200sv_shuffle(self.h, other.h))

    def copy_state(self, src: "_CudaBackend"):
        self._ck(self.lib.b200sv_copy_state(self.h, src.h))

    def get_amplitude(self, perm: int) -> complex:
        import ctypes
        re, im = ctypes.c_double(), ctypes.c_double()
        self._ck(self.lib.b200sv_get_amplitude(self.h, perm, ctypes.byref(re), ctypes.byref(im)))
        return complex(re.value, im.value)

    def set_amplitude(self, perm: int, amp: complex):
        self._ck(self.lib.b200sv_set_amplitude(self.h, perm, amp.real, amp.imag))

    def apply2x2(self, off1, off2, mtrx, pows, nrm, thresh, calc_norm):
        import ctypes
        # the marshalled matrix / power arrays are read-only on the C side and repeat thousands of times per circuit: keep them
        cache = self.__dict__.setdefault("_marshal_cache", {})
        if len(cache) > 8192:
            cache.clear()
        mk = ("m", mtrx[0], mtrx[1], mtrx[2], mtrx[3])
        m8 = cache.get(mk)
        if m8 is None:
            m8 = (ctypes.c_double * 8)()
            for k in range(4):
                m8[2 * k] = mtrx[k].real
                m8[2 * k + 1] = mtrx[k].imag
            cache[mk] = m8
        pk = ("p",) + tuple(pows)
        pw = cache.get(pk)
        if pw is None:
            pw = cache[pk] = (ctypes.c_uint64 * max(len(pows), 1))(*pows)
        if calc_norm:
            out = ctypes.c_double()
            self._ck(self.lib.b200sv_apply2x2(self.h, off1, off2, m8, len(pows), pw, nrm, thresh, ctypes.byref(out)))
            return out.value
        self._ck(self.lib.b200sv_apply2x2(self.h, off1, off2, m8, len(pows), pw, nrm, thresh, None))
        return None

    def apply_gates(self, n, off1, off2, pmasks, mats8):
        """b200sv_apply_gates: n single-target Apply2x2 forms (ctypes arrays) in one ABI call"""
        self._ck(self.lib.b200sv_apply_gates(self.h, n, off1, off2, pmasks, mats8))

    def xmask(self, mask):
        self._ck(self.lib.b200sv_xmask(self.h, mask))

    def phase_parity(self, radians, mask):
        self._ck(self.lib.b200sv_phase_parity(self.h, radians, mask))

    def phase_root_n_mask(self, n, mask):
        self._ck(self.lib.b200sv_phase_root_n_mask(self.h, n, mask))

    def uniform_parity_rz(self, cmask, mask, angle):
        self._ck(self.lib.b200sv_uniform_parity_rz(self.h, cmask, mask, angle))

    def apply_m(self, mask, result, nrm: complex):
        self._ck(self.lib.b200sv_apply_m(self.h, mask, result, nrm.real, nrm.imag))

    def collapse_parity(self, mask, result: bool) -> float:
        import ctypes
        out = ctypes.c_double()
        self._ck(self.lib.b200sv_collapse_parity(self.h, mask, int(result), ctypes.byref(out)))
        return out.value

    def _scalar(self, fn, *args) -> float:
        import ctypes
        out = ctypes.c_double()
        self._ck(fn(self.h, *args, ctypes.byref(out)))
        return out.value

    def prob_mask(self, mask, perm) -> float:
        return self._scalar(self.lib.b200sv_prob_mask, mask, perm)

    def prob_parity(self, mask) -> float:
        return self._scalar(self.lib.b200sv_prob_parity, mask)

    def prob_mask_all(self, mask) -> np.ndarray:
        out = np.empty(1 << bin(mask).count("1"), dtype=self.real)
        self._ck(self.lib.b200sv_prob_mask_all(self.h, mask, out.ctypes.data))
        return out

    def norm(self, thresh) -> float:
        return self._scalar(self.lib.b200sv_norm, float(thresh))

    def normalize(self, nrm, thresh, phase_arg):
        self._ck(self.lib.b200sv_normalize(self.h, float(nrm), float(thresh), float(phase_arg)))

    def inner(self, other: "_CudaBackend") -> complex:
        import ctypes
        re, im = ctypes.c_double(), ctypes.c_double()
        self._ck(self.lib.b200sv_inner(self.h, other.h, ctypes.byref(re), ctypes.byref(im)))
        return complex(re.value, im.value)

    def expectation(self, start, length) -> float:
        return self._scalar(self.lib.b200sv_expectation, start, length)

    def _moments(self, fn, bits, table, ctype, *args):
        import ctypes
        k = len(bits)
        b = (ctypes.c_int * max(k, 1))(*bits)
        t = (ctype * max(2 * k, 1))(*table[:2 * k])
        out = (ctypes.c_double * 3)()
        self._ck(fn(self.h, k, b, t, *args, out))
        return out[0], out[1], out[2]

    def moments_bits(self, bits, perms, offset, center):
        """(S0, S1, S2) of the sum-form weight (b200sv_moments_bits)"""
        import ctypes
        return self._moments(self.lib.b200sv_moments_bits, bits, perms, ctypes.c_uint64, int(offset), float(center))

    def moments_floats(self, bits, weights, center):
        """(S0, S1, S2) of the product-form weight (b200sv_moments_floats)"""
        import ctypes
        return self._moments(self.lib.b200sv_moments_floats, bits, weights, ctypes.c_double, float(center))

    def expectation_pauli(self, x_mask, z_mask):
        """(sum |psi|^2, <psi|P|psi>) of the Pauli string (x_mask, z_mask) (b200sv_expectation_pauli)"""
        import ctypes
        out = (ctypes.c_double * 2)()
        self._ck(self.lib.b200sv_expectation_pauli(self.h, x_mask, z_mask, out))
        return out[0], out[1]

    def reduced_density_matrix(self, qubits) -> np.ndarray:
        """rho on the listed qubits, complex128 of shape (2^k, 2^k) (b200sv_reduced_density_matrix)"""
        import ctypes
        k = len(qubits)
        q = (ctypes.c_int * max(k, 1))(*qubits)
        out = np.empty(2 << (2 * k), dtype=np.float64)
        self._ck(self.lib.b200sv_reduced_density_matrix(self.h, k, q, out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
        return out.view(np.complex128).reshape(1 << k, 1 << k)

    def highest_prob(self) -> int:
        import ctypes
        p = ctypes.c_uint64()
        self._ck(self.lib.b200sv_highest_prob(self.h, ctypes.byref(p)))
        return p.value

    def sample(self, rnd: float) -> int:
        import ctypes
        p = ctypes.c_uint64()
        self._ck(self.lib.b200sv_sample(self.h, float(rnd), ctypes.byref(p)))
        return p.value

    def sample_many(self, rnds) -> list:
        import ctypes
        n = len(rnds)
        r = (ctypes.c_double * max(n, 1))(*[float(x) for x in rnds])
        out = (ctypes.c_uint64 * max(n, 1))()
        self._ck(self.lib.b200sv_sample_many(self.h, n, r, out))
        return [int(out[i]) for i in range(n)]

    def compose(self, other: "_CudaBackend", start: int):
        self._ck(self.lib.b200sv_compose(self.h, other.h, start))

    def decompose(self, start, length, dest: Optional["_CudaBackend"]):
        self._ck(self.lib.b200sv_decompose(self.h, start, length, dest.h if dest is not None else None))

    def dispose_perm(self, start, length, perm):
        self._ck(self.lib.b200sv_dispose_perm(self.h, start, length, perm))

    # ---- QAlu family (include/b200sv.h "QAlu family") ----
    def alu_rol(self, shift, start, length):
        self._ck(self.lib.b200sv_rol(self.h, shift, start, length))

    def alu_inc(self, to_add, start, length, ctrl_mask):
        self._ck(self.lib.b200sv_inc(self.h, to_add, start, length, ctrl_mask))

    def alu_incdecc(self, to_mod, start, length, carry_index):
        self._ck(self.lib.b200sv_incdecc(self.h, to_mod, start, length, carry_index))

    def alu_incs(self, to_add, start, length, overflow_index):
        self._ck(self.lib.b200sv_incs(self.h, to_add, start, length, overflow_index))

    def alu_incdecsc(self, to_mod, start, length, overflow_index, carry_index):
        self._ck(self.lib.b200sv_incdecsc(self.h, to_mod, start, length, overflow_index, carry_index))

    def alu_muldiv(self, inverse, to_mul, start, carry_start, length, ctrl_mask):
        self._ck(self.lib.b200sv_muldiv(self.h, inverse, to_mul, start, carry_start, length, ctrl_mask))

    def alu_modnout(self, kind, to_mod, mod_n, in_start, out_start, length, ctrl_mask):
        self._ck(self.lib.b200sv_modnout(self.h, kind, to_mod, mod_n, in_start, out_start, length, ctrl_mask))

    def alu_indexed(self, kind, index_start, index_length, value_start, value_length, carry_index, carry_in, values: bytes):
        self._ck(self.lib.b200sv_indexed(self.h, kind, index_start, index_length, value_start, value_length, carry_index,
                                        carry_in, values))

    def alu_hash(self, start, length, values: bytes):
        self._ck(self.lib.b200sv_hash(self.h, start, length, values))

    def alu_phase_flip_if_less(self, greater_perm, start, length, flag_index):
        self._ck(self.lib.b200sv_phase_flip_if_less(self.h, greater_perm, start, length, flag_index))

    def set_fusion(self, mode: int):
        self._ck(self.lib.b200sv_set_fusion(self.h, mode))

    def stats(self) -> dict:
        st = self.abi.Stats()
        import ctypes
        self._ck(self.lib.b200sv_get_stats(self.h, ctypes.byref(st)))
        return {f[0]: getattr(st, f[0]) for f in st._fields_}

    def reset_stats(self):
        self._ck(self.lib.b200sv_reset_stats(self.h))

    def timer_begin(self):
        self._ck(self.lib.b200sv_timer_begin(self.h))

    def timer_end(self) -> float:
        return self._scalar(self.lib.b200sv_timer_end)

    def flush_l2(self, nbytes: int):
        self._ck(self.lib.b200sv_flush_l2(self.h, nbytes))


class QEngineCUDA(QEngineHost):
    """The ``Qrack::QEngineCUDA`` slot (reference include/qengine_cuda.hpp:280-284) on the H100 state-vector core."""

    def _make_backend(self, n_qubits: int):
        return _CudaBackend(n_qubits, self.precision, self.deviceId)

    @classmethod
    def over_buffer(cls, device_ptr: int, n_qubits: int, device: int, precision: int = 32, rgp=None):
        """Engine over an externally owned device buffer of 2^n amplitudes (e.g. a torch tensor's data_ptr()).  The
        buffer is used as is (no initialisation) and never freed by the library."""
        q = cls(0, 0, rgp, 1.0 + 0j, False, False, deviceId=device, precision=precision)
        q.be.lib.b200sv_destroy(q.be.h)
        q.be.h = q.be.abi.create(q.be.lib, q.be.device, n_qubits, precision, device_ptr)
        q.qubitCount = n_qubits
        q.runningNorm = REAL1_DEFAULT_ARG
        return q

    def RunCircuit(self, circuit):
        """Whole-circuit submission (SURVEY 8f N4): the recorded single-target gates of a ``qcircuit.QCircuit`` go through
        ``b200sv_apply_gates`` in one ABI call.  Same effect as ``circuit.Run`` gate by gate (QCircuit::Run,
        src/qcircuit.cpp:173-281); needs doNormalize off (QPager/QUnit create their engines that way)."""
        if self.doNormalize:
            raise ValueError("QEngineCUDA::RunCircuit: doNormalize engines take their gates one by one (running-norm bookkeeping)")
        if circuit.GetQubitCount() != self.qubitCount or circuit.precision != self.precision:
            raise ValueError("QEngineCUDA::RunCircuit: circuit width / precision differs from the engine's")
        if self.be.is_zero():
            return
        n, o1, o2, pm, m8 = circuit.packed()
        if n:
            self.be.apply_gates(n, o1, o2, pm, m8)

    def SetDevice(self, dID: int):
        import ctypes
        self.be._ck(self.be.lib.b200sv_set_device(self.be.h, dID))
        self.deviceId = dID
        self.be.device = max(dID, 0)

    def GetDevice(self) -> int:
        return self.be.device

    def isOpenCL(self) -> bool:
        return True
