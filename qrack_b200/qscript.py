"""qscript — the circuit-script text format shared by the CUDA engine, the oracle and the reference harness.

One op per line, ``#`` starts a comment.  Ops are spelled exactly like the reference's public
``QInterface`` methods (reference ``include/qinterface.hpp``) so that the *same file* can be
replayed on (a) ``oracle/_ref/ref_harness_f{32,64}`` = the unmodified reference ``QEngineCPU``,
(b) the plain-C restatement in ``oracle/`` and (c) this package's ``QEngineCUDA`` mirror.  Circuits are
always materialised to a gate list *outside* any simulator (SURVEY.md §8c: never let ``Rand()`` pick gates).

Grammar (tokens are whitespace separated; ``<m8>`` = 8 reals = 4 complex row-major; ``<cs>`` = ``n c0 .. c{n-1}``)::

    qubits N                      create register 0 with N qubits in |0..0>, global phase 1
    reg ID N PERM                 create register ID with N qubits in permutation PERM
    @ID <op ...>                  run <op> on register ID instead of register 0
    TIC / TOC                     start / stop the timed region (Finish() on both sides)

    H|X|Y|Z|S|IS|T|IT|SqrtX q
    CNOT|AntiCNOT|CZ|CY c t       CCNOT c1 c2 t
    Swap|ISwap|SqrtSwap a b       FSim theta phi a b     CSwap|AntiCSwap <cs> a b
    U q theta phi lambda          AI|IAI q azimuth inclination
    Phase q tl.re tl.im br.re br.im          Invert q tr.re tr.im bl.re bl.im
    Mtrx q <m8>                   MCMtrx|MACMtrx <cs> t <m8>       UCMtrx <cs> t perm <m8>
    MCPhase|MACPhase <cs> t tl br            MCInvert|MACInvert <cs> t tr bl
    PhaseRootN n q                CPhaseRootN n c t
    QFT|IQFT start length
    XMask mask   ZMask mask   PhaseParity radians mask   PhaseRootNMask n mask   ZeroPhaseFlip start length
    UniformParityRZ mask angle    CUniformParityRZ <cs> mask angle
    UniformlyControlledSingleBit <cs> t <ss> skipValueMask <m8 per table entry>     (<ss> = n skipPower0 .. skipPower{n-1};
                                  the table has 2^(len(cs) + n) entries)
    UniformlyControlledRY|UniformlyControlledRZ <cs> t angle0 .. angle{2^len(cs)-1}
    INC|DEC value start length
    SetPermutation perm   ForceM q result   ForceMReg start length result
    NormalizeState   UpdateRunningNorm
    LossySave path p b   LossyLoad path            (LossySaveStateVector / LossyLoadStateVector; path has no spaces;
                                                   replayed by the Python engines and dropin/observables_harness.cpp)
    Compose SRC [start]   Decompose start length DST   Dispose start length [perm]   Allocate start length
  queries (each appends one line to the results):
    Prob q   ProbAll perm   ProbReg start length perm   ProbMask mask perm   ProbParity mask
    CProb c t   ACProb c t   GetAmplitude perm   SumSqrDiff OTHER   Norm
    ExpectationBitsAll|VarianceBitsAll <cs> offset
    ExpectationBitsFactorized|VarianceBitsFactorized <cs> offset perm0 .. perm{2n-1}
    ExpectationFloatsFactorized|VarianceFloatsFactorized <cs> weight0 .. weight{2n-1}
    ExpectationPauliAll|VariancePauliAll <cs> pauli0 .. pauli{n-1}        (0 = I, 1 = X, 2 = Z, 3 = Y: include/pauli.hpp)
    ExpectationUnitaryAll|VarianceUnitaryAll <cs> theta0 phi0 lambda0 .. [eigenvalue0 .. eigenvalue{2n-1}]
                                      (the U3 form of ExpVarUnitaryAll)
    ExpectationMatrixAll|VarianceMatrixAll <cs> <m8 per qubit> [eigenvalues]   (its matrix form: ExpectationUnitaryAll /
                                      VarianceUnitaryAll with one 2x2 matrix per qubit)
    GetReducedDensityMatrix <cs>      (the 2 4^n values of rho row-major, interleaved re / im; bit p of a row is qubit p of <cs>)
    HighestProbAllN n                 (the n most probable basis states, most probable first: QInterface::HighestProbAll(n))
"""
from __future__ import annotations

import math
import random
from typing import Callable, Dict, Iterable, List, Sequence, Tuple

QUERY_OPS = {
    "Prob", "ProbAll", "ProbReg", "ProbMask", "ProbParity", "CProb", "ACProb", "GetAmplitude", "SumSqrDiff", "Norm",
    "ExpectationBitsAll", "VarianceBitsAll", "ExpectationBitsFactorized", "VarianceBitsFactorized",
    "ExpectationFloatsFactorized", "VarianceFloatsFactorized", "ExpectationPauliAll", "VariancePauliAll",
    "ExpectationUnitaryAll", "VarianceUnitaryAll", "ExpectationMatrixAll", "VarianceMatrixAll", "GetReducedDensityMatrix",
    "HighestProbAllN",
}


def parse(text: str) -> List[Tuple[int, List[str]]]:
    """Return [(register_id, tokens)] for every non-empty line."""
    out = []
    for line in text.splitlines():
        h = line.find("#")
        if h >= 0:
            line = line[:h]
        toks = line.split()
        if not toks:
            continue
        reg = 0
        if toks[0].startswith("@"):
            reg = int(toks[0][1:])
            toks = toks[1:]
        out.append((reg, toks))
    return out


def _cplx(t: Sequence[str], p: int) -> complex:
    return complex(float(t[p]), float(t[p + 1]))


def _qubits(t: Sequence[str], p: int) -> Tuple[List[int], int]:
    n = int(t[p])
    return [int(x) for x in t[p + 1:p + 1 + n]], p + 1 + n


def _mtrx(t: Sequence[str], p: int) -> List[complex]:
    return [_cplx(t, p + 2 * k) for k in range(4)]


def run(text: str, make_reg: Callable[[int, int], object]) -> Tuple[Dict[int, object], List[Tuple[str, Tuple[float, ...]]]]:
    """Replay a script.  ``make_reg(n_qubits, perm)`` must return an engine object exposing the
    QInterface-named methods of ``qrack_b200.qengine.QEngineHost``.  Returns (registers, results)."""
    regs: Dict[int, object] = {}
    results: List[Tuple[str, Tuple[float, ...]]] = []
    for reg, t in parse(text):
        op = t[0]
        if op == "qubits":
            regs[0] = make_reg(int(t[1]), 0)
            continue
        if op == "reg":
            regs[int(t[1])] = make_reg(int(t[2]), int(t[3]))
            continue
        if op in ("TIC", "TOC"):
            for q in regs.values():
                q.Finish()
            continue
        q = regs[reg]
        if op in ("H", "X", "Y", "Z", "S", "IS", "T", "IT", "SqrtX"):
            getattr(q, op)(int(t[1]))
        elif op in ("CNOT", "AntiCNOT", "CZ", "CY", "Swap", "ISwap", "SqrtSwap"):
            getattr(q, op)(int(t[1]), int(t[2]))
        elif op == "CCNOT":
            q.CCNOT(int(t[1]), int(t[2]), int(t[3]))
        elif op == "FSim":
            q.FSim(float(t[1]), float(t[2]), int(t[3]), int(t[4]))
        elif op in ("CSwap", "AntiCSwap"):
            c, p = _qubits(t, 1)
            getattr(q, op)(c, int(t[p]), int(t[p + 1]))
        elif op == "U":
            q.U(int(t[1]), float(t[2]), float(t[3]), float(t[4]))
        elif op in ("AI", "IAI"):
            getattr(q, op)(int(t[1]), float(t[2]), float(t[3]))
        elif op in ("Phase", "Invert"):
            getattr(q, op)(_cplx(t, 2), _cplx(t, 4), int(t[1]))
        elif op == "Mtrx":
            q.Mtrx(_mtrx(t, 2), int(t[1]))
        elif op in ("MCMtrx", "MACMtrx"):
            c, p = _qubits(t, 1)
            getattr(q, op)(c, _mtrx(t, p + 1), int(t[p]))
        elif op == "UCMtrx":
            c, p = _qubits(t, 1)
            q.UCMtrx(c, _mtrx(t, p + 2), int(t[p]), int(t[p + 1]))
        elif op in ("MCPhase", "MACPhase", "MCInvert", "MACInvert"):
            c, p = _qubits(t, 1)
            getattr(q, op)(c, _cplx(t, p + 1), _cplx(t, p + 3), int(t[p]))
        elif op == "PhaseRootN":
            q.PhaseRootN(int(t[1]), int(t[2]))
        elif op == "CPhaseRootN":
            q.CPhaseRootN(int(t[1]), int(t[2]), int(t[3]))
        elif op in ("QFT", "IQFT", "ZeroPhaseFlip"):
            getattr(q, op)(int(t[1]), int(t[2]))
        elif op in ("XMask", "ZMask"):
            getattr(q, op)(int(t[1]))
        elif op == "PhaseParity":
            q.PhaseParity(float(t[1]), int(t[2]))
        elif op == "PhaseRootNMask":
            q.PhaseRootNMask(int(t[1]), int(t[2]))
        elif op == "UniformParityRZ":
            q.UniformParityRZ(int(t[1]), float(t[2]))
        elif op == "CUniformParityRZ":
            c, p = _qubits(t, 1)
            q.CUniformParityRZ(c, int(t[p]), float(t[p + 1]))
        elif op == "UniformlyControlledSingleBit":
            c, p = _qubits(t, 1)
            skips, p2 = _qubits(t, p + 1)
            v = [float(x) for x in t[p2 + 1:]]
            q.UniformlyControlledSingleBit(c, int(t[p]), [complex(v[2 * k], v[2 * k + 1]) for k in range(len(v) // 2)], skips,
                                           int(t[p2]))
        elif op in ("UniformlyControlledRY", "UniformlyControlledRZ"):
            c, p = _qubits(t, 1)
            getattr(q, op)(c, int(t[p]), [float(x) for x in t[p + 1:]])
        elif op in ("INC", "DEC"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]))
        elif op in ("ROL", "ROR"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]))
        elif op in ("CINC", "CDEC"):
            c, p = _qubits(t, 1)
            getattr(q, op)(int(t[p]), int(t[p + 1]), int(t[p + 2]), c)
        elif op in ("INCC", "DECC", "INCS", "DECS"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]), int(t[4]))
        elif op in ("INCSCc", "DECSCc"):  # carry-only forms
            getattr(q, op[:-1])(int(t[1]), int(t[2]), int(t[3]), int(t[4]))
        elif op in ("INCSC", "DECSC"):  # overflow flag + carry
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]), int(t[4]), int(t[5]))
        elif op in ("MUL", "DIV"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]), int(t[4]))
        elif op in ("CMUL", "CDIV"):
            c, p = _qubits(t, 1)
            getattr(q, op)(int(t[p]), int(t[p + 1]), int(t[p + 2]), int(t[p + 3]), c)
        elif op in ("MULModNOut", "IMULModNOut", "POWModNOut"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]), int(t[4]), int(t[5]))
        elif op in ("CMULModNOut", "CIMULModNOut", "CPOWModNOut"):
            c, p = _qubits(t, 1)
            getattr(q, op)(int(t[p]), int(t[p + 1]), int(t[p + 2]), int(t[p + 3]), int(t[p + 4]), c)
        elif op == "IndexedLDA":
            q.IndexedLDA(int(t[1]), int(t[2]), int(t[3]), int(t[4]), bytes.fromhex(t[5]), True)
        elif op in ("IndexedADC", "IndexedSBC"):
            getattr(q, op)(int(t[1]), int(t[2]), int(t[3]), int(t[4]), int(t[5]), bytes.fromhex(t[6]))
        elif op == "Hash":
            q.Hash(int(t[1]), int(t[2]), bytes.fromhex(t[3]))
        elif op == "PhaseFlipIfLess":
            q.PhaseFlipIfLess(int(t[1]), int(t[2]), int(t[3]))
        elif op == "CPhaseFlipIfLess":
            q.CPhaseFlipIfLess(int(t[1]), int(t[2]), int(t[3]), int(t[4]))
        elif op == "SetPermutation":
            q.SetPermutation(int(t[1]), 1.0 + 0j)
        elif op == "ForceM":
            q.ForceM(int(t[1]), int(t[2]) != 0, True, True)
        elif op == "ForceMReg":
            q.ForceMReg(int(t[1]), int(t[2]), int(t[3]), True, True)
        elif op == "NormalizeState":
            q.NormalizeState()
        elif op == "UpdateRunningNorm":
            q.UpdateRunningNorm()
        elif op == "LossySave":
            q.LossySaveStateVector(t[1], int(t[2]), int(t[3]))
        elif op == "LossyLoad":
            q.LossyLoadStateVector(t[1])
        elif op == "Compose":
            if len(t) > 2:
                q.Compose(regs[int(t[1])], int(t[2]))
            else:
                q.Compose(regs[int(t[1])])
        elif op == "Decompose":
            regs[int(t[3])] = q.Decompose(int(t[1]), int(t[2]))
        elif op == "Dispose":
            if len(t) > 3:
                q.Dispose(int(t[1]), int(t[2]), int(t[3]))
            else:
                q.Dispose(int(t[1]), int(t[2]))
        elif op == "Allocate":
            q.Allocate(int(t[1]), int(t[2]))
        elif op == "Prob":
            results.append((op, (q.Prob(int(t[1])),)))
        elif op == "ProbAll":
            results.append((op, (q.ProbAll(int(t[1])),)))
        elif op == "ProbReg":
            results.append((op, (q.ProbReg(int(t[1]), int(t[2]), int(t[3])),)))
        elif op == "ProbMask":
            results.append((op, (q.ProbMask(int(t[1]), int(t[2])),)))
        elif op == "ProbParity":
            results.append((op, (q.ProbParity(int(t[1])),)))
        elif op in ("CProb", "ACProb"):
            results.append((op, (getattr(q, op)(int(t[1]), int(t[2])),)))
        elif op == "GetAmplitude":
            a = q.GetAmplitude(int(t[1]))
            results.append((op, (a.real, a.imag)))
        elif op == "SumSqrDiff":
            results.append((op, (q.SumSqrDiff(regs[int(t[1])]),)))
        elif op == "Norm":
            q.UpdateRunningNorm()
            results.append((op, (q.GetRunningNorm(),)))
        elif op in ("ExpectationBitsAll", "VarianceBitsAll"):
            c, p = _qubits(t, 1)
            results.append((op, (getattr(q, op)(c, int(t[p])),)))
        elif op in ("ExpectationBitsFactorized", "VarianceBitsFactorized"):
            c, p = _qubits(t, 1)
            results.append((op, (getattr(q, op)(c, [int(x) for x in t[p + 1:]], int(t[p])),)))
        elif op in ("ExpectationFloatsFactorized", "VarianceFloatsFactorized"):
            c, p = _qubits(t, 1)
            results.append((op, (getattr(q, op)(c, [float(x) for x in t[p:]]),)))
        elif op in ("ExpectationUnitaryAll", "VarianceUnitaryAll"):
            c, p = _qubits(t, 1)
            v = [float(x) for x in t[p:]]
            if len(v) > 3 * len(c):  # past the 3 angles per qubit: the eigenvalues
                results.append((op, (getattr(q, op)(c, v[:3 * len(c)], v[3 * len(c):]),)))
            else:
                results.append((op, (getattr(q, op)(c, v),)))
        elif op in ("ExpectationMatrixAll", "VarianceMatrixAll"):
            c, p = _qubits(t, 1)
            v = [float(x) for x in t[p:]]
            mats = [[complex(v[8 * i + 2 * e], v[8 * i + 2 * e + 1]) for e in range(4)] for i in range(len(c))]
            fn = q.ExpectationUnitaryAll if op[0] == "E" else q.VarianceUnitaryAll
            results.append((op, (fn(c, mats, v[8 * len(c):]),)))
        elif op in ("ExpectationPauliAll", "VariancePauliAll"):
            c, p = _qubits(t, 1)
            results.append((op, (getattr(q, op)(c, [int(x) for x in t[p:]]),)))
        elif op == "GetReducedDensityMatrix":
            c, _ = _qubits(t, 1)
            vals = []
            for row in q.GetReducedDensityMatrix(c):
                for z in row:
                    vals += [float(z.real), float(z.imag)]
            results.append((op, tuple(vals)))
        elif op == "HighestProbAllN":
            results.append((op, tuple(float(p) for p in q.HighestProbAllN(int(t[1])))))
        else:
            raise ValueError("qscript: unknown op %r" % op)
    return regs, results


def parse_results(text: str) -> List[Tuple[str, Tuple[float, ...]]]:
    out = []
    for line in text.splitlines():
        t = line.split()
        if t:
            out.append((t[0], tuple(float(x) for x in t[1:])))
    return out


# ---------------------------------------------------------------------------------------------
# Circuit generators (SURVEY.md §8d).  Deterministic given the seed; python's Mersenne twister.
# ---------------------------------------------------------------------------------------------

def random_matching(rng: random.Random, n: int) -> List[Tuple[int, int]]:
    """Random perfect matching of n qubits (the pairing scheme of the reference's
    examples/quantum_volume.cpp:84-88 / test/benchmarks.cpp:4169-4174)."""
    unused = list(range(n))
    pairs = []
    while len(unused) > 1:
        a = unused.pop(rng.randrange(len(unused)))
        b = unused.pop(rng.randrange(len(unused)))
        pairs.append((a, b))
    return pairs


def random_htcnot(n: int, depth: int, seed: int = 20250921, timed: bool = True) -> str:
    """BASELINE configs[0]/[1]: per layer every qubit gets H (p=1/2) else T, then CNOTs on a random
    perfect matching.  n=20, depth=40 -> 1200 gates (C1); n=30 -> 1800 gates (C2)."""
    rng = random.Random(seed)
    lines = ["qubits %d" % n]
    if timed:
        lines.append("TIC")
    for _ in range(depth):
        for q in range(n):
            lines.append(("H %d" if rng.random() < 0.5 else "T %d") % q)
        for a, b in random_matching(rng, n):
            lines.append("CNOT %d %d" % (a, b))
    if timed:
        lines.append("TOC")
    return "\n".join(lines) + "\n"


def random_u3_cnot(n: int, depth: int, seed: int = 7) -> str:
    """C1b: same layering with general U(theta,phi,lambda) single-qubit gates."""
    rng = random.Random(seed)
    lines = ["qubits %d" % n]
    for _ in range(depth):
        for q in range(n):
            lines.append("U %d %.17g %.17g %.17g" % (q, rng.uniform(-math.pi, math.pi), rng.uniform(-math.pi, math.pi),
                                                       rng.uniform(-math.pi, math.pi)))
        for a, b in random_matching(rng, n):
            lines.append("CNOT %d %d" % (a, b))
    return "\n".join(lines) + "\n"


def qft(n: int, seed: int = 11, init: str = "h", timed: bool = True) -> str:
    """BASELINE configs[2] (C3): QFT(0, n) from an H-on-random-bits start (test/benchmarks.cpp:577-602)."""
    rng = random.Random(seed)
    lines = ["qubits %d" % n]
    if init == "perm":
        lines.append("SetPermutation %d" % rng.getrandbits(n))
    else:
        for q in range(n):
            if rng.random() < 0.5:
                lines.append("H %d" % q)
    if timed:
        lines.append("TIC")
    lines.append("QFT 0 %d" % n)
    if timed:
        lines.append("TOC")
    return "\n".join(lines) + "\n"


def quantum_volume(n: int, depth: int | None = None, seed: int = 33, timed: bool = True) -> str:
    """BASELINE configs[3] (C4): examples/quantum_volume.cpp:69-88 — per layer AI(q, theta, phi) on every
    qubit with theta, phi ~ U(-pi, pi), then CNOT on a random matching; depth defaults to n."""
    rng = random.Random(seed)
    depth = n if depth is None else depth
    lines = ["qubits %d" % n]
    if timed:
        lines.append("TIC")
    for _ in range(depth):
        for q in range(n):
            lines.append("AI %d %.17g %.17g" % (q, rng.uniform(-math.pi, math.pi), rng.uniform(-math.pi, math.pi)))
        for a, b in random_matching(rng, n):
            lines.append("CNOT %d %d" % (a, b))
    if timed:
        lines.append("TOC")
    return "\n".join(lines) + "\n"


def grover(n: int, iterations: int, target: int = 3, timed: bool = True) -> str:
    """BASELINE configs[4] (C5): examples/grovers.cpp:24-68 generalised as test/benchmarks.cpp:548-573."""
    lines = ["qubits %d" % n]
    if timed:
        lines.append("TIC")
    for q in range(n):
        lines.append("H %d" % q)
    for _ in range(iterations):
        lines.append("DEC %d 0 %d" % (target, n))
        lines.append("ZeroPhaseFlip 0 %d" % n)
        lines.append("INC %d 0 %d" % (target, n))
        for q in range(n):
            lines.append("H %d" % q)
        lines.append("ZeroPhaseFlip 0 %d" % n)
        for q in range(n):
            lines.append("H %d" % q)
    if timed:
        lines.append("TOC")
    lines.append("ProbAll %d" % target)
    return "\n".join(lines) + "\n"


def count_gate_ops(text: str) -> int:
    """Number of non-query, non-structural ops (what 'gates/sec' counts)."""
    n = 0
    for _, t in parse(text):
        if t[0] in ("qubits", "reg", "TIC", "TOC") or t[0] in QUERY_OPS:
            continue
        n += 1
    return n
