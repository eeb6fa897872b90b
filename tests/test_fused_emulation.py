"""CPU tests of the fused-sweep scheduler and program encoder: the real planner/encoder of libb200sv.so + the host
interpreter of the encoded programs (b200sv_emulate_fused, no device) against the oracle restatement and the golden
fixtures of the compiled reference.  Same tolerances as the GPU parity tests."""
import random

import numpy as np
import pytest

from oracle.restate_engine import QEngineRestate
from qrack_b200 import qscript

import util
from emu_engine import QEngineEmu


def run_emu(text, prec):
    regs, results = qscript.run(text, util.make_factory(QEngineEmu, prec))
    return {k: v.GetQuantumState() for k, v in regs.items()}, results, regs


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("name", [n for n in util.golden_names() if not n.startswith("alu_")])
def test_emulated_sweeps_reproduce_golden_fixtures(name, prec):
    text, regs, results = util.load_golden(name, prec)
    got, gres, _ = run_emu(text, prec)
    util.assert_states_close(got, regs, prec, name)
    util.assert_results_close(gres, results, prec, name)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("gen", ["htcnot", "u3", "qft", "qv", "grover", "htcnot_qft_mc"])
def test_emulated_sweeps_vs_oracle_multi_tile(gen, prec):
    """15-16 qubits: 8-16 tiles per sweep, high tile qubits, outer controls (ballots), DIAG slots, several passes."""
    n = 16 if prec == 32 else 15
    text = {"htcnot": lambda: qscript.random_htcnot(n, 12, seed=5, timed=False),
            "u3": lambda: qscript.random_u3_cnot(n, 5, seed=6),
            "qft": lambda: "qubits %d\nSetPermutation 12345\nH 3\nH 9\nQFT 0 %d\nT 2\nIQFT 1 %d\n" % (n, n, n - 2),
            "qv": lambda: qscript.quantum_volume(n, depth=5, seed=8, timed=False),
            "grover": lambda: qscript.grover(n, 2, target=77, timed=False),
            "htcnot_qft_mc": lambda: (qscript.random_htcnot(15, 8, seed=3, timed=False)
                                      + "QFT 2 9\nCCNOT 1 14 7\nMCPhase 2 3 13 8 0.6 0.8 1 0\n")}[gen]()
    want, _ = util.run_engine(text, QEngineRestate, prec)
    got, _, regs = run_emu(text, prec)
    util.assert_states_close(got, want, prec, gen)
    assert regs[0].be.flushes >= 1          # the gates really went through the planner + emulator


def test_emulation_hook_rejects_bad_arguments():
    import ctypes
    from qrack_b200 import _abi
    lib = _abi.load()
    st = np.zeros(32, dtype=np.complex64)
    one = (ctypes.c_uint64 * 1)(3)
    two = (ctypes.c_uint64 * 1)(0)
    pm = (ctypes.c_uint64 * 1)(3)
    m = (ctypes.c_double * 8)(1, 0, 0, 0, 0, 0, 1, 0)
    # off1 ^ off2 has two bits: not a single-target gate
    assert lib.b200sv_emulate_fused(5, 32, 1, one, two, pm, m, st.ctypes.data_as(ctypes.c_void_p)) == _abi.B200SV_EINVAL
    assert lib.b200sv_emulate_fused(3, 32, 0, None, None, None, None, st.ctypes.data_as(ctypes.c_void_p)) == _abi.B200SV_EINVAL


def _random_mixed_circuit(rng, n, ngates):
    import math
    L = ["qubits %d" % n] + ["H %d" % q for q in range(n) if rng.random() < 0.7]

    def cx():
        a = rng.uniform(0, 2 * math.pi)
        return "%.17g %.17g" % (math.cos(a), math.sin(a))

    def unitary():
        th, ph, la = (rng.uniform(-math.pi, math.pi) for _ in range(3))
        c, s = math.cos(th / 2), math.sin(th / 2)
        m = [c, -s * complex(math.cos(la), math.sin(la)), s * complex(math.cos(ph), math.sin(ph)),
             c * complex(math.cos(ph + la), math.sin(ph + la))]
        return " ".join("%.17g %.17g" % (complex(z).real, complex(z).imag) for z in m)

    for _ in range(ngates):
        r, qs = rng.random(), rng.sample(range(n), 4)
        if r < 0.2:
            L.append("%s %d" % (rng.choice(["H", "T", "X", "S", "Z", "Y", "IT", "SqrtX"]), qs[0]))
        elif r < 0.4:
            L.append("%s %d %d" % (rng.choice(["CNOT", "CZ", "AntiCNOT", "CY"]), qs[0], qs[1]))
        elif r < 0.5:
            L.append("CCNOT %d %d %d" % tuple(qs[:3]))
        elif r < 0.6:
            L.append("U %d %.17g %.17g %.17g" % (qs[0], rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3)))
        elif r < 0.7:
            L.append("MCMtrx 2 %d %d %d %s" % (qs[0], qs[1], qs[2], unitary()))
        elif r < 0.78:
            L.append("MACMtrx 2 %d %d %d %s" % (qs[0], qs[1], qs[2], unitary()))
        elif r < 0.86:
            L.append("MCPhase 2 %d %d %d %s %s" % (qs[0], qs[1], qs[2], cx(), cx()))
        elif r < 0.92:
            L.append("MACInvert 1 %d %d %s %s" % (qs[0], qs[1], cx(), cx()))
        elif r < 0.96:
            L.append("CPhaseRootN %d %d %d" % (rng.randrange(1, 6), qs[0], qs[1]))
        else:
            L.append("UCMtrx 3 %d %d %d %d %d %s" % (qs[0], qs[1], qs[2], qs[3], rng.randrange(8), unitary()))
    return "\n".join(L) + "\n"


def test_emulated_sweeps_fuzz_mixed_gates():
    """Random circuits mixing every single-target form the dispatch produces (controls, anti-controls, phases, inverts,
    uniformly-controlled selections) on 13-17 qubits, both precisions, through planner + encoder + interpreter."""
    rng = random.Random(2025)
    for trial in range(10):
        prec = rng.choice([32, 64])
        n = rng.randrange(13, 18) if prec == 32 else rng.randrange(13, 17)
        text = _random_mixed_circuit(rng, n, rng.randrange(60, 300))
        want, _ = util.run_engine(text, QEngineRestate, prec)
        got, _, _ = run_emu(text, prec)
        util.assert_states_close(got, want, prec, "fuzz %d" % trial)


def _random_gate_arrays(n, n_gates, rng):
    """random single-target gates in the ABI's (off1, off2, pmask, m) form: H, T, X, random unitaries, 0-2 controls of either polarity"""
    import cmath
    import ctypes
    o1, o2, pm, mats = [], [], [], []
    for _ in range(n_gates):
        t = rng.randrange(n)
        ctrls = rng.sample([q for q in range(n) if q != t], rng.choice([0, 0, 1, 1, 2]))
        cval = sum((1 << c) for c in ctrls if rng.random() < 0.7)
        kind = rng.choice("HHTXU")
        if kind == "H":
            m = [2 ** -0.5, 2 ** -0.5, 2 ** -0.5, -(2 ** -0.5)]
        elif kind == "T":
            m = [1, 0, 0, cmath.exp(0.25j * cmath.pi)]
        elif kind == "X":
            m = [0, 1, 1, 0]
        else:
            th, a, b = rng.uniform(0, 3.1), rng.uniform(0, 6.2), rng.uniform(0, 6.2)
            m = [cmath.cos(th), -cmath.exp(1j * a) * cmath.sin(th), cmath.exp(1j * b) * cmath.sin(th),
                 cmath.exp(1j * (a + b)) * cmath.cos(th)]
        o1.append(cval)
        o2.append(cval | (1 << t))
        pm.append((1 << t) | sum(1 << c for c in ctrls))
        mats.extend(x for z in m for x in (complex(z).real, complex(z).imag))
    g = len(o1)
    return (g, (ctypes.c_uint64 * g)(*o1), (ctypes.c_uint64 * g)(*o2), (ctypes.c_uint64 * g)(*pm), (ctypes.c_double * (8 * g))(*mats))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("k,nl,n_gates", [(1, 14, 30), (2, 15, 60), (3, 14, 25), (2, 13, 0), (3, 16, 90)])
def test_emulated_pull_exchange_equals_exchange_then_sweeps(prec, k, nl, n_gates):
    """b200sv_exchange_pull rides on the first fused sweep: the host interpreter of the same programs, reading through the pull
    mapping from W host 'pages', must give bit for bit what the plain exchange (numpy permutation) followed by the same
    flush gives — on every rank, for victim bits anywhere in the page (tile-low, tile-high and outer qubits)."""
    import ctypes
    from qrack_b200 import _abi
    lib = _abi.load()
    rng = random.Random(1000 * k + nl + prec)
    nrng = np.random.default_rng(k * 77 + nl)
    W = 1 << k
    cplx = np.complex64 if prec == 32 else np.complex128
    pages = [(nrng.standard_normal(1 << nl) + 1j * nrng.standard_normal(1 << nl)).astype(cplx) for _ in range(W)]
    lo = 1 if prec == 32 else 0
    vb = rng.sample(range(lo, nl), k)
    vmask = sum(1 << b for b in vb)
    g, o1, o2, pm, mats = _random_gate_arrays(nl, n_gates, rng)
    idx = np.arange(1 << nl, dtype=np.uint64)
    src_rank = np.zeros(1 << nl, dtype=np.int64)
    for b in range(k):
        src_rank |= (((idx >> np.uint64(vb[b])) & np.uint64(1)).astype(np.int64) << b)
    src = (ctypes.c_void_p * W)(*[p.ctypes.data for p in pages])
    vbc = (ctypes.c_int * k)(*vb)
    for rank in range(W):
        dep = sum((1 << vb[b]) for b in range(k) if (rank >> b) & 1)
        src_idx = (idx & np.uint64(~vmask & ((1 << nl) - 1))) | np.uint64(dep)
        want = np.empty(1 << nl, dtype=cplx)
        for r in range(W):
            sel = src_rank == r
            want[sel] = pages[r][src_idx[sel]]
        if g:
            _abi.check(lib, lib.b200sv_emulate_fused(nl, prec, g, o1, o2, pm, mats, want.ctypes.data_as(ctypes.c_void_p)))
        got = np.full(1 << nl, np.nan, dtype=cplx)
        _abi.check(lib, lib.b200sv_emulate_fused_pull(nl, prec, g, o1, o2, pm, mats, k, vbc, rank, src,
                                                      got.ctypes.data_as(ctypes.c_void_p)))
        assert np.array_equal(got, want), (rank, vb)
    # argument checks: the out page may not alias a source, k is bounded by the 8 peers of one box
    assert lib.b200sv_emulate_fused_pull(nl, prec, 0, None, None, None, None, k, vbc, 0, src, ctypes.c_void_p(pages[0].ctypes.data)) \
        == _abi.B200SV_EINVAL
    assert lib.b200sv_emulate_fused_pull(nl, prec, 0, None, None, None, None, 4, vbc, 0, src, None) == _abi.B200SV_EINVAL


@pytest.mark.parametrize("prec", [32, 64])
def test_rank_bits_and_carry_on_the_host_interpreter(prec):
    """b200sv_set_rank_bits + b200sv_flush_carry semantics (the same check body runs on the GPU in tests/test_zz_carry_gpu.py):
    gates with controls / diagonal targets on virtual qubits, one flush vs carry + resubmission, for every rank value."""
    from carry_checks import check_rank_bits_and_carry
    handed = 0
    for seed in range(3):
        handed += check_rank_bits_and_carry(lambda n: QEngineEmu(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec), prec, seed=seed)
    assert handed > 0
