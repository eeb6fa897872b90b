"""CPU pin of the float64 NumPy reference (tests/npref.py): every primitive against the oracle restatement (itself pinned to
the compiled reference by test_oracle_pin.py), and the gate-list reference against the fused planner + encoder run on the host
(b200sv_emulate_fused).  A wrong reference fails here, before any GPU test trusts it."""
import ctypes
import random

import numpy as np
import pytest

from oracle.restate_engine import QEngineRestate, _load as load_oracle
from qrack_b200 import _abi

import npref
import util


def oracle(n, prec, psi):
    o = QEngineRestate(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    o.SetQuantumState(psi)
    return o


def dense(rng, n, prec):
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def amp_close(got, want, prec, what):
    d = float(np.abs(np.asarray(got, dtype=np.complex128) - want).max()) if np.size(want) else 0.0
    assert d <= util.AMP_TOL[prec], "%s: max |delta amp| = %.3e" % (what, d)


def scalar_close(got, want, prec, what):
    assert abs(got - want) <= util.PROB_TOL[prec], "%s: %r vs %r" % (what, got, want)


def thresh_between(psi, q):
    """a threshold halfway between two neighbouring |amp|^2 of psi near quantile q: no amplitude sits on it in either precision"""
    p = np.sort(np.abs(psi.astype(np.complex128)) ** 2)
    i = int(q * (p.size - 1))
    return float(0.5 * (p[i] + p[i + 1]))


def rand_mask(rng, n, k=None):
    k = rng.randrange(1, n + 1) if k is None else k
    m = 0
    for b in rng.sample(range(n), k):
        m |= 1 << b
    return m


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [3, 7, 12])
def test_elementwise_primitives_match_the_oracle(n, prec):
    rng = random.Random(n * 100 + prec)
    nrng = np.random.default_rng(n + prec)
    psi = dense(nrng, n, prec)

    def run(name, *args):
        o = oracle(n, prec, psi)
        ret = getattr(o.be, name)(*args)
        return o.GetQuantumState(), ret

    for _ in range(4):
        t = rng.randrange(n)
        cs = rng.sample([q for q in range(n) if q != t], min(2, n - 1))
        m = npref.round_matrix(npref.random_unitary(rng), prec)
        off1, off2, pm = npref.gate_form(t, cs[:1], cs[1:])
        pows = [1 << b for b in range(n) if (pm >> b) & 1]
        got, _ = run("apply2x2", off1, off2, m, pows, 1.0, 0.0, False)
        amp_close(got, npref.apply2x2(psi, off1, off2, m, pows), prec, "apply2x2")
        nrm = 0.75
        o = oracle(n, prec, psi)
        gnorm = o.be.apply2x2(off1, off2, m, pows, nrm, 1e-4, True)
        want, wnorm = npref.apply2x2(psi, off1, off2, m, pows, nrm, 1e-4)
        amp_close(o.GetQuantumState(), want, prec, "apply2x2 norm")
        scalar_close(gnorm, wnorm, prec, "apply2x2 norm")
        mask = rand_mask(rng, n)
        got, _ = run("xmask", mask)
        assert np.array_equal(got, npref.xmask(psi, mask).astype(got.dtype))
        res = mask & rand_mask(rng, n)
        got, _ = run("apply_m", mask, res, 0.6 - 0.8j)
        amp_close(got, npref.apply_m(psi, mask, res, 0.6 - 0.8j), prec, "apply_m")
        got, kept = run("collapse_parity", mask, True)
        want, wkept = npref.collapse_parity(psi, mask, 1)
        amp_close(got, want, prec, "collapse_parity")
        scalar_close(kept, wkept, prec, "collapse_parity kept")
        r = rng.uniform(-3, 3)
        got, _ = run("phase_parity", r, mask)
        amp_close(got, npref.phase_parity(psi, r, mask), prec, "phase_parity")
        cm = rand_mask(rng, n, rng.randrange(0, n))
        got, _ = run("uniform_parity_rz", cm, mask, r)
        amp_close(got, npref.uniform_parity_rz(psi, cm, mask, r), prec, "uniform_parity_rz")
        k = rng.randrange(2, 9)
        got, _ = run("phase_root_n_mask", k, mask)
        amp_close(got, npref.phase_root_n_mask(psi, k, mask), prec, "phase_root_n_mask")
        th = thresh_between(psi, 0.2)
        got, _ = run("normalize", 0.8, th, 0.7)
        amp_close(got, npref.normalize(psi, 0.8, th, 0.7), prec, "normalize")


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [3, 7, 12])
def test_reductions_match_the_oracle(n, prec):
    rng = random.Random(n * 10 + prec)
    psi = dense(np.random.default_rng(n * 3 + prec), n, prec)
    o = oracle(n, prec, psi)
    for _ in range(6):
        mask = rand_mask(rng, n)
        perm = mask & rand_mask(rng, n)
        scalar_close(o.be.prob_mask(mask, perm), npref.prob_mask(psi, mask, perm), prec, "prob_mask")
        scalar_close(o.be.prob_parity(mask), npref.prob_parity(psi, mask), prec, "prob_parity")
        got = o.be.prob_mask_all(mask)
        assert np.abs(got - npref.prob_mask_all(psi, mask)).max() <= util.PROB_TOL[prec]
    for q, w in enumerate(npref.marginals(psi)):
        scalar_close(o.be.prob_mask(1 << q, 1 << q), w, prec, "marginal %d" % q)
    th = thresh_between(psi, 0.3)
    scalar_close(o.be.norm(th), npref.norm(psi, th), prec, "norm")
    other = oracle(n, prec, dense(np.random.default_rng(99), n, prec))
    z = o.be.inner(other.be)
    w = npref.inner(psi, other.GetQuantumState())
    assert abs(z - w) <= util.PROB_TOL[prec]
    for start, length in ((0, n), (0, 0), (1, n - 1), (n - 1, 1)):
        ex = o.be.expectation(start, length)
        assert abs(ex - npref.expectation(psi, start, length)) <= util.PROB_TOL[prec] * max(1, 1 << length)
    assert o.be.highest_prob() == npref.highest_prob(psi)
    for r in (0.0, 0.3, 0.5, 0.999):
        assert o.be.sample(r) == npref.sample(psi, r, prec)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [4, 9, 12])
def test_structure_matches_the_oracle(n, prec):
    rng = random.Random(n + prec)
    nrng = np.random.default_rng(n * 7 + prec)
    psi = dense(nrng, n, prec)
    for start in sorted({0, 1, n // 2, n}):
        nb = rng.randrange(1, 4)
        b = dense(nrng, nb, prec)
        o = oracle(n, prec, psi)
        o.Compose(oracle(nb, prec, b), start)
        amp_close(o.GetQuantumState(), npref.compose(psi, b, start), prec, "compose at %d" % start)
    # product states (Decompose is exact there) and an entangled one (the formula is defined for any state)
    prod = npref.compose(dense(nrng, n - 2, prec), dense(nrng, 2, prec), 1).astype(psi.dtype)
    for st in (prod, psi):
        for start, length in ((0, 1), (1, 2), (n - 3, 3), (0, n - 1)):
            o = oracle(n, prec, st)
            part = o.Decompose(start, length)
            rem, want_part = npref.decompose(st, start, length, prec)
            amp_close(o.GetQuantumState(), rem, prec, "decompose rem %d %d" % (start, length))
            amp_close(part.GetQuantumState(), want_part, prec, "decompose part %d %d" % (start, length))
        for perm in range(4):
            o = oracle(n, prec, st)
            o.Dispose(1, 2, perm)
            assert np.array_equal(o.GetQuantumState(), npref.dispose_perm(st, 1, 2, perm).astype(st.dtype))
    a, b = psi, dense(nrng, n, prec)
    oa, ob = oracle(n, prec, a), oracle(n, prec, b)
    oa.ShuffleBuffers(ob)
    wa, wb = npref.shuffle(a, b)
    assert np.array_equal(oa.GetQuantumState(), wa.astype(a.dtype)) and np.array_equal(ob.GetQuantumState(), wb.astype(a.dtype))


def oracle_uniformly_controlled(psi, prec, controls, target, mtrxs, skips, skip_value, nrm):
    lib = load_oracle()
    real = ctypes.c_float if prec == 32 else ctypes.c_double
    st = np.array(psi, dtype=np.complex64 if prec == 32 else np.complex128)
    m = np.array(mtrxs, dtype=st.dtype).reshape(-1)
    fn = getattr(lib, "orc_uniformly_controlled_f%d" % prec)
    fn(st.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(st.size.bit_length() - 1), ctypes.c_int(len(controls)),
       (ctypes.c_int * max(1, len(controls)))(*controls), ctypes.c_int(target), m.ctypes.data_as(ctypes.c_void_p),
       ctypes.c_int(len(skips)), (ctypes.c_uint64 * max(1, len(skips)))(*skips), ctypes.c_uint64(skip_value), real(nrm))
    return st


@pytest.mark.parametrize("prec", [32, 64])
def test_uniformly_controlled_matches_the_oracle(prec):
    rng = random.Random(prec)
    n = 8
    psi = dense(np.random.default_rng(4), n, prec)
    for nc, skips, sv, nrm in ((0, [], 0, 1.0), (1, [], 0, 1.0), (2, [2], 2, 0.9), (3, [1, 8], 9, 1.0), (3, [], 0, 1.25)):
        t = rng.randrange(n)
        controls = rng.sample([q for q in range(n) if q != t], nc)
        mt = [npref.round_matrix(npref.random_unitary(rng), prec) for _ in range(1 << (nc + len(skips)))]
        got = oracle_uniformly_controlled(psi, prec, controls, t, mt, skips, sv, nrm)
        amp_close(got, npref.uniformly_controlled(psi, controls, t, mt, skips, sv, nrm), prec, "uc %d %r" % (nc, skips))


def emulate_fused(n, prec, gates, psi):
    k, o1, o2, pm, m8 = npref.pack_gates(gates)
    st = np.array(psi, copy=True)
    rc = _abi.load().b200sv_emulate_fused(n, prec, k, o1, o2, pm, m8, st.ctypes.data_as(ctypes.c_void_p))
    assert rc == _abi.B200SV_OK
    return st


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [13, 16])
@pytest.mark.parametrize("family", ["light", "rotation", "full"])
def test_gate_list_reference_matches_the_emulated_fused_sweeps(family, n, prec):
    rng = random.Random(n * 31 + prec)
    psi = dense(np.random.default_rng(n), n, prec)
    gates = npref.gate_family(family, n, rng)
    amp_close(emulate_fused(n, prec, gates, psi), npref.apply_gates(psi, gates, prec), prec, family)


def test_gate_families_reach_every_fused_op_kind(capfd, monkeypatch):
    """The families of the device sweep test lower to every kind of fused op: Hadamard and rotation STAGEs, two-phase
    (PH2) and general phase (PHGEN) ops, X swaps, general unitaries (GEN_U) and general matrices (GEN_P)."""
    monkeypatch.setenv("B200SV_FUSED_DEBUG", "2")
    n = 14
    psi = dense(np.random.default_rng(1), n, 32)
    seen = {}
    for family in ("light", "rotation", "full"):
        emulate_fused(n, 32, npref.gate_family(family, n, random.Random(5)), psi)
        seen[family] = capfd.readouterr().err
    text = "".join(seen.values())
    for token in ("STAGE(", "PH2.", "PHGEN", "XSWAP.", "GEN_U.", "GEN_P."):
        assert token in text, "no %s op in the lowered families" % token
    assert ", rotation 0)" not in seen["rotation"].splitlines()[0], seen["rotation"].splitlines()[0]


# ---- QAlu maps and the re-page --------------------------------------------------------------------------------------

def check_alu_cases(n, prec, psi, cases):
    for name, args in cases:
        o = oracle(n, prec, psi)
        getattr(o.be, "alu_" + name)(*args)
        got = o.be.get_state()
        want = getattr(npref, name)(psi, *args)
        assert np.array_equal(got, want.astype(got.dtype)), "%s%r at %dq: %d amplitudes differ" % (
            name, args[:7], n, int(np.sum(got != want)))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", list(range(6, 15)))
def test_qalu_reference_matches_the_oracle(n, prec):
    """Every QAlu map of npref on the edge grid of the device test, bit for bit against the oracle restatement (itself pinned
    to the compiled reference by the alu_* golden fixtures): index maps and sign flips of the amplitudes, nothing rounds."""
    psi = dense(np.random.default_rng(40 + n), n, prec)
    check_alu_cases(n, prec, psi, npref.alu_grid(n))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [12, 19])
def test_wide_qalu_reference_matches_the_oracle(n, prec):
    """The wide-register calls of the device test, 2- and 3-byte table entries among them (19 qubits hold a 17-bit value
    register with its index bit and carry)."""
    psi = dense(np.random.default_rng(60 + n), n, prec)
    check_alu_cases(n, prec, psi, npref.alu_wide(n))


def test_forward_maps_must_be_injective():
    """A forward map that sends two sources to one destination has no defined result: the reference refuses it."""
    psi = dense(np.random.default_rng(3), 6, 64)
    with pytest.raises(AssertionError, match="not injective"):
        npref.muldiv(psi, 0, 16, 0, 3, 3, 0)                # 16 * 4 wraps past the 6 bits of register and carry to 0
    with pytest.raises(AssertionError, match="not injective"):
        npref.muldiv(psi, 0, 0, 0, 3, 3, 0)
    with pytest.raises(AssertionError, match="not injective"):
        npref.hash(psi, 0, 2, bytes([0, 1, 1, 2]))


def test_exchange_reference_is_a_rank_permutation():
    """Re-paging twice with the same victim bits is the identity, and every amplitude of every page lands exactly once."""
    nl, k, vb = 7, 2, [5, 1]
    pages = [np.arange(r << nl, (r + 1) << nl).astype(np.complex128) for r in range(1 << k)]
    new = [npref.exchange(pages, k, vb, r) for r in range(1 << k)]
    assert np.array_equal(np.sort(np.concatenate(new).real), np.arange(4 << nl))
    for r in range(1 << k):
        assert np.array_equal(npref.exchange(new, k, vb, r), pages[r])
        # element i: source rank = (bit 5, bit 1) of i, index = i with those bits := this rank's bits
        i = 0b1100010
        assert new[r][i] == pages[3][(i & ~0b100010) | ((r & 1) << 5) | ((r >> 1) << 1)]


def first_sweep_direct_flags(n, prec, gates, capfd, monkeypatch):
    monkeypatch.setenv("B200SV_FUSED_DEBUG", "1")
    capfd.readouterr()
    k, o1, o2, pm, m8 = npref.pack_gates(gates)
    ns, npass, nops = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = _abi.load().b200sv_plan_gates(n, prec, k, o1, o2, pm, m8, ctypes.byref(ns), ctypes.byref(npass), ctypes.byref(nops))
    assert rc == _abi.B200SV_OK
    err = capfd.readouterr().err
    first = next(line for line in err.splitlines() if line.strip().startswith("sweep:"))
    return int(first.split("directIn")[1].split(",")[0]), first


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [13, 16])
def test_pull_gate_lists_take_both_first_pass_paths(n, prec, capfd, monkeypatch):
    """The first sweep of a flush carries a pending pull re-page.  Its first pass reads the source pages either through the
    staged tile copy (stage_in_pull: directIn 0) or with direct per-thread loads (pull_src in the pass: directIn 1); the
    planner decides per sweep.  The two gate lists per family of the device pull test must reach one each."""
    for family in ("light", "rotation", "full"):
        staged, direct = npref.pull_gate_lists(family, n, prec)
        d, line = first_sweep_direct_flags(n, prec, staged, capfd, monkeypatch)
        assert d == 0, (family, "staged", line)
        d, line = first_sweep_direct_flags(n, prec, direct, capfd, monkeypatch)
        assert d == 1, (family, "direct", line)
