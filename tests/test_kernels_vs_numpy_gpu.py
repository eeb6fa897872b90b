"""Every CUDA kernel of libb200sv.so against the float64 NumPy reference (tests/npref.py), at the shapes where its code path
changes: qubit counts on both sides of each size switch, masks of each kind, both precisions.

The reference is always fed the state the kernel read, read back from the engine in its own precision; gate matrices are
rounded to the engine's precision first.  Tolerances: amplitudes util.AMP_TOL (1e-6 fp32 / 1e-12 fp64) against float64,
reductions RED_TOL; exact equality for pure permutations, selections, basis states and sample indices."""
import ctypes
import math
import random

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi

import npref
import util

pytestmark = pytest.mark.gpu

RED_TOL = {32: 2e-6, 64: 1e-12}
# relative L2 error ||got - want|| / ||want|| of a gate list: each lowered op rounds every amplitude once (relative 2^-24 /
# 2^-53), and independent roundings add in quadrature, so a list of a few hundred ops stays near sqrt(ops) * 2^-24 = 1e-6
# (fp32) / 2e-15 (fp64).  The host interpreter of the same sweep programs measures 1.6e-7..3.6e-7 / 5e-16..2.8e-15 on these
# families at 5-18 qubits.  Unlike the absolute amplitude bar, this one does not loosen as amplitudes shrink with n.
REL_TOL = {32: 5e-6, 64: 5e-14}


def engine(n, prec, psi=None, fusion=1, normalize=False):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    q.be.set_fusion(fusion)
    if psi is not None:
        q.SetQuantumState(psi)
    return q


def dense(rng, n, prec):
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return (psi / np.linalg.norm(psi)).astype(np.complex64 if prec == 32 else np.complex128)


def amp_close(got, want, prec, what):
    d = float(np.abs(np.asarray(got, dtype=np.complex128) - want).max()) if np.size(want) else 0.0
    assert d <= util.AMP_TOL[prec], "%s: max |delta amp| = %.3e > %.1e" % (what, d, util.AMP_TOL[prec])


def rel_close(got, want, prec, what):
    want = np.asarray(want, dtype=np.complex128)
    r = float(np.linalg.norm(np.asarray(got, dtype=np.complex128) - want) / np.linalg.norm(want))
    assert r <= REL_TOL[prec], "%s: relative L2 error %.3e > %.1e" % (what, r, REL_TOL[prec])


def red_close(got, want, prec, what):
    assert abs(got - want) <= RED_TOL[prec], "%s: %r vs %r (|delta| %.3e)" % (what, got, want, abs(got - want))


def exact(got, want, what):
    want = np.asarray(want).astype(np.asarray(got).dtype)
    assert np.array_equal(got, want), "%s: %d entries differ" % (what, int(np.sum(got != want)))


# ---------------------------------------------------------------------------------------------------------------
# fused sweep: every size from 5 to 20 qubits and 22, every kernel variant
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("family", ["light", "rotation", "full"])
@pytest.mark.parametrize("n", list(range(5, 21)) + [22])
def test_fused_sweep_every_size(n, family, prec):
    """The whole state is one partial tile up to 13 (fp32) / 12 (fp64) qubits and several tiles above; every qubit is a
    target and a control, so qubit 0, the low and high tile bits and the outer bits all carry gates."""
    rng = random.Random(1000 * n + prec)
    gates = npref.gate_family(family, n, rng)
    q = engine(n, prec, dense(np.random.default_rng(n), n, prec))
    psi = q.GetQuantumState()
    q.be.reset_stats()
    q.be.apply_gates(*npref.pack_gates(gates))
    got = q.GetQuantumState()
    st = q.be.stats()
    assert st["fused_sweeps"] >= 1 and st["single_launches"] == 0, st
    want = npref.apply_gates(psi, gates, prec)
    amp_close(got, want, prec, "%s %dq" % (family, n))
    rel_close(got, want, prec, "%s %dq" % (family, n))


# ---------------------------------------------------------------------------------------------------------------
# marginals: k_prob_all_bits below 2^14 16-byte chunks, k_prob_all_bits2 from there
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
def test_basis_state_marginals_are_exact(prec):
    """Every qubit's Prob on the basis states 2^q and their complements is exactly 0 or 1: pins which index bit each lane,
    warp, block and iteration bit of the marginals sweep stands for."""
    for n in range(3, 25):
        q = engine(n, prec)
        full = (1 << n) - 1
        for b in range(n):
            for perm, want_one in ((1 << b, lambda k: k == b), (full ^ (1 << b), lambda k: k != b)):
                q.SetPermutation(perm)
                got = [q.Prob(k) for k in range(n)]
                want = [1.0 if want_one(k) else 0.0 for k in range(n)]
                assert got == want, (n, b, perm, got)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [3, 8, 13, 14, 15, 16, 20, 24])
def test_dense_marginals(n, prec):
    q = engine(n, prec, dense(np.random.default_rng(n + prec), n, prec))
    want = npref.marginals(q.GetQuantumState())
    for b in range(n):
        red_close(q.Prob(b), want[b], prec, "Prob(%d) at %dq" % (b, n))


@pytest.mark.parametrize("n,prec", [(30, 32), (29, 64)])
def test_full_width_product_state_marginals(n, prec):
    """A product state U(theta_q) |0> on every qubit: Prob(q) = |m10_q|^2 prod_{k != q} (|m00_k|^2 + |m10_k|^2) with the
    engine-rounded matrices.  Qubit 0 of an fp32 state is summed apart from the others in the marginals sweep."""
    rng = random.Random(n)
    mats = [npref.random_unitary(rng) for _ in range(n)]
    q = engine(n, prec)
    q.be.apply_gates(*npref.pack_gates([npref.gate_form(b) + (m,) for b, m in enumerate(mats)]))
    r = [npref.round_matrix(m, prec) for m in mats]
    col = np.array([abs(m[0]) ** 2 + abs(m[2]) ** 2 for m in r])
    for b in range(n):
        want = abs(r[b][2]) ** 2 * np.prod(np.delete(col, b))
        red_close(q.Prob(b), want, prec, "Prob(%d) at %dq" % (b, n))
    del q


# ---------------------------------------------------------------------------------------------------------------
# reductions
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
def test_prob_mask_every_path(prec):
    rng = random.Random(prec)
    for n in (1, 2, 3, 5, 16, 20):
        q = engine(n, prec, dense(np.random.default_rng(n), n, prec))
        psi = q.GetQuantumState()
        masks = [1 << b for b in range(n)]                                  # single bits: memoised from 3 qubits on
        if n >= 16:
            masks += [(1 << 4) | (1 << 9) | (1 << (n - 1)), ((1 << n) - 1) & ~15]   # every bit >= 2^4: subset kernel
            masks += [0b1011, 1 | (1 << (n - 1)), 0x3c5]                   # predicate scan
        for mask in masks:
            for perm in {0, mask, mask & rng.getrandbits(n)}:
                red_close(q.be.prob_mask(mask, perm), npref.prob_mask(psi, mask, perm), prec, "mask %x perm %x" % (mask, perm))


@pytest.mark.parametrize("prec", [32, 64])
def test_prob_mask_all_shared_and_global_bins(prec):
    rng = random.Random(prec)
    for n, k in ((18, 12), (18, 13), (19, 14), (20, 15), (20, 16), (20, 3)):
        q = engine(n, prec, dense(np.random.default_rng(n + k), n, prec))
        psi = q.GetQuantumState()
        mask = sum(1 << b for b in rng.sample(range(n), k))
        got = q.be.prob_mask_all(mask).astype(np.float64)
        d = float(np.abs(got - npref.prob_mask_all(psi, mask)).max())
        assert d <= RED_TOL[prec], (n, k, d)


@pytest.mark.parametrize("prec", [32, 64])
def test_prob_parity_norm_inner_expectation(prec):
    nrng = np.random.default_rng(prec)
    for n in (3, 11, 17):
        a = dense(nrng, n, prec)
        # a few amplitudes planted far below the threshold, which Norm must leave out
        a[[0, (1 << n) - 1, 5]] = (1e-5, 2e-5j, -1e-5)
        q = engine(n, prec, a)
        psi = q.GetQuantumState()
        for mask in (1, 1 << (n - 1), (1 << n) - 1, 0b101 & ((1 << n) - 1)):
            red_close(q.be.prob_parity(mask), npref.prob_parity(psi, mask), prec, "parity %x" % mask)
        thresh = 1e-9
        red_close(q.be.norm(thresh), npref.norm(psi, thresh), prec, "norm")
        red_close(q.be.norm(0.0), npref.norm(psi, 0.0), prec, "norm, no threshold")
        o = engine(n, prec, dense(nrng, n, prec))
        z = q.be.inner(o.be)
        w = npref.inner(psi, o.GetQuantumState())
        red_close(z.real, w.real, prec, "inner re")
        red_close(z.imag, w.imag, prec, "inner im")
        for start, length in ((0, 0), (n - 1, 0), (0, n), (1, n - 1), (n - 1, 1), (n // 2, 2)):
            # the values weigh up to 2^length - 1: the bar scales with them
            got, want = q.be.expectation(start, length), npref.expectation(psi, start, length)
            assert abs(got - want) <= RED_TOL[prec] * max(1, (1 << length) - 1), (start, length, got, want)


@pytest.mark.parametrize("prec", [32, 64])
def test_highest_prob_ties_take_the_lowest_index(prec):
    n = 22
    nrng = np.random.default_rng(3)
    st = (nrng.standard_normal(1 << n) + 1j * nrng.standard_normal(1 << n)) * 1e-4
    top = 0.25 + 0.125j
    ties = [3000001, 1234567, 4000000, 1234568, 77]
    for i in ties:
        st[i] = top
    q = engine(n, prec, st.astype(np.complex64 if prec == 32 else np.complex128))
    assert q.be.highest_prob() == 77
    st[77] = 0
    q.SetQuantumState(st.astype(np.complex64 if prec == 32 else np.complex128))
    assert q.be.highest_prob() == 1234567 == npref.highest_prob(q.GetQuantumState())


# ---------------------------------------------------------------------------------------------------------------
# sampling at exact boundaries (dyadic probabilities: every prefix sum is exact)
# ---------------------------------------------------------------------------------------------------------------

def dyadic_state(n, probs_at, prec):
    """|amp|^2 = 2^-m exactly: 2^-(m/2) for even m, (1 + i) 2^-((m+1)/2) for odd m"""
    st = np.zeros(1 << n, dtype=np.complex128)
    for i, m in probs_at.items():
        st[i] = 2.0 ** (-m // 2) if m % 2 == 0 else (1 + 1j) * 2.0 ** (-(m + 1) // 2)
    return st.astype(np.complex64 if prec == 32 else np.complex128)


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [12, 13, 15, 17])
def test_sample_exact_boundaries(n, prec):
    """b200sv_sample and b200sv_sample_many against MAll's rule: 2^14-amplitude chunks (one chunk below 15 qubits), leading
    and trailing all-zero chunks, rnd equal to a prefix sum, rnd close to 1 over a zero tail, rnd above the total of an
    unnormalised state, the FP_NORM_EPSILON early exit (which fires for fp32 when the prefix comes within 2^-25 of 1) and the
    all-zero state."""
    s = 1 << (n - 3)        # at 17 qubits: chunks 1-3 hold the first case, chunk 0 and chunks 4-7 are empty
    t = 1 << (n - 2)
    cases = [
        {s + 4: 2, s + 6: 3, 2 * s + 2: 3, 3 * s: 1},                     # 1/4, 1/8, 1/8, 1/2 after a zero lead
        # 2^-1 .. 2^-25, then 2^-25 at the end: even indices only, so no fp32 pair sum needs more than 24 bits
        dict([(2 * i + (t if i > 12 else 0), i + 1) for i in range(25)] + [(3 * t + 2, 25)]),
        # total 1/2: rnd 0.5 and 0.6 exceed every prefix, so the search ends at the last nonzero index
        {s + 4: 2, 3 * s: 3, 3 * s + 2: 3},
    ]
    for probs_at in cases:
        st = dyadic_state(n, probs_at, prec)
        q = engine(n, prec, st)
        psi = q.GetQuantumState()
        cum = sorted({float(c) for c in np.cumsum(npref.probs(psi)[sorted(probs_at)])})
        rnds = [0.0, 0.1, 0.5, 0.6, 0.9999999, 1 - 2.0 ** -26, 1 - 2.0 ** -40]
        rnds += cum[:-1] + [math.nextafter(c, 0) for c in cum[:-1]]
        want = [npref.sample(psi, r, prec) for r in rnds]
        got = [q.be.sample(r) for r in rnds]
        assert got == want, (probs_at, rnds, got, want)
        assert q.be.sample_many(rnds) == want
    z = engine(n, prec, np.zeros(1 << n, dtype=np.complex64 if prec == 32 else np.complex128))
    assert z.be.sample(0.5) == (1 << n) - 1 and z.be.sample_many([0.0, 0.5]) == [(1 << n) - 1] * 2
    z.ZeroAmplitudes()
    assert z.be.sample(0.5) == (1 << n) - 1 and z.be.sample_many([0.3]) == [(1 << n) - 1]


# ---------------------------------------------------------------------------------------------------------------
# elementwise kernels
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
def test_apply_m_collapse_parity_xmask(prec):
    rng = random.Random(prec)
    for n in (3, 4, 10, 16):
        psi0 = dense(np.random.default_rng(n), n, prec)
        for mask, res in ((0b101, 0b001), (1, 0), (1, 1), (((1 << n) - 1), 0b10), (1 << (n - 1) | 1, 1 << (n - 1))):
            q = engine(n, prec, psi0)
            q.be.apply_m(mask, res, 0.6 + 0.8j)
            amp_close(q.GetQuantumState(), npref.apply_m(psi0, mask, res, 0.6 + 0.8j), prec, "apply_m %x %x" % (mask, res))
        for mask in (1, 0b110, (1 << n) - 1, 1 << (n - 1)):
            for result in (0, 1):
                q = engine(n, prec, psi0)
                kept = q.be.collapse_parity(mask, bool(result))
                want, wkept = npref.collapse_parity(psi0, mask, result)
                got = q.GetQuantumState()
                amp_close(got, want, prec, "collapse_parity %x" % mask)
                assert not got[want == 0].any()
                red_close(kept, wkept, prec, "kept norm %x" % mask)
        for fusion in (0, 1):
            for mask in (1, 1 << (n - 1), 1 | (1 << (n - 1)), (1 << n) - 1, rng.getrandbits(n) | 1):
                q = engine(n, prec, psi0, fusion=fusion)
                q.be.xmask(mask)
                exact(q.GetQuantumState(), npref.xmask(psi0, mask), "xmask %x fusion %d" % (mask, fusion))


@pytest.mark.parametrize("prec", [32, 64])
def test_phase_kernels(prec):
    for n in (3, 12):
        psi0 = dense(np.random.default_rng(n), n, prec)
        full = (1 << n) - 1
        for mask in (1, 0b110, full):
            q = engine(n, prec, psi0)
            q.be.phase_parity(0.9, mask)
            amp_close(q.GetQuantumState(), npref.phase_parity(psi0, 0.9, mask), prec, "phase_parity %x" % mask)
            for cmask in (0, 1 << (n - 1), 0b1000 & full | 1):
                if cmask & mask:
                    continue
                q = engine(n, prec, psi0)
                q.be.uniform_parity_rz(cmask, mask, -0.4)
                amp_close(q.GetQuantumState(), npref.uniform_parity_rz(psi0, cmask, mask, -0.4), prec, "uprz %x %x" % (cmask, mask))
            for k in range(2, 9):
                q = engine(n, prec, psi0)
                q.be.phase_root_n_mask(k, mask)
                amp_close(q.GetQuantumState(), npref.phase_root_n_mask(psi0, k, mask), prec, "root %d %x" % (k, mask))


@pytest.mark.parametrize("prec", [32, 64])
def test_normalize_with_phase_and_threshold(prec):
    n = 12
    psi0 = dense(np.random.default_rng(5), n, prec) * 1.3
    p = np.sort(np.abs(psi0.astype(np.complex128)) ** 2)
    thresh = float(0.5 * (p[400] + p[401]))      # between two amplitudes: nothing sits on the threshold
    q = engine(n, prec, psi0)
    q.be.normalize(1.69, thresh, 0.75)
    amp_close(q.GetQuantumState(), npref.normalize(psi0, 1.69, thresh, 0.75), prec, "normalize")


@pytest.mark.parametrize("prec", [32, 64])
def test_unfused_apply2x2_paths(prec):
    """k_apply2x2 with fusion off: the fp32 float4 path (qubit 0 not involved), the scalar path, anti-controls
    (off1 != 0) and the NORM variant (floor-zeroing, norm returned)."""
    rng = random.Random(prec)
    for n in (3, 10, 15):
        psi0 = dense(np.random.default_rng(n), n, prec)
        forms = [npref.gate_form(0), npref.gate_form(n - 1), npref.gate_form(1, (0,)), npref.gate_form(0, (), (n - 1,)),
                 npref.gate_form(n - 1, (1,), (0,)), npref.gate_form(2, (), (1,))]
        for off1, off2, pm in forms:
            m = npref.round_matrix(npref.random_unitary(rng), prec)
            pows = [1 << b for b in range(n) if (pm >> b) & 1]
            q = engine(n, prec, psi0, fusion=0)
            q.be.reset_stats()
            q.be.apply2x2(off1, off2, m, pows, 1.0, 0.0, False)
            got = q.GetQuantumState()
            assert q.be.stats()["single_launches"] == 1
            amp_close(got, npref.apply2x2(psi0, off1, off2, m, pows), prec, "apply2x2 %x %x" % (off1, off2))
            # floor threshold in a wide gap between two of the touched output probabilities, about a quarter of the way up:
            # a known set of amplitudes is zeroed, and none sits near the threshold in either precision
            touched = (np.arange(1 << n) & (pm ^ off1 ^ off2)) == off1
            pt = np.sort(npref.probs(npref.apply2x2(psi0, off1, off2, m, pows, 0.9))[touched])
            i0 = int(0.25 * (pt.size - 1))
            i = max(range(i0, min(i0 + 16, pt.size - 1)), key=lambda j: pt[j + 1] / pt[j])
            thresh = float(0.5 * (pt[i] + pt[i + 1]))
            q = engine(n, prec, psi0, normalize=True)
            nrm = q.be.apply2x2(off1, off2, m, pows, 0.9, thresh, True)
            want, wnrm = npref.apply2x2(psi0, off1, off2, m, pows, 0.9, thresh)
            assert np.count_nonzero(want[touched] == 0) == i + 1
            amp_close(q.be.get_state(), want, prec, "apply2x2 NORM %x %x" % (off1, off2))
            red_close(nrm, wnrm, prec, "apply2x2 NORM norm")


# ---------------------------------------------------------------------------------------------------------------
# uniformly controlled single-qubit gates (no Python wrapper: through the C ABI)
# ---------------------------------------------------------------------------------------------------------------

def call_uc(q, controls, target, mtrxs, skips=(), skip_value=0, nrm=1.0, raw=None):
    lib = q.be.lib
    m8 = (ctypes.c_double * (8 * max(1, len(mtrxs))))()
    for k, m in enumerate(mtrxs):
        for j, z in enumerate(m):
            m8[8 * k + 2 * j], m8[8 * k + 2 * j + 1] = complex(z).real, complex(z).imag
    c = (ctypes.c_int * max(1, len(controls)))(*controls)
    s = (ctypes.c_uint64 * max(1, len(skips)))(*skips)
    args = [q.be.h, len(controls), c, target, m8, len(skips), s, skip_value, nrm]
    if raw:
        for i, v in raw.items():
            args[i] = v
    return lib.b200sv_uniformly_controlled(*args)


@pytest.mark.parametrize("prec", [32, 64])
def test_uniformly_controlled(prec):
    rng = random.Random(prec)
    n = 12
    psi0 = dense(np.random.default_rng(2), n, prec)
    cases = [((), 0, (), 0, 1.0), ((0,), 5, (), 0, 1.0), ((11,), 0, (), 0, 1.0), ((3, 9), 6, (), 0, 1.0),
             ((7, 1, 10), 4, (), 0, 0.8), ((2, 8), 11, (2,), 2, 1.0), ((0, 5, 6), 3, (1, 16), 17, 1.1), ((), 9, (1,), 1, 1.0)]
    for controls, t, skips, sv, nrm in cases:
        mt = [npref.round_matrix(npref.random_unitary(rng), prec) for _ in range(1 << (len(controls) + len(skips)))]
        q = engine(n, prec, psi0)
        assert call_uc(q, list(controls), t, mt, list(skips), sv, nrm) == _abi.B200SV_OK
        want = npref.uniformly_controlled(psi0, controls, t, mt, skips, sv, nrm)
        amp_close(q.GetQuantumState(), want, prec, "uc %r -> %d skips %r" % (controls, t, skips))


def test_uniformly_controlled_rejects_bad_arguments():
    q = engine(6, 32, dense(np.random.default_rng(1), 6, 32))
    before = q.GetQuantumState()
    one = [npref.H2]
    EINVAL = _abi.B200SV_EINVAL
    assert call_uc(q, [0] * 16, 1, one, [1 << k for k in range(15)]) == EINVAL   # 2^31 table entries
    assert call_uc(q, [0], 1, one * 4, [2], raw={1: 2 ** 31 - 1}) == EINVAL        # n_controls + n_skip overflows an int
    assert call_uc(q, [0, 2], 1, one * 4, raw={2: None}) == EINVAL                 # null controls
    assert call_uc(q, [0], 1, one * 4, [2], raw={6: None}) == EINVAL               # null skip powers
    assert call_uc(q, [0], 1, one, raw={4: None}) == EINVAL                        # null matrices
    assert call_uc(q, [0], 1, one * 4, [3]) == EINVAL                              # not a power of two
    assert call_uc(q, [0], 1, one * 4, [0]) == EINVAL                              # zero
    assert call_uc(q, [0], 1, one * 4, [4]) == EINVAL                              # outside the 4-entry table
    assert call_uc(q, [0], 1, one * 4, [2], skip_value=4) == EINVAL                # skip value outside the table
    assert call_uc(q, [0], 6, one * 2) == EINVAL                                   # target out of range
    assert call_uc(q, [6], 1, one * 2) == EINVAL                                   # control out of range
    exact(q.GetQuantumState(), before, "state after rejected calls")


# ---------------------------------------------------------------------------------------------------------------
# structure
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
def test_compose_every_start(prec):
    nrng = np.random.default_rng(prec)
    for na, nb in ((5, 3), (19, 3), (12, 1)):
        for start in sorted({0, 1, na // 2, na}):
            a, b = engine(na, prec, dense(nrng, na, prec)), engine(nb, prec, dense(nrng, nb, prec))
            pa, pb = a.GetQuantumState(), b.GetQuantumState()
            a.Compose(b, start)
            amp_close(a.GetQuantumState(), npref.compose(pa, pb, start), prec, "compose %d+%d at %d" % (na, nb, start))


@pytest.mark.parametrize("prec", [32, 64])
def test_dispose_every_perm(prec):
    n = 12
    psi0 = dense(np.random.default_rng(4), n, prec)
    for start in (0, 1, 5, n - 3):
        for length in (1, 2, 3):
            for perm in range(1 << length):
                q = engine(n, prec, psi0)
                q.Dispose(start, length, perm)
                exact(q.GetQuantumState(), npref.dispose_perm(psi0, start, length, perm), "dispose %d %d %d" % (start, length, perm))


def entangled(nrng, n, prec):
    return dense(nrng, n, prec)


def product(nrng, n, start, length, prec):
    part = dense(nrng, length, prec).astype(np.complex128)
    rest = dense(nrng, n - length, prec).astype(np.complex128)
    return npref.compose(rest, part, start).astype(np.complex64 if prec == 32 else np.complex128)


DECOMPOSE_CASES = ([(16, s, l) for l in range(1, 12) for s in sorted({0, 3, 16 - l})]          # part <= 2^11: one pass
                   + [(16, s, l) for l in (13, 14, 15) for s in sorted({0, 1, 16 - l})]      # remainder <= 2^11: one pass
                   + [(24, s, 12) for s in (0, 5, 12)] + [(25, s, 13) for s in (0, 5, 12)])  # both large: two passes


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n,start,length", DECOMPOSE_CASES)
def test_decompose_and_dispose(n, start, length, prec):
    """DecomposeDispose in its three regimes (one pass with a small part, one pass with a small remainder, marginals + two
    rebuilds), with and without a destination, on product and entangled states."""
    nrng = np.random.default_rng(n * 100 + start * 10 + length)
    states = [product(nrng, n, start, length, prec)] + ([entangled(nrng, n, prec)] if n <= 16 else [])
    for st in states:
        q = engine(n, prec, st)
        psi = q.GetQuantumState()
        rem, part = npref.decompose(psi, start, length, prec)
        d = q.Decompose(start, length)
        amp_close(q.GetQuantumState(), rem, prec, "decompose remainder")
        amp_close(d.GetQuantumState(), part, prec, "decompose part")
        q = engine(n, prec, psi)
        q.Dispose(start, length)
        amp_close(q.GetQuantumState(), rem, prec, "dispose remainder")
        del q, d


# ---------------------------------------------------------------------------------------------------------------
# page operations
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", [1, 2, 10])
def test_shuffle_buffers(n, prec):
    nrng = np.random.default_rng(n)
    a0, b0 = dense(nrng, n, prec), dense(nrng, n, prec)
    qa, qb = engine(n, prec, a0), engine(n, prec, b0)
    qa.ShuffleBuffers(qb)
    wa, wb = npref.shuffle(a0, b0)
    exact(qa.GetQuantumState(), wa, "shuffle a")
    exact(qb.GetQuantumState(), wb, "shuffle b")


@pytest.mark.parametrize("prec", [32, 64])
def test_page_get_set_copy_odd_ranges(prec):
    n = 11
    nrng = np.random.default_rng(prec)
    a0, b0 = dense(nrng, n, prec), dense(nrng, n, prec)
    qa, qb = engine(n, prec, a0), engine(n, prec, b0)
    ea = a0.copy()
    for off, ln in ((0, 1), (1, 1), (3, 7), (1023, 1), (1001, 1047), ((1 << n) - 1, 1), (5, (1 << n) - 5)):
        exact(qa.GetAmplitudePage(off, ln), ea[off:off + ln], "get %d %d" % (off, ln))
        page = dense(nrng, 11, prec)[:ln]
        qa.SetAmplitudePage(page, off)
        ea[off:off + ln] = page
        exact(qa.GetQuantumState(), ea, "set %d %d" % (off, ln))
    for src, dst, ln in ((0, 1, 1), (7, 3, 13), (1, 1000, 1), (999, 5, 1049), ((1 << n) - 1, 0, 1)):
        qa.SetAmplitudePage(qb, src, dst, ln)
        ea[dst:dst + ln] = b0[src:src + ln]
        exact(qa.GetQuantumState(), ea, "copy %d %d %d" % (src, dst, ln))
