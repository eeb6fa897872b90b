"""Float64 NumPy reference of every state-vector primitive of include/b200sv.h (test infrastructure).

Plain NumPy on complex128 / float64, written from the header's definitions and the reference lines they cite; nothing here
calls or shares code with the library or the oracle restatement.  Inputs are upcast: callers pass the state the engine
actually holds (read back in its own precision), so that what is left of a difference is the kernel's own arithmetic.
Every function returns new arrays and leaves its arguments alone.
"""
import random

import numpy as np

# REAL1_EPSILON (reference include/common/qrack_types.hpp:206,209) and FP_NORM_EPSILON (= machine epsilon / 4, :263)
REAL1_EPSILON = {32: 1.7763568394002505e-15, 64: 6.310887241768095e-30}
FP_NORM_EPSILON = {32: 2.98023223876953125e-08, 64: 5.551115123125783e-17}


def _c(psi):
    return np.array(psi, dtype=np.complex128)


def _index(n_amps):
    return np.arange(n_amps, dtype=np.int64)


def _parity(x):
    x = np.array(x, dtype=np.uint64)
    p = np.zeros(x.shape, dtype=np.uint64)
    while x.any():
        p ^= x & np.uint64(1)
        x = x >> np.uint64(1)
    return p.astype(np.int64)


def _popcount(x):
    x = np.array(x, dtype=np.uint64)
    c = np.zeros(x.shape, dtype=np.int64)
    while x.any():
        c += (x & np.uint64(1)).astype(np.int64)
        x = x >> np.uint64(1)
    return c


def round_matrix(m4, prec):
    """The matrix the engine applies: its entries rounded to the state's precision (b200sv.cu make_gate_op)."""
    dt = np.complex64 if prec == 32 else np.complex128
    return [complex(z) for z in np.array(m4, dtype=dt)]


# ---- gates ------------------------------------------------------------------------------------------------------

def apply2x2(psi, off1, off2, m4, pows, nrm=1.0, thresh=None):
    """Apply2x2 (state.cpp:392-533): for every base index i with zeros at each power in `pows`,
    (a, b) = (psi[i + off1], psi[i + off2]) -> nrm * (m0 a + m1 b, m2 a + m3 b).  With `thresh` given, amplitudes with
    |.|^2 < thresh are set to zero and (psi, sum of the others' |.|^2 over the touched amplitudes) is returned."""
    out = _c(psi)
    idx = _index(out.size)
    mask = 0
    for p in pows:
        mask |= int(p)
    base = idx[(idx & mask) == 0]
    a, b = out[base + off1], out[base + off2]
    m0, m1, m2, m3 = (complex(z) for z in m4)
    x = nrm * (m0 * a + m1 * b)
    y = nrm * (m2 * a + m3 * b)
    if thresh is None:
        out[base + off1], out[base + off2] = x, y
        return out
    px, py = np.abs(x) ** 2, np.abs(y) ** 2
    x = np.where(px < thresh, 0, x)
    y = np.where(py < thresh, 0, y)
    out[base + off1], out[base + off2] = x, y
    return out, float(px[px >= thresh].sum() + py[py >= thresh].sum())


def gate_form(target, controls=(), anti=()):
    """(off1, off2, pmask) of a single-target gate in the Apply2x2 / b200sv_apply_gates layout: controls must be 1, anti-controls 0."""
    on = 0
    for c in controls:
        on |= 1 << c
    pmask = on | (1 << target)
    for c in anti:
        pmask |= 1 << c
    return on, on | (1 << target), pmask


def apply_gates(psi, gates, prec):
    """A list of (off1, off2, pmask, m4) gates, each matrix rounded to the engine's precision first."""
    out = _c(psi)
    for off1, off2, pmask, m4 in gates:
        pows = [1 << b for b in range(int(pmask).bit_length()) if (pmask >> b) & 1]
        out = apply2x2(out, off1, off2, round_matrix(m4, prec), pows)
    return out


def apply_m(psi, mask, result, nrm):
    """ApplyM (state.cpp:2167-2196): psi[i] = ((i & mask) == result) ? nrm * psi[i] : 0"""
    psi = _c(psi)
    keep = (_index(psi.size) & mask) == result
    return np.where(keep, complex(nrm) * psi, 0)


def collapse_parity(psi, mask, result):
    """ForceMParity's collapse (state.cpp:2083-2091): keep the amplitudes whose parity of (i & mask) is `result`, zero the
    rest.  Returns (psi, kept norm)."""
    psi = _c(psi)
    keep = _parity(_index(psi.size) & mask) == int(result)
    out = np.where(keep, psi, 0)
    return out, float((np.abs(out) ** 2).sum())


def xmask(psi, mask):
    """XMask (state.cpp:965-1007): X on every qubit of mask, psi'[i] = psi[i ^ mask]"""
    psi = _c(psi)
    return psi[_index(psi.size) ^ mask]


def phase_parity(psi, radians, mask):
    """PhaseParity (state.cpp:1009-1054): odd parity of (i & mask) gets e^{i r/2}, even parity e^{-i r/2}"""
    psi = _c(psi)
    odd = _parity(_index(psi.size) & mask) == 1
    return psi * np.where(odd, np.exp(0.5j * radians), np.exp(-0.5j * radians))


def uniform_parity_rz(psi, cmask, mask, angle):
    """UniformParityRZ / CUniformParityRZ (state.cpp:1200-1264): where every control bit is set, odd parity of (i & mask)
    gets e^{i angle}, even parity e^{-i angle}; the rest is untouched"""
    psi = _c(psi)
    idx = _index(psi.size)
    odd = _parity(idx & mask) == 1
    f = np.where(odd, np.exp(1j * angle), np.exp(-1j * angle))
    return np.where((idx & cmask) == cmask, psi * f, psi)


def phase_root_n_mask(psi, n, mask):
    """PhaseRootNMask (state.cpp:1056-1092): psi[i] *= e^{i k theta}, k = popcount(i & mask) mod 2^n, theta = -pi / 2^(n-1).
    The sign is the reference's (DESIGN.md section 4)."""
    psi = _c(psi)
    k = _popcount(_index(psi.size) & mask) % (1 << n)
    return psi * np.exp(1j * k * (-np.pi / (1 << (n - 1))))


def uniformly_controlled(psi, controls, target, mtrxs, skip_powers=(), skip_value_mask=0, nrm=1.0):
    """UniformlyControlledSingleBit (state.cpp:1094-1198): the control bits of each pair's base index, in `controls` order,
    form an index; a zero bit is inserted at each skip power, in the order the caller gives them (state.cpp:1135), and
    skip_value_mask is ORed in; that entry of `mtrxs` (rows of 4 complex) is applied to the pair, times nrm."""
    psi = _c(psi)
    mt = np.array(mtrxs, dtype=np.complex128).reshape(-1, 4)
    idx = _index(psi.size)
    tpow = 1 << target
    base = idx[(idx & tpow) == 0]
    off = np.zeros(base.shape, dtype=np.int64)
    for j, c in enumerate(controls):
        off |= ((base >> c) & 1) << j
    sel = np.zeros(base.shape, dtype=np.int64)
    hi = off
    for p in skip_powers:
        low = hi & (p - 1)
        sel |= low
        hi = (hi ^ low) << 1
    sel = (sel | hi) | skip_value_mask
    m = mt[sel]
    a, b = psi[base], psi[base | tpow]
    out = psi.copy()
    out[base] = nrm * (m[:, 0] * a + m[:, 1] * b)
    out[base | tpow] = nrm * (m[:, 2] * a + m[:, 3] * b)
    return out


def normalize(psi, nrm, thresh, phase):
    """NormalizeState (state.cpp:2198-2248): amplitudes with |.|^2 < thresh (thresh > 0) become 0, then every amplitude is
    multiplied by e^{i phase} / sqrt(nrm)"""
    psi = _c(psi)
    if thresh > 0:
        psi = np.where(np.abs(psi) ** 2 < thresh, 0, psi)
    return psi * (np.exp(1j * phase) / np.sqrt(nrm))


# ---- reductions -------------------------------------------------------------------------------------------------

def probs(psi):
    """|psi|^2 as re^2 + im^2: exact for dyadic amplitudes (np.abs goes through a square root and is not)"""
    psi = _c(psi)
    return psi.real ** 2 + psi.imag ** 2


def prob_mask(psi, mask, perm):
    """sum of |psi[i]|^2 over i with (i & mask) == perm (Prob / ProbReg / ProbMask, state.cpp:1751-1947)"""
    p = probs(psi)
    return float(p[(_index(p.size) & mask) == perm].sum())


def prob_parity(psi, mask):
    """ProbParity (state.cpp:1949-1993): probability of odd parity of (i & mask)"""
    p = probs(psi)
    return float(p[_parity(_index(p.size) & mask) == 1].sum())


def prob_mask_all(psi, mask):
    """ProbMaskAll (qinterface.cpp:423-476): entry k, whose bit j is the j-th lowest bit of mask"""
    p = probs(psi)
    idx = _index(p.size)
    bits = [b for b in range(int(mask).bit_length()) if (mask >> b) & 1]
    key = np.zeros(p.size, dtype=np.int64)
    for j, b in enumerate(bits):
        key |= ((idx >> b) & 1) << j
    return np.bincount(key, weights=p, minlength=1 << len(bits))


def marginals(psi):
    """Prob(q) for every qubit q"""
    p = probs(psi)
    n = p.size.bit_length() - 1
    return np.array([p.reshape(-1, 2, 1 << q)[:, 1, :].sum() for q in range(n)])


def norm(psi, thresh):
    """sum of the |psi|^2 that are >= thresh (UpdateRunningNorm / par_norm, parallel_for.cpp:244-300)"""
    p = probs(psi)
    return float(p[p >= thresh].sum())


def inner(a, b):
    """<a|b> = sum conj(a) b (SumSqrDiff, state.cpp:2109-2165)"""
    return complex(np.vdot(_c(a), _c(b)))


def expectation(psi, start, length):
    """sum of |psi[i]|^2 ((i >> start) & (2^length - 1)) (GetExpectation)"""
    p = probs(psi)
    return float((p * ((_index(p.size) >> start) & ((1 << length) - 1))).sum())


def highest_prob(psi):
    """index of the largest |psi|^2, the lowest one on ties (HighestProbAll, state.cpp:1995-2024)"""
    return int(np.argmax(probs(psi)))


def sample(psi, rnd, prec):
    """MAll's search (state.cpp:2026-2050) on the given probabilities: the first index whose |psi|^2 > REAL1_EPSILON and whose
    cumulative probability exceeds rnd or comes within FP_NORM_EPSILON of 1; else the last such index; else 2^n - 1."""
    p = probs(psi)
    nz = np.flatnonzero(p > REAL1_EPSILON[prec])
    if not nz.size:
        return p.size - 1
    cum = np.cumsum(p[nz])
    hit = np.flatnonzero((cum > rnd) | ((1.0 - cum) <= FP_NORM_EPSILON[prec]))
    return int(nz[hit[0]]) if hit.size else int(nz[-1])


# ---- structure --------------------------------------------------------------------------------------------------

def compose(a, b, start):
    """Compose (state.cpp:1368-1459): b's qubits inserted at `start` of a's, amplitude = a[rest] * b[middle]"""
    a, b = _c(a), _c(b)
    na, nb = a.size.bit_length() - 1, b.size.bit_length() - 1
    lo = a.reshape(1 << (na - start), 1 << start)
    out = lo[:, None, :] * b[None, :, None]
    return out.reshape(1 << (na + nb))


def _split(psi, start, length):
    """view as [high, part, low]: index = (high << (start + length)) | (part << start) | low"""
    psi = _c(psi)
    n = psi.size.bit_length() - 1
    return psi.reshape(1 << (n - start - length), 1 << length, 1 << start)


def decompose(psi, start, length, prec):
    """DecomposeDispose (state.cpp:1551-1696): qubits [start, start + length) leave.  Each factor keeps the marginal
    probabilities of its basis states and, as phase, their probability-weighted mean angle (angles of |amp|^2 <= REAL1_EPSILON
    left out; a mean over total probability <= REAL1_EPSILON stays 0).  Returns (remainder, part)."""
    v = _split(psi, start, length)
    p = np.abs(v) ** 2
    floor = REAL1_EPSILON[prec]
    wang = np.where(p > floor, np.angle(v) * p, 0.0)
    rem_p, part_p = p.sum(axis=1), p.sum(axis=(0, 2))
    rem_a, part_a = wang.sum(axis=1), wang.sum(axis=(0, 2))
    rem_a = np.where(rem_p > floor, rem_a / np.where(rem_p > floor, rem_p, 1), rem_a)
    part_a = np.where(part_p > floor, part_a / np.where(part_p > floor, part_p, 1), part_a)
    rem = (np.sqrt(rem_p) * np.exp(1j * rem_a)).reshape(-1)
    part = np.sqrt(part_p) * np.exp(1j * part_a)
    return rem, part


def dispose_perm(psi, start, length, perm):
    """Dispose(start, length, perm) (state.cpp:1708-1748): the slice where the disposed bits equal perm"""
    return _split(psi, start, length)[:, perm, :].reshape(-1).copy()


def shuffle(a, b):
    """ShuffleBuffers (state.cpp:134-163): swap a's upper half with b's lower half"""
    a, b = _c(a), _c(b)
    h = a.size >> 1
    return np.concatenate([a[:h], b[:h]]), np.concatenate([a[h:], b[h:]])


# ---- QAlu family: basis-index maps (reference src/qengine/arithmetic.cpp) -----------------------------------------
#
# Each function evaluates the reference method's index map over all 2^n indices as uint64 arrays.  The forward forms write
# out[f(i)] = +-in[i], the inverse forms out[i] = in[f(i)], each for the sources i of the method's loop domain: par_for over
# every index, par_for_skip(skipPower, width) over the indices whose `width` bits from skipPower up are zero (bits above the
# top qubit do not exist: parallel_for.cpp:98-100), par_for_mask over the indices with every listed bit zero
# (parallel_for.cpp:118-149).  The destination vector starts zeroed (nStateVec->clear()), so whatever no source writes stays 0.
# A forward map must be injective on its domain, or the result would depend on write order: _move asserts it.
# Arguments are those of include/b200sv.h; the pre-steps the header leaves to the adapter (SetReg, M/X of the carry) are not
# modelled, and the argument checks are the header's, tested separately.

_U1 = np.uint64(1)


def _u(x):
    return np.uint64(int(x) & 0xFFFFFFFFFFFFFFFF)


def _ui(n_amps):
    return np.arange(n_amps, dtype=np.uint64)


def _bits(lo, width):
    """bitRegMaskOcl(lo, width): `width` ones from bit lo up"""
    return _u(((1 << width) - 1) << lo)


def _move(psi, dst, src, sign=None, base=None):
    """out[dst] = sign * psi[src] over the domain, on top of `base` (zeros: nStateVec->clear())"""
    psi = _c(psi)
    dst, src = np.asarray(dst, dtype=np.uint64), np.asarray(src, dtype=np.uint64)
    assert int(dst.max(initial=0)) < psi.size and int(src.max(initial=0)) < psi.size
    hit = np.zeros(psi.size, dtype=bool)
    hit[dst] = True
    assert int(np.count_nonzero(hit)) == dst.size, "the index map is not injective on its domain"
    out = np.zeros_like(psi) if base is None else base
    v = psi[src]
    out[dst] = v if sign is None else sign * v
    return out


def _skip_domain(idx, skip_power_bit, width):
    """par_for_skip(0, 2^n, 2^skip_power_bit, width) (parallel_for.cpp:86-116): indices whose bits
    [skip_power_bit, skip_power_bit + width) are zero; bits above the top qubit do not exist"""
    return idx[(idx & _bits(skip_power_bit, width)) == 0]


def _mask_domain(idx, mask):
    """par_for_mask over the powers of `mask` (parallel_for.cpp:118-149): indices with every bit of mask zero"""
    return idx[(idx & _u(mask)) == 0]


def _proper_subsets(mask):
    """every sub-mask of `mask` but mask itself (CMULDIV :537-547, CModNOut :721-731 copy these patterns unchanged)"""
    bits = [1 << b for b in range(int(mask).bit_length()) if (int(mask) >> b) & 1]
    return [sum(b for j, b in enumerate(bits) if (s >> j) & 1) for s in range((1 << len(bits)) - 1)]


def _overflow_add(a, b, length):
    """isOverflowAdd (functions.cpp:214-233) = two's-complement overflow of a length-bit addition: a and b read as signed
    length-bit integers, the sum leaves [-2^(length-1), 2^(length-1))"""
    half = 1 << (length - 1)
    sa = a.astype(np.int64) - np.where(a >= half, 1 << length, 0)
    sb = int(b) - ((1 << length) if int(b) >= half else 0)
    s = sa + sb
    return (s < -half) | (s >= half)


def table_values(values, length):
    """entries of a classical table: (length + 7) / 8 bytes each, little-endian (the reference reads 1-, 2- and 4-byte
    entries through uint8 / uint16 / uint32 pointers on a little-endian host and assembles other widths byte by byte, low
    byte first: arithmetic.cpp:1045-1071, 1220-1231, 1401-1411, 1489-1499)"""
    nb = (length + 7) >> 3
    raw = np.frombuffer(bytes(values), dtype=np.uint8).reshape(-1, nb).astype(np.uint64)
    v = np.zeros(raw.shape[0], dtype=np.uint64)
    for j in range(nb):
        v |= raw[:, j] << np.uint64(8 * j)
    return v


def rol(psi, shift, start, length):
    """ROL (arithmetic.cpp:23-69): length 0 or shift % length == 0 is a no-op; else the register rotates left by
    shift % length, every index moves (par_for)"""
    psi = _c(psi)
    if not length or not shift % length:
        return psi
    shift %= length
    idx = _ui(psi.size)
    lm, rm = _u((1 << length) - 1), _bits(start, length)
    reg = (idx & rm) >> _u(start)
    o = (reg >> _u(length - shift)) | ((reg << _u(shift)) & lm)
    return _move(psi, (o << _u(start)) | (idx & ~rm), idx)


def inc(psi, to_add, start, length, ctrl_mask=0):
    """INC (:73-118) and CINC (:121-172): reg += to_add mod 2^length (to_add masked to length; 0 is a no-op).  CINC starts
    from a copy of the state (:162) and moves only the indices with every control set (par_for_mask, :164-169)."""
    psi = _c(psi)
    to_add = int(to_add) & ((1 << length) - 1)
    if not length or not to_add:
        return psi
    idx = _ui(psi.size)
    src = idx[(idx & _u(ctrl_mask)) == _u(ctrl_mask)]
    rm = _bits(start, length)
    o = (((src & rm) >> _u(start)) + _u(to_add)) & _u((1 << length) - 1)
    return _move(psi, (o << _u(start)) | (src & ~rm), src, base=psi.copy())


def _add_with_carry(src, to_mod, start, length, carry_mask):
    """outRes of INCDECC / INCDECSC (:211-214, :350-353, :408-411): reg + to_mod, the carry qubit set where it reaches 2^length"""
    rm = _bits(start, length)
    o = ((src & rm) >> _u(start)) + _u(to_mod)
    wrap = o >= _u(1 << length)
    o = np.where(wrap, o - _u(1 << length), o)
    return (o << _u(start)) | (src & ~(rm | _u(carry_mask))) | np.where(wrap, _u(carry_mask), _u(0))


def incdecc(psi, to_mod, start, length, carry_index):
    """INCDECC (:175-218): to_mod masked to length (0 is a no-op); sources with the carry qubit clear (par_for_skip, :208)"""
    psi = _c(psi)
    to_mod = int(to_mod) & ((1 << length) - 1)
    if not length or not to_mod:
        return psi
    src = _skip_domain(_ui(psi.size), carry_index, 1)
    return _move(psi, _add_with_carry(src, to_mod, start, length, 1 << carry_index), src)


def incs(psi, to_add, start, length, overflow_index):
    """INCS (:227-310): reg += to_add mod 2^length over every index; the amplitude changes sign where the signed addition
    overflows AND the overflow qubit is set in the RESULT index (:297-304)"""
    psi = _c(psi)
    to_add = int(to_add) & ((1 << length) - 1)
    if not length or not to_add:
        return psi
    idx = _ui(psi.size)
    rm = _bits(start, length)
    reg = (idx & rm) >> _u(start)
    dst = (((reg + _u(to_add)) & _u((1 << length) - 1)) << _u(start)) | (idx & ~rm)
    ovf = _u(1 << overflow_index)
    flip = _overflow_add(reg, to_add, length) & ((dst & ovf) == ovf)
    return _move(psi, dst, idx, np.where(flip, -1.0, 1.0))


def incdecsc(psi, to_mod, start, length, overflow_index, carry_index):
    """INCDECSC: overflow_index < 0 is the carry-only form (:312-362), where the sign flips wherever the signed addition
    overflows; otherwise (:364-420) only where the overflow qubit is also set in the RESULT index (:413).  to_mod masked to
    length (0 is a no-op); sources with the carry qubit clear (par_for_skip, :346 / :404)."""
    psi = _c(psi)
    to_mod = int(to_mod) & ((1 << length) - 1)
    if not length or not to_mod:
        return psi
    src = _skip_domain(_ui(psi.size), carry_index, 1)
    dst = _add_with_carry(src, to_mod, start, length, 1 << carry_index)
    flip = _overflow_add((src & _bits(start, length)) >> _u(start), to_mod, length)
    if overflow_index >= 0:
        ovf = _u(1 << overflow_index)
        flip &= (dst & ovf) == ovf
    return _move(psi, dst, src, np.where(flip, -1.0, 1.0))


def muldiv(psi, inverse, to_mul, start, carry_start, length, ctrl_mask=0):
    """MULDIV (:422-456) and CMULDIV (:488-551): reg * to_mul (64-bit wrap) split into the low `length` bits (back into the
    register) and the next `length` bits (into the carry register).  inverse = 0 (MUL) writes out[mulRes] = in[orig],
    inverse = 1 (DIV) out[orig] = in[mulRes].  Sources: carry register zero (par_for_skip, :447).  With controls the domain
    also has every control clear (par_for_mask, :529): orig and mulRes get every control set (:532-534), and each other
    control pattern of the source index is copied unchanged (:537-547) — so where the controls are not all set, only
    indices whose carry register reads zero survive; the rest becomes 0.  The forward form is injective only for
    0 < to_mul < 2^length."""
    psi = _c(psi)
    low = (1 << length) - 1
    io, cr = _bits(start, length), _bits(carry_start, length)
    other = _u(psi.size - 1) ^ (io | cr | _u(ctrl_mask))
    src = _mask_domain(_ui(psi.size), int(cr) | int(ctrl_mask))
    m = ((src & io) >> _u(start)) * _u(to_mul)
    mul = ((m & _u(low)) << _u(start)) | (((m >> _u(length)) & _u(low)) << _u(carry_start)) | (src & other) | _u(ctrl_mask)
    orig = src | _u(ctrl_mask)
    dst, frm = (orig, mul) if inverse else (mul, orig)
    for part in _proper_subsets(ctrl_mask):
        dst = np.concatenate([dst, src | _u(part)])
        frm = np.concatenate([frm, src | _u(part)])
    return _move(psi, dst, frm)


def modnout(psi, kind, to_mod, mod_n, in_start, out_start, length, ctrl_mask=0):
    """ModNOut (:595-632) and CModNOut (:670-735); kind 0 MULModNOut (in * to_mod, :634-645), 1 IMULModNOut (the same
    map, inverse direction: out[lcv] = in[map], :647-656), 2 POWModNOut (to_mod ^ in with 64-bit wrap, intPowOcl,
    functions.cpp:77-95, :658-668).  outRes = (k % mod_n) << out_start.  Sources: output register zero (par_for_skip, :620);
    uncontrolled, the "other" bits exclude modMask << out_start, modMask sized from mod_n (:611-613).  Controlled: the
    domain also has every control clear (par_for_mask, :711), every control is set in both indices (:717-719) and each
    other control pattern of the source index is copied unchanged (:721-731): where the controls are not all set, only
    indices whose output register reads zero survive, the rest becomes 0."""
    psi = _c(psi)
    low = (1 << length) - 1
    im = _bits(in_start, length)
    src = _mask_domain(_ui(psi.size), (low << out_start) | int(ctrl_mask))
    x = (src & im) >> _u(in_start)
    if kind == 2:
        tab = np.array([pow(int(to_mod), v, 1 << 64) for v in range(1 << length)], dtype=np.uint64)
        k = tab[x.astype(np.int64)]
    else:
        k = x * _u(to_mod)
    out_res = (k % _u(mod_n)) << _u(out_start)
    if ctrl_mask:
        out_mask = _u(low << out_start)
    else:
        mn = int(mod_n)
        out_mask = _u(((mn if not (mn & (mn - 1)) else 1 << mn.bit_length()) - 1) << out_start)
    other = _u(psi.size - 1) ^ (im | out_mask | _u(ctrl_mask))
    mapped = (src & im) | out_res | (src & other) | _u(ctrl_mask)
    orig = src | _u(ctrl_mask)
    dst, frm = (orig, mapped) if kind == 1 else (mapped, orig)
    for part in _proper_subsets(ctrl_mask):
        dst = np.concatenate([dst, src | _u(part)])
        frm = np.concatenate([frm, src | _u(part)])
    return _move(psi, dst, frm)


def indexed(psi, kind, index_start, index_length, value_start, value_length, carry_index, carry_in, values):
    """IndexedLDA (kind 0, :983-1083), IndexedADC (1, :1086-1260), IndexedSBC (2, :1263-1444), dense branches.  v = the table
    entry the index register selects (table_values).  `carry_in` is the number the formula adds, as the header passes it:
    the reference derives it from measuring the carry qubit, 1 for a set carry in ADC (:1115-1120) but INVERTED in SBC,
    1 for a clear one (:1293-1298).
      LDA: sources with a zero value register (par_for_skip(valueStart, valueLength), :1073), out[lcv | v << value_start].
      ADC: sources with the carry clear (par_for_skip(carry, 1), :1248); value register := v + value + carry_in, the carry
           qubit set where that reaches 2^value_length (:1232-1246).
      SBC: sources with value_length bits from the carry qubit upward clear (par_for_skip(carry, valueLength), :1432) —
           a window that also covers other qubits unless the carry is the top one; value register :=
           value + 2^value_length - (v + carry_in), carry set where that reaches 2^value_length (:1412-1430)."""
    psi = _c(psi)
    vals = table_values(values, value_length)
    idx = _ui(psi.size)
    im, vm = _bits(index_start, index_length), _bits(value_start, value_length)
    if kind == 0:
        src = _skip_domain(idx, value_start, value_length)
        v = vals[((src & im) >> _u(index_start)).astype(np.int64)]
        return _move(psi, src | (v << _u(value_start)), src)
    cmask = _u(1 << carry_index)
    src = _skip_domain(idx, carry_index, 1 if kind == 1 else value_length)
    v = vals[((src & im) >> _u(index_start)).astype(np.int64)]
    cur = (src & vm) >> _u(value_start)
    vp = _u(1 << value_length)
    o = (v + cur + _u(carry_in)) if kind == 1 else (cur + (vp - (v + _u(carry_in))))
    wrap = o >= vp
    o = np.where(wrap, o - vp, o)
    other = _u(psi.size - 1) & ~(im | vm | cmask)
    dst = (o << _u(value_start)) | (src & im) | (src & other) | np.where(wrap, cmask, _u(0))
    return _move(psi, dst, src)


def hash(psi, start, length, values):
    """Hash (:1447-1506): the register's value is replaced by its table entry, every index moves (par_for); injective only
    when the table is a permutation of the register's values"""
    psi = _c(psi)
    vals = table_values(values, length)
    idx = _ui(psi.size)
    rm = _bits(start, length)
    v = vals[((idx & rm) >> _u(start)).astype(np.int64)]
    return _move(psi, (v << _u(start)) | (idx & ~rm), idx)


def phase_flip_if_less(psi, greater_perm, start, length, flag_index):
    """PhaseFlipIfLess (flag_index < 0, :1703-1720) / CPhaseFlipIfLess (:1678-1701): psi[i] = -psi[i] where the register
    value is below greater_perm (and the flag qubit is set)"""
    psi = _c(psi)
    idx = _ui(psi.size)
    hit = ((idx & _bits(start, length)) >> _u(start)) < _u(greater_perm)
    if flag_index >= 0:
        hit &= (idx & _u(1 << flag_index)) != 0
    return np.where(hit, -psi, psi)


# ---- re-page ------------------------------------------------------------------------------------------------------

def exchange(pages, k, victim_bits, rank):
    """This rank's page after the re-page of b200sv_exchange_scatter / b200sv_exchange_pull (include/b200sv.h): the 2^k
    ranks' old pages in rank order; element i comes from the rank whose index bit b is bit victim_bits[b] of i, at index i
    with those bits replaced by this rank's bits.  Returned in the pages' own dtype (a pure selection)."""
    nl = pages[0].size.bit_length() - 1
    idx = _ui(1 << nl)
    src_rank = np.zeros(idx.size, dtype=np.int64)
    vmask = dep = 0
    for b in range(k):
        src_rank |= ((idx >> _u(victim_bits[b])) & _U1).astype(np.int64) << b
        vmask |= 1 << victim_bits[b]
        if (rank >> b) & 1:
            dep |= 1 << victim_bits[b]
    src_idx = ((idx & ~_u(vmask)) | _u(dep)).astype(np.int64)
    want = np.empty(idx.size, dtype=pages[0].dtype)
    for r in range(len(pages)):
        sel = src_rank == r
        want[sel] = pages[r][src_idx[sel]]
    return want


# ---- gate lists of the fused-sweep tests ------------------------------------------------------------------------

def random_unitary(rng):
    th, ph, la = (rng.uniform(-np.pi, np.pi) for _ in range(3))
    c, s = np.cos(th / 2), np.sin(th / 2)
    return [c, -s * np.exp(1j * la), s * np.exp(1j * ph), c * np.exp(1j * (ph + la))]


H2 = [2 ** -0.5, 2 ** -0.5, 2 ** -0.5, -(2 ** -0.5)]
X2 = [0, 1, 1, 0]
SQRTX = [0.5 + 0.5j, 0.5 - 0.5j, 0.5 - 0.5j, 0.5 + 0.5j]


def gate_family(family, n, rng):
    """Gates (off1, off2, pmask, m4) of one family on n qubits; every qubit is a target and a control at least once.
      light:    H, T, S, CZ, CNOT, CCNOT and anti-controlled phases (Hadamard stages, phase and swap ops)
      rotation: an uncontrolled random U on every qubit, twice, with a CZ ring between (rotation stages)
      full:     controlled and anti-controlled random unitaries, X with mixed control polarities (general-matrix ops)"""
    g = []

    def add(m4, t, controls=(), anti=()):
        g.append(gate_form(t, controls, anti) + (list(m4),))

    def other(q, *avoid):
        while True:
            c = rng.randrange(n)
            if c != q and c not in avoid:
                return c

    if family == "light":
        for t in range(n):
            add(H2, t)
        for t in range(n):
            add([1, 0, 0, np.exp(0.25j * np.pi)], t)                      # T
            add(X2, t, (other(t),))                                      # CNOT onto t
            add([1, 0, 0, -1], other(t), (t,))                           # CZ controlled by t
            c1 = other(t)
            add(X2, t, (c1, other(t, c1)))                               # CCNOT
            add([1, 0, 0, 1j], t)                                        # S
            add([1, 0, 0, np.exp(1j * rng.uniform(-3, 3))], t, (), (other(t),))   # anti-controlled phase
            add(H2, t)
    elif family == "rotation":
        for t in range(n):
            add(random_unitary(rng), t)
        for t in range(n):
            add([1, 0, 0, -1], (t + 1) % n, (t,))
        for t in range(n):
            add(random_unitary(rng), t)
    elif family == "full":
        for t in range(n):
            add(random_unitary(rng), t)
        add(random_unitary(rng), 0, (n - 1,))                            # controlled from the top qubit (outer above a tile)
        for t in range(n):
            c1 = other(t)
            if t % 3 == 0:                                               # SqrtX twice is exactly X: left as an X swap
                add(SQRTX, t)
                add(SQRTX, t)
            add(random_unitary(rng), t, (c1,))                           # controlled U
            add(random_unitary(rng), t, (), (other(t),))                 # anti-controlled U
            a1 = other(t, c1)
            add(X2, t, (c1,), (a1,))                                     # X, one control of each polarity
            add(random_unitary(rng), other(t), (t,))                     # t as a control
    else:
        raise ValueError(family)
    return g


def pull_gate_lists(family, n, prec):
    """Two fixed gate lists of one family for the sweep that carries a pull re-page: (staged, direct).  `staged` opens with
    a controlled random unitary on each qubit at 16-byte-chunk bits 0..2 (qubits 1..3 for fp32, whose chunk holds 2
    amplitudes, 0..2 for fp64; general ops, whose targets are register bits), then the family on all n qubits: the first
    pass has several register bits on those chunk bits, so the sweep copies its tiles into shared memory first.  `direct`
    is the family on the qubits above chunk bit 2 only, so the first pass loads its sub-blocks straight from the source
    pages.  test_npref_pin.py checks both choices on the planner's listing."""
    rng = random.Random("pull-%s-%d-%d" % (family, n, prec))
    low = 4 if prec == 32 else 3
    staged = [gate_form(q, (n - 1 - j,)) + (random_unitary(rng),) for j, q in enumerate(range(low - 3, low))]
    staged += gate_family(family, n, rng)
    direct = [(o1 << low, o2 << low, pm << low, m4) for o1, o2, pm, m4 in gate_family(family, n - low, rng)]
    return staged, direct


# ---- QAlu call grids of the QAlu tests ----------------------------------------------------------------------------

def _table(rng, n_entries, length):
    """a classical table of (length + 7) / 8-byte little-endian entries that holds 0 and 2^length - 1"""
    nb = (length + 7) >> 3
    v = [rng.randrange(1 << length) for _ in range(n_entries)]
    v[0] = 0
    v[-1] = (1 << length) - 1
    return b"".join(x.to_bytes(nb, "little") for x in v)


def _perm_table(rng, length):
    """a Hash table that is a permutation of the register's values (Hash is injective only then)"""
    v = list(range(1 << length))
    rng.shuffle(v)
    return b"".join(x.to_bytes((length + 7) >> 3, "little") for x in v)


def _indexed_cases(rng, n, shapes, few=False):
    """IndexedLDA / ADC / SBC calls for each (value_length, index_length) of `shapes` that fits n qubits, with carry_in 0 and
    1 and the carry both the top qubit and below it (where SBC's skip window covers more than the carry); `few`: one LDA,
    one ADC and one SBC per shape"""
    out = []
    for vl, il in shapes:
        if il < 0 or il + vl + 1 > n:
            continue
        tab = _table(rng, 1 << il, vl)
        out.append(("indexed", (0, 0, il, il, vl, 0, 0, tab)))                      # LDA: index low, value above
        if few:
            out.append(("indexed", (1, 0, il, il, vl, n - 1, 1, tab)))              # ADC, carry = the top qubit
            out.append(("indexed", (2, 1, il, 1 + il, vl, 0, 0, tab)))             # SBC, carry = qubit 0: the window covers both registers
            continue
        out.append(("indexed", (0, n - il, il, 0, vl, 0, 0, tab)))                  # LDA: index on the top qubits
        for kind in (1, 2):
            for cin in (0, 1):
                out.append(("indexed", (kind, 0, il, il, vl, n - 1, cin, tab)))     # carry = the top qubit
            out.append(("indexed", (kind, 0, il, il, vl, il + vl, 1, tab)))         # carry right above the value register
            out.append(("indexed", (kind, 1, il, 1 + il, vl, 0, 0, tab)))          # carry = qubit 0, below both registers
    return out


def alu_grid(n, seed=0):
    """(name, args) QAlu calls at the edges of the index maps on an n-qubit (6 <= n) register: name is the npref function
    and, prefixed with alu_, the backend method.  Every forward map here is injective on its domain."""
    rng = random.Random(1000 * n + seed)
    g = []
    # ROL: length 1, 2 and the whole register; shift 0, 1, length - 1 and >= length; at the bottom and the top
    for L in (1, 2, n):
        for shift in sorted({0, 1, L - 1, L, L + 1, 2 * L + 1}):
            for start in sorted({0, n - L}):
                g.append(("rol", (shift, start, L)))
    # INC / CINC: register at qubits 2..4; to_add 0, 1, 2^L - 1 and >= 2^L; controls below, above, at 0 and at n - 1
    s, L = 2, 3
    for to_add in (0, 1, (1 << L) - 1, (1 << L) + 5, (1 << 40) + 3):
        for cm in (0, 1 << 1, 1 << (s + L), 1, 1 << (n - 1), (1 << 0) | (1 << (n - 1))):
            g.append(("inc", (to_add, s, L, cm)))
    g.append(("inc", (5, 0, n, 0)))                                                # the whole register
    g.append(("inc", (3, n - 2, 2, 1)))                                            # register on the top qubits
    # INCDECC / INCS / INCDECSC: length 1 (sign mask 1) and 3; to_add 1, 2^(L-1), 2^L - 1; carry and flag below and above
    for L in (1, 3):
        s = 2
        below, above = (0, 1), (s + L, n - 1)
        for to_add in sorted({1, 1 << (L - 1), (1 << L) - 1}):
            for c in (below[0], above[0]):
                g.append(("incdecc", (to_add, s, L, c)))
                g.append(("incdecsc", (to_add, s, L, -1, c)))
            for o in (below[1], above[1]):
                g.append(("incs", (to_add, s, L, o)))
            for o, c in ((below[1], above[0]), (above[1], below[0]), (below[1], below[0]), (above[1], above[0])):
                g.append(("incdecsc", (to_add, s, L, o, c)))
    g.append(("incdecc", (3, n - 3, 3, 0)))                                        # register on the top qubits
    g.append(("incs", (3, n - 3, 3, n - 1)))                                       # overflow flag inside the register
    # MUL / DIV: the forward form is injective only for 0 < to_mul < 2^L (to_mul = 0 and wrapping products collide), so the
    # grid stays inside that; carry register below the input register and not adjacent to it, or right above it
    for L in (1, 2, 3):
        if 2 * L + 2 > n:
            continue
        for to_mul in sorted({1, 2, 6, (1 << L) - 1} & set(range(1, 1 << L))):
            for inv in (0, 1):
                g.append(("muldiv", (inv, to_mul, L + 1, 0, L, 0)))                # carry at 0, one qubit gap
                g.append(("muldiv", (inv, to_mul, 0, L, L, 0)))                    # carry right above
                g.append(("muldiv", (inv, to_mul, L + 1, 0, L, 1 << (n - 1))))     # controlled from the top qubit
                g.append(("muldiv", (inv, to_mul, 0, L, L, (1 << (2 * L)) | (1 << (n - 1)))))
    # ModNOut, kinds 0..2: mod_n 1, 3, 2^L - 1, 2^L; POWModNOut with base 0 and 1; output below and above the input
    L = 3 if n >= 7 else 2
    for kind in (0, 1, 2):
        for mod_n in (1, 3, (1 << L) - 1, 1 << L):
            for to_mod in ((5, 0, 1) if kind == 2 else (5,)):
                g.append(("modnout", (kind, to_mod, mod_n, L, 0, L, 0)))           # output below the input
                g.append(("modnout", (kind, to_mod, mod_n, 0, L, L, 0)))           # output above
                g.append(("modnout", (kind, to_mod, mod_n, L, 0, L, 1 << (n - 1))))
                g.append(("modnout", (kind, to_mod, mod_n, 0, L, L, (1 << (2 * L)) | (1 << (n - 1)))))
    # Indexed LDA / ADC / SBC: 1- and 2-byte entries; index_length 0 and 1 (the wide shapes are in alu_wide)
    g += _indexed_cases(rng, n, [(vl, il) for vl in (1, 3, 8, 9) for il in (0, 1, 2)])
    # Hash: 1- and 2-byte entries
    for L in (3, 9, 10, 11, 12):
        if L <= n:
            g.append(("hash", (n - L, L, _perm_table(rng, L))))
    # PhaseFlipIfLess: greater_perm 0, 1, inside, 2^L and above; flag none, below and above the register
    s, L = 2, 3
    for gp in (0, 1, 5, 1 << L, (1 << L) + 3, 1 << 63):
        for flag in (-1, 0, n - 1):
            g.append(("phase_flip_if_less", (gp, s, L, flag)))
    g.append(("phase_flip_if_less", (7, 0, n, -1)))
    return g


def alu_wide(n, seed=0):
    """one call per QAlu map with registers as wide as n qubits allow (the grid-stride loop runs from 20 qubits up), plus
    the indexed shapes with 2- and 3-byte entries and 10 index bits"""
    rng = random.Random(7 * n + seed)
    h = n // 2 - 1
    g = [("rol", (n - 3, 0, n)),
         ("inc", ((1 << n) - 7, 0, n, 0)),
         ("inc", (12345, 1, n - 2, (1 << 0) | (1 << (n - 1)))),
         ("incdecc", ((1 << (n - 2)) + 3, 1, n - 1, 0)),
         ("incs", ((1 << (n - 2)) + 3, 0, n - 1, n - 1)),
         ("incdecsc", ((1 << (n - 2)) + 3, 1, n - 1, -1, 0)),
         ("incdecsc", ((1 << (n - 3)) + 1, 0, n - 2, n - 2, n - 1)),
         ("muldiv", (0, (1 << h) - 3, h + 1, 0, h, 0)),
         ("muldiv", (1, (1 << h) - 3, h + 1, 0, h, 1 << (n - 1))),
         ("modnout", (0, 11, (1 << h) - 1, h, 0, h, 0)),
         ("modnout", (1, 11, (1 << h) - 5, 0, h, h, 1 << (n - 1))),
         ("modnout", (2, 3, (1 << h) - 1, h + 1, 0, h, 1 << h)),
         ("hash", (n - 12, 12, _perm_table(rng, 12))),
         ("phase_flip_if_less", (1 << (n - 3), 2, n - 3, 0))]
    g += _indexed_cases(rng, n, [(16, 1), (17, 1), (9, 10), (17, n - 18)], few=True)
    return g


def pack_gates(gates):
    """ctypes arrays in the b200sv_apply_gates layout"""
    import ctypes
    k = len(gates)
    o1 = (ctypes.c_uint64 * k)(*[int(x[0]) for x in gates])
    o2 = (ctypes.c_uint64 * k)(*[int(x[1]) for x in gates])
    pm = (ctypes.c_uint64 * k)(*[int(x[2]) for x in gates])
    m8 = (ctypes.c_double * (8 * k))()
    for i, x in enumerate(gates):
        for j, z in enumerate(x[3]):
            m8[8 * i + 2 * j] = complex(z).real
            m8[8 * i + 2 * j + 1] = complex(z).imag
    return k, o1, o2, pm, m8
