"""Float64 NumPy reference of every state-vector primitive of include/b200sv.h (test infrastructure).

Plain NumPy on complex128 / float64, written from the header's definitions and the reference lines they cite; nothing here
calls or shares code with the library or the oracle restatement.  Inputs are upcast: callers pass the state the engine
actually holds (read back in its own precision), so that what is left of a difference is the kernel's own arithmetic.
Every function returns new arrays and leaves its arguments alone.
"""
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
