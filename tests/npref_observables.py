"""Float64 NumPy reference of the observable sweeps (b200sv_moments_bits / _floats, b200sv_expectation_pauli), written from
their definitions in include/b200sv.h.  Like tests/npref.py it shares no code with the library or the oracle: weights are
built per basis index with NumPy integer arithmetic, the Pauli string is applied as an explicit operator on the state."""
import numpy as np


def _bit(n, q):
    return (np.arange(1 << n, dtype=np.uint64) >> np.uint64(q)) & np.uint64(1)


def _moments(psi, w, center):
    p = np.abs(np.asarray(psi, dtype=np.complex128)) ** 2
    d = w - center
    return float(p.sum()), float((p * d).sum()), float((p * d * d).sum())


def weights_bits(n, bits, perms, offset):
    """w_i = offset + sum_p perms[2p + bit(i, bits[p])] in uint64 (exact; callers keep the largest weight below 2^64),
    then float64"""
    assert int(offset) + sum(max(int(perms[2 * p]), int(perms[2 * p + 1])) for p in range(len(bits))) < 1 << 64
    w = np.full(1 << n, int(offset), dtype=np.uint64)
    for p, b in enumerate(bits):
        w += np.where(_bit(n, b) == 1, np.uint64(int(perms[2 * p + 1])), np.uint64(int(perms[2 * p])))
    return w.astype(np.float64)


def weights_floats(n, bits, weights):
    w = np.ones(1 << n)
    for p, b in enumerate(bits):
        w *= np.where(_bit(n, b) == 1, float(weights[2 * p + 1]), float(weights[2 * p]))
    return w


def moments_bits(psi, bits, perms, offset=0, center=0.0):
    """(S0, S1, S2) = sum |psi_i|^2 (1, w_i - c, (w_i - c)^2) with the sum-form weight"""
    n = int(np.log2(len(psi)))
    return _moments(psi, weights_bits(n, bits, perms, offset), center)


def moments_floats(psi, bits, weights, center=0.0):
    """(S0, S1, S2) with the product-form weight w_i = prod_p weights[2p + bit(i, bits[p])]"""
    n = int(np.log2(len(psi)))
    return _moments(psi, weights_floats(n, bits, weights), center)


def pauli_masks(bits, paulis):
    """(x, z) of a Pauli string with the reference's enum (I = 0, X = 1, Z = 2, Y = 3)"""
    x = z = 0
    for b, p in zip(bits, paulis):
        if p & 1:
            x |= 1 << b
        if p & 2:
            z |= 1 << b
    return x, z


def apply_1q(psi, m, q):
    """the 2x2 matrix m on qubit q (bit q of the index)"""
    psi = np.asarray(psi, dtype=np.complex128)
    v = psi.reshape(-1, 2, 1 << q)
    out = np.empty_like(v)
    out[:, 0, :] = m[0][0] * v[:, 0, :] + m[0][1] * v[:, 1, :]
    out[:, 1, :] = m[1][0] * v[:, 0, :] + m[1][1] * v[:, 1, :]
    return out.reshape(-1)


PAULI = {1: ((0, 1), (1, 0)), 2: ((1, 0), (0, -1)), 3: ((0, -1j), (1j, 0))}


def pauli_expectation(psi, x, z):
    """(sum |psi|^2, <psi|P|psi>) with P the tensor product of the single-qubit X / Y / Z matrices, applied qubit by qubit"""
    psi = np.asarray(psi, dtype=np.complex128)
    phi = psi
    for q in range(int(np.log2(len(psi)))):
        kind = ((x >> q) & 1) | (((z >> q) & 1) << 1)
        if kind:
            phi = apply_1q(phi, PAULI[kind], q)
    return float(np.vdot(psi, psi).real), float(np.vdot(psi, phi).real)


def u3(theta, phi, lam):
    """QInterface::U (src/qinterface/rotational.cpp:18-26)"""
    c, s = np.cos(theta / 2), np.sin(theta / 2)
    return np.array([[c, -np.exp(1j * lam) * s], [np.exp(1j * phi) * s, np.exp(1j * (phi + lam)) * c]])


def _prob1(psi, q):
    return float(np.sum(np.abs(np.asarray(psi, dtype=np.complex128)[_bit(int(np.log2(len(psi))), q) == 1]) ** 2))


def query_value(psi, op, toks):
    """What the QInterface query `op` (tokens as in qrack_b200/qscript.py, after the op) returns on psi, built from the
    functions above: the k = 0 / k = 1 branches over Prob(bits[0]), the sweeps for k >= 2, the reference's unsquared
    VarianceFloatsFactorized sum (qinterface.cpp:653) and the Pauli / Unitary basis changes.  Returns (value, scale, state
    after the query): the scale of the result is sum p |w| for an expectation and sum p (|w| + |m|)^2 for a variance (for
    relative tolerances); the U3 form of ExpVarUnitaryAll (:511-540) applies U(-theta, -phi, -lambda) before the query and
    U(theta, phi, lambda) after it, which is not its inverse, so the state after a Unitary query differs from the one before."""
    v = _query_value(psi, op, toks)
    if op.endswith("UnitaryAll"):
        k = int(toks[0])
        ang = [float(t) for t in toks[1 + k:]]
        for i, b in enumerate(int(t) for t in toks[1:1 + k]):
            psi = apply_1q(apply_1q(psi, u3(-ang[3 * i], -ang[3 * i + 1], -ang[3 * i + 2]), b),
                           u3(ang[3 * i], ang[3 * i + 1], ang[3 * i + 2]), b)
    return v[0], v[1], psi


def _query_value(psi, op, toks):
    k = int(toks[0])
    bits = [int(t) for t in toks[1:1 + k]]
    rest = toks[1 + k:]
    isExp = op.startswith("Expectation")
    if op.endswith("BitsAll") or op.endswith("BitsFactorized"):
        offset = int(rest[0])
        perms = [v for i in range(k) for v in (0, 1 << i)] if op.endswith("BitsAll") else [int(t) for t in rest[1:]]
        if k == 0:
            return 1.0, 1.0
        n = int(np.log2(len(psi)))
        w = weights_bits(n, bits, perms, offset)
        if k == 1:
            pr = _prob1(psi, bits[0])
            v0, v1 = float(perms[0] + offset), float(perms[1] + offset)
            m = v0 * (1 - pr) + v1 * pr
            if isExp:
                return m, abs(v0) * (1 - pr) + abs(v1) * pr
            return (v0 - m) ** 2 * (1 - pr) + (v1 - m) ** 2 * pr, (abs(v0) + abs(m)) ** 2 + (abs(v1) + abs(m)) ** 2
        s0, m, _ = moments_bits(psi, bits, perms, offset)
        p = np.abs(np.asarray(psi, dtype=np.complex128)) ** 2
        if isExp:
            return m, float((p * np.abs(w)).sum())
        return moments_bits(psi, bits, perms, offset, m)[2], float((p * (np.abs(w) + abs(m)) ** 2).sum())
    if op.endswith("PauliAll"):
        # the reference's PauliI-dropping loop (qinterface.cpp:663-670) re-reads the size after each erase and so keeps some
        # PauliI entries; those get the weights (1, -1) without a basis gate, i.e. count as Z
        kept = [(b, int(t)) for b, t in zip(bits, rest)]
        i = 0
        while i < len(kept):
            j = len(kept) - (i + 1)
            if kept[j][1] == 0:
                del kept[j]
            i += 1
        kept = [(b, p if p else 2) for b, p in kept]
        if not kept:
            return 1.0, 1.0
        x, z = pauli_masks([b for b, _ in kept], [p for _, p in kept])
        s0, e = pauli_expectation(psi, x, z)
        if len(kept) == 1:
            pr = (s0 - e) / 2
            m = 1 - 2 * pr
            return (m, 1.0) if isExp else ((1 - m) ** 2 * (1 - pr) + (1 + m) ** 2 * pr, 4.0)
        return (e, s0) if isExp else (e * (1 - s0), 2 * s0)
    if op.endswith("UnitaryAll"):
        ang = [float(t) for t in rest]
        for i, b in enumerate(bits):
            psi = apply_1q(psi, u3(-ang[3 * i], -ang[3 * i + 1], -ang[3 * i + 2]), b)
        weights = [1.0, -1.0] * k
    else:
        weights = [float(t) for t in rest]
    if k == 0:
        return 1.0, 1.0
    n = int(np.log2(len(psi)))
    p = np.abs(np.asarray(psi, dtype=np.complex128)) ** 2
    w = weights_floats(n, bits, weights)
    if k == 1:
        pr = _prob1(psi, bits[0])
        m = weights[0] * (1 - pr) + weights[1] * pr
        if isExp:
            return m, abs(weights[0]) * (1 - pr) + abs(weights[1]) * pr
        return ((weights[0] - m) ** 2 * (1 - pr) + (weights[1] - m) ** 2 * pr,
                (abs(weights[0]) + abs(m)) ** 2 + (abs(weights[1]) + abs(m)) ** 2)
    s0, m, _ = moments_floats(psi, bits, weights)
    if isExp:
        return m, float((p * np.abs(w)).sum())
    return m * (1 - s0), float((p * (np.abs(w) + abs(m)) ** 2).sum())
