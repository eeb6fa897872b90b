"""Float64 NumPy reference of the moments in a per-qubit basis (b200sv_moments_basis) and of the ExpVarUnitaryAll queries built
on it, written from their definitions in include/b200sv.h and src/qinterface/qinterface.cpp:478-540, 620-657, 771-806.  Like
tests/npref.py it shares no code with the library or the oracle: the state is reshaped to one axis per qubit, each listed
qubit's axis is contracted with its 2x2 matrix by einsum, and the weights are broadcast along the same axes."""
import math

import numpy as np


def u3(theta, phi, lam):
    """the matrix of QInterface::U (rotational.cpp:18-26) in float64"""
    c, s = math.cos(theta / 2), math.sin(theta / 2)
    return np.array([[c, -np.exp(1j * lam) * s], [np.exp(1j * phi) * s, np.exp(1j * (phi + lam)) * c]])


def inv2x2(m):
    m = np.asarray(m, dtype=np.complex128).reshape(2, 2)
    det = 1.0 / (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0])
    return det * np.array([[m[1, 1], -m[0, 1]], [-m[1, 0], m[0, 0]]])


def apply(psi, bits, mats):
    """(x)_p mats[p] on qubit bits[p] of psi, in float64"""
    psi = np.asarray(psi, dtype=np.complex128)
    n = int(np.log2(psi.size))
    t = psi.reshape([2] * n)  # axis a is qubit n - 1 - a
    for b, m in zip(bits, mats):
        ax = n - 1 - b
        idx = "".join(chr(ord("a") + i) for i in range(n))
        out = idx[:ax] + "Z" + idx[ax + 1:]
        t = np.einsum("Z%s,%s->%s" % (idx[ax], idx, out), np.asarray(m, dtype=np.complex128).reshape(2, 2), t)
    return t.reshape(-1)


def weight(n, bits, weights):
    """w_i = prod_p weights[2p + bit(i, bits[p])] for every basis state i"""
    w = np.ones([2] * n)
    for p, b in enumerate(bits):
        shape = [1] * n
        shape[n - 1 - b] = 2
        w = w * np.asarray(weights[2 * p:2 * p + 2], dtype=np.float64).reshape(shape)
    return w.reshape(-1)


def moments_basis(psi, bits, mats, weights, center=0.0):
    """(S0, S1, S2) = sum |phi|^2 (1, w - c, (w - c)^2) with phi = (x)_p mats[p] psi, and the scale sum |phi|^2 (1 + |w - c|)^2
    of the three for tolerances"""
    phi = apply(psi, bits, mats)
    p = np.abs(phi) ** 2
    d = weight(int(np.log2(p.size)), bits, weights) - center
    return (float(p.sum()), float((p * d).sum()), float((p * d * d).sum())), float((p * (1 + np.abs(d)) ** 2).sum())


def basis_mats(form, bits, ops):
    """the A_p the reference applies before its query: inv2x2 of each matrix, or U(-theta, -phi, -lambda)"""
    if form == "matrix":
        return [inv2x2(m) for m in ops]
    return [u3(-ops[3 * i], -ops[3 * i + 1], -ops[3 * i + 2]) for i in range(len(bits))]


def exp_var_unitary(psi, isExp, bits, mats, eig=()):
    """(value, scale) of ExpectationUnitaryAll / VarianceUnitaryAll with the basis matrices A_p already formed: the Floats
    query's 1-bit branch (Prob, and a squared variance) or its k >= 2 sums (the variance unsquared, :653)"""
    k = len(bits)
    if not k:
        return 1.0, 1.0
    eig = list(eig) if len(eig) else [1.0, -1.0] * k
    if k == 1:
        (s0, pr, _), _ = moments_basis(psi, bits, mats, [0.0, 1.0])
        pr = min(max(pr, 0.0), 1.0)
        mean = eig[0] * (1 - pr) + eig[1] * pr
        if isExp:
            return mean, abs(eig[0]) + abs(eig[1])
        v0, v1 = eig[0] - mean, eig[1] - mean
        return v0 * v0 * (1 - pr) + v1 * v1 * pr, (abs(eig[0]) + abs(eig[1]) + abs(mean)) ** 2
    (s0, s1, _), scale = moments_basis(psi, bits, mats, eig)
    return (s1 if isExp else s1 - s1 * s0), scale * (1 + abs(s1))


def u3_post_state(psi, bits, angles):
    """the reference's state after a U3-form query: U(theta, phi, lambda) U(-theta, -phi, -lambda) on every listed qubit"""
    net = [u3(*angles[3 * i:3 * i + 3]) @ u3(-angles[3 * i], -angles[3 * i + 1], -angles[3 * i + 2]) for i in range(len(bits))]
    return apply(psi, bits, net)
