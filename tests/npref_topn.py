"""Float64 NumPy reference of the n most probable basis states (b200sv_highest_probs), written from its definition in
include/b200sv.h.  Like tests/npref.py it shares no code with the library or the oracle."""
import numpy as np


def probs(psi):
    """P(i) = min(|psi_i|^2, 1) in double: an fp32 component squared in double is exact, so only the sum rounds; NumPy does not
    contract re * re + im * im into an FMA, so this is the device's key bit for bit in both precisions"""
    psi = np.asarray(psi)
    re, im = psi.real.astype(np.float64), psi.imag.astype(np.float64)
    return np.minimum(re * re + im * im, 1.0)


def order(psi):
    """every index with P > 0, by P descending, then index ascending"""
    p = probs(psi)
    o = np.lexsort((np.arange(len(p)), -p))
    return o[p[o] > 0]


def top_n(psi, n):
    """the n indices of largest P, ties to the smaller index, P = 0 never listed, zero-filled past the last P > 0"""
    o = order(psi)[:n]
    out = np.zeros(n, dtype=np.int64)
    out[:len(o)] = o
    return [int(v) for v in out]
