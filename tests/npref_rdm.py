"""Float64 NumPy reference of the reduced density matrix (b200sv_reduced_density_matrix), written from its definition in
include/b200sv.h.  Like tests/npref.py it shares no code with the library or the oracle: the state is reshaped to one axis per
qubit, the kept axes are moved to the front and rho is the matrix product A A^H."""
import numpy as np


def rdm(psi, qubits):
    """(rho, scale): rho[i, j] = sum_e psi[i, e] conj(psi[j, e]) with bit p of i and j the qubit qubits[p] and e the other
    qubits, as the matrix product A A^H of the state reshaped to (kept, env); scale[i, j] = sum_e |psi[i, e]| |psi[j, e]|,
    the natural size of entry (i, j) for relative tolerances"""
    psi = np.asarray(psi, dtype=np.complex128)
    n, k = int(np.log2(len(psi))), len(qubits)
    t = psi.reshape([2] * n)  # axis a is qubit n - 1 - a
    rows = [n - 1 - q for q in reversed(qubits)]  # row index bit k - 1 (the first axis) is qubits[k - 1]
    a = np.transpose(t, rows + [x for x in range(n) if x not in rows]).reshape(1 << k, -1)
    m = np.abs(a)
    return a @ a.conj().T, m @ m.T
