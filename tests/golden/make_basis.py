"""Writes tests/golden/ref_basis_12q.f32.npz / .f64.npz — and nothing else — from the compiled reference.

dropin/observables_harness.cpp is compiled against the reference's own QEngineCPU (oracle/_ref/f{32,64}/libqrack.a, built by
`make -C oracle ref`) in a temporary directory, exactly as tests/golden/make_observables.py does.  It replays the 12-qubit
U3 + CNOT circuit of the observables fixture, then, one run per query of basis_queries(), that query with the state dumped
after it.  Each file holds
  state     the reference's state after the circuit (complex64 / complex128);
  queries   the query lines, one per result;
  results   one "<op> <value>" line per query, in query order (qscript.parse_results reads it);
  post<q>   for every U3-form expectation query q without eigenvalues, the reference's state after it (the variance and
            the eigenvalues do not change the post-state).

    QRACK_REFERENCE=<reference tree> python tests/golden/make_basis.py
"""
import math
import os
import random
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import oracle_observables  # noqa: E402
from make_observables import compile_harness  # noqa: E402

# k in {1, 2, 3, 5, 12}; qubit 0 listed and not; the top qubit; unsorted lists
SETS = [[3], [0], [7, 8], [11, 0, 5], [0, 7, 8, 11, 5], [9, 2, 4, 1, 10], list(range(12))[::-1]]


def basis_queries(seed=777):
    """every set in both forms (U3 angles, and one 2x2 matrix per qubit: I + a random complex perturbation, so that inv2x2
    is well conditioned and not unitary), expectation and variance, with the default eigenvalues and with given ones"""
    rng = random.Random(seed)
    lines = []
    for bits in SETS:
        cs = "%d %s" % (len(bits), " ".join(map(str, bits)))
        angles = ["%.9g" % rng.uniform(-math.pi, math.pi) for _ in range(3 * len(bits))]
        mats = []
        for _ in bits:
            m = [complex(1.0 if e in (0, 3) else 0.0, 0.0) + 0.6 * complex(rng.uniform(-1, 1), rng.uniform(-1, 1)) for e in range(4)]
            mats += ["%.9g %.9g" % (z.real, z.imag) for z in m]
        eig = ["%.9g" % rng.uniform(-1.5, 1.5) for _ in range(2 * len(bits))]
        for ev in ([], eig):
            for op in ("ExpectationUnitaryAll", "VarianceUnitaryAll"):
                lines.append(" ".join([op, cs] + angles + ev))
            for op in ("ExpectationMatrixAll", "VarianceMatrixAll"):
                lines.append(" ".join([op, cs] + mats + ev))
    return lines


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            cplx = np.complex64 if prec == 32 else np.complex128
            exe = os.path.join(td, "obs_f%d" % prec)
            compile_harness(prec, exe)
            circ = oracle_observables.observables_circuit()
            open(os.path.join(td, "c.qs"), "w").write(circ)
            subprocess.run([exe, os.path.join(td, "c.qs"), "--dump", os.path.join(td, "s.bin")], check=True)
            out = {"state": np.fromfile(os.path.join(td, "s.bin"), dtype=cplx)}
            queries, results = basis_queries(), []
            for q, line in enumerate(queries):
                script, dump = os.path.join(td, "q.qs"), os.path.join(td, "p.bin")
                open(script, "w").write(circ + line + "\n")
                res = subprocess.run([exe, script, "--dump", dump], check=True, capture_output=True, text=True).stdout
                assert len(res.splitlines()) == 1, res
                results.append(res)
                t = line.split()
                if t[0] == "ExpectationUnitaryAll" and len(t) == 2 + 4 * int(t[1]):
                    out["post%d" % q] = np.fromfile(dump, dtype=cplx)
            out["queries"] = np.array("\n".join(queries) + "\n")
            out["results"] = np.array("".join(results))
            fn = os.path.join(HERE, "ref_basis_12q.f%d.npz" % prec)
            np.savez_compressed(fn, **out)
            print("wrote", fn, len(queries), "results")


if __name__ == "__main__":
    main()
