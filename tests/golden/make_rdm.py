"""Writes tests/golden/ref_rdm_12q.f32.npz / .f64.npz — and nothing else — from the compiled reference.

dropin/observables_harness.cpp is compiled against the reference's own QEngineCPU (oracle/_ref/f{32,64}/libqrack.a, built by
`make -C oracle ref`) in a temporary directory, exactly as tests/golden/make_observables.py does, and replays
tests/oracle_rdm.rdm_text(): the 12-qubit U3 + CNOT circuit of the observables fixture, then one
GetReducedDensityMatrix per kept set of oracle_rdm.rdm_queries().  Each file holds
  state    the reference's state after the circuit (complex64 / complex128);
  rho<q>   query q's matrix in the reference's complex type, shape (2^k, 2^k), bit p of a row index = qubit p of the query.

    QRACK_REFERENCE=<reference tree> python tests/golden/make_rdm.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import oracle_rdm  # noqa: E402
from make_observables import compile_harness  # noqa: E402
from qrack_b200 import qscript  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            cplx = np.complex64 if prec == 32 else np.complex128
            exe = os.path.join(td, "obs_f%d" % prec)
            compile_harness(prec, exe)
            circ, full = os.path.join(td, "c.qs"), os.path.join(td, "q.qs")
            open(circ, "w").write(oracle_rdm.rdm_circuit())
            open(full, "w").write(oracle_rdm.rdm_text())
            subprocess.run([exe, circ, "--dump", os.path.join(td, "s.bin")], check=True)
            res = subprocess.run([exe, full], check=True, capture_output=True, text=True).stdout
            state = np.fromfile(os.path.join(td, "s.bin"), dtype=cplx)
            out = {"state": state}
            for q, (op, vals) in enumerate(qscript.parse_results(res)):
                assert op == "GetReducedDensityMatrix"
                v = np.array(vals, dtype=np.float64).view(np.complex128)
                d = int(round(np.sqrt(v.size)))
                out["rho%d" % q] = v.astype(cplx).reshape(d, d)
            fn = os.path.join(HERE, "ref_rdm_12q.f%d.npz" % prec)
            np.savez_compressed(fn, **out)
            print("wrote", fn, len(out) - 1, "matrices")


if __name__ == "__main__":
    main()
