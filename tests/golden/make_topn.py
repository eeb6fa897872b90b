"""Writes tests/golden/ref_topn_12q.f32.npz / .f64.npz — and nothing else — from the compiled reference.

dropin/observables_harness.cpp is compiled against the reference's own QEngineCPU (oracle/_ref/f{32,64}/libqrack.a, built by
`make -C oracle ref`) in a temporary directory, exactly as tests/golden/make_observables.py does, and replays each case of
tests/oracle_topn.topn_cases(): a 12-qubit circuit, then one HighestProbAllN per query size.  Each file holds, per case c,
  state_<c>         the reference's state after the circuit (complex64 / complex128);
  top_<c>_<n>       the reference's HighestProbAll(n) (int64).

    QRACK_REFERENCE=<reference tree> python tests/golden/make_topn.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import oracle_topn  # noqa: E402
from make_observables import compile_harness  # noqa: E402
from qrack_b200 import qscript  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            cplx = np.complex64 if prec == 32 else np.complex128
            exe = os.path.join(td, "obs_f%d" % prec)
            compile_harness(prec, exe)
            out = {}
            for name, circ, sizes in oracle_topn.topn_cases():
                c, full, dump = os.path.join(td, "c.qs"), os.path.join(td, "q.qs"), os.path.join(td, "s.bin")
                open(c, "w").write(circ)
                open(full, "w").write(oracle_topn.topn_text(circ, sizes))
                subprocess.run([exe, c, "--dump", dump], check=True)
                res = subprocess.run([exe, full], check=True, capture_output=True, text=True).stdout
                out["state_" + name] = np.fromfile(dump, dtype=cplx)
                results = qscript.parse_results(res)
                assert len(results) == len(sizes)
                for k, (op, vals) in zip(sizes, results):
                    assert op == "HighestProbAllN" and len(vals) == k
                    out["top_%s_%d" % (name, k)] = np.array(vals, dtype=np.int64)
            fn = os.path.join(HERE, "ref_topn_12q.f%d.npz" % prec)
            np.savez_compressed(fn, **out)
            print("wrote", fn, len(out), "arrays")


if __name__ == "__main__":
    main()
