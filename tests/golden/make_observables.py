"""Writes tests/golden/ref_observables_12q.f32.npz / .f64.npz — and nothing else — from the compiled reference.

dropin/observables_harness.cpp is compiled against the reference's own QEngineCPU (oracle/_ref/f{32,64}/libqrack.a, built by
`make -C oracle ref`) in a temporary directory and replays tests/oracle_observables.observables_text().  Each file holds
  state    the reference's state after the circuit, before the first query (complex64 / complex128);
  results  one "<op> <value>" line per query, in script order (util.load_reference parses it).

    QRACK_REFERENCE=<reference tree> python tests/golden/make_observables.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import oracle_observables  # noqa: E402
from __graft_entry__ import REFERENCE_DEFAULT  # noqa: E402


def compile_harness(prec, out):
    ref = os.environ.get("QRACK_REFERENCE", REFERENCE_DEFAULT)
    lib = os.path.join(ROOT, "oracle", "_ref", "f%d" % prec)
    cmd = ["g++", "-O3", "-std=c++14", "-msse3", "-mfma", "-I" + os.path.join(lib, "include", "common"),
           "-I" + os.path.join(ref, "include"), "-I" + os.path.join(ref, "include", "common"),
           os.path.join(ROOT, "dropin", "observables_harness.cpp"), os.path.join(lib, "libqrack.a"), "-lpthread", "-o", out]
    if prec == 64:
        cmd.insert(1, "-mavx")
    subprocess.run(cmd, check=True)


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            exe = os.path.join(td, "obs_f%d" % prec)
            compile_harness(prec, exe)
            circ, full = os.path.join(td, "c.qs"), os.path.join(td, "q.qs")
            open(circ, "w").write(oracle_observables.observables_circuit())
            open(full, "w").write(oracle_observables.observables_text())
            subprocess.run([exe, circ, "--dump", os.path.join(td, "s.bin")], check=True)
            res = subprocess.run([exe, full], check=True, capture_output=True, text=True).stdout
            state = np.fromfile(os.path.join(td, "s.bin"), dtype=np.complex64 if prec == 32 else np.complex128)
            fn = os.path.join(HERE, "ref_observables_12q.f%d.npz" % prec)
            np.savez_compressed(fn, state=state, results=np.array(res))
            print("wrote", fn, len(res.splitlines()), "results")


if __name__ == "__main__":
    main()
