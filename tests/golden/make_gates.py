"""Generate tests/golden/ref_gates_9q.f{32,64}.npz: the final state the reference's own QEngineCPU returns for each script of
tests/oracle_gates.ref_scripts (two-target gates, (C)UniformParityRZ with controls inside and outside the mask,
UniformlyControlledSingleBit / RY / RZ with skip arguments).  dropin/gates_harness.cpp is compiled against
oracle/_ref/f{32,64}/libqrack.a, which oracle/Makefile builds from the reference sources:

    make -C oracle REF=<reference source tree> ref && python tests/golden/make_gates.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import oracle_gates  # noqa: E402
from __graft_entry__ import REFERENCE_DEFAULT  # noqa: E402


def compile_harness(prec, out):
    ref = os.environ.get("QRACK_REFERENCE", REFERENCE_DEFAULT)
    lib = os.path.join(ROOT, "oracle", "_ref", "f%d" % prec)
    cmd = ["g++", "-O3", "-std=c++14", "-msse3", "-mfma", "-I" + os.path.join(lib, "include", "common"),
           "-I" + os.path.join(ref, "include"), "-I" + os.path.join(ref, "include", "common"),
           os.path.join(ROOT, "dropin", "gates_harness.cpp"), os.path.join(lib, "libqrack.a"), "-lpthread", "-o", out]
    if prec == 64:
        cmd.insert(1, "-mavx")
    subprocess.run(cmd, check=True)


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            exe = os.path.join(td, "gates_f%d" % prec)
            compile_harness(prec, exe)
            out = {}
            for name, text in oracle_gates.ref_scripts().items():
                script, dump = os.path.join(td, name + ".qs"), os.path.join(td, name + ".bin")
                open(script, "w").write(text)
                subprocess.run([exe, script, "--dump", dump], check=True)
                out[name] = np.fromfile(dump, dtype=np.complex64 if prec == 32 else np.complex128)
            fn = os.path.join(HERE, "ref_gates_9q.f%d.npz" % prec)
            np.savez_compressed(fn, **out)
            print("wrote", fn)


if __name__ == "__main__":
    main()
