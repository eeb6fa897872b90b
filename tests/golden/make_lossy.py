"""Writes tests/golden/ref_lossy.f32.npz / .f64.npz — and nothing else — from the compiled reference.

dropin/observables_harness.cpp, compiled against the reference's own QEngineCPU, runs each case of CASES: a U3 + CNOT
circuit, then `LossySave` (which writes the reference's TurboQuant file, QEngineCPU::LossySaveStateVector), and in a second
run `LossyLoad` of that file into a fresh register.  Each file holds, per case c,
  state_<c>    the state that was saved (complex64 / complex128);
  file_<c>     the file the reference wrote (uint8);
  decode_<c>   the state the reference decoded from it.
The file's seed comes from std::random_device, so each regeneration writes other bytes; the tests take the seed from the file.

The codec is specified in plain sequential IEEE arithmetic (qrack_b200/csrc/lossy.cuh).  The reference's build flags include
-mfma, and GCC contracts a * b + c into one FMA by default in C++ (-ffp-contract=fast), which changes the rotation and the
sums in their last bits.  So the harness here is linked against oracle/_ref/f{32,64}/libqrack.a with the two translation units
that hold the codec (src/qengine/state.cpp: QEngineCPU's save / load; src/qinterface/qinterface.cpp: the QInterface default)
recompiled, unmodified, with -ffp-contract=off in front of it.

    QRACK_REFERENCE=<reference tree> python tests/golden/make_lossy.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT]

from __graft_entry__ import REFERENCE_DEFAULT  # noqa: E402
from qrack_b200 import qscript  # noqa: E402

# name -> (qubits, p, b, circuit depth; 0 = |0>)
CASES = {
    "u3_n10_p6_b4": (10, 6, 4, 3),
    "u3_n9_p3_b3": (9, 3, 3, 3),
    "u3_n12_p5_b8": (12, 5, 8, 3),
    "u3_n8_p6_b1": (8, 6, 1, 3),
    "u3_n8_p6_b16": (8, 6, 16, 3),
    "ket0_n10_p6_b4": (10, 6, 4, 0),
    "u3_n4_p6_b4": (4, 6, 4, 2),
}


def circuit(name):
    n, _, _, depth = CASES[name]
    return qscript.random_u3_cnot(n, depth, seed=sum(map(ord, name))) if depth else "qubits %d\n" % n


def compile_harness(prec, out, td):
    ref = os.environ.get("QRACK_REFERENCE", REFERENCE_DEFAULT)
    lib = os.path.join(ROOT, "oracle", "_ref", "f%d" % prec)
    flags = ["-O3", "-std=c++14", "-msse3", "-mfma", "-ffp-contract=off"] + (["-mavx"] if prec == 64 else [])
    inc = ["-I" + os.path.join(lib, "include", "common"), "-I" + os.path.join(ref, "include"),
           "-I" + os.path.join(ref, "include", "common")]
    objs = []
    for src in ("src/qengine/state.cpp", "src/qinterface/qinterface.cpp"):
        o = os.path.join(td, "f%d_%s.o" % (prec, os.path.basename(src)[:-4]))
        subprocess.run(["g++"] + flags + inc + ["-c", os.path.join(ref, src), "-o", o], check=True)
        objs.append(o)
    subprocess.run(["g++"] + flags + inc + [os.path.join(ROOT, "dropin", "observables_harness.cpp")] + objs +
                   [os.path.join(lib, "libqrack.a"), "-lpthread", "-o", out], check=True)


def main():
    with tempfile.TemporaryDirectory() as td:
        for prec in (32, 64):
            cplx = np.complex64 if prec == 32 else np.complex128
            exe = os.path.join(td, "ref_f%d" % prec)
            compile_harness(prec, exe, td)
            out = {}
            for name, (n, p, b, _) in CASES.items():
                f = os.path.join(td, name + ".svtq")
                save, load = os.path.join(td, "save.qs"), os.path.join(td, "load.qs")
                open(save, "w").write(circuit(name) + "LossySave %s %d %d\n" % (f, p, b))
                open(load, "w").write("qubits %d\nLossyLoad %s\n" % (n, f))
                subprocess.run([exe, save, "--dump", os.path.join(td, "s.bin")], check=True)
                out["state_" + name] = np.fromfile(os.path.join(td, "s.bin"), dtype=cplx)
                out["file_" + name] = np.fromfile(f, dtype=np.uint8)
                subprocess.run([exe, load, "--dump", os.path.join(td, "d.bin")], check=True)
                out["decode_" + name] = np.fromfile(os.path.join(td, "d.bin"), dtype=cplx)
            fn = os.path.join(HERE, "ref_lossy.f%d.npz" % prec)
            np.savez_compressed(fn, **out)
            print("wrote", fn, len(out), "arrays")


if __name__ == "__main__":
    main()
