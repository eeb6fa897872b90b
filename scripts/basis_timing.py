"""Times ExpectationUnitaryAll (the matrix form) on the resident state, with CUDA events on the engine's stream
(b200sv_timer_begin/_end):

  * the read-only sweep (b200sv_moments_basis behind the mirror's ExpectationUnitaryAll) against the gate route the reference
    takes (the inverse basis gates, the Floats moments sweep, the gates again), at k in {1, 2, 4, 8, 12} listed qubits (a fixed
    random set containing qubit 0 for odd k), at 30 qubits fp32 and 29 qubits fp64 (8 GiB each): the mean of 20 calls after
    a warm-up, each including its read-back and host synchronise;
  * the sweep's read rate 2^n S / t (S = bytes per amplitude) against the 3.35 TB/s of the H100 SXM data sheet and its
    double-precision flop rate 16 k 2^n / t (k butterfly levels of 8 FMAs per amplitude);

and prints the card's name and power limit beside the numbers.

    python scripts/basis_timing.py [--reps R] [--sizes 30:32,29:64] [--ks 1,2,4,8,12]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from qrack_b200 import QEngineCUDA  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception as e:  # the numbers are still printed, marked as unattributed
        return "unknown (%s)" % e, "unknown"


def timed(q, fn, reps):
    fn()  # warm-up: module load, scratch allocation
    q.be.finish()
    q.be.timer_begin()
    for _ in range(reps):
        fn()
    return q.be.timer_end() / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="30:32,29:64")
    ap.add_argument("--ks", default="1,2,4,8,12")
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power))
    for spec in a.sizes.split(","):
        n, prec = (int(v) for v in spec.split(":"))
        q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
        rng = random.Random(5)
        for b in range(n):
            q.U(b, rng.uniform(0, 3), rng.uniform(-3, 3), rng.uniform(-3, 3))
        q.Finish()
        state_bytes = (1 << n) * (8 if prec == 32 else 16)
        nrng = np.random.default_rng(7)
        for k in (int(v) for v in a.ks.split(",")):
            bits = rng.sample(range(1, n), k - 1) + [0] if k % 2 else rng.sample(range(1, n), k)
            mats = [(np.eye(2) + 0.3 * (nrng.standard_normal((2, 2)) + 1j * nrng.standard_normal((2, 2)))).reshape(-1).tolist()
                    for _ in bits]
            eig = [1.0, -1.0] * k
            t_sweep = timed(q, lambda: q.ExpectationUnitaryAll(bits, mats, eig), a.reps)
            t_gates = timed(q, lambda: q._exp_var_unitary_gates(True, bits, mats, eig, True), a.reps)
            print(json.dumps({"qubits": n, "precision": prec, "k": k, "card": name, "power_limit": power,
                              "sweep_ms": round(t_sweep, 4), "gate_route_ms": round(t_gates, 4),
                              "speedup": round(t_gates / t_sweep, 2),
                              "read_GBps": round(state_bytes / t_sweep / 1e6, 1),
                              "read_share_of_hbm": round(state_bytes / t_sweep / 1e9 / HBM_TBPS, 3),
                              "fp64_GFLOPs": round(16.0 * k * 2.0 ** n / t_sweep / 1e6, 1)}), flush=True)
        del q


if __name__ == "__main__":
    main()
