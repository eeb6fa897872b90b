"""Times GetReducedDensityMatrix on the resident state, with CUDA events on the engine's stream (b200sv_timer_begin/_end):

  * b200sv_reduced_density_matrix at k in {1, 2, 4, 6, 8, 10, 12} kept qubits (a fixed random set containing qubit 0 for
    odd k), at 30 qubits fp32 and 29 qubits fp64 (8 GiB each): the mean of 20 calls after a warm-up, each including its
    read-back and host synchronise; its read rate 2^n S / t (S = bytes per amplitude) and, for k >= 7, where the sweep is
    bound by the double-precision FMAs, its flop rate 8 2^(n + k - 1) / t (the upper triangle of rho);
  * once, for the record, the QInterface default (qinterface.cpp:886-944: one GetAmplitude per environment state and kept
    state pair) at 16 qubits and k = 2, host clock;

and prints the card's name and power limit beside the numbers.

    python scripts/rdm_timing.py [--reps R] [--sizes 30:32,29:64] [--ks 1,2,4,6,8,10,12]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from qrack_b200 import QEngineCUDA  # noqa: E402


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


def qinterface_default(q, qubits):
    """the reference's loop as written, over the engine's GetAmplitude (one device round trip each)"""
    n, k = q.qubitCount, len(qubits)
    env = [b for b in range(n) if b not in qubits]
    out = [[0j] * (1 << k) for _ in range(1 << k)]
    for e in range(1 << len(env)):
        base = sum(1 << b for i, b in enumerate(env) if (e >> i) & 1)
        full = [base | sum(1 << b for p, b in enumerate(qubits) if (i >> p) & 1) for i in range(1 << k)]
        for i in range(1 << k):
            ai = q.GetAmplitude(full[i])
            for j in range(1 << k):
                out[i][j] += ai * q.GetAmplitude(full[j]).conjugate()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="30:32,29:64")
    ap.add_argument("--ks", default="1,2,4,6,8,10,12")
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
        for k in (int(v) for v in a.ks.split(",")):
            kept = rng.sample(range(1, n), k - 1) + [0] if k % 2 else rng.sample(range(1, n), k)
            t = timed(q, lambda: q.be.reduced_density_matrix(kept), a.reps)
            row = {"qubits": n, "precision": prec, "k": k, "card": name, "power_limit": power, "ms": round(t, 4),
                   "read_GBps": round(state_bytes / t / 1e6, 1)}
            if k >= 7:
                row["GFLOPs"] = round(8.0 * 2.0 ** (n + k - 1) / t / 1e6, 1)
            print(json.dumps(row), flush=True)
        del q
    q = QEngineCUDA(16, 0, random.Random(1), 1.0 + 0j, False, False, precision=32)
    for b in range(16):
        q.U(b, 0.3 * b, 0.1, -0.2)
    t0 = time.perf_counter()
    qinterface_default(q, [3, 9])
    t_loop = time.perf_counter() - t0
    t_kernel = timed(q, lambda: q.be.reduced_density_matrix([3, 9]), a.reps)
    print(json.dumps({"qubits": 16, "precision": 32, "k": 2, "card": name, "power_limit": power,
                      "qinterface_default_s": round(t_loop, 3), "sweep_ms": round(t_kernel, 4)}))


if __name__ == "__main__":
    main()
