"""Times one observable query on the resident state, with CUDA events on the engine's stream (b200sv_timer_begin/_end):

  * one ExpectationPauliAll term through the read-only sweep (b200sv_expectation_pauli);
  * the same term through the gate route of the QInterface default (qinterface.cpp:715-769): H / IS.H basis gates, the
    Floats moments sweep with weights (1, -1), the gates undone — the gates queued and fused exactly as in a circuit;
  * the moments sweep (b200sv_moments_floats, every qubit listed) and its read bandwidth: 2^n amplitudes read once.

at 30 qubits fp32 and 29 qubits fp64 (8 GiB each), and prints the card's name and power limit beside the numbers.

    python scripts/observables_timing.py [--reps R] [--sizes 30:32,29:64]
"""
import argparse
import json
import os
import random
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="30:32,29:64")
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
        # one Hamiltonian-like term: X on 0 and n/2, Y on 3 and n-1, Z on 1, 2 and n-2, I elsewhere
        term = {0: 1, n // 2: 1, 3: 3, n - 1: 3, 1: 2, 2: 2, n - 2: 2}
        bits, paulis = list(term), list(term.values())
        x = sum(1 << b for b, p in term.items() if p & 1)
        z = sum(1 << b for b, p in term.items() if p & 2)

        def gate_route():
            for b, p in term.items():
                if p == 1:
                    q.H(b)
                elif p == 3:
                    q.IS(b)
                    q.H(b)
            q.be.moments_floats(bits, [1.0, -1.0] * len(bits), 0.0)
            for b, p in term.items():
                if p == 1:
                    q.H(b)
                elif p == 3:
                    q.H(b)
                    q.S(b)

        e_kernel = q.ExpectationPauliAll(bits, paulis)
        t_pauli = timed(q, lambda: q.be.expectation_pauli(x, z), a.reps)
        t_route = timed(q, gate_route, a.reps)
        allbits = list(range(n))
        weights = [1.0, -1.0] * n
        t_mom = timed(q, lambda: q.be.moments_floats(allbits, weights, 0.0), a.reps)
        state_bytes = (1 << n) * (8 if prec == 32 else 16)
        print(json.dumps({"qubits": n, "precision": prec, "card": name, "power_limit": power,
                          "pauli_term_readonly_ms": round(t_pauli, 4), "pauli_term_gate_route_ms": round(t_route, 4),
                          "moments_sweep_ms": round(t_mom, 4), "moments_sweep_read_GBps": round(state_bytes / t_mom / 1e6, 1),
                          "pauli_expectation": e_kernel}))
        del q


if __name__ == "__main__":
    main()
