"""Times the top-n select under a tie key (b200sv_highest_probs_keyed) against the plain one (b200sv_highest_probs) on the
resident state, with CUDA events on the engine's stream (b200sv_timer_begin/_end):

  * the three states of scripts/topn_timing.py (a random dense state, the uniform superposition, GHZ) at 30 qubits fp32 and
    29 qubits fp64 (8 GiB each), n in {2, 64, 4096, 2^20};
  * the keyed call uses what a page of the sharded engine passes: the qubits scattered over key_bits = qubits + 1 positions
    and an XOR, so the keyed kernels look up t(i) in their byte tables;
  * plain and keyed alternate in blocks of --reps calls, --rounds times, after a warm-up of each; the mean per call of each
    block, and the keyed / plain ratio of the medians;
  * before timing, the keyed call with the identity map must return the plain list, and the mapped call the same P list.

It prints the card's name and power limit beside the numbers.

    python scripts/topn_keyed_timing.py [--reps R] [--rounds K] [--sizes 30:32,29:64] [--ns 2,64,4096,1048576]
"""
import argparse
import json
import os
import random
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from qrack_b200 import QEngineCUDA  # noqa: E402
from topn_timing import card, prepare  # noqa: E402


def block(q, fn, reps):
    """mean ms per call over `reps` calls, CUDA events around the block (each call ends in its read-back)"""
    q.be.finish()
    q.be.timer_begin()
    for _ in range(reps):
        fn()
    return q.be.timer_end() / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--sizes", default="30:32,29:64")
    ap.add_argument("--ns", default="2,64,4096,1048576")
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power), flush=True)
    rng = np.random.default_rng(1)
    for spec in a.sizes.split(","):
        nq, prec = (int(v) for v in spec.split(":"))
        bits = nq + 1
        pos = [int(v) for v in rng.permutation(bits)[:nq]]
        xr = int(rng.integers(0, 1 << bits))
        for kind in ("random", "uniform", "ghz"):
            q = QEngineCUDA(nq, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
            prepare(q, kind, nq)
            for n in (int(v) for v in a.ns.split(",")):
                plain = lambda: q.be.highest_probs(n)  # noqa: E731
                keyed = lambda: q.be.highest_probs_keyed(n, bits, pos, xr)  # noqa: E731
                ident_keys, ident_probs = q.be.highest_probs_keyed(n, nq, None, 0)
                _, mapped_probs = keyed()
                same = ([int(v) for v in ident_keys] == plain()) and np.array_equal(ident_probs, mapped_probs)
                ts = {"plain": [], "keyed": []}
                for r in range(a.rounds):
                    order = ("plain", "keyed") if r % 2 == 0 else ("keyed", "plain")
                    for which in order:
                        ts[which].append(block(q, plain if which == "plain" else keyed, a.reps))
                row = {"qubits": nq, "precision": prec, "state": kind, "n": n, "card": name, "power_limit": power,
                       "plain_ms": [round(t, 3) for t in ts["plain"]], "keyed_ms": [round(t, 3) for t in ts["keyed"]],
                       "keyed_over_plain": round(statistics.median(ts["keyed"]) / statistics.median(ts["plain"]), 4),
                       "lists_agree": same}
                print(json.dumps(row), flush=True)
            del q


if __name__ == "__main__":
    main()
