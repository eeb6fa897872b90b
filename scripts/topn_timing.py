"""Times HighestProbAll(n) on the resident state, with CUDA events on the engine's stream (b200sv_timer_begin/_end):

  * b200sv_highest_probs at n in {2, 64, 4096, 2^20} on three states at 30 qubits fp32 and 29 qubits fp64 (8 GiB each): a
    random dense state (H / T / CNOT layers), the uniform superposition and GHZ.  The mean of 20 calls after a warm-up, each
    including the read-backs and the host sort; the full-state reads per call, counted from one profiled call by kernel
    role (k_topn_stats / k_topn_hist / k_topn_collect on the state; the same kernels on the candidate buffer do not read
    it) and checked against the kernel_launches delta; the read rate reads x 8 GiB / t;
  * once, for the record, the QInterface default (qinterface.cpp:962-1003: one ProbAll per basis state, insertion into the
    n best) at 16 qubits and n = 64, through the Python mirror, host clock;

and prints the card's name and power limit beside the numbers.

    python scripts/topn_timing.py [--reps R] [--sizes 30:32,29:64] [--ns 2,64,4096,1048576]
"""
import argparse
import json
import os
import random
import re
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


def kernel_roles(fn, calls=3):
    """(kernels recorded, of which read the state) over `calls` calls, from the kernel names torch.profiler records: the source
    is the first template argument, 0 / 1 = an fp32 / fp64 state, 2 = the candidate buffer"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "k_topn_" in e.name]
    return len(names), sum(1 for s in names if re.search(r"<[01][,>]", s))


def prepare(q, kind, n):
    if kind == "uniform":
        for b in range(n):
            q.H(b)
    elif kind == "ghz":
        q.H(0)
        for b in range(1, n):
            q.CNOT(0, b)
    else:
        for layer in range(2):
            for b in range(n):
                q.H(b)
                q.T(b)
            for b in range(layer, n - 1, 2):
                q.CNOT(b, b + 1)
    q.Finish()


def qinterface_default(q, n):
    """the reference's loop as written (early exit included), over the engine's ProbAll (one device round trip each)"""
    tot, best = 0.0, [(0, 0.0)] * n
    for p in range(q.maxQPower):
        prob = q.ProbAll(p)
        tot += prob
        for t in range(n):
            if prob > best[t][1]:
                best[t + 1:] = best[t:n - 1]
                best[t] = (p, prob)
                break
        if best[-1][1] > 1.0 - tot:
            break
    return [p for p, _ in best]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="30:32,29:64")
    ap.add_argument("--ns", default="2,64,4096,1048576")
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power))
    for spec in a.sizes.split(","):
        nq, prec = (int(v) for v in spec.split(":"))
        state_bytes = (1 << nq) * (8 if prec == 32 else 16)
        for kind in ("random", "uniform", "ghz"):
            q = QEngineCUDA(nq, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
            prepare(q, kind, nq)
            for n in (int(v) for v in a.ns.split(",")):
                before = q.be.stats()["kernel_launches"]
                q.be.highest_probs(n)
                launches = q.be.stats()["kernel_launches"] - before
                kernels, reads = kernel_roles(lambda: q.be.highest_probs(n))
                t = timed(q, lambda: q.be.highest_probs(n), a.reps)
                row = {"qubits": nq, "precision": prec, "state": kind, "n": n, "card": name, "power_limit": power,
                       "ms": round(t, 3), "launches": launches}
                if kernels == 3 * launches:
                    row["state_reads"] = reads // 3
                    row["read_GBps"] = round(reads // 3 * state_bytes / t / 1e6, 1)
                else:  # the profile lost kernels: no read count rather than a wrong one
                    row["profiled_kernels_of_3_calls"] = kernels
                print(json.dumps(row), flush=True)
            del q
    q = QEngineCUDA(16, 0, random.Random(1), 1.0 + 0j, False, False, precision=32)
    prepare(q, "random", 16)
    t0 = time.perf_counter()
    qinterface_default(q, 64)
    t_loop = time.perf_counter() - t0
    t_kernel = timed(q, lambda: q.be.highest_probs(64), a.reps)
    print(json.dumps({"qubits": 16, "precision": 32, "n": 64, "card": name, "power_limit": power,
                      "qinterface_default_s": round(t_loop, 3), "select_ms": round(t_kernel, 4)}))


if __name__ == "__main__":
    main()
