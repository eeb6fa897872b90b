"""Times MAll's search for many shots (b200sv_sample_many) on a dense random state (scripts/topn_timing.py's "random": H / T /
CNOT layers) at 30 qubits fp32 and 29 qubits fp64 (8 GiB each), shots in {1, 10^3, 10^5, 10^6}:

  * the b200sv_sample_many call, CUDA events on the engine's stream around a block of calls, read-back of the picks
    included (b200sv_timer_begin/_end); the same call of an older build of the library (--parent-lib, e.g. one built from
    the parent commit) on the same device buffer, alternating with this build block by block, so both are timed under the
    same conditions.  Both must return the same picks for the same seeded rnds at every size;
  * the kernels' own times, k_chunk_sums and k_sample_search, from one more call per size and shot count, all of them in a
    single torch.profiler session after the timed blocks (rows are printed after it);
  * state reads per call: one for the chunk sums, plus at most the share of 2^14-amplitude chunks that hold a pick;
  * MultiShotMeasureMask over every qubit end to end (host clock; it includes drawing the rnds in Python);

and prints the card's name and power limit beside the numbers.

    python scripts/sample_timing.py [--parent-lib PATH] [--rounds K] [--sizes 30:32,29:64] [--shots 1,1000,100000,1000000]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from qrack_b200 import QEngineCUDA  # noqa: E402
from topn_timing import card, prepare  # noqa: E402

PD = ctypes.POINTER(ctypes.c_double)
PU = ctypes.POINTER(ctypes.c_uint64)


class Build:
    """one build of libb200sv.so and a state handle of it over a device buffer (this build: the engine's own handle)"""

    def __init__(self, lib, h):
        self.lib, self.h = lib, h

    def sample_many(self, rnds, out):
        rc = self.lib.b200sv_sample_many(self.h, rnds.size, rnds.ctypes.data_as(PD), out.ctypes.data_as(PU))
        assert rc == 0, rc

    def block(self, rnds, out, reps):
        """mean ms per call over `reps` calls, CUDA events around the block"""
        self.lib.b200sv_finish(self.h)
        self.lib.b200sv_timer_begin(self.h)
        for _ in range(reps):
            self.sample_many(rnds, out)
        ms = ctypes.c_double()
        assert self.lib.b200sv_timer_end(self.h, ctypes.byref(ms)) == 0
        return ms.value / reps


def parent_build(path, q, nq, prec):
    """the older library's handle over the engine's device buffer (read-only use on both sides)"""
    lib = ctypes.CDLL(path)
    for fn in ("b200sv_create_external", "b200sv_sample_many", "b200sv_timer_begin", "b200sv_timer_end", "b200sv_finish",
               "b200sv_destroy"):
        getattr(lib, fn).restype = ctypes.c_int
    lib.b200sv_create_external.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
    lib.b200sv_sample_many.argtypes = [ctypes.c_void_p, ctypes.c_int, PD, PU]
    lib.b200sv_timer_end.argtypes = [ctypes.c_void_p, PD]
    for fn in ("b200sv_timer_begin", "b200sv_finish", "b200sv_destroy"):
        getattr(lib, fn).argtypes = [ctypes.c_void_p]
    ptr, h = ctypes.c_void_p(), ctypes.c_void_p()
    assert q.be.lib.b200sv_device_ptr(q.be.h, ctypes.byref(ptr)) == 0
    dev = ctypes.c_int()
    assert q.be.lib.b200sv_device(q.be.h, ctypes.byref(dev)) == 0
    assert lib.b200sv_create_external(dev.value, nq, prec, ptr, ctypes.byref(h)) == 0
    return Build(lib, h)


KERNELS = ("k_chunk_sums", "k_sample_search")


def kernel_ms(calls):
    """{kernel: ms} of each call in `calls`, from ONE torch.profiler session over all of them (later sessions of one process
    dropped kernel records): every call launches k_chunk_sums then k_sample_search, so the kernels, in launch order, pair up
    with the calls in order.  A session that recorded another count gives no times rather than misassigned ones."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for fn in calls:
            fn()
            torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if any(k in e.name for k in KERNELS)), key=lambda e: e.time_range.start)
    if len(ev) != 2 * len(calls):
        return [{"profile_recorded_kernels": len(ev), "expected": 2 * len(calls)}] * len(calls)
    out = []
    for i in range(len(calls)):
        pair = ev[2 * i:2 * i + 2]
        assert [k for e in pair for k in KERNELS if k in e.name] == list(KERNELS)
        out.append({k: round(e.time_range.elapsed_us() / 1e3, 4) for k, e in zip(KERNELS, pair)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--sizes", default="30:32,29:64")
    ap.add_argument("--shots", default="1,1000,100000,1000000")
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power), flush=True)
    rows, calls, keep = [], [], []
    for spec in a.sizes.split(","):
        nq, prec = (int(v) for v in spec.split(":"))
        q = QEngineCUDA(nq, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
        prepare(q, "random", nq)
        new = Build(q.be.lib, q.be.h)
        old = parent_build(a.parent_lib, q, nq, prec) if a.parent_lib else None
        nchunks = max(1, (1 << nq) >> 14)
        for shots in (int(v) for v in a.shots.split(",")):
            rnds = np.random.default_rng(shots).random(shots)
            out_new = np.zeros(shots, dtype=np.uint64)
            out_old = np.zeros(shots, dtype=np.uint64)
            new.sample_many(rnds, out_new)  # warm-up, and the picks to compare
            reps = 20 if shots <= 1000 else (5 if shots <= 100000 else 1)
            row = {"qubits": nq, "precision": prec, "shots": shots, "card": name, "power_limit": power}
            if old is not None:
                old.sample_many(rnds, out_old)
                row["picks_identical"] = bool(np.array_equal(out_new, out_old))
            ts = {"new": [], "parent": []}
            rounds = a.rounds if (old is None or shots < 1000000) else 2
            for r in range(rounds):
                order = ("new", "parent") if r % 2 == 0 else ("parent", "new")
                for which in order:
                    if which == "new":
                        ts["new"].append(new.block(rnds, out_new, reps))
                    elif old is not None:
                        ts["parent"].append(old.block(rnds, out_old, reps))
            row["sample_many_ms"] = [round(t, 3) for t in ts["new"]]
            if old is not None:
                row["parent_sample_many_ms"] = [round(t, 3) for t in ts["parent"]]
                row["parent_over_new"] = round(statistics.median(ts["parent"]) / statistics.median(ts["new"]), 3)
            calls.append(lambda new=new, rnds=rnds, out=out_new: new.sample_many(rnds, out))
            row["state_reads_at_most"] = round(1 + np.unique(out_new >> np.uint64(14)).size / nchunks, 4)
            t0 = time.perf_counter()
            res = q.MultiShotMeasureMask([1 << b for b in range(nq)], shots)
            row["multishot_all_qubits_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
            assert sum(res.values()) == shots
            rows.append(row)
        if old is not None:
            old.lib.b200sv_destroy(old.h)
        keep.append(q)  # profiled at the end, in one session
    for row, ms in zip(rows, kernel_ms(calls)):
        row["kernel_ms"] = ms
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
