"""Times the lossy checkpoint pair (b200sv_lossy_save / b200sv_lossy_load, p = 6, b = 4) on the resident state:

  * kernel time: the k_lossy_encode / k_lossy_decode launches of one save and one load, summed from a torch.profiler trace
    with CUDA activities (a separate run from the end-to-end timing);
  * end to end: host clock around LossySave / LossyLoad (file written to and read from a temporary directory), mean of
    --reps calls after a warm-up;
  at 26, 28 and 30 qubits fp32 and 29 qubits fp64 (a U3 layer and CNOTs, so every block is dense);
  * for contrast, the reference's codec on the host (the StateVectorTurboQuant code the QInterface default runs, here through
    the reference's QEngineCPU compiled into dropin/_build) at --host-qubits, when that build is present;

and prints the card's name and power limit beside the numbers, one JSON line per measurement.

    python scripts/lossy_timing.py [--reps R] [--sizes 26:32,28:32,30:32,29:64] [--host-qubits 18]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
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


def prepare(n, prec):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    rng = random.Random(n)
    for t in range(n):
        q.U(t, rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3))
    for t in range(0, n - 1, 2):
        q.CNOT(t, t + 1)
    q.Finish()
    return q


def kernel_ms(q, path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        q.be.lossy_save(path, 6, 4, 12345)
        q.be.lossy_load(path)
        torch.cuda.synchronize()
    out = {"k_lossy_encode": 0.0, "k_lossy_decode": 0.0}
    for e in prof.key_averages():
        for k in out:
            if k in e.key:
                out[k] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="26:32,28:32,30:32,29:64")
    ap.add_argument("--host-qubits", type=int, default=18)
    a = ap.parse_args()
    name, power = card()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "state.svtq")
        for spec in a.sizes.split(","):
            n, prec = (int(x) for x in spec.split(":"))
            q = prepare(n, prec)
            q.be.lossy_save(path, 6, 4, 12345)  # warm-up: module load, staging allocation, page cache
            q.be.lossy_load(path)
            q.Finish()
            ts, tl = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                q.be.lossy_save(path, 6, 4, 12345)
                ts.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                q.be.lossy_load(path)
                q.Finish()
                tl.append(time.perf_counter() - t0)
            k = kernel_ms(q, path)
            nblocks = 1 << (n - 6)
            print(json.dumps({"qubits": n, "precision": prec, "file_bytes": os.path.getsize(path),
                              "save_s": [round(x, 3) for x in ts], "load_s": [round(x, 3) for x in tl],
                              "encode_kernel_ms": round(k["k_lossy_encode"], 2), "decode_kernel_ms": round(k["k_lossy_decode"], 2),
                              # 128 x 128 multiply-adds per block, each a separate multiply and add
                              "encode_gflops": round(2 * nblocks * 128 * 128 / (k["k_lossy_encode"] * 1e6), 1)
                              if k["k_lossy_encode"] else None,
                              "gpu": name, "power_limit": power}), flush=True)
            del q
        harness = os.path.join(ROOT, "dropin", "_build", "observables_b200_f32")
        if os.path.exists(harness):
            # --engine cpu: the reference's own QEngineCPU, compiled unchanged into the drop-in build.  Host clock around the
            # harness process, less the same process with the circuit alone.
            n = a.host_qubits
            env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "qrack_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
            circ = "qubits %d\n" % n + "".join("U %d 0.3 0.2 0.1\n" % t for t in range(n))
            scripts = {"base": circ, "save": circ + "LossySave %s 6 4\n" % path, "load": "qubits %d\nLossyLoad %s\n" % (n, path)}
            wall = {}
            for what, text in scripts.items():
                sp = os.path.join(td, what + ".qs")
                open(sp, "w").write(text)
                t0 = time.perf_counter()
                subprocess.run([harness, sp, "--engine", "cpu"], capture_output=True, check=True, env=env)
                wall[what] = time.perf_counter() - t0
            print(json.dumps({"qubits": n, "precision": 32, "save_s": round(wall["save"] - wall["base"], 3),
                              "load_s": round(wall["load"] - wall["base"], 3),
                              "engine": "reference QEngineCPU codec on the host (drop-in build, --engine cpu)",
                              "gpu": name, "power_limit": power}), flush=True)

if __name__ == "__main__":
    main()
