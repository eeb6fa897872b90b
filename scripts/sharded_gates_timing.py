"""Cost of FSim / ISwap layers on the sharded engine.

Host (no GPU): replays one layer of each kind through QEngineSharded's real scheduler with the data-free shard of
scripts/shard_sweep_count.py and the real fused planner, and prints the exchanges and sweeps the layer costs.  A two-target
gate is queued as CNOT, a single-target gate and CNOT, so a layer of them on 30 local + k rank qubits should cost what a
layer of single-target gates on the same qubits costs: one exchange when a rank-bit qubit is touched, and a few sweeps.

GPU (`--gpu`): times a 30-qubit FSim random circuit on the sharded engine, W ranks as W processes on one device (the
tests' one-device harness), and prints the card's name and power limit with the time.  Without `--gpu`, or without a device,
every time is "not measured"."""
import argparse
import os
import random
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from qrack_b200 import qscript  # noqa: E402

import shard_sweep_count  # noqa: E402


def layer(n, kind, seed):
    """U3 on every qubit, then `kind` on a random matching"""
    rng = random.Random(seed)
    text = "qubits %d\n" % n
    for q in range(n):
        text += "U %d %.17g %.17g %.17g\n" % (q, rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3))
    for a, b in qscript.random_matching(rng, n):
        text += ("FSim %.17g %.17g %d %d\n" % (rng.uniform(-3, 3), rng.uniform(-3, 3), a, b)) if kind == "FSim" else \
            ("%s %d %d\n" % (kind, a, b))
    return text


def host_counts(worlds, layers=4):
    print("host: exchanges and fused sweeps per layer (the real scheduler and planner, 30 local qubits, rank 0)")
    for world in worlds:
        k = world.bit_length() - 1
        n = 30 + k
        for kind in ("CNOT", "ISwap", "FSim"):
            text = "qubits %d\n" % n + "".join(layer(n, kind, s).split("\n", 1)[1] for s in range(layers))
            ex, rows = shard_sweep_count.windows(30, world, 0, text)
            print("  world %d %-5s: %.2f exchanges, %.2f sweeps per layer (%d layers)"
                  % (world, kind, ex / layers, sum(r[1] for r in rows) / layers, layers))


def _ranks(rank, world, dist, n, layers, prec, out):
    import numpy as np
    import torch
    from qrack_b200.sharded import QEngineSharded, cuda_engine_factory
    dev = torch.device("cuda", 0)
    q = QEngineSharded(n, 0, random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank, device=dev,
                       make_engine=cuda_engine_factory(0, prec), p2p=True)
    text = "".join(layer(n, "FSim", s).split("\n", 1)[1] for s in range(layers))
    qscript.run("qubits %d\n" % n + text, lambda nq, p: q)   # warm-up: every kernel compiled and loaded
    q.Finish()
    dist.barrier()
    t0 = time.perf_counter()
    qscript.run("qubits %d\n" % n + text, lambda nq, p: q)
    q.Finish()
    dist.barrier()
    dt = time.perf_counter() - t0
    if rank == 0:
        np.save(out, np.array([dt, q.be.exchanges]))


def gpu_time(n, world, layers, prec):
    import numpy as np
    import tempfile
    import torch
    if not torch.cuda.is_available():
        print("gpu: %d-qubit FSim circuit over %d ranks: not measured (no device)" % (n, world))
        return
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
    import one_device
    import subprocess
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name(0)
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "t.npy")
        one_device.spawn(_ranks, world, n, layers, prec, out)
        dt, ex = np.load(out)
    gates = layers * (n + n // 2)
    print("gpu (%s): %d-qubit fp%d FSim circuit, %d layers (%d gates) over %d ranks on one device: %.3f s, %.1f ms per layer, "
          "%d exchanges in all (warm-up included)" % (card, n, prec, layers, gates, world, dt, 1e3 * dt / layers, ex))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--qubits", type=int, default=30)
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--layers", type=int, default=8)
    args = ap.parse_args()
    host_counts([2, 8])
    if args.gpu:
        gpu_time(args.qubits, args.world, args.layers, 32)
    else:
        print("gpu: %d-qubit FSim circuit over %d ranks: not measured" % (args.qubits, args.world))
