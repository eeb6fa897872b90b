"""Times the cross-page Pauli sweep (b200sv_expectation_pauli_pair) against the local one (b200sv_expectation_pauli) on one
GPU, with CUDA events on the engine's stream (b200sv_timer_begin/_end), mean of R calls after a warm-up.  The partner is a
second page on the same device.  Read rate = the bytes each sweep must read over its time: two pages for the pair sweep, one
for the local sweep, against the 3.35 TB/s HBM3 data-sheet figure.  The card's name and power limit are printed beside the
numbers.

With >= 2 GPUs it also times the sharded end-to-end ExpectationPauliAll with X on a rank-bit qubit in pull mode (the partner
page read through its peer mapping), max over ranks, and prints "not measured" for that row otherwise.

    python scripts/sharded_pauli_timing.py [--reps R] [--sizes 28:32,30:32,29:64] [--shard-local 28]
"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from qrack_b200 import QEngineCUDA, _abi  # noqa: E402

HBM = 3.35e12


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


def random_state(n, prec, seed):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, False, False, precision=prec)
    rng = random.Random(seed)
    for b in range(n):
        q.U(b, rng.uniform(0, 3), rng.uniform(-3, 3), rng.uniform(-3, 3))
    for b in range(0, n - 1, 2):
        q.CNOT(b, b + 1)
    q.Finish()
    return q


def _shard_worker(rank, world, port, nl, reps, out_path):
    import torch
    import torch.distributed as dist
    os.environ["B200SV_SHARD_PULL"] = "1"
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from qrack_b200.sharded import QEngineSharded
        k = world.bit_length() - 1
        n = nl + k
        q = QEngineSharded(n, 0, random.Random(1), 1.0 + 0j, precision=32, dist=dist, world=world, rank=rank,
                           device=torch.device("cuda", rank), p2p=True)
        for b in range(n):
            q.H(b)
        q.Finish()
        rq = [b for b in range(n) if q.be.perm[b] >= nl][0]
        loc = [b for b in range(n) if q.be.perm[b] < nl]
        bits, paulis = [rq, loc[0], loc[len(loc) // 2]], [1, 3, 2]
        q.ExpectationPauliAll(bits, paulis)  # warm-up
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            q.ExpectationPauliAll(bits, paulis)
        t1.record()
        t1.synchronize()
        ms = torch.tensor([t0.elapsed_time(t1) / reps], device=torch.device("cuda", rank))
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        if rank == 0:
            with open(out_path, "w") as f:
                json.dump({"world": world, "qubits": n, "local_qubits": nl, "ms": ms.item(), "exchanges": q.be.exchanges}, f)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="28:32,30:32,29:64")
    ap.add_argument("--shard-local", type=int, default=28)
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power))
    lib = _abi.load()
    for spec in a.sizes.split(","):
        n, prec = (int(v) for v in spec.split(":"))
        q, p = random_state(n, prec, 5), random_state(n, prec, 6)
        ptr = ctypes.c_void_p()
        _abi.check(lib, lib.b200sv_device_ptr(p.be.h, ctypes.byref(ptr)))
        top = n - 1  # the pair sweep's x: what stays of a rank-bit X / Y once the rank part is split off
        x, z = (1 << top) | 1 | (1 << (n // 2)), 0b110 | (1 << (n - 2))
        t_pair = timed(q, lambda: q.be.expectation_pauli_pair(ptr.value, x, z), a.reps)
        t_local = timed(q, lambda: q.be.expectation_pauli(x, z), a.reps)
        page = (1 << n) * (8 if prec == 32 else 16)
        print(json.dumps({"qubits": n, "precision": prec, "card": name, "power_limit": power,
                          "pair_sweep_ms": round(t_pair, 4), "pair_read_TBps": round(2 * page / t_pair / 1e9, 3),
                          "pair_share_of_hbm": round(2 * page / (t_pair * 1e-3) / HBM, 3),
                          "local_sweep_ms": round(t_local, 4), "local_read_TBps": round(page / t_local / 1e9, 3),
                          "local_share_of_hbm": round(page / (t_local * 1e-3) / HBM, 3)}))
        del q, p
    import torch
    ng = torch.cuda.device_count()
    if ng < 2:
        print(json.dumps({"sharded_expectation_pauli_rank_bit_x": "not measured (needs >= 2 GPUs)"}))
        return
    import tempfile
    import socket
    import torch.multiprocessing as mp
    world = 1 << (min(ng, 8).bit_length() - 1)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "shard.json")
        mp.spawn(_shard_worker, args=(world, port, a.shard_local, a.reps, out), nprocs=world, join=True)
        r = json.load(open(out))
    r.update({"card": name, "power_limit": power, "mode": "pull", "sharded_expectation_pauli_rank_bit_x_ms": round(r.pop("ms"), 4)})
    print(json.dumps(r))


if __name__ == "__main__":
    main()
