"""W ranks of the sharded engine as W processes on ONE CUDA device (test infrastructure).

The ranks talk over a loopback gloo group (NCCL refuses two ranks on one device).  `StagedDist` is the `dist` the engine
is given: it stages every collective and point-to-point transfer of a CUDA tensor through host copies and passes the rest
through, and its barrier synchronises the device first.  The P2P exchange (qrack_b200.sharded.P2PShardBuffers) relies on
a stream-ordered barrier: a peer's page may be read once every rank's queued sweeps on it have run, which a plain host
barrier does not guarantee.  CUDA IPC works between processes on the same device, so the P2P pages, their peer mappings,
the push scatter and the pull gather run unmodified; peer pointers map the other processes' pages.

What this harness cannot see: stream-ordering races between ranks (its barrier synchronises the whole device) and the
NCCL branch of the exchange."""
import datetime
import os
import socket

import torch
import torch.distributed as tdist
import torch.multiprocessing as mp

# one failing rank must not leave the others blocked in a collective for gloo's default 30 minutes
TIMEOUT = datetime.timedelta(seconds=120)


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _Staged:
    """a point-to-point transfer in flight: the host buffer stays referenced until wait(), which then copies a received
    buffer into its destination tensor"""

    def __init__(self, work, host, dst=None):
        self.work, self.host, self.dst = work, host, dst

    def wait(self, timeout=None):
        self.work.wait()
        if self.dst is not None:
            self.dst.copy_(self.host)
            self.dst = None
        return True

    def is_completed(self):
        return self.dst is None and self.work.is_completed()


class _P2POp:
    def __init__(self, op, tensor, peer, group=None, tag=0):
        self.op, self.tensor, self.peer = op, tensor, peer


class StagedDist:
    """torch.distributed for ranks that share one device over gloo: CUDA tensors go through host copies, `barrier()`
    synchronises `device` first (no synchronisation without a CUDA device); everything else is torch.distributed's"""

    P2POp = _P2POp

    def __init__(self, device=None):
        self.device = device if device is not None and torch.device(device).type == "cuda" else None

    def __getattr__(self, name):
        return getattr(tdist, name)

    def get_backend(self, group=None):
        return "gloo"

    def barrier(self, group=None):
        if self.device is not None:
            torch.cuda.synchronize(self.device)
        tdist.barrier()

    def all_reduce(self, tensor, op=tdist.ReduceOp.SUM, group=None, async_op=False):
        host = tensor.cpu()
        tdist.all_reduce(host, op=op)
        if host is not tensor:
            tensor.copy_(host)

    def all_gather(self, tensor_list, tensor, group=None, async_op=False):
        host = [torch.empty_like(t, device="cpu") for t in tensor_list]
        tdist.all_gather(host, tensor.cpu())
        for t, h in zip(tensor_list, host):
            t.copy_(h)

    def isend(self, tensor, dst, group=None, tag=0):
        host = tensor.to("cpu", copy=True)      # a snapshot: the source may be overwritten before the peer receives it
        return _Staged(tdist.isend(host, dst, tag=tag), host)

    def irecv(self, tensor, src=None, group=None, tag=0):
        host = torch.empty_like(tensor, device="cpu")
        return _Staged(tdist.irecv(host, src, tag=tag), host, tensor)

    def batch_isend_irecv(self, p2p_op_list):
        return [op.op(op.tensor, op.peer) for op in p2p_op_list]


def _entry(rank, world, port, use_cuda, staged, fn, args):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    device = None
    if use_cuda:
        torch.cuda.set_device(0)
        device = torch.device("cuda", 0)
    tdist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    try:
        fn(rank, world, StagedDist(device) if staged else tdist, *args)
    finally:
        tdist.destroy_process_group()


def spawn(fn, world, *args, use_cuda=True, staged=True):
    """fn(rank, world, dist, *args) in `world` processes over one loopback gloo group, every rank on cuda:0 (use_cuda) or
    on the CPU; dist is a StagedDist (staged) or torch.distributed itself.  `fn` must be a module-level function.  Returns
    when every rank has; a failing rank's exception is raised here after the others have been terminated."""
    for attempt in range(3):  # the rendezvous port can be taken between probing and binding
        try:
            mp.spawn(_entry, args=(world, free_port(), use_cuda, staged, fn, args), nprocs=world, join=True)
            return
        except Exception as e:
            if "EADDRINUSE" not in str(e) or attempt == 2:
                raise
