"""One-process-per-GPU sharding of one state vector: the multi-GPU analogue of the reference's ``QPager``.

Partition (reference ``include/qpager.hpp:60-69``, ``src/qpager.cpp:57-67``): with ``W = 2^k`` ranks the top ``k`` index
bits are the rank, every rank holds one page of ``2^(n-k)`` amplitudes.  What differs from QPager is how a gate on a
device-index ("meta") qubit is served.  QPager does swap–compute–swap with two half-page ``ShuffleBuffers`` per gate
(``src/qpager.cpp:425-432``); here the engine keeps a *logical→physical qubit map* and, when a non-diagonal gate needs a
qubit that currently lives in the rank bits, does **one all-to-all that exchanges all k rank bits with the top k local
bits** (each rank keeps 1/W of its page and ships the rest over NVLink/NVSwitch — NCCL ``all_to_all_single``), choosing
the qubits that become the new rank bits with Belady's rule over the queued gate list (farthest next non-diagonal use).
Everything else needs no data motion: gates on local qubits run on the local engine (the fused sweep), diagonal gates on
rank-bit qubits are per-rank scalars or predicated local phases, controls on rank-bit qubits just select which ranks run
(QPager's meta-controlled cases, ``src/qpager.cpp:452-593``), scalars (Prob, norms) are one ``all_reduce``.  The observable
moments and Pauli strings are per-rank read-only sweeps and one ``all_reduce`` too; a Pauli string with X or Y on a rank-bit
qubit pairs each page with one partner page, read in place or received into the spare buffer, with no exchange.
``HighestProbAll(n)`` is a per-rank radix select whose ties go to the smaller LOGICAL index, then one ``all_gather`` of every
rank's best min(n, page) entries and a merge.  ``MultiShotMeasureMask`` over more than 16 qubits samples every shot as
``MAll``'s search would: each rank searches its page on the device for the shots that land there, returning logical indices,
and one ``all_reduce`` of a slot per shot gathers them.  A two-target gate (ISwap, SqrtSwap, FSim, CSwap, ...) is queued as
CNOT, a single-target gate, CNOT, so it is scheduled, deferred and fused like any other gate; ``(C)UniformParityRZ`` is a
per-rank sign of the angle on the local parity kernel; ``UniformlyControlledSingleBit`` turns rank-bit controls into skip
powers of the local kernel's table and makes a rank-bit target local with the scheduler's exchange.

``QEngineSharded`` derives from ``QEngineHost`` — the same gate dispatch mirror as ``QEngineCUDA`` — and supplies a
backend whose primitives are distributed, so the gate-level ``QInterface`` methods (H, T, CNOT, MC/MAC gates, the Swap family,
FSim, (C)UniformParityRZ, UniformlyControlledSingleBit / RY / RZ, QFT, INC/DEC,
ZeroPhaseFlip, Prob*, ForceM, M, MAll, MultiShotMeasureMask, HighestProbAll, HighestProbAll(n), ProbMaskAll,
Expectation/Variance{BitsAll, BitsFactorized, FloatsFactorized, PauliAll}, ExpectationUnitaryAll past 12 qubits, …) work
unchanged on top of it.  Primitives
that are not sharded (Compose/Decompose, ForceMParity, SumSqrDiff, the register expectation primitive, the
per-qubit basis sweep behind ExpectationUnitaryAll up to 12 qubits, reduced density matrices, the single-vector top-n
primitive ``highest_probs``, lossy checkpoints, the native QAlu sweeps, page ops) raise ``NotImplementedError`` identically
on every rank.  The local engine and the communicator are injected: ``QEngineCUDA`` over a torch CUDA buffer +
NCCL on the GPU box; the oracle restatement over a torch CPU buffer + gloo in the CPU tests.
"""
from __future__ import annotations

import math
import os
import random
from typing import Callable, List, Optional, Sequence

import numpy as np

from .qengine import QEngineHost, REAL1_DEFAULT_ARG, X_MTRX, lower_two_target


def _bits(mask: int):
    q = 0
    while mask:
        if mask & 1:
            yield q
        mask >>= 1
        q += 1


class ShardBuffers:
    """Two page-sized torch buffers (real view, interleaved re/im) + the local engine bound to the active one."""

    def __init__(self, n_local: int, precision: int, device, make_engine: Callable):
        import torch
        self.torch = torch
        self.nl = n_local
        self.precision = precision
        self.rdtype = torch.float32 if precision == 32 else torch.float64
        self.device = device
        self.buf = torch.zeros(2 << n_local, dtype=self.rdtype, device=device)
        self.scratch = torch.empty(2 << n_local, dtype=self.rdtype, device=device)
        self.make_engine = make_engine
        self.engine = make_engine(self.buf, n_local)
        self.retired_stats = {}

    def _retire(self):
        st = getattr(self.engine.be, "stats", None)
        if st is not None:
            for k, v in st().items():
                self.retired_stats[k] = self.retired_stats.get(k, 0) + v

    def stats(self) -> dict:
        """kernel/launch counters of every local engine this page has had (a new one is bound after each exchange)"""
        out = dict(self.retired_stats)
        st = getattr(self.engine.be, "stats", None)
        if st is not None:
            for k, v in st().items():
                out[k] = out.get(k, 0) + v
        return out

    needs_top = True  # the all-to-all exchanges the TOP k local bits: victims must be moved there first
    min_victim_bit = 0
    chunk_floor = 0   # local swaps bring any local qubit to the top

    def zero_live(self):
        self.buf.zero_()

    def local_host(self, cplx) -> np.ndarray:
        return self.buf.cpu().numpy().view(cplx)

    def exchange(self, dist, world, rank, k, victim_bits):
        """all k rank bits <-> top k local bits: chunk j of this page goes to rank j and lands there as chunk `rank`"""
        src, dst = self.buf, self.scratch
        if dist.get_backend() == "nccl":
            self.engine.be.flush()  # NCCL runs on the same (torch current) stream as the engine: stream order suffices
            dist.all_to_all_single(dst, src)
        else:
            self.engine.Finish()
            chunk = src.numel() // world
            reqs = []
            for peer in range(world):
                if peer == rank:
                    dst[peer * chunk:(peer + 1) * chunk].copy_(src[peer * chunk:(peer + 1) * chunk])
                else:
                    reqs.append(dist.isend(src[peer * chunk:(peer + 1) * chunk], peer))
                    reqs.append(dist.irecv(dst[peer * chunk:(peer + 1) * chunk], peer))
            for r in reqs:
                r.wait()
        self.swap()
        return src.numel() * src.element_size() * (world - 1) // world

    def partner_page(self, dist, world, rank, partner):
        """`partner`'s current page, readable by the local engine: the two ranks swap whole pages into their `scratch`
        buffers (rank <-> partner is a perfect matching, so every rank sends and receives exactly once).  The live page is
        not written; `scratch` holds nothing between exchanges."""
        if dist.get_backend() == "nccl":
            self.engine.be.flush()  # same stream as NCCL's send (see exchange)
        else:
            self.engine.Finish()
        reqs = dist.batch_isend_irecv([dist.P2POp(dist.isend, self.buf, partner), dist.P2POp(dist.irecv, self.scratch, partner)])
        for r in reqs:
            r.wait()
        return self.scratch.data_ptr()

    def swap(self):
        """the exchange wrote into `scratch`: make it the live page"""
        self.buf, self.scratch = self.scratch, self.buf
        rebind = getattr(self.engine.be, "rebind_external", None)
        if rebind is not None:
            rebind(self.buf.data_ptr())  # same handle, same stream: ordered behind the exchange
            self.engine.runningNorm = REAL1_DEFAULT_ARG
        else:
            self.engine.Finish()
            self._retire()
            self.engine = self.make_engine(self.buf, self.nl)


class P2PShardBuffers:
    """CUDA pages owned by libb200sv (cudaMalloc, exported with CUDA IPC) + the fused NVLink re-page kernel
    (b200sv_exchange_scatter): the k rank bits are exchanged with ANY k local qubits in one pass that reads the page once
    and stores straight into the peers' pages — no local pre-permutation, no NCCL staging."""

    needs_top = False
    min_victim_bit = 8  # keep >= 2 KB contiguous runs per destination (preferred)
    # the re-page kernels move whole 16-byte chunks: an fp32 chunk holds qubit 0, which can never be a victim (hard floor)
    CHUNK_FLOOR = {32: 1, 64: 0}

    def __init__(self, n_local: int, precision: int, device_index: int, dist, world: int, rank: int):
        import ctypes
        import torch
        from . import _abi
        from .qengine import QEngineCUDA
        self.chunk_floor = self.CHUNK_FLOOR[precision]
        self.torch, self.dist, self.world, self.rank = torch, dist, world, rank
        self.lib = _abi.load()
        self.abi = _abi
        self.nl, self.precision, self.dev = n_local, precision, device_index
        self.device = torch.device("cuda", device_index)
        self.nbytes = (1 << n_local) * (8 if precision == 32 else 16)
        self.pages = []
        for _ in range(2):
            p = ctypes.c_void_p()
            _abi.check(self.lib, self.lib.b200sv_alloc_page(device_index, self.nbytes, ctypes.byref(p)))
            self.pages.append(p.value)
        # exchange the IPC handles of both pages
        mine = torch.zeros(2, 64, dtype=torch.uint8)
        for i, p in enumerate(self.pages):
            hb = (ctypes.c_ubyte * 64)()
            _abi.check(self.lib, self.lib.b200sv_ipc_export(device_index, ctypes.c_void_p(p), hb))
            mine[i] = torch.tensor(list(hb), dtype=torch.uint8)
        allh = [torch.empty(2, 64, dtype=torch.uint8, device=self.device) for _ in range(world)]
        dist.all_gather(allh, mine.to(self.device))
        self.peer_pages = []  # [rank][page] -> device pointer valid in THIS process
        for r in range(world):
            if r == rank:
                self.peer_pages.append(list(self.pages))
                continue
            ptrs = []
            hr = allh[r].cpu()
            for i in range(2):
                hb = (ctypes.c_ubyte * 64)(*hr[i].tolist())
                p = ctypes.c_void_p()
                _abi.check(self.lib, self.lib.b200sv_ipc_import(device_index, hb, ctypes.byref(p)))
                ptrs.append(p.value)
            self.peer_pages.append(ptrs)
        self.live = 0
        self.pull = os.environ.get("B200SV_SHARD_PULL", "1") != "0"  # 0: the push kernel (b200sv_exchange_scatter), one pass per exchange
        self.engine = QEngineCUDA.over_buffer(self.pages[0], n_local, device_index, precision, random.Random(1))
        self.engine.be.set_stream(torch.cuda.current_stream(self.device).cuda_stream)
        self.zero_live()
        dist.barrier()

    def zero_live(self):
        self.engine.be.zero()

    def local_host(self, cplx) -> np.ndarray:
        return self.engine.be.get_state()

    def stats(self) -> dict:
        return self.engine.be.stats()

    def exchange(self, dist, world, rank, k, victim_bits):
        import ctypes
        other = 1 - self.live
        vb = (ctypes.c_int * k)(*victim_bits)
        be = self.engine.be
        if self.pull and k <= 3:
            # PULL mode (b200sv_exchange_pull): nothing moves now.  The first fused sweep of the next window reads its tiles straight
            # from the ranks' current pages through the peer mappings and writes this rank's other page, so the re-page costs no pass
            # of its own.  Ordering: the flush puts the old window's last sweeps (and an earlier pending pull, which still reads the
            # peers' previous pages) on the stream, the stream-ordered barrier then says every rank's current page is final and
            # nobody reads my other page any more; the current pages stay untouched until the barrier of the next exchange.
            be.flush()
            dist.barrier()
            src = (ctypes.c_void_p * world)(*[self.peer_pages[r][self.live] for r in range(world)])
            be._ck(self.lib.b200sv_exchange_pull(be.h, k, vb, rank, src, ctypes.c_void_p(self.pages[other])))
            self.live = other
            self.engine.runningNorm = REAL1_DEFAULT_ARG
            return self.nbytes * (world - 1) // world
        dst = (ctypes.c_void_p * world)(*[self.peer_pages[r][other] for r in range(world)])
        be._ck(self.lib.b200sv_exchange_scatter(be.h, k, vb, rank, dst))
        # every rank's stores into my `other` page are complete once the stream-ordered barrier has completed everywhere
        dist.barrier()
        self.live = other
        be.rebind_external(self.pages[other])
        self.engine.runningNorm = REAL1_DEFAULT_ARG
        return self.nbytes * (world - 1) // world

    def partner_page(self, dist, world, rank, partner):
        """`partner`'s current page through its peer mapping, no copy.  The flush puts this rank's queue (and a pending pull
        gather) on the stream; after the stream-ordered barrier every rank's current page is final.  The caller's all-reduce
        after the read is the closing barrier: no rank writes its page again before every partner has read it."""
        self.engine.be.flush()
        dist.barrier()
        return self.peer_pages[partner][self.live]


def cuda_engine_factory(device_index: int, precision: int = 32):
    """local engine = QEngineCUDA over the torch buffer, running on torch's current stream"""
    def make(buf, n_local):
        import torch
        from .qengine import QEngineCUDA
        q = QEngineCUDA.over_buffer(buf.data_ptr(), n_local, device_index, precision, random.Random(1))
        q.be.set_stream(torch.cuda.current_stream(torch.device("cuda", device_index)).cuda_stream)
        return q
    return make


def _table_index(offset: int, skip_powers) -> int:
    """UniformlyControlledSingleBit's table index of a control offset: a zero bit inserted at each skip power, in the
    order given (state.cpp:1130-1137)"""
    i, hi = 0, offset
    for p in skip_powers:
        low = hi & (p - 1)
        i |= low
        hi = (hi ^ low) << 1
    return i | hi


class _Gate:
    __slots__ = ("t", "cmask", "cval", "m", "diag")

    def __init__(self, t, cmask, cval, m):
        self.t, self.cmask, self.cval, self.m = t, cmask, cval, m
        self.diag = (m[1] == 0 and m[2] == 0)


def rank_walk(tots, rnds):
    """_ShardedBackend.sample's walk over the page totals for every rnd at once: (the rank whose page it searches, the rnd
    it passes there), the rank -1 where every page is zero.  np.cumsum adds in order, so cum holds the doubles of sample's
    running sum (a page with total 0 adds 0.0, which changes nothing).  Past the total, the last nonzero page is searched
    with rnd - (cum - tots[last]): the total less that page, not the sum of the pages before it."""
    tots = np.asarray(tots, dtype=np.float64)
    rnds = np.asarray(rnds, dtype=np.float64)
    live = tots > 0
    if not live.any():
        return np.full(rnds.size, -1, dtype=np.int64), rnds.copy()
    cum = np.cumsum(np.where(live, tots, 0.0))
    before = np.concatenate(([0.0], cum[:-1]))
    hit = live[None, :] & (cum[None, :] > rnds[:, None])
    found = hit.any(axis=1)
    last = int(np.flatnonzero(live)[-1])
    pick = np.where(found, hit.argmax(axis=1), last).astype(np.int64)
    res = np.where(found, rnds - before[pick], rnds - (cum[-1] - tots[last]))
    return pick, res


def merge_top_n(keys: np.ndarray, probs: np.ndarray, n: int) -> list:
    """the n keys of largest P among (keys, probs) pairs, ties to the smaller key; P = 0 (and padding) never listed, the
    list zero-filled past the last P > 0"""
    live = probs > 0
    keys, probs = keys[live], probs[live]
    o = np.lexsort((keys, -probs))[:n]
    return [int(v) for v in keys[o]] + [0] * (n - o.size)


class _ShardedBackend:
    """Backend primitives (see qengine.QEngineHost) over W ranks; indices and masks arrive in LOGICAL qubit order."""

    def __init__(self, n_qubits: int, precision: int, shard: Optional[ShardBuffers], dist, world: int, rank: int):
        self.n = n_qubits
        self.precision = precision
        self.dist = dist
        self.world = world
        self.rank = rank
        self.k = int(round(math.log2(world))) if world > 1 else 0
        assert (1 << self.k) == world, "world size must be a power of two"
        self.nl = n_qubits - self.k
        self.shard = shard
        self.cplx = np.complex64 if precision == 32 else np.complex128
        self.real = np.float32 if precision == 32 else np.float64
        self.perm = list(range(n_qubits))  # logical qubit -> physical index bit (>= nl: rank bit)
        self.pending: List[_Gate] = []
        self.defer_exchanges = os.environ.get("B200SV_SHARD_DEFER", "1") != "0"
        self.exchanges = 0
        self.exchange_bytes = 0
        self.local_swaps = 0
        self._batch = []  # local single-target gates waiting for ONE b200sv_apply_gates call (SURVEY N4)
        # X gates are never executed: |psi_logical> = X^{xinv} |psi_stored>.  An X (XMask) toggles bits of `xinv`; every later
        # gate is conjugated (control polarities flip, a target's matrix becomes X m X), every index that goes to or comes
        # from the stored state is XORed.  QInterface::MACWrapper (include/qinterface.hpp:179-189) wraps each anti-controlled
        # gate of INC/DEC/ZeroPhaseFlip in XMask ... XMask: on rank-bit qubits those would each cost a page exchange.
        self.xinv = 0

    # ---- helpers ------------------------------------------------------------------------------------------------
    @property
    def loc(self):
        return self.shard.engine

    def _pmask(self, mask: int) -> int:
        out = 0
        for q in _bits(mask):
            out |= 1 << self.perm[q]
        return out

    def _pindex(self, idx: int) -> int:
        out = 0
        for q in _bits(idx):
            out |= 1 << self.perm[q]
        return out

    def _stored(self, idx: int, mask: Optional[int] = None) -> int:
        """logical basis index -> the logical-qubit-ordered index of the STORED vector (pending X inversions applied)"""
        return idx ^ (self.xinv if mask is None else (self.xinv & mask))

    def _split(self, pmask: int):
        lm = pmask & ((1 << self.nl) - 1)
        return lm, pmask >> self.nl

    def _allreduce(self, vals: Sequence[float]) -> List[float]:
        if self.world == 1:
            return list(vals)
        torch = self.shard.torch
        t = torch.tensor(list(vals), dtype=torch.float64, device=self.shard.device)
        self.dist.all_reduce(t)
        return t.tolist()

    # ---- lifecycle / trivial --------------------------------------------------------------------------------------
    def resize_zero(self, n):
        raise NotImplementedError("sharded states have a fixed width")

    def finish(self):
        self.flush()
        self.loc.Finish()

    def is_zero(self) -> bool:
        return False

    def zero(self):
        self.pending.clear()
        self.loc.Finish()
        self.shard.zero_live()

    def set_permutation(self, perm: int, phase: complex):
        self.pending.clear()
        self.xinv = 0
        self.perm = list(range(self.n))
        self.loc.Finish()
        self.shard.zero_live()
        if (perm >> self.nl) == self.rank:
            self.loc.SetAmplitude(perm & ((1 << self.nl) - 1), phase)
        self.loc.runningNorm = REAL1_DEFAULT_ARG

    # ---- gates ------------------------------------------------------------------------------------------------------
    def apply2x2(self, off1, off2, mtrx, pows, nrm, thresh, calc_norm):
        if calc_norm or nrm != 1.0:
            raise NotImplementedError("doNormalize is not supported on the sharded engine (QPager forces it off too)")
        pmask = 0
        for p in pows:
            pmask |= p
        diff = off1 ^ off2
        if diff and not (diff & (diff - 1)):
            t = diff.bit_length() - 1
            m = list(mtrx)
            if off1 & diff:  # off1 holds the |1> branch
                m = [m[3], m[2], m[1], m[0]]
            cmask = pmask & ~diff
            if not cmask and m[0] == 0 and m[3] == 0 and m[1] == 1 and m[2] == 1:
                self.xinv ^= 1 << t                             # a bare X: one more inversion, nothing to execute
                return None
            cval = (off1 & ~diff) ^ (self.xinv & cmask)      # control polarities see the stored bits
            if (self.xinv >> t) & 1:
                m = [m[3], m[2], m[1], m[0]]                    # X m X
            self.pending.append(_Gate(t, cmask, cval, m))
            return None
        if bin(diff).count("1") == 2 and pmask == diff and mtrx[0] == 0 and mtrx[3] == 0 and mtrx[1] == 1 and mtrx[2] == 1:
            # uncontrolled Swap: relabel, no data motion (QPager::Swap does the same for meta qubits)
            self.flush()
            a, b = [q for q in _bits(diff)]
            self.perm[a], self.perm[b] = self.perm[b], self.perm[a]
            xa, xb = (self.xinv >> a) & 1, (self.xinv >> b) & 1
            if xa != xb:                                        # the pending inversions travel with the qubits
                self.xinv ^= (1 << a) | (1 << b)
            return None
        if bin(diff).count("1") == 2:
            # ISwap, SqrtSwap, FSim, controlled Swap ...: CNOT(p -> q), the gate on p, CNOT(p -> q) (lower_two_target).  Both
            # are non-diagonal targets, so a rank-bit target costs the one deferred exchange a single-target gate on it costs
            for o1, o2, pm, m in lower_two_target(off1, off2, pmask, mtrx):
                self.apply2x2(o1, o2, list(m), [pm], 1.0, thresh, False)
            return None
        raise NotImplementedError("Apply2x2 forms with more than two targets are not sharded")

    def xmask(self, mask):
        self.xinv ^= mask   # never executed: see __init__

    def phase_parity(self, radians, mask):
        self.flush()
        lm, gm = self._split(self._pmask(mask))
        sign = -1.0 if (bin(self.rank & gm).count("1") & 1) else 1.0
        if bin(self.xinv & mask).count("1") & 1:
            sign = -sign                                         # parity of the logical bits = stored parity ^ parity of the inversions
        if lm:
            self.loc.PhaseParity(sign * radians, lm)
        else:  # all qubits are rank bits: a per-rank scalar, e^{+i r/2} for odd parity, e^{-i r/2} for even (state.cpp:1035-1051)
            ang = (radians / 2) if sign < 0 else -(radians / 2)
            ph = complex(math.cos(ang), math.sin(ang))
            self.loc.Mtrx([ph, 0j, 0j, ph], 0)

    def uniform_parity_rz(self, cmask, mask, angle):
        """(C)UniformParityRZ: odd parity of the logical mask bits gets e^{i angle}, even parity e^{-i angle}, where every
        control is 1 (state.cpp:1200-1264).  Diagonal, so no exchange: the stored parity is the local bits' parity, this
        rank's rank-bit parity and the parity of the pending inversions on the mask; each odd one flips the angle's sign.
        Rank-bit controls select the ranks that run.  The kernel wants every local control's STORED bit to be 1, so a
        pending inversion on a local control is executed first (a local X) and cleared."""
        self.flush()
        for c in _bits(cmask & self.xinv):
            if self.perm[c] < self.nl:
                self._local_gate([], 0, list(X_MTRX), self.perm[c])
                self.xinv ^= 1 << c
        self._submit_batch()
        for c in _bits(cmask):
            pc = self.perm[c]
            if pc >= self.nl and ((self.rank >> (pc - self.nl)) & 1) == ((self.xinv >> c) & 1):
                return   # a rank-bit control that is 0 on this rank
        lc, _ = self._split(self._pmask(cmask))
        lm, gm = self._split(self._pmask(mask))
        if (bin(self.rank & gm).count("1") + bin(self.xinv & mask).count("1")) & 1:
            angle = -angle
        if lm or lc:
            self.loc.be.uniform_parity_rz(lc, lm, angle)
        else:  # no local bit in the mask, no local control: the parity is even on the page, a per-page scalar e^{-i angle}
            ph = complex(math.cos(angle), -math.sin(angle))
            self.loc.Mtrx([ph, 0j, 0j, ph], 0)

    def uniformly_controlled(self, controls, target, mtrxs, skip_powers, skip_value_mask, nrm):
        """UniformlyControlledSingleBit over the pages (state.cpp:1094-1198).  Table index of a pair = the controls' logical
        bits (controls[j] -> bit j) with zeros inserted at the skip powers, then skip_value_mask ORed in; control j lands on
        table bit pos[j].  On this rank:
          * a rank-bit control has one value: it becomes a skip power at pos[j], and its value goes into the skip value mask;
          * a local control with a pending inversion reads its stored bit flipped: entry e is served from entry e ^ 2^pos[j]
            (the table is permuted on the host; a position the skip value mask already sets is read as 1 either way);
          * a pending inversion on the target conjugates every matrix by X.
        A target on a rank bit is made local first, by the scheduler's exchange."""
        self.flush()
        if self.perm[target] >= self.nl:
            self._exchange([], 0)
        pos = [_table_index(1 << j, skip_powers).bit_length() - 1 for j in range(len(controls))]
        lctrls, lpos, flip, svm = [], [], 0, skip_value_mask
        for j, c in enumerate(controls):
            x, pc = (self.xinv >> c) & 1, self.perm[c]
            if pc >= self.nl:
                if ((self.rank >> (pc - self.nl)) & 1) ^ x:
                    svm |= 1 << pos[j]
            else:
                lctrls.append(pc)
                lpos.append(pos[j])
                flip |= x << pos[j]
        table = np.asarray(mtrxs, dtype=np.complex128).reshape(-1, 4)
        flip &= ~skip_value_mask
        if flip:
            table = table[np.arange(table.shape[0], dtype=np.int64) ^ flip]
        if (self.xinv >> target) & 1:
            table = table[:, ::-1]                              # X m X
        bits = len(controls) + len(skip_powers)
        skips = [1 << b for b in range(bits) if b not in lpos]  # ascending: the local controls fill the other positions in order
        self.loc.be.uniformly_controlled(lctrls, self.perm[target], table, skips, svm, nrm)

    def phase_root_n_mask(self, n, mask):
        if self.xinv & mask:
            # popcount of the LOGICAL bits is not a function of the stored popcount: the mask phase is the product of the
            # single-qubit PhaseRootN gates, which the gate path conjugates correctly
            rad = -math.pi / (1 << (n - 1))
            ph = complex(math.cos(rad), math.sin(rad))
            for q in _bits(mask):
                self.apply2x2(0, 1 << q, [1 + 0j, 0j, 0j, ph], [1 << q], 1.0, 0.0, False)
            return
        self.flush()
        lm, gm = self._split(self._pmask(mask))
        steps = bin(self.rank & gm).count("1")
        if lm:
            self.loc.PhaseRootNMask(n, lm)
        if steps:
            rad = -math.pi / (1 << (n - 1)) * steps
            ph = complex(math.cos(rad), math.sin(rad))
            self.loc.Mtrx([ph, 0j, 0j, ph], 0)

    def apply_m(self, mask, result, nrm: complex):
        self.flush()
        lm, gm = self._split(self._pmask(mask))
        lr, gr = self._split(self._pindex(self._stored(result, mask)))
        if (self.rank & gm) != gr:
            self.loc.Finish()
            self.shard.zero_live()
        elif lm:
            self.loc.be.apply_m(lm, lr, nrm)
        else:
            self.loc.Mtrx([nrm, 0j, 0j, nrm], 0)

    # ---- reductions -------------------------------------------------------------------------------------------------
    def prob_mask(self, mask, perm) -> float:
        self.flush()
        lm, gm = self._split(self._pmask(mask))
        lr, gr = self._split(self._pindex(self._stored(perm, mask)))
        v = 0.0
        if (self.rank & gm) == gr:
            v = self.loc.be.prob_mask(lm, lr) if lm else self.loc.be.norm(0.0)
        return self._allreduce([v])[0]

    def prob_parity(self, mask) -> float:
        self.flush()
        lm, gm = self._split(self._pmask(mask))
        odd_rank = bin(self.rank & gm).count("1") & 1
        tot = self.loc.be.norm(0.0)
        podd = self.loc.be.prob_parity(lm) if lm else 0.0
        if bin(self.xinv & mask).count("1") & 1:
            odd_rank ^= 1                                        # odd logical parity = even stored parity
        return self._allreduce([(tot - podd) if odd_rank else podd])[0]

    def norm(self, thresh) -> float:
        self.flush()
        return self._allreduce([self.loc.be.norm(thresh)])[0]

    def normalize(self, nrm, thresh, phase_arg):
        self.flush()
        self.loc.be.normalize(nrm, thresh, phase_arg)

    def get_amplitude(self, perm: int) -> complex:
        self.flush()
        p = self._pindex(self._stored(perm))
        a = 0j
        if (p >> self.nl) == self.rank:
            a = self.loc.GetAmplitude(p & ((1 << self.nl) - 1))
        re, im = self._allreduce([a.real, a.imag])
        return complex(re, im)

    def set_amplitude(self, perm: int, amp: complex):
        self.flush()
        p = self._pindex(self._stored(perm))
        if (p >> self.nl) == self.rank:
            self.loc.SetAmplitude(p & ((1 << self.nl) - 1), amp)

    def get_state(self) -> np.ndarray:
        """full state in LOGICAL order on every rank (tests / small n only)"""
        self.flush()
        self.loc.Finish()
        torch = self.shard.torch
        mine = np.ascontiguousarray(self.shard.local_host(self.cplx))
        if self.world > 1:
            local = torch.from_numpy(mine.view(self.real)).to(self.shard.device)
            parts = [torch.empty_like(local) for _ in range(self.world)]
            self.dist.all_gather(parts, local)
            phys = torch.cat(parts).cpu().numpy().view(self.cplx)
        else:
            phys = mine
        # phys index bit perm[q] holds logical qubit q: transpose the 2^n tensor accordingly
        t = phys.reshape([2] * self.n)  # axis 0 = most significant physical bit (n-1)
        axes = [self.n - 1 - self.perm[q] for q in range(self.n - 1, -1, -1)]
        v = np.ascontiguousarray(t.transpose(axes)).reshape(-1)
        if self.xinv:
            v = v[np.arange(v.size, dtype=np.int64) ^ self.xinv]   # logical[i] = stored[i ^ xinv]
        return v

    def get_probs(self):
        s = self.get_state()
        return (s.real.astype(self.real) ** 2 + s.imag.astype(self.real) ** 2).astype(self.real)

    # ---- sampling (SURVEY N1): on-device per rank, one small collective for the choice of rank -----------------------
    def _logical_index(self, phys: int) -> int:
        out = 0
        for q in range(self.n):
            if (phys >> self.perm[q]) & 1:
                out |= 1 << q
        return out

    def _gather_scalars(self, vals: Sequence[float]) -> List[List[float]]:
        """every rank's `vals`, indexed [rank][i] (an all_reduce of a one-hot-by-rank matrix)"""
        w = len(vals)
        flat = [0.0] * (self.world * w)
        flat[self.rank * w:(self.rank + 1) * w] = list(vals)
        red = self._allreduce(flat)
        return [red[r * w:(r + 1) * w] for r in range(self.world)]

    def sample(self, rnd: float) -> int:
        """MAll's search (state.cpp:2026-2050) over the sharded vector: the pages are walked in PHYSICAL order (rank-major),
        so for a given `rnd` the outcome is a valid sample of |psi|^2 but not index-for-index the single-engine one once the
        qubit map has been permuted by exchanges."""
        self.flush()
        tots = [t[0] for t in self._gather_scalars([self.loc.be.norm(0.0)])]
        cum, pick, last_nz = 0.0, None, None
        for r in range(self.world):
            if tots[r] > 0:
                last_nz = r
                if cum + tots[r] > rnd:
                    pick = r
                    break
                cum += tots[r]
        if pick is None:
            if last_nz is None:
                return (1 << self.n) - 1
            pick, cum = last_nz, cum - tots[last_nz]
        idx = 0.0
        if self.rank == pick:
            idx = float((pick << self.nl) | self.loc.be.sample(rnd - cum))
        phys = int(round(self._allreduce([idx])[0]))
        return self._logical_index(phys) ^ self.xinv

    def sample_many(self, rnds) -> list:
        """[sample(rnd) for rnd in rnds] with one search per rank: every rank walks the page totals for every rnd
        (rank_walk), searches its own page for its shots' residual rnds, keyed so that it returns logical indices (the key
        of highest_probs_merged), and one all_reduce of a slot per shot, filled by the rank that searched it, gives every
        rank the list.  Nothing is written and nothing is exchanged."""
        self.flush()
        tots = [t[0] for t in self._gather_scalars([self.loc.be.norm(0.0)])]
        pick, res = rank_walk(tots, rnds)
        if pick.size and pick[0] < 0:
            return [(1 << self.n) - 1] * pick.size
        out = np.zeros(pick.size, dtype=np.int64)
        mine = pick == self.rank
        if mine.any():
            inv = {p: q for q, p in enumerate(self.perm)}                 # physical bit -> logical qubit
            xr = self.xinv
            for g in range(self.k):
                if (self.rank >> g) & 1:
                    xr ^= 1 << inv[self.nl + g]
            keys = self.loc.be.sample_keyed(res[mine], self.n, [inv[b] for b in range(self.nl)], xr)
            out[mine] = np.asarray(keys, dtype=np.uint64).view(np.int64)
        if self.world > 1:
            torch = self.shard.torch
            t = torch.from_numpy(out).to(self.shard.device)
            self.dist.all_reduce(t)
            out = t.cpu().numpy()
        return out.tolist()

    def highest_prob(self) -> int:
        self.flush()
        li = self.loc.be.highest_prob()
        a = self.loc.GetAmplitude(li)
        rows = self._gather_scalars([a.real * a.real + a.imag * a.imag, float((self.rank << self.nl) | li)])
        best = max(range(self.world), key=lambda r: (rows[r][0], -r))
        return self._logical_index(int(round(rows[best][1]))) ^ self.xinv

    def prob_mask_all(self, mask: int) -> np.ndarray:
        self.flush()
        qs = [q for q in range(self.n) if (mask >> q) & 1]           # logical mask qubits, ascending = output bit order
        lm, _ = self._split(self._pmask(mask))
        loc = self.loc.be.prob_mask_all(lm) if lm else np.array([self.loc.be.norm(0.0)])
        lbits = [b for b in range(self.nl) if (lm >> b) & 1]          # physical local mask bits, ascending = loc's bit order
        where = {self.perm[q]: j for j, q in enumerate(qs)}           # physical bit -> output bit
        fixed = 0
        for q in qs:
            if self.perm[q] >= self.nl and (self.rank >> (self.perm[q] - self.nl)) & 1:
                fixed |= 1 << where[self.perm[q]]
        out = np.zeros(1 << len(qs), dtype=np.float64)
        for j in range(loc.size):
            o = fixed
            for i, b in enumerate(lbits):
                if (j >> i) & 1:
                    o |= 1 << where[b]
            out[o] += float(loc[j])
        res = np.asarray(self._allreduce(out.tolist()), dtype=self.real)
        flip = 0
        for j, q in enumerate(qs):
            if (self.xinv >> q) & 1:
                flip |= 1 << j
        if flip:
            res = res[np.arange(res.size, dtype=np.int64) ^ flip]   # logical outcome = stored outcome ^ inversions on the mask
        return res

    # ---- observables: per-rank sweeps + one all_reduce; nothing is written and the qubit map does not change ----------------
    def _obs_split(self, bits, table):
        """Per listed qubit, its (bit 0, bit 1) table pair swapped where the qubit has a pending inversion (logical bit =
        stored bit ^ xinv bit).  Returns the local physical qubits with their pairs, and the entries this rank's fixed value
        of every listed rank-bit qubit selects."""
        lbits, ltab, fixed = [], [], []
        for p, q in enumerate(bits):
            pair = [table[2 * p], table[2 * p + 1]]
            if (self.xinv >> q) & 1:
                pair.reverse()
            pq = self.perm[q]
            if pq >= self.nl:
                fixed.append(pair[(self.rank >> (pq - self.nl)) & 1])
            else:
                lbits.append(pq)
                ltab += pair
        return lbits, ltab, fixed

    def moments_bits(self, bits, perms, offset, center):
        """(S0, S1, S2) of the sum-form weight: a listed rank-bit qubit adds a constant on this page, folded into the offset
        (the global bound on offset + the largest perms bounds every rank's)"""
        self.flush()
        lbits, lperms, fixed = self._obs_split(bits, perms)
        s = self.loc.be.moments_bits(lbits, lperms, offset + sum(fixed), center)
        return tuple(self._allreduce(list(s)))

    def moments_floats(self, bits, weights, center):
        """(S0, S1, S2) of the product-form weight: the listed rank-bit qubits give a per-page factor f, multiplied into the
        first local qubit's pair, or (no local qubit listed) w = f on the whole page"""
        self.flush()
        lbits, lw, fixed = self._obs_split(bits, weights)
        f = 1.0
        for v in fixed:
            f *= v
        if lbits:
            lw[0] *= f
            lw[1] *= f
            s = self.loc.be.moments_floats(lbits, lw, center)
        else:
            s0 = self.loc.be.moments_floats([], [], center)[0]
            d = f - center
            s = (s0, s0 * d, s0 * d * d)
        return tuple(self._allreduce(list(s)))

    def expectation_pauli(self, x, z):
        """(S0, <psi|P|psi>) of the logical Pauli string (x, z).

        Pending inversions: psi_logical = X^xinv psi_stored and X Z X = -Z, X Y X = -Y, so on the stored state the string
        carries sign = (-1)^popcount(xinv & z).  With X, Z the physical masks and J = (r, j) (rank r, local index j),
        P|J> = i^|X&Z| (-1)^popcount(J & Z) |J ^ X>, hence
            E = sum_J conj(psi[J ^ X]) i^|X&Z| (-1)^popcount(J & Z) psi[J]
              = sum_r i^|X&Z| (-1)^popcount(r & Z_r) T_r,  T_r = sum_j conj(psi_{r ^ X_r}[j ^ X_l]) (-1)^popcount(j & Z_l) psi_r[j],
        since popcount(J & Z) = popcount(r & Z_r) + popcount(j & Z_l) and J ^ X = (r ^ X_r, j ^ X_l).  E is real (P is
        Hermitian), so summing the real parts of every rank's share gives E.  X_r = 0: T_r is this page's own term and the
        local sweep returns i^|X&Z| T_r.  X_r != 0: T_r pairs this page with rank r ^ X_r's page (k_pauli_pair); that page
        is read where it lies (peer mapping) or sent into `scratch`, never written."""
        self.flush()
        sign = -1.0 if (bin(self.xinv & z).count("1") & 1) else 1.0
        px, pz = self._pmask(x), self._pmask(z)
        xl, xr = self._split(px)
        zl, zr = self._split(pz)
        if bin(self.rank & zr).count("1") & 1:
            sign = -sign
        if not xr:
            s0, e = self.loc.be.expectation_pauli(xl, zl)
            return tuple(self._allreduce([s0, sign * e]))
        page = self.shard.partner_page(self.dist, self.world, self.rank, self.rank ^ xr)
        t, s0 = self.loc.be.expectation_pauli_pair(page, xl, zl)
        t *= (1, 1j, -1, -1j)[bin(px & pz).count("1") & 3]
        return tuple(self._allreduce([s0, sign * t.real]))

    # ---- top n: a keyed select per rank + one all_gather; nothing is written and the qubit map does not change ----------
    def highest_probs_merged(self, n: int) -> list:
        """HighestProbAll(n) over the pages: the n logical indices of largest P = min(|psi|^2, 1), ties to the smaller logical
        index, zero-filled past the last P > 0; the same list on every rank.

        Every rank orders its page by one key, (P desc, t asc) with t(j) = the logical index of its local index j: local
        physical bit b is logical qubit inv[b], this rank's rank bits and the pending inversions are a constant XOR, so
        t(j) = _logical_index((rank << nl) | j) ^ xinv, the index sample / highest_prob report.  Under a key shared by
        every rank the global top n lies in the union of each rank's top min(n, 2^nl), so one all_gather of those (key, P)
        pairs, zero-padded to a fixed size, and a merge give it exactly."""
        self.flush()
        inv = {p: q for q, p in enumerate(self.perm)}                     # physical bit -> logical qubit
        xr = self.xinv
        for g in range(self.k):
            if (self.rank >> g) & 1:
                xr ^= 1 << inv[self.nl + g]
        m = min(n, 1 << self.nl)
        keys, probs = self.loc.be.highest_probs_keyed(m, self.n, [inv[b] for b in range(self.nl)], xr)
        mine = np.stack([np.asarray(keys, dtype=np.uint64).view(np.int64), np.asarray(probs, dtype=np.float64).view(np.int64)])
        if self.world > 1:
            torch = self.shard.torch
            local = torch.from_numpy(np.ascontiguousarray(mine)).to(self.shard.device)
            parts = [torch.empty_like(local) for _ in range(self.world)]
            self.dist.all_gather(parts, local)
            mine = torch.cat(parts, 1).cpu().numpy()
        return merge_top_n(mine[0].view(np.uint64), mine[1].view(np.float64), n)

    _UNSUPPORTED = ("collapse_parity", "inner", "expectation",
                    "moments_basis", "reduced_density_matrix", "highest_probs", "lossy_save", "lossy_load",
                    "compose", "decompose", "dispose_perm", "get_page", "set_page", "copy_page", "shuffle", "copy_state", "clone")

    def __getattr__(self, name):
        # primitives the sharded backend does not provide fail the same way on every rank, before any collective of theirs
        if name in _ShardedBackend._UNSUPPORTED or name.startswith("alu_"):
            raise NotImplementedError("QEngineSharded: backend primitive %r is not sharded (use the gate-level QInterface form, "
                                      "or QPager over the drop-in)" % name)
        raise AttributeError(name)

    # ---- scheduling -------------------------------------------------------------------------------------------------
    def flush(self):
        """Run the queued gates.  Gates whose target is a rank-bit qubit need an exchange; instead of exchanging at the
        first one, it is DEFERRED together with everything that does not commute with a deferred gate, and the scan goes
        on executing every later gate that does commute (shared qubits used diagonally — as control or phase — by both,
        the rule of the fused scheduler).  One exchange then serves the whole deferred set; the reference's QPager pays
        a swap-compute-swap per such gate (src/qpager.cpp:425-432).  ``defer_exchanges = False`` restores in-order
        execution (exchange at the first blocked gate)."""
        ops, self.pending = self.pending, []
        while ops:
            deferred: List[_Gate] = []
            blocked_t = blocked_d = 0
            for idx, g in enumerate(ops):
                if g.diag:
                    uses_t, uses_d = 0, g.cmask | (1 << g.t)
                else:
                    uses_t, uses_d = 1 << g.t, g.cmask
                runnable = g.diag or self.perm[g.t] < self.nl
                conflict = bool((uses_t & (blocked_t | blocked_d)) or (uses_d & blocked_t))
                if runnable and not conflict:
                    self._run_local(g)
                    continue
                if not self.defer_exchanges:
                    deferred = ops[idx:]
                    break
                deferred.append(g)
                blocked_t |= uses_t
                blocked_d |= uses_d
            self._submit_batch()
            if not deferred:
                break
            # the first deferred gate is blocked only by its rank-bit target: after the exchange it can run
            self._exchange(deferred, 0)
            ops = deferred

    def _local_gate(self, ctrls, cperm, m, pt):
        """UCMtrx(ctrls, m, pt, cperm) on the local engine; batched when its backend takes whole gate lists"""
        be = getattr(self.loc, "be", None)
        if be is None or not hasattr(be, "apply_gates"):
            self.loc.UCMtrx(ctrls, m, pt, cperm)
            return
        off1, pmask = 0, 1 << pt
        for j, c in enumerate(ctrls):
            pmask |= 1 << c
            if (cperm >> j) & 1:
                off1 |= 1 << c
        self._batch.append((off1, off1 | (1 << pt), pmask, m))

    def _submit_batch(self):
        g, self._batch = self._batch, []
        if not g:
            return
        import ctypes
        n = len(g)
        m8 = (ctypes.c_double * (8 * n))()
        k = 0
        for x in g:
            for z in x[3]:
                z = complex(z)
                m8[k] = z.real
                m8[k + 1] = z.imag
                k += 2
        self.loc.be.apply_gates(n, (ctypes.c_uint64 * n)(*[x[0] for x in g]), (ctypes.c_uint64 * n)(*[x[1] for x in g]),
                                (ctypes.c_uint64 * n)(*[x[2] for x in g]), m8)

    def _run_local(self, g: _Gate):
        nl = self.nl
        ctrls, cperm = [], 0
        for c in _bits(g.cmask):
            pc = self.perm[c]
            want = (g.cval >> c) & 1
            if pc >= nl:
                if ((self.rank >> (pc - nl)) & 1) != want:
                    return  # a rank-bit control that is not satisfied on this rank: nothing to do
            else:
                if want:
                    cperm |= 1 << len(ctrls)
                ctrls.append(pc)
        pt = self.perm[g.t]
        if pt < nl:
            self._local_gate(ctrls, cperm, g.m, pt)
            return
        # diagonal gate on a rank-bit qubit: this rank sees one diagonal entry
        d = g.m[3] if ((self.rank >> (pt - nl)) & 1) else g.m[0]
        if d == 1:
            return
        if ctrls:
            # a controlled scalar: fold the last control into the matrix (a phase on that qubit under the other controls)
            last = ctrls[-1]
            want_last = (cperm >> (len(ctrls) - 1)) & 1
            rest_perm = cperm & ((1 << (len(ctrls) - 1)) - 1)
            m = [1 + 0j, 0j, 0j, d] if want_last else [d, 0j, 0j, 1 + 0j]
            self._local_gate(ctrls[:-1], rest_perm, m, last)
        else:
            self._local_gate([], 0, [d, 0j, 0j, d], 0)

    def _exchange(self, ops: List[_Gate], i: int):
        """make every rank-bit qubit local: all k rank bits <-> top k local bits, victims chosen by Belady's rule"""
        k, nl, n = self.k, self.nl, self.n
        inv = {p: q for q, p in enumerate(self.perm)}  # physical bit -> logical qubit
        far = {}
        horizon = len(ops)
        for q in range(n):
            if self.perm[q] < nl:
                far[q] = horizon + 1
        for j in range(i, len(ops)):
            g = ops[j]
            if not g.diag and g.t in far and far[g.t] > horizon:
                far[g.t] = j
        # k local logical qubits with the farthest next non-diagonal use (ties: higher physical position = cheaper), on
        # physical bits >= min_victim_bit when the page has k of them, else on any bit >= chunk_floor (never below it)
        lo = self.shard.min_victim_bit if (nl - self.shard.min_victim_bit) >= k else self.shard.chunk_floor
        cands = [q for q in far if self.perm[q] >= lo]
        victims = sorted(cands, key=lambda q: (-far[q], -self.perm[q]))[:k]
        if self.shard.needs_top:
            # bring the victims to the top k local positions with local swaps, then exchange bit nl-k+b <-> rank bit b
            top = list(range(nl - k, nl))
            need = [v for v in victims if self.perm[v] < nl - k]
            free_top = [p for p in top if inv[p] not in victims]
            for v, p in zip(need, free_top):
                pv = self.perm[v]
                other = inv[p]
                self.loc.Swap(pv, p)
                self.local_swaps += 1
                self.perm[v], self.perm[other] = p, pv
                inv[p], inv[pv] = v, other
            vbits = top
        else:
            vbits = sorted(self.perm[v] for v in victims)
        if self.world > 1:
            self.exchange_bytes += self.shard.exchange(self.dist, self.world, self.rank, k, vbits)
        self.exchanges += 1
        for b in range(k):
            pl, pg = vbits[b], nl + b
            ql, qg = inv[pl], inv[pg]
            self.perm[ql], self.perm[qg] = pg, pl
            inv[pl], inv[pg] = qg, ql


class QEngineSharded(QEngineHost):
    """QPager-like engine over `world` ranks; constructed collectively by every rank with the same arguments.  Queries
    (Prob*, MAll, MultiShotMeasureMask, HighestProbAll(n), the Expectation / Variance family) return the same value on
    every rank, and the read-only ones leave the pages and the qubit map alone."""

    def __init__(self, qBitCount: int, initState: int = 0, rgp=None, phaseFac=None, doNorm: bool = False,
                 randomGlobalPhase: bool = False, precision: int = 32, dist=None, world: int = 1, rank: int = 0,
                 device=None, make_engine: Optional[Callable] = None, p2p: bool = False, **kw):
        if doNorm:
            raise ValueError("QEngineSharded: doNormalize is not supported (QPager forces it off as well)")
        self._dist, self._world, self._rank = dist, world, rank
        self._device, self._make_engine, self._p2p = device, make_engine, p2p
        if rgp is None and world > 1:
            # measurement outcomes are drawn per rank after an all-reduced probability: every rank must draw the SAME numbers.
            # Rank 0 picks the seed, everybody adopts it.
            import random as _random
            box = [_random.SystemRandom().getrandbits(62) if rank == 0 else 0]
            dist.broadcast_object_list(box, src=0)
            rgp = _random.Random(box[0])
        super().__init__(qBitCount, initState, rgp, 1.0 + 0j if phaseFac is None else phaseFac, False, randomGlobalPhase,
                         precision=precision)

    def _make_backend(self, n_qubits: int):
        k = int(round(math.log2(self._world))) if self._world > 1 else 0
        floor = P2PShardBuffers.CHUNK_FLOOR[self.precision] if self._p2p else ShardBuffers.chunk_floor
        if n_qubits - k - floor < k:
            # an exchange trades the k rank bits for k local qubits on bits >= floor: the page must hold that many
            raise ValueError("QEngineSharded: %d qubits over %d ranks leave %d local qubits at or above bit %d, fewer than "
                             "the %d an exchange needs; use fewer ranks or more qubits"
                             % (n_qubits, self._world, max(n_qubits - k - floor, 0), floor, k))
        if self._p2p:
            shard = P2PShardBuffers(n_qubits - k, self.precision, self._device.index, self._dist, self._world, self._rank)
        else:
            shard = ShardBuffers(n_qubits - k, self.precision, self._device, self._make_engine)
        return _ShardedBackend(n_qubits, self.precision, shard, self._dist, self._world, self._rank)

    def _has_alu(self) -> bool:
        return False  # INC/DEC take the gate-level QInterface form (src/qinterface/arithmetic.cpp:20-51); other QAlu members raise

    def flush(self):
        self.be.flush()

    def _highest_probs(self, n: int) -> list:
        return self.be.highest_probs_merged(n)
