"""Two-target gates (ISwap, SqrtSwap, FSim, CSwap, AntiCSwap), (C)UniformParityRZ and UniformlyControlledSingleBit / RY / RZ on
the sharded engine (gloo worlds 2 and 4, CPU), against the float64 oracle; the NumPy identity behind the two-target lowering;
and QCircuit recording the two-target forms.

Every gate script starts from a state whose rank-bit qubits have not been touched yet, so the qubit map is the identity
when its first gates are queued: qubits 7 and 8 are rank bits at world 4, qubit 8 at world 2.  The gates then sit on local
qubits, on one rank bit and on two, with controls on both sides and pending X inversions (XMask) on targets and controls."""
import math
import os
import random

import numpy as np
import pytest

from qrack_b200 import qscript
from qrack_b200.qengine import lower_two_target

import one_device
import oracle_gates
import util

N = 9


def _u3(rng):
    th, ph, la = (rng.uniform(-math.pi, math.pi) for _ in range(3))
    c, s = math.cos(th / 2), math.sin(th / 2)
    m = [complex(c), -np.exp(1j * la) * s, np.exp(1j * ph) * s, np.exp(1j * (ph + la)) * c]
    return " ".join("%.17g %.17g" % (z.real, z.imag) for z in m)


def _prep(n, seed):
    """U3 on qubits 0..n-3 (local at world 4) and a CNOT chain among them: the rank-bit qubits stay untouched"""
    rng = random.Random(seed)
    lines = ["qubits %d" % n]
    lines += ["U %d %.17g %.17g %.17g" % (q, rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3)) for q in range(n - 2)]
    lines += ["CNOT %d %d" % (q, q + 1) for q in range(n - 3)]
    return "\n".join(lines) + "\n"


def _uc(rng, controls, target, skips=(), svm=0):
    size = 1 << (len(controls) + len(skips))
    return ("UniformlyControlledSingleBit %d %s %d %d %s %d " % (len(controls), " ".join(map(str, controls)), target, len(skips),
                                                                 " ".join(map(str, skips)), svm)
            + " ".join(_u3(rng) for _ in range(size)) + "\n").replace("  ", " ")


def _mixed(n, seed):
    """every family on random qubits after the qubit map has been scrambled by exchanges, pending inversions throughout"""
    rng = random.Random(seed)
    text = qscript.random_u3_cnot(n, 2, seed=seed)
    for _ in range(40):
        a, b, c, d = rng.sample(range(n), 4)
        kind = rng.randrange(9)
        if kind == 0:
            text += "XMask %d\n" % rng.getrandbits(n)
        elif kind == 1:
            text += "%s %d %d\n" % (rng.choice(["ISwap", "SqrtSwap", "Swap"]), a, b)
        elif kind == 2:
            text += "FSim %.17g %.17g %d %d\n" % (rng.uniform(-3, 3), rng.uniform(-3, 3), a, b)
        elif kind == 3:
            text += "%s 2 %d %d %d %d\n" % (rng.choice(["CSwap", "AntiCSwap"]), c, d, a, b)
        elif kind == 4:
            text += "UniformParityRZ %d %.17g\n" % (rng.getrandbits(n) | 1, rng.uniform(-3, 3))
        elif kind == 5:
            text += "CUniformParityRZ 2 %d %d %d %.17g\n" % (c, d, rng.getrandbits(n) & ~((1 << c) | (1 << d)), rng.uniform(-3, 3))
        elif kind == 6:
            text += _uc(rng, [b, c], a, *(([1 << rng.randrange(3)], rng.getrandbits(3)) if rng.random() < 0.5 else ()))
        elif kind == 7:
            text += "%s 2 %d %d %d %s\n" % (rng.choice(["UniformlyControlledRY", "UniformlyControlledRZ"]), b, c, a,
                                            " ".join("%.17g" % rng.uniform(-3, 3) for _ in range(4)))
        else:
            text += "H %d\nCNOT %d %d\n" % (a, b, c)
    return text


def gate_scripts(n=N):
    """name -> script; the probes at the end read the state without changing it"""
    rng = random.Random(11)
    r, r2 = n - 1, n - 2                       # rank bits at world 4 (r2 local at world 2)
    two = (_prep(n, 1) + "XMask %d\n" % ((1 << r) | (1 << 3) | (1 << 5))
           + "ISwap 0 1\nSqrtSwap 2 %d\nISwap %d %d\nFSim 0.7 -1.3 %d 4\nFSim -2.1 0.4 %d %d\n" % (r, r2, r, r, r2, r)
           + "CSwap 2 3 %d 5 6\nCSwap 2 0 %d %d 1\nAntiCSwap 1 %d 2 4\nAntiCSwap 2 1 %d %d %d\nSqrtSwap %d %d\n"
           % (r, r2, r, r, r2, 6, r, r2, 0)
           + "".join("H %d\n" % q for q in range(n)) + "ISwap 0 %d\nCSwap 1 4 %d 2\nFSim 1.1 0.2 3 %d\n" % (r, r2, r))
    prz = (_prep(n, 2) + "XMask %d\n" % ((1 << r) | (1 << 2) | (1 << 4))
           + "UniformParityRZ %d 0.37\n" % ((1 << r) | (1 << r2) | 0b10110)
           + "UniformParityRZ %d -1.1\n" % ((1 << r) | (1 << r2))
           + "CUniformParityRZ 2 2 %d %d 0.9\n" % (r, (1 << r2) | 0b1001)
           + "CUniformParityRZ 1 %d %d 0.55\n" % (r2, 1 << r)
           + "CUniformParityRZ 2 4 0 %d -0.8\n" % (1 << r)
           + "CUniformParityRZ 1 4 %d 1.3\n" % 0b1000110
           + "".join("H %d\n" % q for q in range(n)) + "UniformParityRZ %d 0.21\n" % ((1 << n) - 1))
    uc = (_prep(n, 3) + "XMask %d\n" % ((1 << r) | (1 << r2) | (1 << 1) | (1 << 2))
          + _uc(rng, [1, 3], 0) + _uc(rng, [2, r, 4], 5) + _uc(rng, [r2, 1], 6, [2], 1) + _uc(rng, [3, r, 2], r2, [8, 1], 5)
          + _uc(rng, [0], r, [2, 1], 3) + _uc(rng, [r, r2], 3)
          + "UniformlyControlledRY 2 %d 1 0 0.3 -0.7 1.9 2.4\n" % r + "UniformlyControlledRZ 3 0 %d 5 2 %s\n"
          % (r2, " ".join("%.3f" % (0.4 * k - 1.1) for k in range(8)))
          + "".join("H %d\n" % q for q in range(n)) + _uc(rng, [0, r, 5], 7, [1], 0))
    out = {"two_target": two, "parity_rz": prz, "uc": uc, "mixed": _mixed(n, 5), "mixed2": _mixed(n, 6)}
    probes = "".join("Prob %d\n" % q for q in range(n)) + "ProbParity %d\nGetAmplitude 5\nNorm\n" % ((1 << n) - 1)
    return {k: v + probes for k, v in out.items()}


def golden_scripts():
    """the misc_8q fixture and the scripts of the reference gate fixture (tests/golden/ref_gates_9q.*.npz)"""
    out = {"misc_8q": open(os.path.join(util.GOLDEN, "misc_8q.qs")).read()}
    out.update({"ref_" + k: v for k, v in oracle_gates.ref_scripts().items()})
    return out


def ref_gates(prec):
    """name -> the state the reference's QEngineCPU returned for oracle_gates.ref_scripts()[name]"""
    return dict(np.load(os.path.join(util.GOLDEN, "ref_gates_9q.f%d.npz" % prec)))


LOG_KIND = {"2q": 0, "uc": 1, "prz": 2}


def _instrument(be, log):
    """log, at the call, how many of the gate's targets / mask bits / controls are rank bits"""
    a2, uc, prz = be.apply2x2, be.uniformly_controlled, be.uniform_parity_rz

    def rank_bits(mask):
        return sum(1 for q in range(be.n) if (mask >> q) & 1 and be.perm[q] >= be.nl)

    def apply2x2(off1, off2, *a):
        if bin(off1 ^ off2).count("1") == 2:
            log.append(("2q", rank_bits(off1 ^ off2)))
        return a2(off1, off2, *a)

    def uniformly_controlled(controls, target, *a):
        log.append(("uc", rank_bits(1 << target), rank_bits(sum(1 << c for c in controls))))
        return uc(controls, target, *a)

    def uniform_parity_rz(cmask, mask, angle):
        log.append(("prz", rank_bits(mask), bin(mask).count("1") - rank_bits(mask), rank_bits(cmask)))
        return prz(cmask, mask, angle)
    be.apply2x2, be.uniformly_controlled, be.uniform_parity_rz = apply2x2, uniformly_controlled, uniform_parity_rz


def engine_maker(rank, world, dist, prec, local, mode=None):
    """make(n, perm) for qscript.run: the sharded engine over the oracle restatement ("restate"), the fused-planner
    emulation ("emu") or CUDA pages ("cuda": P2P pages in push / pull mode, torch pages in staged mode)"""
    import random as _random

    from qrack_b200 import sharded

    if local == "emu":
        class Eng(sharded.QEngineSharded):
            def _make_backend(self, n_qubits):
                k = world.bit_length() - 1
                return sharded._ShardedBackend(n_qubits, prec, oracle_gates.EmuGatesShard(n_qubits - k, prec, dist, world, rank),
                                               dist, world, rank)
        return lambda n, perm: Eng(n, perm, _random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world, rank=rank,
                                   device="cpu")
    if local == "restate":
        return lambda n, perm: sharded.QEngineSharded(n, perm, _random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world,
                                                      rank=rank, device="cpu", make_engine=oracle_gates.restate_factory(prec))
    import torch
    os.environ["B200SV_SHARD_PULL"] = "0" if mode == "push" else "1"
    dev = torch.device("cuda", 0)
    return lambda n, perm: sharded.QEngineSharded(n, perm, _random.Random(1), 1.0 + 0j, precision=prec, dist=dist, world=world,
                                                  rank=rank, device=dev, make_engine=sharded.cuda_engine_factory(0, prec),
                                                  p2p=mode != "staged")


def run_ranks(rank, world, dist, prec, local, mode, out):
    """every gate script and the golden script on this rank; saves the states, query results, exchange counts and the log"""
    make = engine_maker(rank, world, dist, prec, local, mode)
    log = []

    def make_logged(n, perm):
        q = make(n, perm)
        _instrument(q.be, log)
        return q
    save = {}
    for name, text in dict(gate_scripts(), **golden_scripts()).items():
        regs, results = qscript.run(text, make_logged)
        save[name + "_state"] = regs[0].GetQuantumState()
        save[name + "_results"] = np.array([v for _, vals in results for v in vals], dtype=np.float64)
        save[name + "_exchanges"] = regs[0].be.exchanges
        del regs
    # one row per distinct entry: kind, then its counts, padded with -1
    save["log"] = np.array(sorted({(LOG_KIND[e[0]],) + e[1:] + (-1,) * (4 - len(e)) for e in log}), dtype=np.int64)
    np.savez(os.path.join(out, "gates.%d.npz" % rank), **save)


def oracle64(text):
    regs, results = qscript.run(text, util.make_factory(oracle_gates.QEngineRestateGates, 64))
    return regs[0].GetQuantumState(), np.array([v for _, vals in results for v in vals], dtype=np.float64)


def check_ranks(z, world, prec):
    """every rank returned the same states and values; the gate scripts match the float64 oracle, the golden script its
    fixture; at world 4 the scripts put two-target gates on 0, 1 and 2 rank bits, uniformly controlled targets on local
    and rank-bit qubits and parity masks without local bits.  Returns the largest |delta amp| against the oracle."""
    for r in range(1, world):
        for key in z[0]:
            assert np.array_equal(z[r][key], z[0][key]), "rank %d differs from rank 0 in %s" % (r, key)
    worst = 0.0
    for name, text in gate_scripts().items():
        want, wres = oracle64(text)
        d = float(np.abs(z[0][name + "_state"].astype(np.complex128) - want).max())
        assert d <= util.AMP_TOL[prec], "%s: max |delta amp| = %.3e" % (name, d)
        bound = util.PROB_TOL[prec] + 2 * float(np.linalg.norm(z[0][name + "_state"].astype(np.complex128) - want))
        e = float(np.abs(z[0][name + "_results"] - wres).max())
        assert e <= bound, "%s: max |delta query| = %.3e" % (name, e)
        worst = max(worst, d)
    _, regs, results = util.load_golden("misc_8q", prec)
    util.assert_states_close({0: z[0]["misc_8q_state"]}, {0: regs[0]}, prec, "misc_8q")
    want = np.array([v for _, vals in results for v in vals], dtype=np.float64)
    e = float(np.abs(z[0]["misc_8q_results"] - want).max())
    assert e <= util.PROB_TOL[prec], "misc_8q: max |delta query| = %.3e" % e
    for name, st in ref_gates(prec).items():
        util.assert_states_close({0: z[0]["ref_" + name + "_state"]}, {0: st}, prec, "reference " + name)
    if world == 4:
        seen = [tuple(int(v) for v in row) for row in z[0]["log"]]
        two, uc, prz = ([row[1:] for row in seen if row[0] == LOG_KIND[k]] for k in ("2q", "uc", "prz"))
        for k in (0, 1, 2):
            assert (k, -1, -1) in two, ("two-target gate on %d rank bits" % k, seen)
        assert any(e[0] == 1 for e in uc) and any(e[0] == 0 and e[1] > 0 for e in uc), seen     # target / control on rank bits
        assert any(e[1] == 0 for e in prz) and any(e[2] > 0 for e in prz), seen                 # no local mask bit / rank control
    return worst


@pytest.mark.parametrize("local", ["restate", "emu"])
@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_gates_match_the_oracle(world, prec, local, tmp_path):
    one_device.spawn(run_ranks, world, prec, local, None, str(tmp_path), use_cuda=False, staged=False)
    z = [dict(np.load(str(tmp_path / ("gates.%d.npz" % r)))) for r in range(world)]
    check_ranks(z, world, prec)


def _exchange_counts(rank, world, dist, out):
    make = engine_maker(rank, world, dist, 32, "restate")
    q = make(N, 0)
    for b in range(N - 2):
        q.H(b)
    q.Finish()

    def rank_qubits():
        return [l for l in range(N) if q.be.perm[l] >= q.be.nl]

    def local_qubits():
        return [l for l in range(N) if q.be.perm[l] < q.be.nl]
    steps = [lambda: (q.ISwap(0, 1), q.SqrtSwap(2, 5), q.FSim(0.3, 0.2, 1, 3), q.CSwap([2, 4], 5, 6), q.AntiCSwap([0], 3, 4)),
             lambda: (q.Swap(N - 1, 0), q.Swap(N - 2, N - 1)),
             lambda: q.ISwap(rank_qubits()[0], local_qubits()[0]),
             lambda: q.ISwap(*rank_qubits()),
             lambda: q.CSwap([rank_qubits()[0]], *local_qubits()[:2]),
             lambda: q.H(rank_qubits()[0])]
    counts = [q.be.exchanges]
    for step in steps:
        step()
        q.Finish()
        counts.append(q.be.exchanges)
    if rank == 0:
        np.save(out, np.diff(counts))


def test_exchange_counts(tmp_path):
    """local two-target gates and an uncontrolled Swap add no exchange; a two-target gate with one or two rank-bit targets
    adds exactly one, as a single-target gate on a rank bit does; a rank-bit control alone adds none"""
    out = str(tmp_path / "counts.npy")
    one_device.spawn(_exchange_counts, 4, out, use_cuda=False, staged=False)
    assert np.load(out).tolist() == [0, 0, 1, 1, 0, 1]


def _apply2x2(psi, off1, off2, m, pmask):
    """QEngineCPU::Apply2x2 on a NumPy state: m on (i | off1, i | off2) for every i with no bit of pmask set"""
    psi = psi.copy()
    i = np.arange(psi.size, dtype=np.int64)
    base = i[(i & pmask) == 0]
    a, b = psi[base | off1], psi[base | off2]
    psi[base | off1] = m[0] * a + m[1] * b
    psi[base | off2] = m[2] * a + m[3] * b
    return psi


def test_two_target_lowering_identity():
    """Apply2x2(off1, off2, m, pows) with two target bits equals CNOT(p -> q), the single-target form on p, CNOT(p -> q)
    (qengine.lower_two_target), for random offsets, controls, control values and matrices on 6 qubits, both target-pair
    kinds (|01>, |10> and |00>, |11>)"""
    rng = np.random.default_rng(7)
    n = 6
    for _ in range(300):
        a, b = rng.choice(n, 2, replace=False)
        diff = (1 << int(a)) | (1 << int(b))
        cmask = int(rng.integers(0, 1 << n)) & ~diff
        cval = int(rng.integers(0, 1 << n)) & cmask
        x = int(rng.choice([0, 1 << int(a), 1 << int(b), diff]))
        off1, off2 = cval | x, cval | (x ^ diff)
        m = rng.standard_normal(4) + 1j * rng.standard_normal(4)
        psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
        want = _apply2x2(psi, off1, off2, m, cmask | diff)
        got = psi
        for o1, o2, pm, mm in lower_two_target(off1, off2, cmask | diff, m):
            assert bin(o1 ^ o2).count("1") == 1 and (o1 & ~pm) == 0 and (o2 & ~pm) == 0
            got = _apply2x2(got, o1, o2, np.asarray(mm), pm)
        assert np.abs(got - want).max() <= 1e-12, (off1, off2, cmask)
