"""The top-n radix select on the GPU (b200sv_highest_probs) against the float64 NumPy reference (tests/npref_topn.py), exactly:
the keys are computed by one rule on both sides (include/b200sv.h), so every list must be identical, ties and zero fill
included.  Also its argument errors, what it leaves alone (the state, the memoised marginals), the Python mirror against the
oracle's literal ProbAll loop, full-size analytic states, and the C++ drop-in against the compiled reference."""
import ctypes
import heapq
import math
import os
import random
import subprocess

import numpy as np
import pytest

from qrack_b200 import QEngineCUDA, _abi, qscript

import npref_topn as no
import oracle_topn as ot
import test_topn_cpu as tcpu
import util

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 5, 12, 17, 22, 26]
STATES = ["dense", "uniform", "blocks", "zeros", "half_norm", "over_one"]


def engine(n, prec, psi=None, normalize=False):
    q = QEngineCUDA(n, 0, random.Random(1), 1.0 + 0j, normalize, False, precision=prec)
    if psi is not None:
        q.SetQuantumState(psi)
    return q


def make_state(kind, n, prec, seed=0):
    rng = np.random.default_rng(1000 * n + seed)
    dim = 1 << n
    cplx = np.complex64 if prec == 32 else np.complex128
    if kind == "uniform":
        return np.full(dim, 1.0 / math.sqrt(dim), dtype=cplx)
    if kind == "blocks":
        # H on the low half of the qubits: blocks of exactly equal amplitudes
        lo = n // 2
        hi = rng.standard_normal(dim >> lo) + 1j * rng.standard_normal(dim >> lo)
        hi = (hi / np.linalg.norm(hi)).astype(cplx)
        return np.repeat(hi, 1 << lo) * cplx(1.0 / math.sqrt(1 << lo))
    psi = rng.standard_normal(dim) + 1j * rng.standard_normal(dim)
    if kind == "zeros":
        psi[rng.random(dim) < 0.9] = 0
        psi[0] = 0
    psi = psi / max(np.linalg.norm(psi), 1e-300)
    if kind == "half_norm":
        psi = psi * math.sqrt(0.5)
    if kind == "over_one":
        # several moduli above 1: P is clamped to 1, a tie that goes to the smaller index
        for i, v in zip(rng.choice(dim, size=min(dim, 5), replace=False), (1.5, -2.0j, 1.1 + 0.5j, 3.0, 1.0)):
            psi[i] = v
    return psi.astype(cplx)


def sizes_for(n, psi):
    nz = int(np.count_nonzero(psi))
    ks = {2, 3, 64, 1000}
    if nz < (1 << n):
        ks.add(min(nz + 7, 1 << n))  # more than the nonzero count: the zero fill
    if n <= 22:
        ks.add(1 << n)
    return sorted(k for k in ks if k <= (1 << n))


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_topn_vs_numpy(n, prec):
    for kind in (STATES if n <= 22 else ["dense", "uniform", "zeros"]):
        q = engine(n, prec, make_state(kind, n, prec))
        psi = q.be.get_state()
        order = no.order(psi)
        for k in sizes_for(n, psi):
            got = np.array(q.be.highest_probs(k), dtype=np.int64)
            want = np.zeros(k, dtype=np.int64)
            want[:min(k, len(order))] = order[:k]
            assert np.array_equal(got, want), (kind, n, k, np.flatnonzero(got != want)[:5])
        assert np.array_equal(q.be.get_state(), psi), kind


@pytest.mark.parametrize("prec", [32, 64])
def test_read_only_zero_state_queued_gates_and_marginals(prec):
    n = 11
    q = engine(n, prec, make_state("dense", n, prec, 2))
    for b in range(n):
        q.H(b)
        q.T(b)
    # queued, unflushed gates are part of the state the query sees
    got = q.be.highest_probs(50)
    psi = q.GetQuantumState()
    assert got == no.top_n(psi, 50)
    # bit-identical state; memoised marginals survive without a new launch
    p3 = q.Prob(3)
    before = q.be.stats()["kernel_launches"]
    q.be.highest_probs(200)
    mid = q.be.stats()["kernel_launches"]
    assert mid > before
    assert q.Prob(3) == p3 and q.Prob(7) >= 0
    assert q.be.stats()["kernel_launches"] == mid
    assert np.array_equal(q.GetQuantumState(), psi)
    # the zero state: zeros without a launch
    q.ZeroAmplitudes()
    q.be.reset_stats()
    assert q.be.highest_probs(5) == [0] * 5
    assert q.be.stats()["kernel_launches"] == 0


@pytest.mark.parametrize("prec", [32, 64])
def test_every_einval_and_the_edge_rules(prec):
    n = 6
    q = engine(n, prec, make_state("dense", n, prec, 3))
    psi = q.GetQuantumState()
    lib, h = q.be.lib, q.be.h
    out = (ctypes.c_uint64 * 128)()
    assert lib.b200sv_highest_probs(h, 3, None) == _abi.B200SV_EINVAL
    assert lib.b200sv_highest_probs(h, 65, out) == _abi.B200SV_EINVAL
    assert lib.b200sv_highest_probs(h, 0, None) == 0 and lib.b200sv_highest_probs(h, 0, out) == 0
    assert lib.b200sv_highest_probs(h, 64, out) == 0 and list(out[:64]) == no.top_n(psi, 64)
    with pytest.raises(ValueError):
        q.HighestProbAllN(65)
    assert q.HighestProbAllN(0) == []
    assert q.HighestProbAllN(1) == [q.HighestProbAll()]
    assert np.array_equal(q.GetQuantumState(), psi)


@pytest.mark.parametrize("prec", [32, 64])
def test_mirror_matches_the_oracle_loop_with_normalize(prec):
    """doNormalize on and a state made unnormalised by SetAmplitude: both normalise first (the reference's first ProbAll
    does), so on the normalised state the exact list and the reference's loop agree up to near-ties"""
    n = 10
    psi0 = make_state("dense", n, prec, 4)
    regs = []
    for cls in (QEngineCUDA, ot.QEngineRestateTopn):
        r = cls(n, 0, random.Random(1), 1.0 + 0j, True, False, precision=prec)
        r.SetQuantumState(psi0)
        r.SetAmplitude(5, 0.3 + 0.2j)
        r.SetAmplitude(700, -0.25j)
        regs.append(r)
    for k in (2, 3, 17, 100):
        got, want = regs[0].HighestProbAllN(k), regs[1].HighestProbAllN(k)
        p = no.probs(regs[0].be.get_state())
        assert abs(float(no.probs(regs[0].be.get_state()).sum()) - 1.0) < 1e-5
        assert got == no.top_n(regs[0].be.get_state(), k)
        tcpu.assert_same_up_to_near_ties(want, got, p, no.probs(regs[1].GetQuantumState()), prec, k)


def _ry_product(n, seed):
    """angles of a product of RY rotations whose 65 largest probabilities differ pairwise by more than 1e-4 relative, and those
    65 states, most probable first: each qubit has a major outcome, and a state's log-probability is the sum of the majors' minus
    the penalties ln(major / minor) of the qubits it flips; subsets come out in increasing penalty sum from a heap"""
    rng = random.Random(seed)
    th = [rng.uniform(0.15, 1.2) * (1 if rng.random() < 0.5 else -1) + (math.pi if rng.random() < 0.3 else 0) for _ in range(n)]
    c2 = [math.cos(t / 2) ** 2 for t in th]
    major = [0 if c >= 0.5 else 1 for c in c2]
    pen = sorted((math.log(max(c, 1 - c) / min(c, 1 - c)), q) for q, c in enumerate(c2))
    d = [x for x, _ in pen]
    heap, out = [(d[0], (0,))], [((), 0.0)]
    while len(out) < 65:
        s, sub = heapq.heappop(heap)
        out.append((sub, s))
        j = sub[-1]
        if j + 1 < n:
            heapq.heappush(heap, (s + d[j + 1], sub + (j + 1,)))
            heapq.heappush(heap, (s - d[j] + d[j + 1], sub[:-1] + (j + 1,)))
    sums = [s for _, s in out]
    gap = min(b - a for a, b in zip(sums, sums[1:]))
    perms = []
    for sub, _ in out:
        flip = {pen[j][1] for j in sub}
        perms.append(sum((major[q] ^ (q in flip)) << q for q in range(n)))
    return th, perms, gap


@pytest.mark.parametrize("n,prec", [(30, 32), (29, 64)])
def test_full_size_analytic(n, prec):
    # GHZ: two states of probability 1/2, then the zero fill
    q = engine(n, prec)
    q.H(0)
    for b in range(1, n):
        q.CNOT(0, b)
    assert q.HighestProbAllN(3) == [0, (1 << n) - 1, 0]
    del q
    # a product of RY rotations: the top 64 from the per-qubit factors
    th, perms, gap = _ry_product(n, 7)
    assert gap > 1e-4  # ln P differs by more than 1e-4 between neighbours: gate rounding (~n 2^-24) cannot reorder them
    q = engine(n, prec)
    for b in range(n):
        q.U(b, th[b], 0.0, 0.0)
    assert q.HighestProbAllN(64) == perms[:64]


# ---- the C++ drop-in (dropin/_build, built when the reference sources are present) -------------------------------------
B = os.path.join(util.ROOT, "dropin", "_build")


def test_dropin_topn_matches_the_compiled_reference(tmp_path):
    exe = os.path.join(B, "observables_b200_f32")
    if not os.path.exists(exe):
        pytest.skip("dropin/_build not built (needs the reference sources: QRACK_REFERENCE)")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.join(util.ROOT, "qrack_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    z = tcpu._fixture(32)
    for name, circ, sizes in ot.topn_cases():
        c, full, dump = tmp_path / "c.qs", tmp_path / "q.qs", tmp_path / "s.bin"
        c.write_text(circ)
        full.write_text(ot.topn_text(circ, sizes))
        subprocess.run([exe, str(c), "--engine", "cuda", "--dump", str(dump)], check=True, timeout=600, env=env)
        out = subprocess.run([exe, str(full), "--engine", "cuda"], check=True, capture_output=True, text=True, timeout=600,
                             env=env).stdout
        mine = np.fromfile(str(dump), dtype=np.complex64)
        p_ref, p_mine = no.probs(z["state_" + name]), no.probs(mine)
        # the drop-in's gates round differently from the reference's: two entries may swap where the reference's probabilities
        # are closer than twice the largest difference between the two states' probabilities
        slack = 2 * float(np.abs(p_mine - p_ref).max())
        got = qscript.parse_results(out)
        assert len(got) == len(sizes)
        for k, (op, vals) in zip(sizes, got):
            assert op == "HighestProbAllN"
            vals = [int(v) for v in vals]
            assert vals == no.top_n(mine, k), (name, k)
            tcpu.assert_same_up_to_near_ties(vals, list(z["top_%s_%d" % (name, k)]), p_ref, p_mine, 32, (name, k), slack)
