"""The lossy checkpoint codec without a GPU: the NumPy reference (tests/npref_lossy.py) against the C++ standard's check value,
against the library's host rotation (b200sv_lossy_rotation) and against the files and decodes of the compiled reference
(tests/golden/ref_lossy.*.npz, tests/golden/make_lossy.py), all bit for bit; plus the qscript ops and the sharded backend's
refusal."""
import os
import sys

import numpy as np
import pytest

from qrack_b200 import _abi, qscript
from qrack_b200.sharded import _ShardedBackend

import npref_lossy as nl

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lossy  # noqa: E402

CASES = sorted(make_lossy.CASES)


def fixture(prec):
    return np.load(os.path.join(HERE, "golden", "ref_lossy.f%d.npz" % prec))


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_mt19937_64_check_value():
    # [rand.predef]: the 10000th consecutive invocation of a default-constructed mt19937_64 produces 9981545732273789042
    assert int(nl.MT19937_64().draw(10000)[-1]) == 9981545732273789042


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("d", [4, 8, 16, 32, 64, 128])
def test_library_rotation_equals_numpy(prec, d):
    real = np.float32 if prec == 32 else np.float64
    for seed in (0, 5489, 0xFEEDFACECAFEBEEF):
        R = _abi.lossy_rotation(_abi.load(), d, prec, seed)
        assert bits_equal(R, nl.rotation(d, seed, real)), (d, seed)
        Rm = R.reshape(d, d).astype(np.float64)
        assert np.abs(Rm @ Rm.T - np.eye(d)).max() < (1e-4 if prec == 32 else 1e-12)


def test_fixtures_cover_the_cases():
    for prec in (32, 64):
        z = fixture(prec)
        for name in CASES:
            n, p, b, _ = make_lossy.CASES[name]
            cap, fp, fb, rec = nl.parse(z["file_" + name].tobytes(), prec)
            assert (cap, fp, fb) == (1 << n, p, b)
            assert len(np.unique(rec["seed"])) == 1  # the reference writes one seed per file
    # buckets straddling two words, a single padded block, 1 and 16 bits
    assert any((2 << p) * b % 64 and 64 % b for (_, p, b, _) in make_lossy.CASES.values())
    assert any(p > n for (n, p, _, _) in make_lossy.CASES.values())


@pytest.mark.parametrize("prec", [32, 64])
@pytest.mark.parametrize("name", CASES)
def test_numpy_reencodes_and_decodes_the_reference_files(prec, name):
    z = fixture(prec)
    _, p, b, _ = make_lossy.CASES[name]
    data = z["file_" + name].tobytes()
    seed = int(nl.parse(data, prec)[3]["seed"][0])
    assert nl.encode(z["state_" + name], p, b, seed) == data
    assert bits_equal(nl.decode(data, prec), z["decode_" + name])


def test_zero_blocks_decode_to_noise():
    # |0>: every block but the first is the zero block, which the reference decodes to nonzero values (kept as is)
    z = fixture(32)
    dec = z["decode_ket0_n10_p6_b4"]
    assert np.abs(dec[64:]).min() > 0


def test_script_ops_round_trip():
    calls = []

    class Rec:
        def LossySaveStateVector(self, f, p, b):
            calls.append(("save", f, p, b))

        def LossyLoadStateVector(self, f):
            calls.append(("load", f))

    _, res = qscript.run("qubits 3\nLossySave /tmp/a.svtq 5 3\nLossyLoad /tmp/a.svtq\n", lambda n, p: Rec())
    assert calls == [("save", "/tmp/a.svtq", 5, 3), ("load", "/tmp/a.svtq")] and res == []


def test_sharded_backend_refuses_the_primitives():
    be = _ShardedBackend.__new__(_ShardedBackend)
    for name in ("lossy_save", "lossy_load"):
        with pytest.raises(NotImplementedError):
            getattr(be, name)
