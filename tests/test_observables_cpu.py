"""The observable queries on the CPU: the float64 reference (tests/npref_observables.py) and the literal QInterface loops of
the oracle (tests/oracle_observables.py) against what the compiled reference returned (tests/golden/ref_observables_12q.*),
and the query ops of the script format."""
import os
import re

import pytest

from qrack_b200 import qscript

import npref_observables as no
import oracle_observables as oo
import util

# Relative to the scale of each result (sum p |w| for an expectation, sum p (|w| + |m|)^2 for a variance).  The reference adds
# the 2^12 terms of each query one by one in real1_f (float in the fp32 build, qinterface.cpp:573,612,653,804): each add rounds
# by up to 2^-24 (fp32) / 2^-53 (fp64) of the running sum, which grows to the scale.  Measured on the stored reference state:
# 1.9e-6 (fp32) and 4.4e-15 (fp64) at worst over the 48 queries; the bars sit just above.
REF_REL_TOL = {32: 5e-6, 64: 2e-14}


def _queries():
    return [t for _, t in qscript.parse(oo.observables_queries())]


@pytest.mark.parametrize("prec", [32, 64])
def test_npref_matches_the_compiled_reference(prec):
    ref = util.load_reference("observables_12q", prec)
    psi = ref["state"]
    assert len(ref["results"]) == len(_queries()) == 48
    for (op, (got,)), t in zip(ref["results"], _queries()):
        assert op == t[0]
        want, scale, psi = no.query_value(psi, t[0], t[1:])
        assert abs(got - want) <= REF_REL_TOL[prec] * scale, (t, got, want, scale)


@pytest.mark.parametrize("prec", [32, 64])
def test_oracle_loops_match_the_compiled_reference(prec):
    ref = util.load_reference("observables_12q", prec)
    regs, results = util.run_engine(oo.observables_text(), oo.QEngineRestateObs, prec)
    psi = ref["state"]
    for (gop, (got,)), (wop, (want,)), t in zip(results, ref["results"], _queries()):
        assert gop == wop == t[0]
        _, scale, psi = no.query_value(psi, t[0], t[1:])
        assert abs(got - want) <= REF_REL_TOL[prec] * scale, (t, got, want, scale)


def test_unsquared_floats_variance_is_the_reference_behaviour():
    """VarianceFloatsFactorized for k >= 2 is sum p (w - mean), i.e. ~0 on a normalised state, in the reference too"""
    ref = util.load_reference("observables_12q", 64)
    vals = [v for (op, (v,)), t in zip(ref["results"], _queries()) if op == "VarianceFloatsFactorized" and int(t[1]) >= 2]
    assert vals and all(abs(v) < 1e-12 for v in vals)


def test_query_ops_round_trip():
    """every query op parses, is a query of the script format, dispatches to the method of the same name, and its result
    line is read back; the C++ harness handles the same op names"""
    text = oo.observables_text()
    calls = []

    class Rec:
        def __getattr__(self, name):
            def f(*args):
                calls.append((name, args))
                return 0.25
            return f

    _, results = qscript.run(text, lambda n, p: Rec())
    ops = [t[0] for t in _queries()]
    assert set(ops) <= qscript.QUERY_OPS and len(set(ops)) == 10
    calls = [c for c in calls if c[0] in qscript.QUERY_OPS]
    assert [r[0] for r in results] == ops == [c[0] for c in calls]
    assert qscript.parse_results("".join("%s %.17g\n" % (op, v[0]) for op, v in results)) == results
    assert qscript.count_gate_ops(text) == qscript.count_gate_ops(oo.observables_circuit())
    src = open(os.path.join(util.ROOT, "dropin", "observables_harness.cpp")).read()
    assert set(ops) <= set(re.findall(r'op == "(\w+)"', src))
    # argument shapes: (bits, perms, offset), (bits, offset), (bits, weights / paulis / angles)
    byname = dict(reversed(calls))  # the first call of each op (k = 1)
    assert byname["ExpectationBitsFactorized"][2] == 1001 and len(byname["ExpectationBitsFactorized"][1]) == 2
    assert byname["ExpectationBitsAll"] == ([3], 0)
    assert len(byname["ExpectationUnitaryAll"][1]) == 3 * len(byname["ExpectationUnitaryAll"][0])
