"""The encoder's floating-point analysis, intermediate by intermediate, on the CPU.

tests/exact_analysis.py restates ResidueGenerator in numpy; oracle/sela_oracle.c restates it in C.  Both are
compared here bitwise with the compiled reference on every analysis unit of tests/analysis_corpus.py: the
normalised autocorrelation, the order and q.  The raw reflection coefficients and the mean are not observable
in the reference, so for those the two restatements are compared with each other.  The GPU tests
(test_analysis_trace.py) then hold the CUDA encoder to these values.
"""
import numpy as np
import pytest

import analysis_corpus
import exact_analysis as ea
import oracle_lib as ol


@pytest.fixture(scope="module")
def units():
    return analysis_corpus.all_units()


@pytest.fixture(scope="module")
def model(units):
    return ea.analyse(units)


@pytest.fixture(scope="module")
def port(units):
    P = ol.load("port")
    return [P.lpc_analyse(u, want_internals=True) for u in units]


def _rows_differing(a, b):
    return np.nonzero(~ea.same_bits(a, b).reshape(len(a), -1).all(axis=1))[0]


def test_corpus_runs_every_path(units, model):
    assert units.shape[0] > 2800
    assert units.min() < -32768 and units.max() > 32767                 # 17-bit difference units
    assert np.isnan(model["ac"][:, 1]).sum() >= 3                        # silence: lag 0 is 0
    assert len(np.unique(model["order"])) >= 90
    # the quantiser sees values across its range at q[0] and q[1]
    assert np.ptp(model["q"][:, 0]) > 100 and np.ptp(model["q"][model["order"] > 1, 1]) > 100


def test_model_equals_port(units, model, port):
    """Every intermediate, including the two the reference does not expose (the mean and k)."""
    for name, key in [("mean", "mean"), ("ac", "ac"), ("k", "refl")]:
        theirs = np.array([p[key] for p in port])
        assert _rows_differing(model[name], theirs).size == 0, name
    assert np.array_equal(model["order"], [p["order"] for p in port])
    for i, p in enumerate(port):
        assert np.array_equal(model["q"][i, :p["order"]], p["q"]), i


def _ref_exposing_ac():
    R = ol.load("ref")
    if "ac" not in R.internals:
        pytest.skip("oracle/_ref/libsela_ref.so was built from an older oracle/ref_shim.cpp that does not expose "
                    "the autocorrelation, and the reference sources are not here to rebuild it")
    return R


@pytest.mark.ref
def test_model_and_port_equal_reference_autocorrelation(units, model, port):
    R = _ref_exposing_ac()
    ac_ref = np.array([R.lpc_analyse(u, want_internals=True)["ac"] for u in units])
    assert _rows_differing(model["ac"], ac_ref).size == 0
    assert _rows_differing(np.array([p["ac"] for p in port]), ac_ref).size == 0


@pytest.mark.ref
def test_model_and_port_equal_reference(units, model, port):
    R = ol.load("ref")
    ref = [R.lpc_analyse(u, want_internals=True) for u in units]
    order = np.array([r["order"] for r in ref])
    assert np.array_equal(model["order"], order)
    assert np.array_equal([p["order"] for p in port], order)
    for i, r in enumerate(ref):
        assert np.array_equal(model["q"][i, :r["order"]], r["q"]), i
        assert np.array_equal(port[i]["q"], r["q"]), i
        assert not model["q"][i, r["order"]:].any(), i
        assert r["refl"] is None and r["mean"] is None   # the reference does not expose them


def test_corpus_sees_reordered_sums(units, model):
    """The corpus must be able to see an edit that keeps the maths and changes the rounding, at the
    intermediates, where (order, q) almost never show it.  Constant units are left out: there every term of a
    lag sum is the same product, and the DC tests cover their mean."""
    varying = ~(units == units[:, :1]).all(axis=1)
    two_chains = ea.analyse(units[varying], lag_chains=2)
    changed = _rows_differing(two_chains["ac"], model["ac"][varying]).size
    assert changed >= 0.9 * varying.sum(), (changed, varying.sum())
    reciprocal = ea.analyse(units[varying], schur_reciprocal=True)
    changed = _rows_differing(reciprocal["k"], model["k"][varying]).size
    assert changed >= 0.9 * varying.sum(), (changed, varying.sum())


def test_quantiser_probes_model_equals_port():
    k = ea.quantiser_probes()
    expected = ea.quantiser_expected(k)
    assert np.array_equal(ol.load("port").quantise_probe(k), expected)
    # the probes straddle every step: each level of q[0] and q[1] and every |k| side of 0.05 occurs
    assert set(expected[:, 0]) >= set(range(-64, 65)) and set(expected[:, 1]) >= set(range(-64, 65))
    assert set(expected[:, 3]) == {0, 1}
    # one ulp either side of a step lands on both levels
    steps = ea.first_reaching(lambda x: ea.quantise(x)[0], np.arange(-63, 65))
    below = ea.quantise(np.nextafter(steps, -2.0))[0]
    assert np.array_equal(ea.quantise(steps)[0], np.arange(-63, 65)) and np.array_equal(below, np.arange(-64, 64))
