"""The batch encoder's floating-point analysis, intermediate by intermediate, against the reference.

order, q and the Q35 predictor are floors and thresholds of doubles, so the CUDA analysis must round exactly as
the reference does.  The encoded words show a rounding difference only when some 64*k lands within a few ulps of
an integer or some |k| within a few ulps of 0.05, so these tests compare the intermediates themselves.
codec.encode_trace runs the production encoder with the tracing instantiation of its analysis kernel, which
records every analysis unit's mean, normalised autocorrelation, reflection coefficients, order, q and
predictor.  Each is compared bitwise (NaN equals NaN; +0 and -0 differ) on every unit of
tests/analysis_corpus.py: mono, stereo with the 17-bit difference unit, 3 and 8 channels.
  ac                the port, tests/exact_analysis.py and the compiled reference (where its library exposes ac)
  order, q, c       the compiled reference (the port where it is not built; test_exact_analysis pins the two)
  k, mean           the port and tests/exact_analysis.py (the reference does not expose them)
The quantiser and the order threshold are also probed on their own at every step of q[0], q[1] and q[i >= 2]
and at 0.05, since a trace only reaches those steps by chance.
Run on the H100:  python -m pytest tests -m gpu -q
"""
import numpy as np
import pytest

import analysis_corpus
import exact_analysis as ea
import oracle_lib as ol
import sela_b200
from sela_b200 import codec

pytestmark = pytest.mark.gpu

MAX_ORDER = 100


@pytest.fixture(scope="module")
def runs():
    """Per batch: its name, PCM, channels, the encoder's (descs, words, trace), and the CPU answers per unit."""
    O, P = ol.best(), ol.load("port")
    out = []
    for name, pcm, channels in analysis_corpus.batches():
        units = analysis_corpus.units(pcm, channels)
        descs, words, trace = codec.encode_trace(pcm, channels)
        ref = [O.lpc_analyse(u, want_internals=True) for u in units]
        port = [P.lpc_analyse(u, want_internals=True) for u in units]
        out.append(dict(name=name, pcm=pcm, channels=channels, units=units, descs=descs, words=words, trace=trace,
                        ref=ref, port=port, model=ea.analyse(units)))
    return out


def _padded(rows, width, dtype):
    out = np.zeros((len(rows), width), dtype)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return out


def _check_bits(runs, field, expected_of):
    """Compare trace[field] bitwise with expected_of(run) on every unit; report the units that differ per batch."""
    bad = []
    for r in runs:
        got, want = r["trace"][field], expected_of(r)
        rows = np.nonzero(~ea.same_bits(got, want).reshape(len(got), -1).all(axis=1))[0]
        if rows.size:
            u = rows[0]
            col = np.nonzero(~ea.same_bits(got[u], want[u]).reshape(-1))[0][0] if np.ndim(got[u]) else 0
            g, w = np.ravel(got[u])[col], np.ravel(want[u])[col]
            bad.append("%s: %d of %d units differ; first unit %d at [%d]: %r (%016x) vs %r (%016x)" % (
                r["name"], rows.size, len(got), u, col, g, np.float64(g).view(np.uint64), w,
                np.float64(w).view(np.uint64)))
    assert not bad, "\n".join(bad)


def test_trace_covers_every_unit_kind(runs):
    kinds = {(r["channels"], r["trace"].size) for r in runs}
    assert {c for c, _ in kinds} == {1, 2, 3, 8}
    for r in runs:
        assert r["trace"].size == r["units"].shape[0]
        assert not r["trace"]["reserved"].any()
    stereo = [r for r in runs if r["channels"] == 2]
    assert any(np.abs(r["units"][2::3]).max() > 32767 for r in stereo)   # 17-bit difference units traced


def test_mean_matches_restatements(runs):
    _check_bits(runs, "mean", lambda r: np.array([p["mean"] for p in r["port"]]))
    _check_bits(runs, "mean", lambda r: r["model"]["mean"])


def test_autocorrelation_matches_restatements(runs):
    _check_bits(runs, "ac", lambda r: np.array([p["ac"] for p in r["port"]]))
    _check_bits(runs, "ac", lambda r: r["model"]["ac"])


def test_autocorrelation_matches_reference(runs):
    if runs[0]["ref"][0]["ac"] is None:
        pytest.skip("the reference library was built from an older oracle/ref_shim.cpp that does not expose the "
                    "autocorrelation; test_autocorrelation_matches_restatements still compares it with the port")
    _check_bits(runs, "ac", lambda r: np.array([x["ac"] for x in r["ref"]]))


def test_reflection_coefficients_match_restatements(runs):
    _check_bits(runs, "k", lambda r: np.array([p["refl"] for p in r["port"]]))
    _check_bits(runs, "k", lambda r: r["model"]["k"])


def test_order_and_q_match_reference(runs):
    for r in runs:
        order = np.array([x["order"] for x in r["ref"]])
        bad = np.nonzero(r["trace"]["order"] != order)[0]
        assert bad.size == 0, "%s: order differs on %d units, first %d" % (r["name"], bad.size, bad[0])
        q = _padded([x["q"] for x in r["ref"]], MAX_ORDER, np.int32)
        bad = np.nonzero((r["trace"]["q"] != q).any(axis=1))[0]
        assert bad.size == 0, "%s: q differs on %d units, first %d" % (r["name"], bad.size, bad[0])


def test_predictor_matches_reference(runs):
    for r in runs:
        c = _padded([x["c"] for x in r["ref"]], MAX_ORDER + 1, np.int64)
        bad = np.nonzero((r["trace"]["c"] != c).any(axis=1))[0]
        assert bad.size == 0, "%s: c differs on %d units, first %d" % (r["name"], bad.size, bad[0])


def test_trace_leaves_the_same_stream(runs):
    """The tracing kernel is the production kernel plus stores: same descriptors and words as encode_frames."""
    for r in runs:
        descs, words = sela_b200.encode_frames(r["pcm"], r["channels"])
        assert r["descs"].tobytes() == descs.tobytes(), r["name"]
        assert np.array_equal(r["words"], words), r["name"]


def test_quantiser_at_its_steps():
    k = ea.quantiser_probes()
    got = codec.quantise_probe(k)
    expected = ea.quantiser_expected(k)
    assert np.array_equal(ol.load("port").quantise_probe(k), expected)
    bad = np.nonzero((got != expected).any(axis=1))[0]
    assert bad.size == 0, "%d of %d probes differ, first k = %r (%016x): %s vs %s" % (
        bad.size, k.size, k[bad[0]], k[bad[0]:bad[0] + 1].view(np.uint64)[0], got[bad[0]], expected[bad[0]])
