"""Keeps the edge corpus (tests/edge_signals.py) honest: the oracle, built with gcov coverage (tests/oracle_coverage.py),
encodes every case, and the corpus must span the global-gain range 16-bit input can reach.  Which branches the corpus
(with every other input the GPU tests compare with the oracle) takes is accounted for in tests/branch_ledger.py, whose
REQUIRED list holds the data-dependent branches the corpus was written for."""
import hashlib

import pytest

import edge_signals
import oracle_coverage

IDS = ["edge/" + edge_signals.case_id(c) for c in edge_signals.CASES]


@pytest.fixture(scope="module")
def coverage(tmp_path_factory):
    so = oracle_coverage.build(str(tmp_path_factory.mktemp("oracle_cov")))
    res = oracle_coverage.run(so, IDS, trace_frames=max(c[4] for c in edge_signals.CASES) + 8)
    return [dict(res[i], case=i) for i in IDS]


def test_corpus_spans_the_reachable_gain_range(coverage):
    """+-1 LSB input at the highest bitrates drives the global gain as low as 16-bit input can (about 60), full-scale noise
    at the lowest native bitrates as high as it can (about 224); every case is a native configuration (no resampling)."""
    runs = coverage
    assert all(edge_signals.ratio(c) == 1 for c in edge_signals.CASES)
    assert min(r["gmin"] for r in runs) <= 66, min(r["gmin"] for r in runs)
    assert max(r["gmax"] for r in runs) >= 222, max(r["gmax"] for r in runs)


def test_coverage_build_encodes_like_the_oracle(coverage, oracle):
    """The instrumented -O0 build is only a witness if it computes what the oracle computes."""
    runs = coverage
    for c, r in zip(edge_signals.CASES, runs):
        l, rr = edge_signals.signal(c)
        assert hashlib.sha256(oracle.encode_stream(c[1], c[2], c[3], l, rr)[0]).hexdigest() == r["sha"], r["case"]
