"""Accounts for every branch of the oracle's per-frame path (tests/branch_ledger.py): the oracle, built with gcov coverage,
encodes every input the GPU tests compare with it (tests/oracle_inputs.py), and each branch outcome of the per-frame
functions of lj_psy.cpp, lj_mdct.cpp, lj_quant.cpp and lj_bitstream.cpp must be taken by some input or listed in the ledger
with its reason -- and a listed outcome must not be taken.  A GPU copy of a branch no input takes would be unchecked by
the GPU tests whatever it did."""
import collections
import re
import shutil
import subprocess

import pytest

import branch_ledger
import oracle_coverage
import oracle_inputs


@pytest.fixture(scope="module")
def reports(tmp_path_factory):
    ver = subprocess.run([shutil.which("gcov") or "gcov", "--version"], capture_output=True, text=True).stdout
    major = int(re.search(r"(\d+)\.\d+\.\d+", ver).group(1))
    if major != branch_ledger.GCC_MAJOR:
        pytest.fail("the ledger's branch indices are gcov %d's; this is gcov %d, which may number branches differently: "
                    "re-derive the indices with it" % (branch_ledger.GCC_MAJOR, major))
    so = oracle_coverage.build(str(tmp_path_factory.mktemp("oracle_cov")))
    oracle_coverage.run(so, [r[0] for r in oracle_inputs.runs()])
    return {src: oracle_coverage.report(so, src) for src in branch_ledger.SOURCES}


def _in_scope(reports):
    """{(source, function, statement, n): (line number, [taken counts])} for every per-frame line with branches"""
    out = {}
    for src, lines in reports.items():
        seen = collections.Counter()
        for num, ln in enumerate(lines, 1):
            if not ln.branches or ln.func in branch_ledger.INIT_FUNCTIONS or any(t in ln.src for t in branch_ledger.TRACE_TAPS):
                continue
            stmt = ln.src.strip()
            out[(src, ln.func, stmt, seen[(ln.func, stmt)])] = (num, ln.branches)
            seen[(ln.func, stmt)] += 1
    return out


def test_ledger_entries_are_well_formed():
    keys = [e[:4] for e in branch_ledger.LEDGER]
    assert len(keys) == len(set(keys)), [k for k, n in collections.Counter(keys).items() if n > 1]
    for src, func, stmt, n, untaken, kind, reason in branch_ledger.LEDGER:
        assert src in branch_ledger.SOURCES and untaken and list(untaken) == sorted(set(untaken)), (src, func, stmt)
        assert kind in ("a", "b", "c", "open") and len(reason) > 10, (src, func, stmt)


def test_every_untaken_outcome_is_in_the_ledger(reports):
    """fails, naming the branch, when an outcome no input takes is not listed"""
    ledger = {e[:4]: e for e in branch_ledger.LEDGER}
    bad = []
    for key, (num, branches) in _in_scope(reports).items():
        untaken = tuple(i for i, b in enumerate(branches) if b == 0)
        listed = ledger[key][4] if key in ledger else ()
        missing = [i for i in untaken if i not in listed]
        if missing:
            bad.append("%s:%d %s(): %r -- branch %s never taken (counts %s)" % (key[0], num, key[1], key[2], missing, branches))
    assert not bad, "untaken branch outcomes that the ledger does not account for:\n" + "\n".join(bad)


def test_every_ledger_entry_is_still_untaken(reports):
    """fails when a listed outcome is taken (the entry is stale) or its statement is gone"""
    scope = _in_scope(reports)
    bad = []
    for src, func, stmt, n, untaken, kind, _ in branch_ledger.LEDGER:
        if (src, func, stmt, n) not in scope:
            bad.append("%s %s(): %r (#%d) not found among the branch lines" % (src, func, stmt, n))
            continue
        num, branches = scope[(src, func, stmt, n)]
        taken = [i for i in untaken if i >= len(branches) or branches[i] > 0]
        if taken:
            bad.append("%s:%d %s(): %r -- listed branch %s is taken (counts %s)" % (src, num, func, stmt, taken, branches))
    assert not bad, "ledger entries that no longer hold:\n" + "\n".join(bad)


@pytest.mark.parametrize("target", branch_ledger.REQUIRED, ids=[t[3] for t in branch_ledger.REQUIRED])
def test_corpus_takes_every_branch(reports, target):
    src, anchor, stmt, what = target
    ln = oracle_coverage.find(reports[src], anchor, stmt)
    assert ln.count and ln.branches, "%s: line not executed (%s)" % (what, stmt)
    assert all(b > 0 for b in ln.branches), "%s: branch counts %s" % (what, ln.branches)
