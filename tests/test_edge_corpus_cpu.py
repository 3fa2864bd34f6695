"""Keeps the edge corpus (tests/edge_signals.py) honest: the oracle, built with gcov coverage into a temporary directory,
encodes every case, and the data-dependent branches the corpus exists for must all have been taken both ways.  The
GPU copies of these branches are only checked where an input reaches them, so a corpus that silently stopped reaching
them would leave tests/test_gpu_edges.py green for the wrong reason.  Statements are found by their source text (and,
where the same text occurs more than once, by the nearest unique line before it), not by line number."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

import edge_signals
import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))

# (file, anchor or None, statement, what it is).  With an anchor, the statement is the first line with that text after the
# anchor line.  Every branch gcov reports on the statement's line must have been taken.
#
# Not listed: the global-gain clamps of bin_search_StepSize (gain < 0 -> 0, gain > 255 -> 255) and the exit of its follow-up
# loop at gain 255.  From a true in-state (the previous granule's gain, step 2 or 4) no 16-bit input reaches them: the
# smallest nonzero input (+-1 LSB clicks) still lands near gain 60, and full-scale noise at 8 kbps near 224, where every
# line already quantizes to 0.  On the GPU they are reached from speculative start gains (tests/test_gpu_speculation.py).
TARGETS = [
    ("lj_quant.cpp", "cod_info->scalefac[sfb]++;", "if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];",
     "amp_scalefac_bands raises xrpow_max"),
    ("lj_quant.cpp", "double amp = e->ipow20[202];", "if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];",
     "inc_subblock_gain raises xrpow_max in the sfb21 region"),
    ("lj_psy.cpp", None, "if (e->blocktype_old[chn] == STOP_TYPE) e->blocktype_old[chn] = SHORT_TYPE;",
     "block-type FSM rewrites STOP -> SHORT (an attack one granule after a short block ended)"),
    ("lj_psy.cpp", None, "if (ns_attacks[0] != 0 && e->lastAttacks[chn] != 0) ns_attacks[0] = 0;",
     "an attack in sub-block 0 is suppressed by the previous granule's lastAttacks"),
]

_RUNNER = r"""
import hashlib, json, sys
import numpy as np
sys.path.insert(0, sys.argv[2])
import oracle_lib, edge_signals
oracle_lib.ORACLE_SO = sys.argv[1]
res = []
for c in edge_signals.CASES:
    kind, ch, sr, kbps, frames = c
    l, r = edge_signals.signal(c)
    b, _, tr = oracle_lib.encode_stream(ch, sr, kbps, l, r, trace_frames=frames + 8)
    G = 2 if sr >= 32000 else 1
    g = tr["global_gain"][:, :G, :ch]
    res.append({"case": edge_signals.case_id(c), "sha": hashlib.sha256(b).hexdigest(), "gmin": int(g.min()), "gmax": int(g.max()),
                "native": oracle_lib.out_samplerate(ch, sr, kbps) == sr})
print(json.dumps(res))
"""


def _parse_gcov(path):
    """[(count or None, source text, [branch taken counts])] per source line of a `gcov -b` report."""
    lines = []
    for raw in open(path, encoding="utf-8", errors="replace"):
        m = re.match(r"\s*([^:]+):\s*(\d+):(.*)$", raw.rstrip("\n"))
        if m:
            cnt, num, src = m.group(1).strip(), int(m.group(2)), m.group(3)
            if num == 0:
                continue
            c = None if cnt == "-" else 0 if cnt.startswith("#") or cnt.startswith("=") else int(cnt.rstrip("*"))
            lines.append([c, src, []])
            continue
        m = re.match(r"branch\s+\d+\s+(taken (\d+)|never executed)", raw)
        if m and lines:
            lines[-1][2].append(int(m.group(2)) if m.group(2) else 0)
    return lines


def _find(lines, anchor, stmt):
    start = 0
    if anchor is not None:
        hits = [i for i, ln in enumerate(lines) if anchor in ln[1]]
        assert len(hits) == 1, "anchor %r found %d times" % (anchor, len(hits))
        start = hits[0] + 1
    hits = [i for i in range(start, len(lines)) if lines[i][1].strip() == stmt]
    assert hits, "statement %r not found" % stmt
    if anchor is None:
        assert len(hits) == 1, "statement %r found %d times: give it an anchor" % (stmt, len(hits))
    return lines[hits[0]]


@pytest.fixture(scope="module")
def coverage(tmp_path_factory):
    gcov = shutil.which("gcov")
    if gcov is None:
        pytest.fail("gcov (part of gcc) is needed to check the edge corpus")
    # the compiler installed beside gcov: its coverage runtime and data format match gcov's
    cxx = os.path.join(os.path.dirname(gcov), "g++")
    cxx = cxx if os.path.exists(cxx) else "g++"
    d = tmp_path_factory.mktemp("oracle_cov")
    for f in os.listdir(oracle_lib.ORACLE_DIR):
        if f.endswith((".cpp", ".h")) or f == "Makefile":
            shutil.copy(os.path.join(oracle_lib.ORACLE_DIR, f), d)
    mk = open(os.path.join(d, "Makefile")).read()
    flags = re.search(r"^CXXFLAGS\s*=\s*(.*)$", mk, re.M).group(1)
    # -O0 keeps one gcov branch per source-level outcome; the numerics flags stay (the bytes are compared below)
    subprocess.check_call(["make", "-s", "-C", str(d), "CXX=" + cxx, "CXXFLAGS=" + flags.replace("-O2", "-O0") + " --coverage"])
    out = subprocess.run([sys.executable, "-c", _RUNNER, str(d / "liblamejs_oracle.so"), HERE], check=True, capture_output=True,
                         text=True, cwd=str(d)).stdout
    runs = json.loads(out.strip().splitlines()[-1])
    reports = {}
    for src in sorted({t[0] for t in TARGETS}):
        gcda = [f for f in os.listdir(d) if f.endswith(src[:-4] + ".gcda")]
        assert len(gcda) == 1, (src, os.listdir(d))
        subprocess.run([gcov, "-b", "-c", gcda[0]], check=True, capture_output=True, cwd=str(d))
        reports[src] = _parse_gcov(os.path.join(d, src + ".gcov"))
    return runs, reports


@pytest.mark.parametrize("target", TARGETS, ids=[t[3] for t in TARGETS])
def test_corpus_takes_every_branch(coverage, target):
    _, reports = coverage
    src, anchor, stmt, what = target
    count, _, branches = _find(reports[src], anchor, stmt)
    assert count and branches, "%s: line not executed (%s)" % (what, stmt)
    assert all(b > 0 for b in branches), "%s: branch counts %s" % (what, branches)


def test_corpus_spans_the_reachable_gain_range(coverage):
    """+-1 LSB input at the highest bitrates drives the global gain as low as 16-bit input can (about 60), full-scale noise
    at the lowest native bitrates as high as it can (about 224); every case is a native configuration (no resampling)."""
    runs, _ = coverage
    assert all(r["native"] for r in runs), [r["case"] for r in runs if not r["native"]]
    assert min(r["gmin"] for r in runs) <= 66, min(r["gmin"] for r in runs)
    assert max(r["gmax"] for r in runs) >= 222, max(r["gmax"] for r in runs)


def test_coverage_build_encodes_like_the_oracle(coverage, oracle):
    """The instrumented -O0 build is only a witness if it computes what the oracle computes."""
    import hashlib

    runs, _ = coverage
    for c, r in zip(edge_signals.CASES, runs):
        l, rr = edge_signals.signal(c)
        assert hashlib.sha256(oracle.encode_stream(c[1], c[2], c[3], l, rr)[0]).hexdigest() == r["sha"], r["case"]
