"""The oracle built with gcov coverage, and its reports: what tests/test_edge_corpus_cpu.py and tests/test_branch_ledger_cpu.py
use to show which branches of the oracle the test inputs take.

build() copies the oracle's sources and tests/oracle_f32.cpp into a directory and compiles them at -O0 with --coverage
(the oracle's numerics flags stay, so the build encodes what the oracle encodes); run() encodes streams with it in worker
processes, which add their counts to the same .gcda files as they exit; report() runs `gcov -b` on one source and
parses it.  Statements are found by their source text and the function they are in, never by line number."""
import json
import os
import re
import shutil
import subprocess
import sys

import oracle_f32
import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))
SO = "liboracle_cov.so"


def _tools():
    gcov = shutil.which("gcov")
    if gcov is None:
        raise RuntimeError("gcov (part of gcc) is needed to measure the oracle's branch coverage")
    # the compiler installed beside gcov: its coverage runtime and data format match gcov's
    cxx = os.path.join(os.path.dirname(gcov), "g++")
    return gcov, (cxx if os.path.exists(cxx) else "g++")


def build(d):
    """compiles the coverage build into directory `d` (oracle/ and tests/ below it); returns the library's path"""
    _, cxx = _tools()
    od, td = os.path.join(d, "oracle"), os.path.join(d, "tests")
    os.makedirs(od)
    os.makedirs(td)
    for f in os.listdir(oracle_lib.ORACLE_DIR):
        if f.endswith((".cpp", ".h")):
            shutil.copy(os.path.join(oracle_lib.ORACLE_DIR, f), od)
    shutil.copy(os.path.join(HERE, "oracle_f32.cpp"), td)
    # -O0 keeps one gcov branch per source-level outcome; the numerics flags stay (the bytes are compared with the oracle's)
    flags = [f for f in oracle_f32.CXXFLAGS if not f.startswith("-O")] + ["-O0", "--coverage"]
    so = os.path.join(d, SO)
    subprocess.check_call([cxx] + flags + ["-shared", "-o", so, os.path.join(td, "oracle_f32.cpp")] +
                          [os.path.join(od, s) for s in oracle_f32.SRCS] + ["-lm"], cwd=d)
    return so


_WORKER = r"""
import hashlib, json, sys
sys.path.insert(0, sys.argv[2])
import oracle_f32, oracle_inputs, oracle_lib
oracle_f32._lib = oracle_f32.bind(sys.argv[1])
want = set(json.loads(sys.argv[3]))
res = {}
for rid, ch, sr, kbps, calls in oracle_inputs.runs():
    if rid not in want:
        continue
    enc = oracle_f32.Encoder(ch, sr, kbps, trace_frames=int(sys.argv[4]))
    out = bytearray()
    try:
        for l, r in calls():
            out += enc.encode_buffer(l, r)
        out += enc.flush()
        thrown = False
    except oracle_lib.LamejsThrows:
        thrown = True
    row = {"sha": hashlib.sha256(bytes(out)).hexdigest(), "thrown": thrown}
    if int(sys.argv[4]):
        g = enc.traces()["global_gain"][:, :2 if oracle_lib.out_samplerate(ch, sr, kbps) >= 32000 else 1, :ch]
        row["gmin"], row["gmax"] = int(g.min()), int(g.max())
    enc.close()
    res[rid] = row
print(json.dumps(res))
"""


def run(so, ids, workers=None, trace_frames=0):
    """encodes the oracle_inputs.runs() streams named in `ids` with the coverage build `so`, spread over worker processes;
    returns {id: {"sha": sha256 of the bytes up to where lamejs throws, "thrown": bool, and with trace_frames > 0 (at
    least the longest stream's frames) "gmin" / "gmax", the global gains}}"""
    ids = list(ids)
    workers = workers or max(1, min(8, os.cpu_count() or 1))
    procs = []
    for k in range(workers):
        part = ids[k::workers]
        if part:
            procs.append(subprocess.Popen([sys.executable, "-c", _WORKER, so, HERE, json.dumps(part), str(trace_frames)],
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                                          cwd=os.path.dirname(so)))
    res = {}
    for p in procs:
        out, err = p.communicate()
        if p.returncode:
            raise RuntimeError("coverage worker failed:\n" + err[-4000:])
        res.update(json.loads(out.strip().splitlines()[-1]))
    return res


class Line:
    __slots__ = ("count", "src", "func", "branches")

    def __init__(self, count, src, func):
        self.count, self.src, self.func, self.branches = count, src, func, []


def report(so, src):
    """the `gcov -b` report of oracle source `src` of the coverage build `so`, after run(): [Line] per source line, with the
    execution count (None: no code), the text, the enclosing function's name (without its parameters) and the taken count
    of each branch gcov reports on the line, in gcov's order"""
    gcov, _ = _tools()
    d = os.path.dirname(so)
    gcda = os.path.join(d, "%s-%s.gcda" % (SO, src[:-4]))
    assert os.path.exists(gcda), (src, sorted(os.listdir(d)))
    out = os.path.join(d, "gcov_" + src[:-4])
    os.makedirs(out, exist_ok=True)
    subprocess.run([gcov, "-b", "-c", "-m", "-o", d, gcda], check=True, capture_output=True, cwd=out)
    return parse(os.path.join(out, src + ".gcov"))


def parse(path):
    lines, func = [], None
    for raw in open(path, encoding="utf-8", errors="replace"):
        raw = raw.rstrip("\n")
        m = re.match(r"\s*([^:]+):\s*(\d+):(.*)$", raw)
        if m:
            cnt, num, src = m.group(1).strip(), int(m.group(2)), m.group(3)
            if num == 0:
                continue
            c = None if cnt == "-" else 0 if cnt.startswith("#") or cnt.startswith("=") else int(cnt.rstrip("*"))
            lines.append(Line(c, src, func))
            continue
        m = re.match(r"function (.+?) called \d+", raw)
        if m:
            func = re.sub(r"\(.*$", "", m.group(1)).split("::")[-1]
            continue
        m = re.match(r"branch\s+\d+\s+(taken (\d+)|never executed)", raw)
        if m and lines and not raw.endswith("(throw)"):      # the exception edge of a call, not a source-level outcome
            lines[-1].branches.append(int(m.group(2)) if m.group(2) else 0)
    return lines


def find(lines, anchor, stmt):
    """the Line of statement `stmt` (its whole stripped text); with an anchor (the text of a unique line), the first such
    statement after the anchor, else the only one"""
    start = 0
    if anchor is not None:
        hits = [i for i, ln in enumerate(lines) if anchor in ln.src]
        assert len(hits) == 1, "anchor %r found %d times" % (anchor, len(hits))
        start = hits[0] + 1
    hits = [i for i in range(start, len(lines)) if lines[i].src.strip() == stmt]
    assert hits, "statement %r not found" % stmt
    if anchor is None:
        assert len(hits) == 1, "statement %r found %d times: give it an anchor" % (stmt, len(hits))
    return lines[hits[0]]
