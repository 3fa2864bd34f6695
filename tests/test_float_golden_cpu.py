"""The oracle's Float32 store (tests/oracle_f32.cpp) and the ReplayGain restatement fed with Float32 (replaygain_ref_f32)
against lamejs itself with Float32Array / Array / mixed Int16Array and Float32Array input
(tests/golden/lamejs_float_golden.json, made by tests/golden/make_lamejs_float_golden.py)."""
import hashlib
import json
import os

import numpy as np
import pytest

import float_signals as FS
import oracle_f32
import oracle_lib
import replaygain_ref as RG
import replaygain_ref_f32 as RGF

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))
# lamejs's frame size is a fraction at these output rates; its own tagged stream then differs from LAME's (test_tag_oracle.py)
FRACTIONAL = (44100, 22050, 11025)


def out_rate(c):
    return oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"])


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_oracle_matches_lamejs(name):
    c = GOLDEN[name]
    _, _, calls = FS.case_signal(c)
    assert calls[-1] is None and None not in calls[:-1]
    b, sizes, _, _ = oracle_f32.encode_calls(c["channels"], c["samplerate"], c["kbps"], calls[:-1], write_vbr_tag=c["rg"])
    if c["rg"] and out_rate(c) in FRACTIONAL:
        return
    assert sizes == c["sizes"], name
    assert hashlib.sha256(b).hexdigest() == c["sha256"], name


@pytest.mark.parametrize("name", sorted(n for n in GOLDEN if GOLDEN[n]["rg"]))
def test_replaygain_restatement_matches_lamejs(name):
    c = GOLDEN[name]
    l, r, _ = FS.case_signal(c)
    sched = [("flush",) if s[0] < 0 else ("enc", s[0]) for s in c["schedule"]]
    res = RGF.analyze_calls(c["channels"], c["samplerate"], c["kbps"], l, r, sched)
    sums = np.concatenate([w[:, :2] for w in res.windows]) if res.windows else np.zeros((0, 2), np.uint64)
    assert len(sums) == c["windows"]
    assert hashlib.sha256(np.ascontiguousarray(sums, dtype="<u8").tobytes()).hexdigest() == c["windows_sha256"]
    assert res.radio == c["radio_gain"]


def test_golden_covers_the_issue():
    g = GOLDEN.values()
    rates = {c["samplerate"] for c in g if out_rate(c) == c["samplerate"]}
    assert rates == {8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000}
    assert {(c["channels"], c["samplerate"]) for c in g} >= {(ch, sr) for ch in (1, 2) for sr in rates}
    assert any(out_rate(c) != c["samplerate"] for c in g)
    assert {c["kind"] for c in g} == set(FS.KINDS)
    assert any(t == "i" for c in g for s in c["schedule"] for t in s[1:]) and any(t == "a" for c in g for s in c["schedule"] for t in s[1:])
    assert any(c["rg"] and out_rate(c) != c["samplerate"] for c in g) and any(c["rg"] and c["kind"] == "mixed" for c in g)
    assert any(0 < s[0] < 10 for c in g for s in c["schedule"])
