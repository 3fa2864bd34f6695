"""Float32 input on the CPU: the oracle's Float32 store (tests/oracle_f32.cpp) against its Int16 path, and js/index.js's
dispatch by array type under the JavaScript engine with the stubbed ffi of tests/test_js_shim.py."""
import json
import os
import re
import sys
import tempfile

import numpy as np
import pytest

import oracle_f32
import oracle_lib
import resample_tap
from synth import make_signal


def _stream(ch, sr, kb, n, seed, chunk):
    l, r = make_signal("noise", n, sr, seed=seed)
    return l, (r if ch == 2 else None), chunk


@pytest.mark.parametrize("sr", resample_tap.RATES)
def test_integer_valued_floats_equal_int16(sr):
    """an integer-valued Float32 sample stores exactly what the Int16 sample stores: every configuration (the 29 resampled
    ones with a second, longer signal) gives the Int16 bytes and per-call sizes"""
    resampled = set(resample_tap.resampled_configs())
    for ch, s, kb in resample_tap.all_configs():
        if s != sr:
            continue
        runs = [(4000, 1500)] + ([(9 * 1152 + 333, 777)] if (ch, s, kb) in resampled else [])
        for n, chunk in runs:
            l, r, chunk = _stream(ch, sr, kb, n, kb + ch, chunk)
            try:
                want = oracle_lib.encode_stream(ch, sr, kb, l, r, chunk=chunk)
            except ValueError:
                with pytest.raises(ValueError):
                    oracle_f32.Encoder(ch, sr, kb)
                continue
            got = oracle_f32.encode_stream(ch, sr, kb, l.astype(np.float32), None if r is None else r.astype(np.float32), chunk=chunk)
            assert got[0] == want[0] and got[1] == want[1], (ch, sr, kb, n)


def test_fractions_reach_the_bytes():
    """the Float32 path keeps what an Int16 cast drops: Web-Audio-style x * 32767 with fractions differs from its truncation"""
    l, r = make_signal("sweep", 8 * 1152, 44100, seed=1)
    x = (l.astype(np.float64) / 32768.0 * 0.7 * 32767.0).astype(np.float32)
    x = x + np.float32(0.37)
    a = oracle_f32.encode_stream(1, 44100, 128, x, None)[0]
    b = oracle_f32.encode_stream(1, 44100, 128, x.astype(np.int16), None)[0]
    assert a != b


def test_mixed_calls_on_one_encoder():
    """Int16 calls and Float32 calls on one encoder: the Float32 calls of integer values change nothing"""
    l, r = make_signal("noise", 7000, 48000, seed=4)
    calls_i = [(l[:3000], r[:3000]), (l[3000:], r[3000:])]
    calls_m = [(l[:3000], r[:3000]), (l[3000:].astype(np.float32), r[3000:].astype(np.float32))]
    a = oracle_f32.encode_calls(2, 48000, 160, calls_i)
    b = oracle_f32.encode_calls(2, 48000, 160, calls_m)
    assert a[0] == b[0] and a[1] == b[1]


DRIVER = r"""
(function () {
  var m = module.exports;
  var e = new m.Mp3Encoder(2, 44100, 128);
  e.encodeBuffer(new Int16Array(1152), new Int16Array(1152));
  e.encodeBuffer(new Float32Array(1152), new Float32Array(1152));
  e.encodeBuffer([0.5, -0.25, 3], [1, 2, 3]);
  e.encodeBuffer(new Int16Array(4), new Float32Array(4));
  e.seek(3, new Float32Array(1328), new Float32Array(1328));
  e.seek(3, new Int16Array(1328), new Int16Array(1328));
  e.close();
  var decl = {}; Object.keys(__lib.__decl).forEach(function (k) { decl[k] = __lib.__decl[k][1].length; });
  return JSON.stringify({calls: __calls, decl: decl, f32: [Float32Array.from([0.1])[0]]});
})();
"""


def test_js_shim_dispatches_by_array_type():
    import test_js_shim as T
    sys.path.insert(0, os.path.join(T.ROOT, "tools", "jsrun"))
    import ref_lamejs
    if not ref_lamejs.qt_dir() or not os.path.exists(os.path.join(ref_lamejs.qt_dir(), "libQt6Qml.so.6")):
        pytest.skip("no JavaScript engine in this environment")
    shim = open(os.path.join(T.ROOT, "js", "index.js")).read()
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "shim.js")
        open(p, "w").write(T.STUBS + shim + DRIVER)
        o = json.loads(ref_lamejs.run_js([p]))
    assert [c[0] for c in o["calls"]] == ["mp3b200_create", "mp3b200_encode", "mp3b200_encode_f32", "mp3b200_encode_f32",
                                          "mp3b200_encode_f32", "mp3b200_seek_f32", "mp3b200_seek", "mp3b200_destroy"]
    hdr = open(os.path.join(T.ROOT, "include", "mp3b200.h")).read()
    for name, nargs in o["decl"].items():
        m = re.search(r"\b%s\s*\(([^;]*?)\)\s*;" % name, hdr, re.S)
        assert m, name
        assert len([x for x in m.group(1).split(",") if x.strip() and x.strip() != "void"]) == nargs, name
    for name, n in o["calls"]:
        assert n == o["decl"][name], (name, n)
