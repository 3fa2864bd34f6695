"""js/index.js's ReplayGain surface (options.findReplayGain, replayGain(), Mp3Encoder.albumGain) executed under the JavaScript
engine against the stubbed ffi of tests/test_js_shim.py: it calls the C-ABI in order, with the arity include/mp3b200.h
declares."""
import json
import os
import re
import sys
import tempfile

import pytest

import test_js_shim as T

DRIVER = r"""
(function () {
  var m = module.exports;
  var e = new m.Mp3Encoder(2, 44100, 128, {writeVbrTag: true, findReplayGain: true});
  e.encodeBuffer(new Int16Array(1152), new Int16Array(1152));
  e.flush();
  var g = e.replayGain();
  var a = m.Mp3Encoder.albumGain([e]);
  e.close();
  var decl = {}; Object.keys(__lib.__decl).forEach(function (k) { decl[k] = __lib.__decl[k][1].length; });
  return JSON.stringify({calls: __calls, decl: decl, exports: Object.keys(m), g: g});
})();
"""


def test_replaygain_calls():
    sys.path.insert(0, os.path.join(T.ROOT, "tools", "jsrun"))
    import ref_lamejs
    if not ref_lamejs.qt_dir() or not os.path.exists(os.path.join(ref_lamejs.qt_dir(), "libQt6Qml.so.6")):
        pytest.skip("no JavaScript engine in this environment")
    stubs = T.STUBS.replace("alloc: function () {", "writePointer: function () {}, alloc: function () {")
    shim = open(os.path.join(T.ROOT, "js", "index.js")).read()
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "shim.js")
        open(p, "w").write(stubs + shim + DRIVER)
        o = json.loads(ref_lamejs.run_js([p]))
    assert o["exports"] == ["Mp3Encoder", "WavHeader"]
    assert [c[0] for c in o["calls"]] == ["mp3b200_create", "mp3b200_set_write_vbr_tag", "mp3b200_lametag_size", "mp3b200_set_find_replay_gain",
                                          "mp3b200_encode", "mp3b200_flush", "mp3b200_get_replay_gain", "mp3b200_album_gain", "mp3b200_destroy"]
    assert o["g"] is None                    # the stub reports no title (0)
    hdr = open(os.path.join(T.ROOT, "include", "mp3b200.h")).read()
    for name, nargs in o["decl"].items():
        m = re.search(r"\b%s\s*\(([^;]*?)\)\s*;" % name, hdr, re.S)
        assert m, name
        assert len([x for x in m.group(1).split(",") if x.strip() and x.strip() != "void"]) == nargs, name
    for name, n in o["calls"]:
        assert n == o["decl"][name], (name, n)
