#!/usr/bin/env python3
"""Generates tests/golden/lamejs_replaygain_golden.json: what REAL lamejs (/root/reference under Qt's QJSEngine, the
driver of tools/jsrun/tag_probe.py) computes with gfp.findReplayGain = true and the tag on.

lamejs's ReplayGain path does not run as shipped.  The names it leaves unbound are bound here, without touching the
source text: MAX_ORDER, GAIN_ANALYSIS_OK / _ERROR, INIT_GAIN_ANALYSIS_OK / _ERROR, GAIN_NOT_ENOUGH_SAMPLES (GainAnalysis.js),
GainAnalysis and NEQ (BitStream.js:784), and common.Arrays.ill (GainAnalysis.js:332, a typo for Arrays.fill).  One
statement is given its Java meaning by a single in-memory substitution: `i = cursamples / 8` (GainAnalysis.js:441) becomes
`i = 0 | (cursamples / 8)`, the integer division of GainAnalysis.java; the JavaScript division leaves a fraction there
(the first segment of a call has 10 samples) and `while ((i--) != 0)` never ends.  An observing hook, inserted in front
of the RMS computation of each completed window, records lsum and rsum; it changes nothing.

Per case: the stream's SHA-256, the finished tag frame, gfc.RadioGain after every flush, and the SHA-256 of the window
sums (float64 bits, little-endian, lsum and rsum per window, all titles in order).

  python tests/golden/make_lamejs_replaygain_golden.py      # a few minutes, 8 processes
The fixtures travel to the GPU box; the engine and /root/reference do not."""
import hashlib
import json
import os
import sys
import tempfile
from concurrent.futures import ProcessPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tools", "jsrun"))
from synth import make_signal  # noqa: E402

_JAVA_DIVISION = ("i = cursamples / 8;", "i = 0 | (cursamples / 8);")
_WINDOW_HOOK = ("/* Get the Root Mean Square (RMS) for this set of samples */",
                "if (typeof __rg_win === 'function') __rg_win(rgData);\n                ")

_BINDINGS = r"""
common.Arrays.ill = common.Arrays.fill;
var MAX_ORDER = GainAnalysis.MAX_ORDER, GAIN_ANALYSIS_OK = GainAnalysis.GAIN_ANALYSIS_OK, GAIN_ANALYSIS_ERROR = GainAnalysis.GAIN_ANALYSIS_ERROR,
 INIT_GAIN_ANALYSIS_OK = GainAnalysis.INIT_GAIN_ANALYSIS_OK, INIT_GAIN_ANALYSIS_ERROR = GainAnalysis.INIT_GAIN_ANALYSIS_ERROR,
 GAIN_NOT_ENOUGH_SAMPLES = GainAnalysis.GAIN_NOT_ENOUGH_SAMPLES, NEQ = BitStream.NEQ;
var __rgw = [], __f64 = new Float64Array(2), __u8 = new Uint8Array(__f64.buffer);
function __rg_win(g) { __f64[0] = g.lsum; __f64[1] = g.rsum; for (var i = 0; i < 16; i++) __rgw.push(__u8[i]); }
"""

_LOOP = r"""
 var L=__unhex(__HEXL), R=__CH==2?__unhex(__HEXR):L, pos=0, radio=[];
 var hex=[], sizes=[];
 for (var s=0;s<__SCHED.length;s++){
   if (__SCHED[s]>=0){ var l=L.subarray(pos,pos+__SCHED[s]), r=R.subarray(pos,pos+__SCHED[s]); pos+=__SCHED[s];
     var buf=new Int8Array(0|(1.25*l.length+7200+2880)); var k=lame.lame_encode_buffer(gfp,l,r,l.length,buf,0,buf.length);
     sizes.push(k); hex.push(__tohex(buf,k)); }
   else { var fb=new Int8Array(7200+4*2880); var k2=lame.lame_encode_flush(gfp,fb,0,fb.length); sizes.push(k2); hex.push(__tohex(fb,k2));
     radio.push(gfc.RadioGain); }
 }
"""


def _driver():
    import tag_probe as T
    d = T._TAG_DRIVER
    for old, new in [
        ("var Tables=__require('Tables.js');\n", "var Tables=__require('Tables.js');\n" + _BINDINGS),
        ("gfp.bWriteVbrTag=true;", "gfp.bWriteVbrTag=true; gfp.findReplayGain=true;"),
        ("return JSON.stringify({rc:rc,", "return JSON.stringify({radio:radio, find_rg:gfc.findReplayGain, rgw:__tohex(__rgw,__rgw.length), rc:rc,"),
    ]:
        assert d.count(old) == 1, old
        d = d.replace(old, new)
    a = d.index(" var L=__unhex(__HEXL)")
    b = d.index(" var tag=new Int8Array(2880)")
    return d[:a] + _LOOP + d[b:]


def lamejs_replaygain(channels, samplerate, kbps, left, right, schedule, fdlibm=False):
    """schedule: list of call sizes, -1 = flush().  Returns the engine's JSON as a dict (bytes / tag / windows decoded)."""
    import ref_lamejs as R
    src = R.modules_loader_source(hooks=False)
    for old, new in (_JAVA_DIVISION, (_WINDOW_HOOK[0], _WINDOW_HOOK[1] + _WINDOW_HOOK[0])):
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    with tempfile.TemporaryDirectory() as td:
        files = [os.path.join(R.HERE, "fdlibm.js")] if fdlibm else []
        p = os.path.join(td, "modules.js")
        open(p, "w").write(src)
        files.append(p)
        d = os.path.join(td, "drive.js")
        with open(d, "w") as f:
            f.write('var __HEXL="%s"; var __HEXR="%s"; var __CH=%d, __SR=%d, __KBPS=%d, __CHUNK=0, __SCHED=%s;\n'
                    % (R._hex16(left), R._hex16(right if right is not None else left), channels, samplerate, kbps, json.dumps(schedule)))
            f.write(_driver())
        files.append(d)
        o = json.loads(R.run_js(files))
    o["bytes"] = bytes.fromhex(o.pop("hex"))
    o["tag"] = bytes.fromhex(o["tag"])
    o["rgw"] = bytes.fromhex(o["rgw"])
    return o


def cases():
    c = {}

    def add(name, kind, ch, sr, kbps, n, seed, sched, fdlibm=False):
        c[name] = dict(kind=kind, channels=ch, samplerate=sr, kbps=kbps, samples=n, seed=seed, schedule=sched, fdlibm=fdlibm)

    def whole(n):
        return [n, -1]

    def chunks(n, step):
        return [min(step, n - i) for i in range(0, n, step)] + [-1]

    def odd(n):
        out, i, k = [], 0, 0
        while i < n:
            s = min((7, 333, 1000)[k % 3], n - i)
            out.append(s)
            i += s
            k += 1
        return out + [-1]

    # the tag must fit the frame (InitVbrTag), or lamejs switches the analysis off: no mono resampled configuration qualifies
    native = [(2, 48000, 128), (2, 44100, 128), (1, 32000, 64), (2, 24000, 64), (1, 22050, 64), (2, 16000, 40),
              (1, 12000, 32), (2, 11025, 32), (1, 8000, 24)]
    for i, (ch, sr, kb) in enumerate(native):
        n = sr * 3 // 4 + 101
        add("noise_%d_%d_whole" % (ch, sr), "noise", ch, sr, kb, n, 60 + i, whole(n))
        add("sweep_%d_%d_1152" % (ch, sr), "sweep", ch, sr, kb, n, 70 + i, chunks(n, 1152))
        add("white_%d_%d_odd" % (ch, sr), "white", ch, sr, kb, n, 80 + i, odd(n))
    for i, (ch, sr, kb) in enumerate([(2, 48000, 64), (2, 48000, 40), (2, 32000, 24), (2, 16000, 24)]):
        n = sr * 3 // 4 + 57
        add("rs_noise_%d_%d_%d_whole" % (ch, sr, kb), "noise", ch, sr, kb, n, 90 + i, whole(n))
        add("rs_sweep_%d_%d_%d_odd" % (ch, sr, kb), "sweep", ch, sr, kb, n, 95 + i, odd(n))
    add("silence_2_44100", "silence", 2, 44100, 128, 30000, 0, chunks(30000, 1152))
    add("silence_1_8000", "silence", 1, 8000, 24, 9000, 0, whole(9000))
    add("short_1_48000", "noise", 1, 48000, 128, 40, 101, whole(40))              # one window, flush zeros included
    add("short_2_48000_none", "noise", 2, 48000, 128, 0, 102, [-1])               # nothing but the flush: less than one window
    add("short_1_32000_none", "noise", 1, 32000, 64, 0, 105, [-1])
    add("twice_2_44100", "noise", 2, 44100, 128, 60000, 103, [20000, 13, -1, 27000, 10000, 2987, -1])
    add("twice_1_24000", "sweep", 1, 24000, 64, 30000, 104, [9, 15000, -1, 14991, -1])
    for i, (ch, sr, kb) in enumerate([(2, 44100, 128), (1, 22050, 64), (2, 48000, 64)]):
        n = sr // 2 + 33
        add("fdlibm_noise_%d_%d_%d" % (ch, sr, kb), "noise", ch, sr, kb, n, 110 + i, odd(n), fdlibm=True)
    return c


def _run(item):
    name, c = item
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], seed=c["seed"])
    o = lamejs_replaygain(c["channels"], c["samplerate"], c["kbps"], l, r if c["channels"] == 2 else None, c["schedule"], fdlibm=c["fdlibm"])
    assert o["find_rg"] and o["write_tag"], name
    n = int(-(-o["tag_ret"] // 1))                  # a fractional frame size in JavaScript at 44.1 / 22.05 / 11.025 kHz
    return name, dict(c, rc=o["rc"], sizes=o["sizes"], bytes=len(o["bytes"]), sha256=hashlib.sha256(o["bytes"]).hexdigest(),
                      tag=o["tag"][:n].hex(), radio_gain=o["radio"], windows=len(o["rgw"]) // 16,
                      windows_sha256=hashlib.sha256(o["rgw"]).hexdigest())


def main():
    out = {}
    with ProcessPoolExecutor(8) as ex:
        for name, r in ex.map(_run, cases().items()):
            out[name] = r
            print(name, r["radio_gain"], r["windows"], flush=True)
    with open(os.path.join(HERE, "lamejs_replaygain_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
