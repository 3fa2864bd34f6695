#!/usr/bin/env python3
"""Generates tests/golden/lamejs_float_golden.json: what REAL lamejs (/root/reference under Qt's QJSEngine) produces when
encodeBuffer is given Float32Arrays, plain Arrays of numbers, or Int16Arrays and Float32Arrays in turn.

The driver is the one of make_lamejs_replaygain_golden.py (lamejs's modules, lame_encode_buffer / lame_encode_flush called
per scheduled call, the unbound ReplayGain names bound, the Java division substituted in memory, a window hook that only
records), with gfp.bWriteVbrTag and gfp.findReplayGain off (Mp3Encoder's settings, index.js:107) unless a case asks for
ReplayGain.  The samples travel as hex of their float64 bits: every kind but "array" holds Float32 values, so that is the
hex of Float32 bit patterns widened exactly; "array" holds doubles, which lamejs rounds at its Float32Array store.

Signals and call schedules come from tests/float_signals.py; a case stores (kind, samples, rate, seed, schedule) and what
lamejs returned: per-call sizes, the stream's SHA-256, and for ReplayGain cases the tag frame, gfc.RadioGain after every
flush and the SHA-256 of the window sums.

  python tests/golden/make_lamejs_float_golden.py      # a few minutes, 8 processes
The fixtures travel to the GPU box; the engine and /root/reference do not."""
import hashlib
import json
import os
import sys
import tempfile
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tools", "jsrun"))
import float_signals as FS  # noqa: E402
import oracle_lib  # noqa: E402
import make_lamejs_replaygain_golden as RGM  # noqa: E402

_HELPERS = r"""
function __unhex64(h){ var n=h.length/16, u=new Uint8Array(8*n); for(var i=0;i<8*n;i++) u[i]=parseInt(h.substr(2*i,2),16);
  return new Float64Array(u.buffer); }
function __as(X,pos,k,t){ var s=X.subarray(pos,pos+k);
  if (t=="f") return new Float32Array(s); if (t=="i") return new Int16Array(s); return Array.prototype.slice.call(s); }
"""

_LOOP = r"""
 var L=__unhex64(__HEXL), R=__CH==2?__unhex64(__HEXR):L, pos=0, radio=[];
 var hex=[], sizes=[];
 for (var s=0;s<__SCHED.length;s++){
   if (__SCHED[s][0]>=0){ var k0=__SCHED[s][0], t=__SCHED[s][1], l=__as(L,pos,k0,t), r=__as(R,pos,k0,t); pos+=k0;
     var buf=new Int8Array(0|(1.25*k0+7200+2880)); var k=lame.lame_encode_buffer(gfp,l,r,k0,buf,0,buf.length);
     sizes.push(k); hex.push(__tohex(buf,k)); }
   else { var fb=new Int8Array(7200+4*2880); var k2=lame.lame_encode_flush(gfp,fb,0,fb.length); sizes.push(k2); hex.push(__tohex(fb,k2));
     radio.push(gfc.RadioGain); }
 }
"""


def _driver(rg):
    import tag_probe as T
    d = T._TAG_DRIVER
    flags = "gfp.bWriteVbrTag=true; gfp.findReplayGain=true;" if rg else "gfp.bWriteVbrTag=false;"
    for old, new in [
        ("var Tables=__require('Tables.js');\n", "var Tables=__require('Tables.js');\n" + RGM._BINDINGS + _HELPERS),
        ("gfp.bWriteVbrTag=true;", flags),
        ("return JSON.stringify({rc:rc,", "return JSON.stringify({radio:radio, find_rg:gfc.findReplayGain, rgw:__tohex(__rgw,__rgw.length), rc:rc,"),
    ]:
        assert d.count(old) == 1, old
        d = d.replace(old, new)
    a = d.index(" var L=__unhex(__HEXL)")
    b = d.index(" var tag=new Int8Array(2880)")
    return d[:a] + _LOOP + d[b:]


def _hex64(a):
    return np.ascontiguousarray(a, dtype="<f8").tobytes().hex()


def lamejs_float(channels, samplerate, kbps, left, right, schedule, rg, driver=None):
    """runs lamejs on one case; `driver` (default _driver) makes the driver's source from `rg`"""
    import ref_lamejs as R
    src = R.modules_loader_source(hooks=False)
    for old, new in (RGM._JAVA_DIVISION, (RGM._WINDOW_HOOK[0], RGM._WINDOW_HOOK[1] + RGM._WINDOW_HOOK[0])):
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "modules.js")
        open(p, "w").write(src)
        d = os.path.join(td, "drive.js")
        with open(d, "w") as f:
            f.write('var __HEXL="%s"; var __HEXR="%s"; var __CH=%d, __SR=%d, __KBPS=%d, __CHUNK=0, __SCHED=%s;\n'
                    % (_hex64(left), _hex64(right), channels, samplerate, kbps, json.dumps(schedule)))
            f.write((driver or _driver)(rg))
        o = json.loads(R.run_js([p, d]))
    o["bytes"] = bytes.fromhex(o.pop("hex"))
    o["tag"] = bytes.fromhex(o["tag"])
    o["rgw"] = bytes.fromhex(o["rgw"])
    return o


# (channels, rate, kbps) lamejs encodes at the input rate: every rate and channel count, two bitrates each
NATIVE = [(1, 48000, 128), (2, 48000, 320), (1, 44100, 128), (2, 44100, 192), (1, 32000, 48), (2, 32000, 128),
          (1, 24000, 48), (2, 24000, 160), (1, 22050, 64), (2, 22050, 96), (1, 16000, 24), (2, 16000, 64),
          (1, 12000, 16), (2, 12000, 48), (1, 11025, 24), (2, 11025, 56), (1, 8000, 8), (2, 8000, 24)]
# integer-ratio resampled configurations: ratios 2, 3, 4 and 6, mono and stereo
RESAMPLED = [(2, 48000, 64), (1, 48000, 8), (2, 44100, 48), (1, 32000, 16), (2, 16000, 24), (1, 24000, 8)]
# ReplayGain needs the tag to fit (InitVbrTag)
RG = [(2, 44100, 128), (1, 22050, 64), (2, 48000, 64), (1, 8000, 24), (2, 16000, 40)]


def cases():
    c = {}

    def add(name, kind, cfg, n, seed, ragged, rg=False):
        ch, sr, kb = cfg
        c[name] = dict(kind=kind, channels=ch, samplerate=sr, kbps=kb, samples=n, seed=seed,
                       schedule=FS.schedule(kind, n, ragged, seed), rg=rg)

    kinds = [k for k in FS.KINDS if k != "mixed"]
    for i, cfg in enumerate(NATIVE):
        fs = 1152 if cfg[1] >= 32000 else 576
        for j in range(2):
            kind = kinds[(i + 3 * j) % len(kinds)]
            add("%s_%d_%d_%d_%s" % (kind, cfg[0], cfg[1], cfg[2], "ragged" if j else "whole"), kind, cfg, 5 * fs + 211, 10 * i + j, j == 1)
    for i, cfg in enumerate(RESAMPLED):
        n = 4 * 576 * (cfg[1] // oracle_lib.out_samplerate(*cfg)) + 331
        for j, kind in enumerate(("webaudio", "x4") if i % 2 == 0 else ("unit", "dither")):
            add("rs_%s_%d_%d_%d_%s" % (kind, cfg[0], cfg[1], cfg[2], "ragged" if j else "whole"), kind, cfg, n, 200 + 10 * i + j, j == 1)
    for i, cfg in enumerate([(2, 44100, 128), (1, 22050, 64), (2, 48000, 64), (1, 8000, 8)]):
        fs = 1152 if cfg[1] >= 32000 else 576
        add("mixed_%d_%d_%d" % cfg, "mixed", cfg, 6 * fs + 99, 300 + i, True)
        add("array_%d_%d_%d" % cfg, "array", cfg, 3 * fs + 17, 310 + i, True)
    for i, cfg in enumerate(RG):
        n = cfg[1] * 3 // 4 + 101
        add("rg_webaudio_%d_%d_%d" % cfg, "webaudio", cfg, n, 400 + i, i % 2 == 1, rg=True)
        add("rg_unit_%d_%d_%d" % cfg, "unit", cfg, n, 410 + i, i % 2 == 0, rg=True)
    add("rg_mixed_2_44100_128", "mixed", (2, 44100, 128), 44100 * 3 // 4 + 7, 420, True, rg=True)
    return c


def _run(item):
    name, c = item
    l, r, _ = FS.case_signal(c)
    o = lamejs_float(c["channels"], c["samplerate"], c["kbps"], l, r if r is not None else l, c["schedule"], c["rg"])
    assert bool(o["find_rg"]) == c["rg"], name
    rec = dict(c, rc=o["rc"], sizes=o["sizes"], bytes=len(o["bytes"]), sha256=hashlib.sha256(o["bytes"]).hexdigest())
    if c["rg"]:
        n = int(-(-o["tag_ret"] // 1))
        rec.update(tag=o["tag"][:n].hex(), radio_gain=o["radio"], windows=len(o["rgw"]) // 16,
                   windows_sha256=hashlib.sha256(o["rgw"]).hexdigest())
    return name, rec


def main():
    out = {}
    with ProcessPoolExecutor(8) as ex:
        for name, r in ex.map(_run, cases().items()):
            out[name] = r
            print(name, r["bytes"], r.get("radio_gain"), flush=True)
    with open(os.path.join(HERE, "lamejs_float_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
