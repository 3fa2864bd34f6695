#!/usr/bin/env python3
"""Generates tests/golden/lamejs_wav_golden.json: what REAL lamejs (unmodified reference under Qt's QJSEngine,
tools/jsrun/ref_lamejs.py) makes of whole WAV files, run the way worker-example/worker.js runs one but with the whole file
in one call:

  w = lamejs.WavHeader.readHeader(new DataView(f));  v = new Int16Array(f, w.dataOffset, w.dataLen / 2);
  stereo: left / right = new Int16Array(w.dataLen / (2 * w.channels)), left[i] = v[2 i], right[i] = v[2 i + 1];
  e = new lamejs.Mp3Encoder(w.channels, w.sampleRate, kbps);  mp3 = e.encodeBuffer(left, right) ++ e.flush()

For each hand-made file of corpus() it records the outcome: the header, the view's and the channels' lengths and the
MP3's size and SHA-256, or what lamejs returns / throws and at which step.  The files themselves are rebuilt by corpus()
(tests import it) and pinned by their SHA-256.  The 8-bit and float files, which the library refuses, are run too: their
bytes are what lamejs makes of them (Int16 noise).

  python tests/golden/make_lamejs_wav_golden.py      # ~1 minute, 8 processes
The fixtures are committed: the tests need neither the engine nor the reference."""
import hashlib
import json
import os
import struct
import sys
import tempfile
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
from synth import make_signal  # noqa: E402


def fmt(ch, sr, n=16, tag=1, bits=16):
    body = struct.pack("<HHIIHH", tag, ch, sr, sr * ch * bits // 8, ch * bits // 8, bits) + b"\0" * (n - 16)
    return b"fmt " + struct.pack("<I", n) + body


def riff(chunks, magic=b"RIFF"):
    body = b"WAVE" + b"".join(chunks)
    return magic + struct.pack("<I", len(body)) + body


def pcm(ch, sr, frames, seed, kind="noise"):
    """interleaved little-endian Int16 frames of a synth signal"""
    l, r = make_signal(kind, frames, sr, seed=seed)
    x = np.stack([l, r], axis=1)[:, :ch] if ch else np.zeros((0, 1), np.int16)
    return np.ascontiguousarray(x, dtype="<i2").tobytes()


def data(payload, n=None):
    return b"data" + struct.pack("<I", len(payload) if n is None else n) + payload


LIST = b"LIST" + struct.pack("<I", 26) + b"INFOISFT" + struct.pack("<I", 14) + b"Lavf58.29.100\0"


def corpus():
    """name -> (wav bytes, kbps, resample): mono and stereo at every MPEG-1 / 2 / 2.5 rate lamejs encodes natively, one
    48 kHz file lamejs resamples by 2, and the header and view edge cases"""
    c = {}

    def add(name, wav, kbps, resample=False):
        c[name] = (wav, kbps, resample)

    add("mono_8k", riff([fmt(1, 8000), data(pcm(1, 8000, 3001, 1))]), 32)
    add("stereo_16k", riff([fmt(2, 16000), data(pcm(2, 16000, 3500, 2, "sweep"))]), 64)
    add("mono_22k", riff([fmt(1, 22050), data(pcm(1, 22050, 4000, 3, "octave"))]), 64)
    add("stereo_24k", riff([fmt(2, 24000), data(pcm(2, 24000, 3333, 4))]), 64)
    add("mono_32k", riff([fmt(1, 32000), data(pcm(1, 32000, 4608, 5, "burst"))]), 128)
    add("stereo_44k", riff([fmt(2, 44100), data(pcm(2, 44100, 5000, 6))]), 128)
    add("stereo_48k", riff([fmt(2, 48000), data(pcm(2, 48000, 4700, 7, "white"))]), 192)
    add("stereo_48k_resampled", riff([fmt(2, 48000), data(pcm(2, 48000, 6000, 8))]), 64, True)   # lamejs encodes at 24 kHz
    add("stereo_44k_fmt18", riff([fmt(2, 44100, 18), data(pcm(2, 44100, 2500, 9))]), 128)
    add("mono_44k_list_before_data", riff([fmt(1, 44100), LIST, data(pcm(1, 44100, 2500, 10))]), 96)
    # two odd-length chunks: lamejs does not pad chunks, and 3 + 5 leaves the data region at an even offset
    add("stereo_32k_odd_chunks_even_offset",
        riff([fmt(2, 32000), b"junk" + struct.pack("<I", 3) + b"abc", b"pad " + struct.pack("<I", 5) + b"defgh",
              data(pcm(2, 32000, 2200, 11))]), 160)
    add("stereo_44k_odd_offset", riff([fmt(2, 44100), b"junk" + struct.pack("<I", 3) + b"abc", data(pcm(2, 44100, 1000, 12))]), 128)
    add("stereo_44k_empty_data", riff([fmt(2, 44100), data(b"")]), 128)
    add("mono_22k_odd_data_len", riff([fmt(1, 22050), data(pcm(1, 22050, 1500, 13) + b"\x7f")]), 48)
    add("stereo_24k_data_len_4k_plus_2", riff([fmt(2, 24000), data(pcm(2, 24000, 1700, 14) + b"\x01\x02")]), 64)
    add("stereo_44k_truncated_data", riff([fmt(2, 44100), data(pcm(2, 44100, 900, 15), n=4 * 2000)]), 128)
    add("stereo_44k_streaming_len", riff([fmt(2, 44100), data(pcm(2, 44100, 900, 16), n=0xFFFFFFFF)]), 128)
    add("truncated_header", riff([fmt(2, 44100), data(pcm(2, 44100, 100, 17))])[:30], 128)
    add("not_riff", riff([fmt(2, 44100), data(pcm(2, 44100, 100, 18))], magic=b"RIFX"), 128)
    add("extended_fmt_40", riff([fmt(2, 44100, 40, 0xFFFE), data(pcm(2, 44100, 100, 19))]), 128)
    add("zero_channels", riff([fmt(0, 44100), data(pcm(2, 44100, 100, 20))]), 128)
    # the 16-bit deviation: lamejs reads these as Int16 all the same
    add("mono_44k_8bit", riff([fmt(1, 44100, bits=8), data(bytes((np.arange(4000) * 7 % 256).astype(np.uint8)))]), 128)
    add("stereo_44k_float32", riff([fmt(2, 44100, tag=3, bits=32),
                                    data(np.sin(np.arange(2 * 1500) / 9.0).astype("<f4").tobytes())]), 128)
    # a rate lamejs resamples by a non-integer ratio (44.1 kHz mono at 8 kbps encodes at 8 kHz)
    add("mono_44k_8kbps", riff([fmt(1, 44100), data(pcm(1, 44100, 3000, 21))]), 8)
    return c


_DRIVER = r"""
function __tohex(b){ var s=[]; for(var i=0;i<b.length;i++){ var v=b[i]&255; s.push((v<16?"0":"")+v.toString(16)); } return s.join(""); }
(function(){
  var h=__HEX, n=h.length/2, ab=new ArrayBuffer(n), u=new Uint8Array(ab);
  for (var i=0;i<n;i++) u[i]=parseInt(h.substr(2*i,2),16);
  var step='readHeader', w, o={};
  try {
    w = lamejs.WavHeader.readHeader(new DataView(ab));
    if (w === undefined) return JSON.stringify({step: step, undefined: true});
    o.header = {dataOffset: w.dataOffset, dataLen: w.dataLen, channels: w.channels, sampleRate: w.sampleRate};
    step = 'view';
    var v = new Int16Array(ab, w.dataOffset, w.dataLen / 2);
    o.view_len = v.length;
    step = 'split';
    var left = w.channels === 1 ? v : new Int16Array(w.dataLen / (2 * w.channels));
    var right = w.channels === 2 ? new Int16Array(w.dataLen / (2 * w.channels)) : undefined;
    if (w.channels > 1) for (var i = 0; i < left.length; i++) { left[i] = v[i * 2]; right[i] = v[i * 2 + 1]; }
    o.left_len = left.length; o.right_len = right ? right.length : -1;
    step = 'encode';
    var e = new lamejs.Mp3Encoder(w.channels, w.sampleRate, __KBPS);
    var a = e.encodeBuffer(left, right), b = e.flush();
    o.hex = __tohex(a) + __tohex(b);
  } catch (err) {
    o.step = step; o.throws = (typeof err === 'string') ? err : (err && err.name ? err.name : String(err));
  }
  return JSON.stringify(o);
})();
"""


def run(item):
    sys.path.insert(0, os.path.join(ROOT, "tools", "jsrun"))
    import ref_lamejs as R
    name, (wav, kbps, resample) = item
    with tempfile.TemporaryDirectory() as td:
        d = os.path.join(td, "drive.js")
        with open(d, "w") as f:
            f.write('var __HEX="%s"; var __KBPS=%d;\n' % (wav.hex(), kbps) + _DRIVER)
        o = json.loads(R.run_js([os.path.join(R.REF, "lame.all.js"), d]))
    if "hex" in o:
        mp3 = bytes.fromhex(o.pop("hex"))
        o.update(mp3_bytes=len(mp3), mp3_sha256=hashlib.sha256(mp3).hexdigest())
    o.update(wav_sha256=hashlib.sha256(wav).hexdigest(), wav_bytes=len(wav), kbps=kbps, resample=resample)
    return name, o


def main():
    sys.path.insert(0, os.path.join(ROOT, "tools", "jsrun"))
    import ref_lamejs as R
    R.build()                                  # once, before the workers run it
    with ProcessPoolExecutor(8) as ex:
        out = dict(ex.map(run, corpus().items()))
    with open(os.path.join(HERE, "lamejs_wav_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print({k: (v.get("throws") or ("undefined" if v.get("undefined") else v.get("mp3_bytes"))) for k, v in out.items()})


if __name__ == "__main__":
    main()
