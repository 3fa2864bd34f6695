#!/usr/bin/env python3
"""Generates tests/golden/lamejs_loud_golden.json: what REAL lamejs (/root/reference under Qt's QJSEngine) does with loud
Float32 input -- samples from 16 x full scale up to the largest Float32 that stays finite after the configuration's scale --
in every MPEG version, mono and stereo, at the lowest and highest bitrate each rate encodes without resampling, and in two
integer-ratio resampled configurations.

The driver is make_lamejs_float_golden.py's (lamejs_float), with every scheduled lame_encode_buffer / lame_encode_flush
call wrapped in try/catch.  Past the magnitude at which a frame's bits no longer fit its slot, format_bitstream's
consistency check (BitStream.js:856-885) calls System.err.println, which common.js does not define, and the call throws.
A case stores its input as (kind, magnitude, samples, rate, seed, schedule) (tests/float_signals.py) and what lamejs
returned: the sizes of the calls before the one that threw, the index of that call (null if none threw), the error text,
the SHA-256 of the bytes, and for ReplayGain cases that did not throw, the tag frame and gfc.RadioGain after the flush.

  make -C tools/jsrun && python tests/golden/make_lamejs_loud_golden.py      # a few minutes, 8 processes
The fixtures travel to the GPU box; the engine and /root/reference do not."""
import hashlib
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import float_signals as FS  # noqa: E402
import oracle_f32  # noqa: E402
import oracle_lib  # noqa: E402
import make_lamejs_float_golden as FG  # noqa: E402

_CALL = " var buf=new Int8Array(0|(1.25*k0+7200+2880)); var k=lame.lame_encode_buffer(gfp,l,r,k0,buf,0,buf.length);"
_FLUSH = " var fb=new Int8Array(7200+4*2880); var k2=lame.lame_encode_flush(gfp,fb,0,fb.length);"


def _driver(rg):
    """FG's driver with each call in try/catch; the loop stops at the call that throws"""
    d = FG._driver(rg)
    for old, new in [
        (" var hex=[], sizes=[];\n", " var hex=[], sizes=[], thrown=null, err=null;\n"),
        (_CALL, " var buf=new Int8Array(0|(1.25*k0+7200+2880)), k;\n"
                " try { k=lame.lame_encode_buffer(gfp,l,r,k0,buf,0,buf.length); } catch(e){ thrown=s; err=String(e); break; }"),
        (_FLUSH, " var fb=new Int8Array(7200+4*2880), k2;\n"
                 " try { k2=lame.lame_encode_flush(gfp,fb,0,fb.length); } catch(e){ thrown=s; err=String(e); break; }"),
        ("return JSON.stringify({", "return JSON.stringify({thrown:thrown, err:err, "),
    ]:
        assert d.count(old) == 1, old
        d = d.replace(old, new)
    return d


def native(samplerate, channels):
    """(lowest, highest) bitrate Mp3Encoder encodes at `samplerate` without resampling"""
    kb = [k for k in (8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160, 192, 224, 256, 320)
          if oracle_lib.out_samplerate(channels, samplerate, k) == samplerate]
    return kb[0], kb[-1]


# one rate of each MPEG version; the resampled ones by 2 (MPEG-1 -> MPEG-2) and 4 (MPEG-1 -> MPEG-2.5)
RATES = (44100, 22050, 8000)
RESAMPLED = ((2, 44100, 48), (1, 32000, 8))
RG = ((2, 32000, 128), (1, 8000, 24))      # ReplayGain needs the tag (InitVbrTag); integral frame sizes (test_tag_oracle.py)


def configs():
    out = []
    for sr in RATES:
        for ch in (1, 2):
            lo, hi = native(sr, ch)
            out += [(ch, sr, lo), (ch, sr, hi)]
    return out + list(RESAMPLED)


def cases():
    c = {}

    def add(kind, mag, cfg, n, seed, ragged, rg=False):
        ch, sr, kb = cfg
        enc = oracle_f32.Encoder(ch, sr, kb)
        scale = oracle_f32.lib().lj_get_scale(enc.h)
        enc.close()
        name = "%s%s_%s_%d_%d_%d_%s" % ("rg_" if rg else "", kind, mag if mag == "max" else "%g" % mag, ch, sr, kb,
                                        "ragged" if ragged else "whole")
        c[name] = dict(kind=kind, magnitude=mag, channels=ch, samplerate=sr, kbps=kb, samples=n, seed=seed, scale=scale,
                       schedule=FS.schedule("f", n, ragged, seed), rg=rg)

    ladder = sorted(FS.LOUD_MAGNITUDES[:-1] + FS.LOUD_FINE) + ["max"]
    for i, cfg in enumerate(configs()):
        fs = 1152 if cfg[1] >= 32000 else 576
        n = 3 * fs * (cfg[1] // oracle_lib.out_samplerate(*cfg)) + 211
        for j in range(2):
            kind = FS.LOUD_KINDS[(i + 2 * j) % len(FS.LOUD_KINDS)]
            for k, mag in enumerate(ladder):
                add(kind, mag, cfg, n, 1000 + 10 * i + j, (j + k) % 2 == 1)
    # the rate loop stops at the first gain whose largest line fits IXMAX_VAL = 8206, a step of 2^-3/16 below the one that
    # does not: lines of 8191 and up (13 linbits) need a magnitude tuned to the signal.  This one quantises a line to 8201.
    add("nyquist", 401200, (2, 22050, 320), 3 * 576 + 211, 1000 + 10 * 7, False)
    for i, cfg in enumerate(RG):
        for mag in (4096, 2 ** 18, 1e6, 2 ** 24, 1e20):
            add("burst" if i == 0 else "noise", mag, cfg, cfg[1] // 4 + 101, 2000 + i, i == 1, rg=True)
    return c


def _run(item):
    name, c = item
    l, r, _ = FS.loud_case_signal(c)
    o = FG.lamejs_float(c["channels"], c["samplerate"], c["kbps"], l, r if r is not None else l, c["schedule"], c["rg"],
                        driver=_driver)
    rec = dict(c, rc=o["rc"], sizes=o["sizes"], thrown=o["thrown"], error=o["err"], bytes=len(o["bytes"]),
               sha256=hashlib.sha256(o["bytes"]).hexdigest())
    if c["rg"] and o["thrown"] is None:
        n = int(-(-o["tag_ret"] // 1))
        rec.update(tag=o["tag"][:n].hex(), radio_gain=o["radio"])
    return name, rec


def main():
    out = {}
    with ProcessPoolExecutor(8) as ex:
        for name, r in ex.map(_run, cases().items()):
            out[name] = r
            print(name, r["bytes"], r["thrown"], r["error"], flush=True)
    with open(os.path.join(HERE, "lamejs_loud_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
