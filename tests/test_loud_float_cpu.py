"""Loud Float32 input against lamejs itself (tests/golden/lamejs_loud_golden.json, made by
tests/golden/make_lamejs_loud_golden.py): samples from 16 x full scale up to the largest Float32 that stays finite after the
configuration's scale.  Past the magnitude at which a frame's bits no longer fit its slot, lamejs throws out of the call
that encodes that frame (format_bitstream's consistency check, BitStream.js:856-885); the oracle must throw at the same
call and agree on every byte before it."""
import hashlib
import json
import os

import numpy as np
import pytest

import float_signals as FS
import mp3_parse
import oracle_f32
import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
LINBITS13 = (23, 31)               # the Huffman tables whose escape carries 13 linbits (lines up to IXMAX_VAL = 8206)
GATE = 2.0 ** 40                   # MP3_F32_MAX_SAMPLE (lamejs_b200/csrc/k_resample.cuh): the library refuses louder samples
FLOAT_TAPS = ("xr", "en_l", "thm_l", "en_s", "thm_s", "xrpow_max")


def out_rate(c):
    return oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"])


def gated(c):
    """the library refuses the case's input at its gate (any sample beyond GATE once scaled)"""
    return FS.loud_peak(c) > GATE


# scalefactor band edges of the MPEG-2 rates (ISO/IEC 13818-3, table B.2); mp3_parse.py holds MPEG-1's
_SFB_LSF = {
    22050: ([0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576],
            [0, 4, 8, 12, 18, 24, 32, 42, 56, 74, 100, 132, 174, 192]),
    24000: ([0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 114, 136, 162, 194, 232, 278, 332, 394, 464, 540, 576],
            [0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 136, 180, 192]),
    16000: ([0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576],
            [0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192]),
}


def region_tables(t, gr, ch, sr):
    """the table each big-value line of granule gr, channel ch is coded with (the region split of mp3_parse.py)"""
    sfl, sfs = _SFB_LSF[sr] if sr in _SFB_LSF else (mp3_parse._SFB_L[sr], mp3_parse._SFB_S[sr])
    bv, bt = int(t["big_values"][gr][ch]), int(t["blocktype"][gr][ch])
    if bt == 2:
        r1, r2 = min(3 * sfs[3], bv), bv
    elif bt != 0:
        r1, r2 = min(sfl[8], bv), bv
    else:
        r1 = min(sfl[t["region0"][gr][ch] + 1], bv)
        r2 = min(sfl[t["region0"][gr][ch] + t["region1"][gr][ch] + 2], bv)
    ts = t["table_select"][gr][ch]
    return np.array([ts[0 if i < r1 else 1 if i < r2 else 2] for i in range(bv)], dtype=np.int32)


def run_oracle(c, trace_frames=0):
    """(bytes, per-call sizes, index of the call that threw or None, encoder traces, gain clamps)"""
    _, _, calls = FS.loud_case_signal(c)
    enc = oracle_f32.Encoder(c["channels"], c["samplerate"], c["kbps"], trace_frames, write_vbr_tag=c["rg"])
    out, sizes, thrown = bytearray(), [], None
    for i, call in enumerate(calls):
        try:
            b = enc.flush() if call is None else enc.encode_buffer(*call)
        except oracle_lib.LamejsThrows:
            thrown = i
            break
        sizes.append(len(b))
        out += b
    if thrown is not None:         # lamejs's encoder is unusable after the throw; the oracle refuses every later call
        with pytest.raises(oracle_lib.LamejsThrows):
            enc.flush()
    tr = enc.traces().copy() if trace_frames else None
    clamps = enc.L.lj_gain_clamps(enc.h)
    enc.close()
    return bytes(out), sizes, thrown, tr, clamps


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_oracle_matches_lamejs(name):
    c = GOLDEN[name]
    b, sizes, thrown, _, _ = run_oracle(c)
    assert thrown == c["thrown"], name
    assert sizes == c["sizes"], name
    assert hashlib.sha256(b).hexdigest() == c["sha256"], name
    assert (c["error"] is None) == (thrown is None)


def test_ladder_reaches_the_corners():
    """The ladder exists for the top of the gain range; it must keep reaching it."""
    gain255 = linbits13 = clamps = 0
    throws = set()
    for c in GOLDEN.values():
        if c["thrown"] is not None:
            throws.add("mpeg1" if oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"]) >= 32000 else "lsf")
        if gated(c) or c["magnitude"] < 4096:
            continue
        _, _, _, tr, n = run_oracle(c, trace_frames=64)
        clamps += n
        for t in tr:
            for gr in range(2):
                for ch in range(c["channels"]):
                    gain255 += t["global_gain"][gr][ch] == 255
                    ix = np.abs(t["l3_enc"][gr][ch])
                    if ix.max() >= 8191:
                        tab = region_tables(t, gr, ch, out_rate(c))
                        big = np.nonzero(ix[:len(tab)] >= 8191)[0]
                        assert len(big) and np.isin(tab[big], LINBITS13).all(), c   # only 13 linbits code such a line
                        linbits13 += 1
    assert gain255 > 0 and clamps > 0 and linbits13 > 0, (gain255, clamps, linbits13)
    assert throws == {"mpeg1", "lsf"}


def test_intermediates_are_finite_below_the_gate_and_overflow_above_it():
    """What the library's input gate rests on.  Up to the gate every intermediate lamejs computes -- MDCT lines, masking
    energies and thresholds, xrpow_max -- is finite, in every frame including the one lamejs throws on.  From 1e15 x full
    scale up its masking energies overflow Float32, from 1e30 up its MDCT lines too, and lamejs still returns bytes for some
    of those streams."""
    below = 0
    energies, lines, encoded = set(), set(), set()
    for name, c in sorted(GOLDEN.items()):
        _, _, thrown, tr, _ = run_oracle(c, trace_frames=64)
        bad = {k for k in FLOAT_TAPS if not np.isfinite(tr[k]).all()}
        big = c["magnitude"] == "max" or c["magnitude"] >= 1e15
        if not big:
            assert not bad, name                   # up to 1e9 x full scale, refused or not
            below += 0 if gated(c) else len(tr)
            continue
        assert gated(c), name
        if bad & {"en_l", "en_s"}:
            energies.add(c["magnitude"])
        if "xr" in bad:
            lines.add(c["magnitude"])
            assert c["magnitude"] == "max" or c["magnitude"] >= 1e30, name
        if bad and thrown is None:
            encoded.add(name)
    assert below > 1000 and 1e15 in energies and min(m for m in lines if m != "max") == 1e30 and encoded


def test_golden_covers_the_ladder():
    g = list(GOLDEN.values())
    assert {c["kind"] for c in g} == set(FS.LOUD_KINDS)
    assert {c["magnitude"] for c in g} >= set(FS.LOUD_MAGNITUDES) | set(FS.LOUD_FINE)
    rates = {oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"]) for c in g}
    assert {r >= 32000 for r in rates} == {True, False} and min(rates) <= 12000          # MPEG-1, 2 and 2.5
    assert any(oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"]) != c["samplerate"] for c in g)
    assert any(c["thrown"] not in (None, 0) and c["sizes"] and sum(c["sizes"]) > 0 for c in g)   # bytes, then a throw
    assert any(c["rg"] and c["thrown"] is None for c in g) and any(c["rg"] and c["thrown"] is not None for c in g)
    assert any(c["thrown"] is None and c["magnitude"] == "max" for c in g)    # lamejs encodes some of the loudest input
