"""The oracle's quant row trace (lj_set_quant_row_trace: xrq, xrpow, have, what lj_iteration_loop hands outer_loop)
against plain numpy from the frame trace (no GPU).  tests/quant_rows.py compares the device's rows with these fields bit for
bit, so they must mean what they say:
  xrq    the MDCT's xr of the granule (frame trace), short blocks reordered band by band (init_outer_loop: for each band, its
         lines of window 0, then of window 1, then of window 2), and above the last line that psfb21_analogsilence keeps in
         the pseudo bands (long blocks: lines from sfb_l[21] up; short blocks: each window's part of band 12) set to 0
  xrpow  init_xrpow's float32 store of sqrt(|x| sqrt(|x|)) evaluated in double, every line
  have   the granule has energy: sum |xr| > 1e-20, which is where calc_xmin ran; xrpow_max is the largest xrpow"""
import numpy as np
import pytest

import edge_signals
import mp3_parse
import psy_rows
from synth import make_signal

BT_SHORT = 2
# scalefactor band tables (ISO/IEC 11172-3, 13818-3): sfb_l[21] (start of the long blocks' pseudo bands) and sfb_s
SFB_L21 = {44100: 418, 48000: 384, 32000: 550, 22050: 522, 24000: 540, 16000: 522}
SFB_S = {**mp3_parse._SFB_S,
         22050: [0, 4, 8, 12, 18, 24, 32, 42, 56, 74, 100, 132, 174, 192],
         24000: [0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 136, 180, 192],
         16000: [0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192]}

CASES = [c for c in edge_signals.CASES if c[0] in ("square", "clicks1", "click_pairs", "hf_tone", "silent_right", "lsb_dither",
                                                   "loud_silent")]


def reorder(xr, sfb_s):
    """init_outer_loop's short-block order of a granule's 576 lines"""
    out = []
    for b in range(13):
        for w in range(3):
            out += [xr[3 * l + w] for l in range(sfb_s[b], sfb_s[b + 1])]
    return np.array(out, np.float32)


def silence_regions(short, sfb_s, l21):
    """the line ranges psfb21_analogsilence walks down from their top"""
    if not short:
        return [(l21, 576)]
    w = sfb_s[13] - sfb_s[12]
    return [(3 * sfb_s[12] + w * k, 3 * sfb_s[12] + w * (k + 1)) for k in range(3)]


def check_rows(tr, G, ch, sr, label):
    """returns (granules, short granules, granules with lines zeroed by the analog-silence rule, granules without energy)"""
    counts = np.zeros(4, int)
    for f in range(len(tr)):
        for gr in range(G):
            for c in range(ch):
                t = tr[f]
                short = t["blocktype"][gr, c] == BT_SHORT
                xr = t["xr"][gr, c]
                pre = reorder(xr, SFB_S[sr]) if short else xr.copy()
                got = t["xrq"][gr, c]
                where = (label, f, gr, c)
                zeroed = False
                for lo, hi in silence_regions(short, SFB_S[sr], SFB_L21[sr]):
                    # lines above the highest one kept are 0, the others unchanged
                    kept = np.nonzero(got[lo:hi] != 0)[0]
                    top = lo + (kept[-1] + 1 if len(kept) else 0)
                    assert not got[top:hi].any(), where
                    zeroed |= bool(pre[top:hi].any())
                    pre[top:hi] = 0
                assert np.array_equal(got.view(np.uint32), pre.view(np.uint32)), where
                t64 = np.abs(got.astype(np.float64))
                want = np.sqrt(t64 * np.sqrt(t64)).astype(np.float32)
                assert np.array_equal(t["xrpow"][gr, c].view(np.uint32), want.view(np.uint32)), where
                have = t64.sum() > 1e-20
                assert t["have"][gr, c] == int(have), where
                assert have == bool(t["xmin"][gr, c].any()), where             # calc_xmin ran: ATH > 0 in every band
                assert t["xrpow_max"][gr, c] == float(want.max()), where
                counts += [1, short, zeroed, not have]
    return counts


@pytest.mark.parametrize("case", CASES, ids=edge_signals.case_id)
def test_quant_trace_rows_edge_corpus(oracle, case):
    kind, ch, sr, kb, frames = case
    l, r = edge_signals.signal(case)
    _, _, tr = oracle.encode_stream(ch, sr, kb, l, r, trace_frames=frames + 8)
    n, short, zeroed, silent = check_rows(tr, 2 if sr >= 32000 else 1, ch, sr, edge_signals.case_id(case))
    assert n > 0
    if kind in ("square", "clicks1", "click_pairs"):
        assert short > 0
    if kind == "silent_right":
        assert silent > 0


def test_quant_trace_rows_reach_every_rule(oracle):
    """quiet noise, silence and bursts at every MPEG-1 and LSF rate: between them, short granules, granules without energy
    and lines zeroed by the analog-silence rule"""
    total = np.zeros(4, int)
    for i, (ch, sr, kb) in enumerate(psy_rows.native_configs()):
        if sr not in SFB_L21:
            continue
        G = 2 if sr >= 32000 else 1
        n = 30 * 576 * G
        l, r = psy_rows.k2_signal(("mixed", "quiet1", "silence")[i % 3], n, 900 + i)
        if i % 3 == 0:
            l, r = make_signal("burst", n, sr, 900 + i)
        _, _, tr = oracle.encode_stream(ch, sr, kb, l, r if ch == 2 else None, trace_frames=40)
        total += check_rows(tr, G, ch, sr, (ch, sr, kb))
    assert (total[1:] > 0).all(), total
