"""The oracle's own record of the quantizer's carried state is consistent (no GPU): each frame starts from the OldValue /
CurrentStep the previous frame ended with; the state after gr0 (MPEG-1) and at the frame's end follow from the bin search's
rule CurrentStep = (start - gain >= 4) ? 4 : 2 wherever a granule had energy, and equal the state before it where the rate
loop was skipped; and OracleEncoder.state() is what the next call starts from -- the traced start state, ATH adjustment and
masking of that call's first frame."""
import numpy as np
import pytest

import edge_signals
from synth import make_signal

CASES = [("burst", 2, 44100, 128, 60), ("silence", 2, 44100, 128, 8), ("sine", 1, 48000, 320, 40),
         ("noise", 2, 22050, 64, 70), ("burst", 1, 8000, 16, 60), ("sweep", 2, 32000, 160, 40)]


def _chain(tr, G, ch, label):
    ov = {"in": tr["old_value_in"], "mid": tr["old_value_mid"], "out": tr["old_value_out"]}
    cs = {"in": tr["cur_step_in"], "mid": tr["cur_step_mid"], "out": tr["cur_step_out"]}
    assert (ov["in"][0] == 180).all() and (cs["in"][0] == 4).all(), label
    assert np.array_equal(ov["in"][1:], ov["out"][:-1]), label
    assert np.array_equal(cs["in"][1:], cs["out"][:-1]), label
    if G == 1:
        assert not ov["mid"].any() and not cs["mid"].any(), label
    # one bin search per granule with energy: (start, step) -> (gain, (start - gain >= 4) ? 4 : 2); no search, no change
    steps = [("in", "mid"), ("mid", "out")] if G == 2 else [("in", "out")]
    searched = 0
    for gr, (a, b) in enumerate(steps):
        have = (tr["xmin"][:, gr, :ch] != 0).any(axis=-1)          # calc_xmin ran (ATH > 0 in every band)
        assert np.array_equal(have, tr["xrpow_max"][:, gr, :ch] > 0), label
        rule = np.where(ov[a][:, :ch] - ov[b][:, :ch] >= 4, 4, 2)
        assert np.array_equal(np.where(have, rule, cs[a][:, :ch]), cs[b][:, :ch]), (label, a, b)
        assert np.array_equal(np.where(have, ov[b][:, :ch], ov[a][:, :ch]), ov[b][:, :ch]), (label, a, b)
        searched += int(have.sum())
    return searched


@pytest.mark.parametrize("kind,ch,sr,kbps,frames", CASES)
def test_oracle_state_chain(oracle, kind, ch, sr, kbps, frames):
    fs = 1152 if sr >= 32000 else 576
    G = fs // 576
    l, r = make_signal(kind, frames * fs + 211, sr, 31)
    _, _, tr = oracle.encode_stream(ch, sr, kbps, l, r if ch == 2 else None, trace_frames=frames + 8)
    searched = _chain(tr, G, ch, kind)
    if kind != "silence":
        assert searched > frames * G * ch // 2
    # the new fields are filled: max_nonzero_coeff in range, xmin only on the psymax bands (21 long, 36 short)
    assert ((tr["max_nonzero_coeff"] >= 0) & (tr["max_nonzero_coeff"] <= 575)).all()
    short = tr["blocktype"][:, :G, :ch] == 2
    xm = tr["xmin"][:, :G, :ch]
    assert not xm[~short][:, 21:].any() and not xm[short][:, 36:].any()


def test_oracle_state_chain_edge_corpus(oracle):
    for c in edge_signals.CASES:
        kind, ch, sr, kbps, frames = c
        l, r = edge_signals.signal(c)
        _, _, tr = oracle.encode_stream(ch, sr, kbps, l, r, trace_frames=frames + 8)
        _chain(tr, 2 if sr >= 32000 else 1, ch, edge_signals.case_id(c))


@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 22050, 32)])
def test_state_is_what_the_next_call_starts_from(oracle, cfg):
    ch, sr, kbps = cfg
    l, r = make_signal("burst", 40000, sr, 5)
    r = r if ch == 2 else None
    enc = oracle.OracleEncoder(ch, sr, kbps, trace_frames=200)
    st0 = enc.state()
    assert st0["frames_done"] == 0 and (st0["old_value"] == 180).all() and (st0["current_step"] == 4).all()
    checked = 0
    for lo in range(0, 36000, 3001):
        st = enc.state()
        n0 = len(enc.traces())
        enc.encode_buffer(l[lo:lo + 3001], None if r is None else r[lo:lo + 3001])
        tr = enc.traces()
        assert enc.state()["frames_done"] == len(tr)
        if len(tr) == n0:
            continue
        first = tr[n0]
        assert np.array_equal(first["old_value_in"], st["old_value"]) and np.array_equal(first["cur_step_in"], st["current_step"])
        if n0 > 0:                 # the masking the psy model hands the next granule (gfc.en / gfc.thm), bit for bit
            for k in ("en_l", "thm_l", "en_s", "thm_s"):
                assert np.array_equal(first[k][0, :ch].view(np.uint32), st[k][:ch].view(np.uint32)), k
            checked += 1
        last = tr[-1]
        now = enc.state()
        assert now["ath_adjust"] == last["ath_adjust"]
        assert np.array_equal(now["old_value"], last["old_value_out"]) and np.array_equal(now["current_step"], last["cur_step_out"])
    assert checked >= 8
    enc.flush()
    assert enc.state()["mf_samples_to_encode"] == 0
    enc.close()
