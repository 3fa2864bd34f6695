"""The short-block half of the psy model runs only for the units whose short thresholds a short granule reads (DESIGN.md 2):
the stage taps with the encoder's skipping equal the oracle wherever the rule says the values are read, the short list holds
exactly the units the rule names, and streaming handles cut just before short granules still equal the oracle."""
import numpy as np
import pytest

import edge_signals
import oracle_f32
from stage_taps import bits_equal
from synth import bursts

pytestmark = pytest.mark.gpu

BT_SHORT = 2
SKIP_TAPS = ("blocktype", "en_l", "thm_l", "en_s", "thm_s", "bytes")


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


def read_rows(bt):
    """R per unit u of bt (units x channels): the quantizer of granule u + 1 reads its en_s / thm_s, or u is the last unit"""
    U = len(bt)
    return [u == U - 1 or bool((bt[u + 1] == BT_SHORT).any()) for u in range(U)]


def short_units(bt):
    """(unit, channel) pairs the short list must hold: units u >= -1 with R(u) or R(u + 1)"""
    R = read_rows(bt)
    return bt.shape[1] * sum(1 for u in range(-1, len(bt)) if (u >= 0 and R[u]) or (u + 1 < len(bt) and R[u + 1]))


def check_skipping(M, g, tr, ref, G, ch, label):
    """taps run with the encoder's skipping: bytes and long masking equal the oracle everywhere; en_s / thm_s of granule u
    (the masking of unit u - 1) wherever the rule computes it -- every granule a short block reads, and the first (the halo
    row, carried or start values); the short list's length equals the rule's count from the oracle's block types"""
    assert g["bytes"].tobytes() == ref, label
    want_bt = tr["blocktype"][:, :G, :ch]
    assert np.array_equal(g["blocktype"], want_bt), label
    for k in ("en_l", "thm_l"):
        assert bits_equal(g[k], tr[k][:, :G, :ch]), (label, k)
    bt = want_bt.reshape(-1, ch)
    rows = [u for u in range(len(bt)) if u == 0 or (bt[u] == BT_SHORT).any()]
    for k in ("en_s", "thm_s"):
        got, want = g[k].reshape(len(bt), ch, -1), tr[k][:, :G, :ch].reshape(len(bt), ch, -1)
        assert bits_equal(got[rows], want[rows]), (label, k)
    assert M.debug_short_units() == short_units(bt), label
    return bt


EDGE = [c for c in edge_signals.CASES if c[0] in ("square", "click_pairs", "loud_silent", "clicks1", "clicks3", "clicks5")]


@pytest.mark.parametrize("case", EDGE, ids=edge_signals.case_id)
def test_taps_with_skipping_edge_corpus(M, oracle, case):
    """short granules first in the stream, on both sides of frame boundaries, in long runs and near the end; MPEG-1 and
    LSF, mono and stereo"""
    kind, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(ch, sr, kb)
    F = M.stream_frames(len(l), ch, sr, kb)
    ref, _, tr = oracle.encode_stream(ch, sr, kb, l, r, trace_frames=F + 2)
    g = M.debug_stages(ch, sr, kb, l, r, want=SKIP_TAPS, skip_short=True)
    bt = check_skipping(M, g, tr, ref, G, ch, edge_signals.case_id(case))
    assert (bt == BT_SHORT).any()
    # and the taps without skipping still compute every unit
    M.debug_stages(ch, sr, kb, l, r, want=("en_s",))
    assert M.debug_short_units() == ch * (len(bt) + 1)


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 44100, 128), (2, 22050, 64), (1, 16000, 32)])
def test_taps_with_skipping_bursts(M, oracle, ch, sr, kb):
    """the bench's c5 signal (bursts): a quarter of the units do the short half"""
    fs = 576 * M.granules_per_frame(ch, sr, kb)
    n = 120 * fs + 333
    l, r = bursts(n, 0xC5)
    r = r if ch == 2 else None
    F = M.stream_frames(n, ch, sr, kb)
    ref, _, tr = oracle.encode_stream(ch, sr, kb, l, r, trace_frames=F + 2)
    g = M.debug_stages(ch, sr, kb, l, r, want=SKIP_TAPS, skip_short=True)
    bt = check_skipping(M, g, tr, ref, M.granules_per_frame(ch, sr, kb), ch, "bursts %d/%d/%d" % (ch, sr, kb))
    assert (bt == BT_SHORT).any()


def test_taps_with_skipping_float32_and_resampled(M, oracle):
    """Float32 input (k_stage_f32, fractional samples) and a configuration lamejs resamples (k_resample)"""
    fs = 576 * M.granules_per_frame(2, 44100, 128)
    n = 120 * fs + 333
    l, r = bursts(n, 0xC5)
    l = l.astype(np.float32) * np.float32(0.75)
    r = r.astype(np.float32) + np.float32(0.25)
    F = M.stream_frames(n, 2, 44100, 128)
    ref, _, tr = oracle_f32.encode_stream(2, 44100, 128, l, r, trace_frames=F + 2)
    g = M.debug_stages(2, 44100, 128, l, r, want=SKIP_TAPS, skip_short=True)
    assert (check_skipping(M, g, tr, ref, 2, 2, "float32") == BT_SHORT).any()
    case = ("clicks1", 2, 48000, 64, 56)
    assert case in edge_signals.RESAMPLED_CASES
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(2, 48000, 64, resample=True)
    F = M.stream_frames(len(l), 2, 48000, 64, resample=True)
    ref, _, tr = oracle.encode_stream(2, 48000, 64, l, r, trace_frames=F + 2)
    g = M.debug_stages(2, 48000, 64, l, r, want=SKIP_TAPS, skip_short=True, resample=True)
    assert (check_skipping(M, g, tr, ref, G, 2, "resampled") == BT_SHORT).any()


@pytest.mark.parametrize("case", [("clicks1", 2, 44100, 128, 56), ("click_pairs", 1, 16000, 32, 120)], ids=edge_signals.case_id)
def test_handles_cut_before_short_granules(M, oracle, case):
    """a streaming handle whose calls end just before a short granule: the carried masking row (halo) decides the next
    call's first granule; export / import round trips there, and the stream cut into segments, equal the oracle"""
    from lamejs_b200 import sharding

    kind, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(ch, sr, kb)
    fs = 576 * G
    F = M.stream_frames(len(l), ch, sr, kb)
    want, _, tr = oracle.encode_stream(ch, sr, kb, l, r, trace_frames=F + 2)
    bt = tr["blocktype"][:, :G, :ch].reshape(-1, ch)
    shorts = [u for u in range(1, len(bt)) if (bt[u] == BT_SHORT).any() and not (bt[u - 1] == BT_SHORT).any()]
    assert len(shorts) >= 3
    rr = r if ch == 2 else None
    # granule u is encoded by the call that completes frame u // G; lamejs holds 1152 + 576 samples back before the
    # first frame (encoder delay + MDCT lookahead), so frame f completes once (f + 1) * fs + fs // 2 + 48 samples are in
    for u in shorts[:3] + shorts[-2:]:
        f = u // G
        for cut in (f * fs + 576 + fs // 2, f * fs + 576 + fs // 2 + 48, (f + 1) * fs):
            cut = min(max(cut, 1), len(l) - 1)
            a = M.Mp3Encoder(ch, sr, kb)
            out = a.encodeBuffer(l[:cut], None if rr is None else rr[:cut])
            blob = a.export_state()
            a.close()
            b = M.Mp3Encoder(ch, sr, kb)
            b.import_state(blob)
            assert b.export_state() == blob
            mid = cut + (len(l) - cut) // 3
            out += b.encodeBuffer(l[cut:mid], None if rr is None else rr[cut:mid])
            out += b.encodeBuffer(l[mid:], None if rr is None else rr[mid:]) + b.flush()
            b.close()
            assert out == want, (u, cut)
    for nseg, warmup in ((3, 8), (5, 1)):
        got, _ = sharding.encode_stream_segments_local(lambda: M.Mp3Encoder(ch, sr, kb), l, rr, fs, nseg, warmup)
        assert got == want, (nseg, warmup)
    assert M.encode_streams(ch, sr, kb, [l], None if rr is None else [rr])[0] == want
