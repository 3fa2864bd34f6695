"""Integer-ratio resampling without a GPU: the FIR model the GPU kernel implements, checked against what the oracle's
resampler writes, and the host logic (acceptance set, output rate, byte counts) of MP3B200_RESAMPLE."""
import numpy as np
import pytest

import oracle_lib as O
import resample_tap as T
from synth import make_signal

INT = T.resampled_configs(integer=True)
FRAC = T.resampled_configs(integer=False)


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    lamejs_b200.lib()
    return lamejs_b200


def ratio_of(ch, sr, kb):
    return sr // O.out_samplerate(ch, sr, kb)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_configuration_inventory():
    """29 of the 78 resampling (channels, rate, kbps) combinations have an integer ratio, and they are these rate pairs"""
    assert (len(INT), len(FRAC)) == (29, 49)
    pairs = {(sr, O.out_samplerate(ch, sr, kb)) for ch, sr, kb in INT}
    assert pairs == {(48000, 24000), (44100, 22050), (48000, 16000), (32000, 16000), (48000, 8000), (32000, 8000), (24000, 8000),
                     (16000, 8000)}


def schedules(n, seed):
    rng = np.random.default_rng(seed)
    rand = []
    while sum(rand) < n:
        rand.append(int(min(n - sum(rand), rng.integers(0, 3000))))
    return {"whole": None, "577": [577] * (n // 577) + [n % 577], "1152": [1152] * (n // 1152) + [n % 1152], "random": rand}


@pytest.mark.parametrize("cfg", INT, ids=lambda c: "%d_%d_%d" % c)
def test_fir_model_equals_oracle_resampler(cfg):
    """Every value lamejs's resampler writes, in every chunking (flush included), is the 33-tap FIR of the zero-extended
    scaled input, bit for bit; after P input samples there are max(0, ceil((P - 16) / r)) of them; and the bytes do not
    depend on the chunking."""
    ch, sr, kb = cfg
    r = ratio_of(*cfg)
    n = 23 * 1152 + 77
    l, rt = make_signal("burst", n, sr, 5)
    rt = np.roll(rt, 13)                               # L != R
    x = [l, rt][:ch]
    first = None
    for name, calls in schedules(n, sr + kb + ch).items():
        y, h, scale, data = T.record(ch, sr, kb, l, rt, calls)
        for c in range(ch):
            assert same_bits(T.fir(x[c], h, scale, r, y.shape[1]), y[c]), (name, c)
        first = data if first is None else first
        assert data == first, name
        y_open, _, _, _ = T.record(ch, sr, kb, l, rt, calls, flush=False)
        assert y_open.shape[1] == T.outputs_after(n, r), name
    # one sample per call on a short stream, incl. the first outputs (P = 16, 17, 18)
    m = 1500
    for p in (0, 15, 16, 17, 18, 19, 40, m):
        y_open, h, scale, _ = T.record(ch, sr, kb, l[:p], rt[:p], [1] * p, flush=False) if p else (np.zeros((ch, 0)), 0, 0, 0)
        assert y_open.shape[1] == T.outputs_after(p, r), p
    y, h, scale, data = T.record(ch, sr, kb, l[:m], rt[:m], [1] * m)
    for c in range(ch):
        assert same_bits(T.fir(x[c][:m], h, scale, r, y.shape[1]), y[c])
    assert data == T.record(ch, sr, kb, l[:m], rt[:m])[3]


@pytest.mark.parametrize("cfg", [(2, 44100, 64), (1, 48000, 48), (2, 32000, 48), (1, 22050, 16)], ids=lambda c: "%d_%d_%d" % c)
def test_fir_model_does_not_describe_fractional_ratios(cfg):
    """The comparison above can tell the cases apart: for a non-integer ratio the recorded values are not the FIR of any
    integer stride, and the count formula fails too."""
    ch, sr, kb = cfg
    assert cfg in FRAC
    n = 6 * 1152 + 77
    l, rt = make_signal("burst", n, sr, 5)
    y, h, scale, _ = T.record(ch, sr, kb, l, rt, [1152] * (n // 1152) + [n % 1152])
    for r in (1, 2):
        assert not same_bits(T.fir(l, h, scale, r, y.shape[1]), y[0])
    y_open, _, _, _ = T.record(ch, sr, kb, l, rt, [1152] * (n // 1152) + [n % 1152], flush=False)
    out = O.out_samplerate(ch, sr, kb)
    assert y_open.shape[1] not in (T.outputs_after(n, int(round(sr / out))), T.outputs_after(n, int(sr // out)))


def test_acceptance_set_and_output_rate(M):
    """Over the 342 combinations: with the flag, exactly the native and integer-ratio configurations are accepted, with the
    oracle's byte count; without it nothing changes; mp3b200_out_samplerate is the oracle's output rate."""
    l, r = make_signal("noise", 2000, 48000, 1)
    for ch, sr, kb in T.all_configs():
        out = O.out_samplerate(ch, sr, kb)
        assert M.out_samplerate(ch, sr, kb) == out, (ch, sr, kb)
        native = out == sr
        accepted = native or (ch, sr, kb) in INT
        got = M.stream_bytes(ch, sr, kb, len(l), resample=True)
        if accepted:
            want = len(O.encode_stream(ch, sr, kb, l, r if ch == 2 else None)[0])
            assert got == want, (ch, sr, kb)
        else:
            assert got == -1, (ch, sr, kb)
        assert M.stream_bytes(ch, sr, kb, len(l)) == (got if native else -1), (ch, sr, kb)
    assert M.out_samplerate(3, 44100, 128) == 0


def _sweep_lengths(r, every):
    top = 4 * 576 * r + 1500
    edges = set(range(0, 60))
    for k in range(1, 8):                      # inputs around the frame and flush edges, in input samples
        for base in (r * (576 * k) + 16, r * (576 * k - 1104) + 16, r * (576 * k + 752 - 528) + 16):
            edges.update(range(max(0, base - 2 * r - 2), base + 2 * r + 3))
    return sorted(x for x in (set(range(0, top + 1, every)) | edges) if x <= top)


# one configuration per ratio takes every length (the FIFO depends on the ratio only); every configuration takes the edges
SWEEP_FULL = {}
for _c in INT:
    SWEEP_FULL.setdefault(ratio_of(*_c), _c)


@pytest.mark.parametrize("cfg", INT, ids=lambda c: "%d_%d_%d" % c)
def test_stream_bytes_sweep_matches_oracle(M, cfg):
    """Input lengths from 0 to 4 output frames * r + 1500 samples, incl. 16, 17, 18 (the first output) and the frame / flush
    edges: mp3b200_stream_bytes_ex is the length of the oracle's encodeBuffer(n) + flush().  Every length for one
    configuration per ratio, the edges and every 37th length for the others."""
    ch, sr, kb = cfg
    r = ratio_of(*cfg)
    for n in _sweep_lengths(r, 1 if SWEEP_FULL[r] == cfg else 37):
        data, _, _ = O.encode_stream(ch, sr, kb, np.zeros(n, dtype=np.int16), None)
        assert M.stream_bytes(ch, sr, kb, n, resample=True) == len(data), n


@pytest.fixture(scope="module")
def resampled_corpus():
    """per case of edge_signals.RESAMPLED_CASES: (what the oracle's resampler wrote, gfp.scale, the oracle's frame trace)"""
    import edge_signals as E

    out = []
    for c in E.RESAMPLED_CASES:
        kind, ch, sr, kb, frames = c
        l, r = E.signal(c)
        y, _, scale, data = T.record(ch, sr, kb, l, r)
        ref, _, tr = O.encode_stream(ch, sr, kb, l, r, trace_frames=frames + 8)
        assert ref == data
        out.append((c, y, scale, tr))
    return out


def test_resampled_edge_corpus_spread():
    """The resampled edge cases are integer-ratio configurations over the ratios 2, 3, 4 and 6, mono and stereo, MPEG-2 and
    MPEG-2.5 output; they are sized in output frames times the ratio; the native corpus stays native."""
    import edge_signals as E

    assert all(E.ratio(c) == 1 for c in E.CASES)
    assert all(c[1:4] in INT for c in E.RESAMPLED_CASES)
    assert {E.ratio(c) for c in E.RESAMPLED_CASES} == {2, 3, 4, 6}
    assert {c[1] for c in E.RESAMPLED_CASES} == {1, 2}
    outs = {O.out_samplerate(*c[1:4]) for c in E.RESAMPLED_CASES}
    assert 8000 in outs and outs & {16000, 22050, 24000}
    for c in E.RESAMPLED_CASES:
        r = E.ratio(c)
        assert len(E.signal(c)[0]) == r * (576 * c[4] + 211), c


def test_resampled_edge_corpus_reaches_what_int16_never_is(resampled_corpus):
    """What the resampler makes of the corpus: the filter's overshoot takes squares, DC, clicks and clipped sines past the
    Int16 range on many cases (beyond 43,000 for the click trains); +-1 LSB input becomes fractional samples (the shares
    measured when the corpus was made: about 91 % for dither, 10 % for sparse clicks, with no sample above 1.5); the
    input-rate Nyquist tone and the tone above the output's Nyquist frequency are mostly filtered out; and over the list
    the encoder takes all four block types.  Keeps the corpus from silently going tame."""
    over, peak_all, blocktypes = [], 0.0, set()
    for c, y, scale, tr in resampled_corpus:
        kind, ch = c[0], c[1]
        peak = float(np.abs(y).max())
        peak_all = max(peak_all, peak)
        frac = float(np.mean(y != np.round(y)))
        assert scale == np.float64(0.95), c                          # every integer-ratio preset scales its input
        if peak > 32768:
            over.append(c)
        if kind == "lsb_dither":
            assert frac >= 0.90 and peak <= 1.5, (c, frac, peak)
        if kind == "lsb_clicks":
            assert frac >= 0.09 and peak <= 1.5, (c, frac, peak)
        if kind in ("nyquist", "hf_tone"):
            assert peak < 9000, (c, peak)                              # measured: 2,466 .. 7,783 of 32,767 in
        blocktypes |= set(np.unique(tr["blocktype"][:, :1, :ch]).tolist())
    assert len(over) >= 15, over
    assert {c[0] for c in over} >= {"square", "dc_max", "dc_min", "clicks1", "click_pairs", "clipped_sine"}
    assert peak_all >= 43000, peak_all
    assert blocktypes == {0, 1, 2, 3}, blocktypes
