"""Float32 input on the GPU (include/mp3b200.h "Float32 input"): every entry point against the oracle's Float32 store
(tests/oracle_f32.cpp), and integer-valued Float32 input against the Int16 path."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import edge_signals  # noqa: E402
import oracle_f32  # noqa: E402
import oracle_inputs  # noqa: E402
import resample_tap  # noqa: E402
import stage_taps  # noqa: E402
from synth import make_signal  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


CFGS = oracle_inputs.FLOAT_CFGS
KINDS = oracle_inputs.FLOAT_KINDS
float_signal = oracle_inputs.float_signal


def accepted(M, cfg):
    ch, sr, kb = cfg
    return M.stream_bytes(ch, sr, kb, 1000, resample=True) >= 0


def resampled(M, cfg):
    return M.out_samplerate(*cfg) != cfg[1]


def oracle_tagged(ch, sr, kb, calls):
    b, sizes, _, tag = oracle_f32.encode_calls(ch, sr, kb, calls, write_vbr_tag=True)
    return (tag + b[len(tag):]) if tag else b


@pytest.mark.parametrize("sr", resample_tap.RATES)
def test_integer_valued_floats_give_the_int16_bytes(M, sr):
    """every accepted configuration, resampled ones included: whole streams (host and tagged) and handles with ragged
    calls give, from integer-valued Float32 samples, exactly the bytes and per-call sizes of the Int16 samples"""
    for cfg in resample_tap.all_configs():
        ch, s, kb = cfg
        if s != sr or not accepted(M, cfg):
            continue
        rs = resampled(M, cfg)
        l, r = make_signal("burst", 9000 + kb, sr, seed=kb)
        lf, rf = l.astype(np.float32), r.astype(np.float32)
        rr, rrf = (r, rf) if ch == 2 else (None, None)
        want = M.encode_streams(ch, sr, kb, [l, l[:777]], None if ch == 1 else [r, r[:777]], resample=rs)
        got = M.encode_streams(ch, sr, kb, [lf, lf[:777]], None if ch == 1 else [rf, rf[:777]], resample=rs)
        assert got == want, cfg
        if not rs:
            assert M.encode_streams_tagged(ch, sr, kb, [lf], [rf] if ch == 2 else None) == \
                M.encode_streams_tagged(ch, sr, kb, [l], [r] if ch == 2 else None), cfg
        runs = []
        for x, y in ((l, rr), (lf, rrf)):
            e = M.Mp3Encoder(ch, sr, kb, resample=rs)
            runs.append([e.encodeBuffer(x[i:i + 1333], None if y is None else y[i:i + 1333]) for i in range(0, len(x), 1333)]
                        + [e.flush()])
            e.close()
        assert runs[0] == runs[1], cfg


def _calls(l, r, sizes):
    out, i = [], 0
    for k in sizes:
        out.append((l[i:i + k], None if r is None else r[i:i + k]))
        i += k
    if i < len(l):
        out.append((l[i:], None if r is None else r[i:]))
    return out


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: "%d-%d-%d" % c)
def test_entry_points_match_the_oracle(M, cfg):
    """Float32 input with fractions, out of range and denormal: host whole streams, a handle with a ragged call schedule
    (bytes and per-call sizes), a batch, tagged streams and the device path all equal the oracle's Float32 store"""
    import torch

    ch, sr, kb = cfg
    rs = resampled(M, cfg)
    fs = 576 * M.granules_per_frame(ch, sr, kb, resample=rs) * (sr // M.out_samplerate(ch, sr, kb))
    n = 6 * fs + 123
    sigs = oracle_inputs.float_entry_signals(cfg)
    assert len(sigs[0][0]) == n
    wants = [oracle_f32.encode_stream(ch, sr, kb, l, r if ch == 2 else None)[0] for l, r in sigs]
    got = M.encode_streams(ch, sr, kb, [l for l, _ in sigs], [r for _, r in sigs] if ch == 2 else None, resample=rs)
    for k, g, w in zip(KINDS, got, wants):
        assert g == w, (cfg, k)
    # a handle: ragged calls, one Int16 call in the middle
    l, r = sigs[0]
    rr = r if ch == 2 else None
    calls = _calls(l, rr, [1, 700, fs - 1, fs + 1, 16, 3 * fs])
    li, ri = calls[2]
    calls[2] = (np.round(li).astype(np.int16), None if ri is None else np.round(ri).astype(np.int16))
    wb, wsizes, _, _ = oracle_f32.encode_calls(ch, sr, kb, calls)
    e = M.Mp3Encoder(ch, sr, kb, resample=rs)
    gout = [e.encodeBuffer(x, y) for x, y in calls] + [e.flush()]
    e.close()
    assert [len(b) for b in gout] == wsizes and b"".join(gout) == wb, cfg
    # a batch of three handles, one of them in Int16 mode throughout
    encs = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(3)]
    li16 = np.round(sigs[1][0] * 32767).astype(np.int16)
    parts = [[], [], []]
    for i in range(0, n, 2 * fs + 5):
        lefts = [sigs[0][0][i:i + 2 * fs + 5], sigs[2][0][i:i + 2 * fs + 5], li16[i:i + 2 * fs + 5]]
        rights = [sigs[0][1][i:i + 2 * fs + 5], sigs[2][1][i:i + 2 * fs + 5], li16[i:i + 2 * fs + 5]] if ch == 2 else None
        for j, b in enumerate(M.encode_batch(encs, lefts, rights)):
            parts[j].append(b)
    for j, b in enumerate(M.flush_batch(encs)):
        parts[j].append(b)
    for e in encs:
        e.close()
    assert b"".join(parts[0]) == wants[0] and b"".join(parts[1]) == wants[2], cfg
    assert b"".join(parts[2]) == oracle_f32.encode_stream(ch, sr, kb, li16, li16 if ch == 2 else None)[0], cfg
    # tagged whole streams
    if not rs:
        got_t = M.encode_streams_tagged(ch, sr, kb, [l], [r] if ch == 2 else None)[0]
        assert got_t == oracle_tagged(ch, sr, kb, [(l, rr)]), cfg
    # the device path: one float32 allocation
    ns = [len(x) for x, _ in sigs]
    nb = [M.stream_bytes(ch, sr, kb, k, resample=rs) for k in ns]
    pcm = np.concatenate([np.concatenate([x, y]) if ch == 2 else x for x, y in sigs]).astype(np.float32)
    pcm_off = np.concatenate([[0], np.cumsum([k * ch for k in ns])[:-1]])
    out_off = np.concatenate([[0], np.cumsum(nb)[:-1]])
    d_pcm = torch.from_numpy(pcm).cuda()
    d_out = torch.zeros(sum(nb), dtype=torch.uint8, device="cuda")
    M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off, resample=rs, float32=True)
    out = d_out.cpu().numpy()
    for i, k in enumerate(KINDS):
        assert out[out_off[i]:out_off[i] + nb[i]].tobytes() == wants[i], (cfg, k)


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: "%d-%d-%d" % c)
def test_stage_taps_match_the_oracle(M, cfg):
    """every stage tap of Float32 input -- xr, block types, masking, ATH adjust, l3_enc, side info and the quantizer state --
    bit-equal to the oracle's traces"""
    ch, sr, kb = cfg
    rs = resampled(M, cfg)
    G = M.granules_per_frame(ch, sr, kb, resample=rs)
    n = (sr // M.out_samplerate(ch, sr, kb)) * (12 * 576 * G + 211) + 5
    assert n == oracle_inputs.float_tap_samples(cfg)
    for kind in oracle_inputs.FLOAT_TAP_KINDS:
        l, r = float_signal(kind, n, sr, 7)
        rr = r if ch == 2 else None
        F = M.stream_frames(n, ch, sr, kb, resample=rs)
        ref, _, tr = oracle_f32.encode_stream(ch, sr, kb, l, rr, trace_frames=F + 2)
        assert len(tr) == F
        g = M.debug_stages(ch, sr, kb, l, rr, want=stage_taps.ALL_TAPS, resample=rs)
        stage_taps.compare(g, tr, ref, G, ch, "%s %d/%d/%d" % (kind, ch, sr, kb))


@pytest.mark.parametrize("cfg", [c for c in resample_tap.resampled_configs()][::3])
def test_resampler_tap_matches_the_model(M, cfg):
    """debug_resample_f32 equals the integer-ratio FIR model on Float32 input bit for bit, and the oracle's recorded
    resampler output on integer-valued input"""
    ch, sr, kb = cfg
    r = sr // M.out_samplerate(ch, sr, kb)
    l, rt = float_signal("webaudio", 5000, sr, 3)
    _, h, scale, _ = resample_tap.record(ch, sr, kb, np.zeros(3000, np.int16))
    y = M.debug_resample(ch, sr, kb, l, rt if ch == 2 else None)
    for c, x in enumerate([l, rt][:ch]):
        want = resample_tap.fir(x.astype(np.float64), h, scale, r, y.shape[1])
        assert np.array_equal(y[c].view(np.uint32), want.view(np.uint32)), (cfg, c)
    li = np.round(l).astype(np.int16)
    yi = M.debug_resample(ch, sr, kb, li)
    yf = M.debug_resample(ch, sr, kb, li.astype(np.float32))
    assert np.array_equal(yi.view(np.uint32), yf.view(np.uint32))


def test_replaygain_of_float_input(M):
    """ReplayGain of Float32 input: integer values give the Int16 windows, gains and tagged streams; on fractional input a
    handle fed in ragged calls ends its title with the whole-stream gain and tag"""
    for ch, sr, kb, rs in ((2, 44100, 128, False), (1, 22050, 64, False), (2, 48000, 64, True)):
        l, r = make_signal("sweep", 3 * sr, sr, seed=5)
        a = M.debug_replaygain(ch, sr, kb, l, r if ch == 2 else None, resample=rs)
        b = M.debug_replaygain(ch, sr, kb, l.astype(np.float32), r.astype(np.float32) if ch == 2 else None, resample=rs)
        assert np.array_equal(a["sums"].view(np.uint64), b["sums"].view(np.uint64)) and a["title_db"] == b["title_db"]
        assert np.array_equal(a["idx"], b["idx"])
        si = M.encode_streams_replaygain(ch, sr, kb, [l, l[:20000]], [r, r[:20000]] if ch == 2 else None, resample=rs)
        sf = M.encode_streams_replaygain(ch, sr, kb, [l.astype(np.float32), l[:20000].astype(np.float32)],
                                         [r.astype(np.float32), r[:20000].astype(np.float32)] if ch == 2 else None, resample=rs)
        assert si == sf
        x, y = float_signal("webaudio", 3 * sr, sr, 11)
        whole, title, album = M.encode_streams_replaygain(ch, sr, kb, [x], [y] if ch == 2 else None, resample=rs)
        e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs, find_replay_gain=True)
        parts = [e.encodeBuffer(x[i:i + 4099], y[i:i + 4099] if ch == 2 else None) for i in range(0, len(x), 4099)]
        parts.append(e.flush())
        tag = e.lametag_frame()
        assert e.replay_gain[0] == title[0]
        e.close()
        stream = b"".join(parts)
        assert tag + stream[len(tag):] == whole[0]


@pytest.mark.parametrize("case", oracle_inputs.EDGE_AS_FLOAT_CASES, ids=edge_signals.case_id)
def test_edge_corpus_as_floats(M, case):
    """edge corpus cases as integer-valued floats give the Int16 bytes; the same signals / 32768 (Web Audio's range) equal
    the oracle's Float32 store"""
    _, ch, sr, kb, _ = case
    rs = edge_signals.ratio(case) > 1
    l, rr = edge_signals.signal(case)
    want = M.encode_streams(ch, sr, kb, [l], None if rr is None else [rr], resample=rs)
    got = M.encode_streams(ch, sr, kb, [l.astype(np.float32)], None if rr is None else [rr.astype(np.float32)], resample=rs)
    assert got == want, case
    lf, rf = oracle_inputs.edge_as_float(case)
    got = M.encode_streams(ch, sr, kb, [lf], None if rf is None else [rf], resample=rs)[0]
    assert got == oracle_f32.encode_stream(ch, sr, kb, lf, rf)[0], case


def test_state_blobs_and_mixed_calls(M):
    """a handle switches to Float32 mode at its first Float32 call; its blob then carries Float32 samples under its own
    magic, and a handle that imports it continues exactly; a blob taken in Int16 mode still has the Int16 magic"""
    for ch, sr, kb, rs in ((2, 44100, 128, False), (2, 48000, 64, True), (1, 16000, 32, False)):
        fs = 576 * M.granules_per_frame(ch, sr, kb, resample=rs) * (sr // M.out_samplerate(ch, sr, kb))
        x, y = float_signal("x1.5", 8 * fs + 99, sr, 4)
        yy = y if ch == 2 else None
        xi = np.round(x / 2).astype(np.int16)
        yi = np.round(y / 2).astype(np.int16) if ch == 2 else None
        want = oracle_f32.encode_calls(ch, sr, kb, [(xi[:fs], None if yi is None else yi[:fs]),
                                                   (x[fs:5 * fs], None if yy is None else yy[fs:5 * fs]),
                                                   (xi[5 * fs:], None if yi is None else yi[5 * fs:])])[0]
        a = M.Mp3Encoder(ch, sr, kb, resample=rs)
        out = a.encodeBuffer(xi[:fs], None if yi is None else yi[:fs])
        blob_i = a.export_state()
        assert blob_i[:4] in (b"M3S1", b"M3R1")
        out += a.encodeBuffer(x[fs:5 * fs], None if yy is None else yy[fs:5 * fs])
        blob = a.export_state()
        assert blob[:4] == (b"M3G1" if rs else b"M3F1")
        b = M.Mp3Encoder(ch, sr, kb, resample=rs)
        b.import_state(blob)
        assert b.export_state() == blob
        rest_a = a.encodeBuffer(xi[5 * fs:], None if yi is None else yi[5 * fs:]) + a.flush()
        rest_b = b.encodeBuffer(xi[5 * fs:], None if yi is None else yi[5 * fs:]) + b.flush()
        assert rest_a == rest_b and out + rest_a == want
        c = M.Mp3Encoder(ch, sr, kb, resample=rs)                # an Int16 blob sets Int16 mode again
        c.import_state(blob)
        c.import_state(blob_i)
        assert c.export_state() == blob_i
        for e in (a, b, c):
            e.close()


def test_non_finite_input_is_refused(M):
    """NaN and infinities are refused before anything runs, by every host entry point; the handle's blob is unchanged; the
    device path finds them on the device"""
    import torch

    l, r = float_signal("webaudio", 5000, 44100, 2)
    for bad in (np.nan, np.inf, -np.inf):
        x = l.copy()
        x[1234] = bad
        with pytest.raises(M.Mp3B200Error):
            M.encode_streams(2, 44100, 128, [l, x], [r, r])
        with pytest.raises(M.Mp3B200Error):
            M.encode_streams_replaygain(2, 44100, 128, [x], [r])
        e = M.Mp3Encoder(2, 44100, 128)
        e.encodeBuffer(l[:3000], r[:3000])
        blob = e.export_state()
        with pytest.raises(M.Mp3B200Error):
            e.encodeBuffer(l[3000:4000], x[1000:2000])
        assert e.export_state() == blob
        e.close()
        with pytest.raises(M.Mp3B200Error):
            M.encode_streams_tagged(2, 44100, 128, [x], [r])
        a, b = M.Mp3Encoder(2, 44100, 128), M.Mp3Encoder(2, 44100, 128)
        a.encodeBuffer(l[:3000], r[:3000])
        blobs = [a.export_state(), b.export_state()]
        with pytest.raises(M.Mp3B200Error):                    # encode_batch_f32: the whole call is refused
            M.encode_batch([a, b], [l[3000:4000], x[1000:2000]], [r[3000:4000], r[3000:4000]])
        assert [a.export_state(), b.export_state()] == blobs
        with pytest.raises(M.Mp3B200Error):                    # seek_f32
            b.seek(3, x[:1328], r[:1328])
        assert b.export_state() == blobs[1]
        a.close()
        b.close()
        for ch, sr, kb, rs in ((2, 44100, 128, False), (2, 48000, 64, True)):     # the device path finds them on the device
            d_pcm = torch.from_numpy(np.concatenate([x, r])).cuda()
            d_out = torch.zeros(M.stream_bytes(ch, sr, kb, len(x), resample=rs), dtype=torch.uint8, device="cuda")
            with pytest.raises(M.Mp3B200Error):
                M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [len(x)], d_out.data_ptr(), [0], resample=rs, float32=True)
    # a Float32 blob that carries a non-finite sample is refused, and the importing handle is left as it was
    e = M.Mp3Encoder(2, 44100, 128)
    e.encodeBuffer(l[:3000], r[:3000])
    blob = bytearray(e.export_state())
    blob[-4:] = np.array([np.nan], dtype=np.float32).tobytes()
    f = M.Mp3Encoder(2, 44100, 128)
    before = f.export_state()
    with pytest.raises(M.Mp3B200Error):
        f.import_state(bytes(blob))
    assert f.export_state() == before
    e.close()
    f.close()


@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 22050, 64), (2, 48000, 64)], ids=lambda c: "%d-%d-%d" % c)
def test_handle_soak_mixed_calls_and_blobs(M, cfg):
    """random schedules of Int16, Float32 and float64 calls of random sizes on a handle that is repeatedly exported and
    continued by a fresh handle importing its blob: bytes and per-call sizes equal the oracle's"""
    ch, sr, kb = cfg
    rs = M.out_samplerate(ch, sr, kb) != sr
    rng = np.random.default_rng(sum(cfg))
    x, y = float_signal("webaudio", 30 * 1152 + 777, sr, 5)
    calls, pos = [], 0
    while pos < len(x):
        k = int(min(len(x) - pos, rng.choice([1, 5, 333, 576, 1151, 1152, 1153, 2304, 5000])))
        t = rng.choice(["i", "f", "d"])
        a, b = x[pos:pos + k], y[pos:pos + k]
        if t == "i":
            a, b = np.round(a).astype(np.int16), np.round(b).astype(np.int16)
        elif t == "d":
            a, b = a.astype(np.float64) + 1e-4, b.astype(np.float64)
        calls.append((a, b if ch == 2 else None))
        pos += k
    wb, wsizes, _, _ = oracle_f32.encode_calls(ch, sr, kb, calls)
    e = M.Mp3Encoder(ch, sr, kb, resample=rs)
    out = []
    for i, (a, b) in enumerate(calls):
        out.append(e.encodeBuffer(a, b))
        if rng.random() < 0.3:
            blob = e.export_state()
            e.close()
            e = M.Mp3Encoder(ch, sr, kb, resample=rs)
            e.import_state(blob)
            assert e.export_state() == blob
    out.append(e.flush())
    e.close()
    assert [len(b) for b in out] == wsizes and b"".join(out) == wb, cfg


@pytest.mark.parametrize("nseg", [2, 4])
def test_segments_of_float_input(M, nseg):
    """seek on Float32 input (seek_f32) and encode_stream_segments_local give the single encoder's stream"""
    from lamejs_b200 import sharding
    for ch, sr, kb in ((2, 44100, 128), (1, 22050, 32)):
        fs = 576 * M.granules_per_frame(ch, sr, kb)
        l, r = float_signal("webaudio", 40 * fs + 517, sr, 12)
        want = oracle_f32.encode_stream(ch, sr, kb, l, r if ch == 2 else None)[0]
        got, redone = sharding.encode_stream_segments_local(lambda: M.Mp3Encoder(ch, sr, kb), l, r if ch == 2 else None, fs, nseg, 8)
        assert got == want, (ch, sr, kb, nseg, redone)
