"""GPU parity tests proper: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.
Bit-exact for everything: bytes, quantised lines, side info -- and also for the float32 intermediates (MDCT
spectrum, masking energies/thresholds), i.e. relative tolerance 0 (the north-star 1e-5 is only an alarm level)."""
import hashlib

import numpy as np
import pytest

import mp3_parse
import oracle_inputs
import stage_taps
from stage_taps import bits_equal
from synth import make_signal, white, octave_hold, bursts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


@pytest.mark.parametrize("kind,ch,sr,kbps,frames", oracle_inputs.STAGE_PARITY_CASES)
def test_stage_parity(M, oracle, kind, ch, sr, kbps, frames):
    l, r = oracle_inputs.stage_parity_signal((kind, ch, sr, kbps, frames))
    F = M.stream_frames(len(l))
    ref, _, tr = oracle.encode_stream(ch, sr, kbps, l, r, trace_frames=F + 2)
    g = M.debug_stages(ch, sr, kbps, l, r, want=stage_taps.ALL_TAPS)
    stage_taps.compare(g, tr, ref, 2, ch)      # every tap, all 15 side-info columns, relative tolerance 0


def test_mdct_alone_with_forced_block_types(M, oracle):
    """K1 in isolation: every granule forced through each window type (NORM/START/SHORT/STOP)."""
    l, r = make_signal("noise", 24 * 1152, 44100, 2)
    F = M.stream_frames(len(l))
    _, _, tr = oracle.encode_stream(2, 44100, 128, l, r, trace_frames=F + 2)
    g = M.debug_stages(2, 44100, 128, l, r, force_blocktype=tr["blocktype"].astype(np.int32), want=("xr",))
    assert bits_equal(g["xr"], tr["xr"])


def test_batch_of_ragged_streams(M, oracle):
    """Many independent streams of different (including tiny / empty-ish) lengths in one launch sequence."""
    lens = [0, 1, 700, 1376, 1377, 5000, 1152 * 7, 1152 * 31 + 5, 1152 * 64]
    ls, rs, refs = [], [], []
    for i, n in enumerate(lens):
        l, r = white(n, 0x5EED0003 + i) if i % 2 else make_signal("noise", n, 44100, i)
        ls.append(l); rs.append(r)
        refs.append(oracle.encode_stream(2, 44100, 128, l, r)[0])
    outs = M.encode_streams(2, 44100, 128, ls, rs)
    for n, o, ref in zip(lens, outs, refs):
        assert o == ref, n


def test_handle_api_matches_lamejs_call_pattern(M, oracle):
    """Mp3Encoder(chunked encodeBuffer + flush): per-call byte counts and bytes equal the oracle's, for README-style
    1152 chunking, odd chunk sizes, and reuse after flush."""
    l, r = make_signal("burst", 40 * 1152 + 77, 44100, 9)
    for chunk in (1152, 777, 5000):
        enc = M.Mp3Encoder(2, 44100, 128)
        ref = oracle.OracleEncoder(2, 44100, 128)
        for i in range(0, len(l), chunk):
            a = enc.encodeBuffer(l[i:i + chunk], r[i:i + chunk])
            b = ref.encode_buffer(l[i:i + chunk], r[i:i + chunk])
            assert a == b, (chunk, i)
        assert enc.flush() == ref.flush()
        assert enc.flush() == b"" == ref.flush()
        a = enc.encodeBuffer(l[:3000], r[:3000]) + enc.flush()
        b = ref.encode_buffer(l[:3000], r[:3000]) + ref.flush()
        assert a == b
        enc.close(); ref.close()


def test_c2_full_size_sweep_10k_frames(M, oracle, books):
    """BASELINE config #2 at full size: stereo 44.1k/128k, 10 000 frames of sine sweep, one stream.  Checked three
    ways: (i) byte-exact against the oracle (it finishes in seconds), (ii) size-independent properties -- closed-form
    length, sync words at closed-form offsets, sampled frames parse with exact bit accounting, (iii) causality:
    a prefix of the stream encodes to a prefix of the bytes (frame k only depends on PCM up to 1152k+1375)."""
    n = 10000 * 1152
    l, r = make_signal("sweep", n, 44100)
    out = M.encode_streams(2, 44100, 128, [l], [r])[0]
    F = M.stream_frames(n)
    assert F == 10001 and len(out) == M.stream_bytes(2, 44100, 128, n)
    off, lag = 0, 42300
    for k in range(F):
        lag -= 42300
        pad = 0
        if lag < 0:
            lag += 44100; pad = 1
        assert out[off] == 0xFF and out[off + 1] == 0xFB and out[off + 2] == (0x90 | (pad << 1)), k
        if k % 997 == 0:
            f = mp3_parse.parse_frame(out, off, books)
            assert f["frame_len"] == 417 + pad
        off += 417 + pad
    assert off == len(out)
    m = 300 * 1152
    pre = M.encode_streams(2, 44100, 128, [l[:m]], [r[:m]])[0]
    keep = M.stream_bytes(2, 44100, 128, m - 1376 - 1152)      # frames not touched by the flush padding of the prefix
    assert pre[:keep] == out[:keep]
    ref = oracle.encode_stream(2, 44100, 128, l, r)[0]
    assert hashlib.sha256(out).hexdigest() == hashlib.sha256(ref).hexdigest()


def test_c3_white_noise_320k_streams(M, oracle):
    """BASELINE config #3 shape (stereo 48k/320k white noise, streams of 1000 frames, counter offset j*2^32);
    4 of the 100 streams are checked against the oracle, all against the closed-form length."""
    S, n = 8, 1000 * 1152
    ls, rs = [], []
    for j in range(S):
        l, r = white(n, 0x5EED0003, offset=j << 32)
        ls.append(l); rs.append(r)
    outs = M.encode_streams(2, 48000, 320, ls, rs)
    for j in range(S):
        assert len(outs[j]) == M.stream_bytes(2, 48000, 320, n) == 1001 * 960
    for j in (0, 3, 5, 7):
        assert outs[j] == oracle.encode_stream(2, 48000, 320, ls[j], rs[j])[0], j


def test_c4_mono_octave_streams_and_c5_bursts(M, oracle):
    ls = [octave_hold(400 * 1152, 0x5EED0004 + 16 * j) for j in range(6)]
    outs = M.encode_streams(1, 44100, 128, ls)
    for j in (0, 5):
        assert outs[j] == oracle.encode_stream(1, 44100, 128, ls[j], None)[0]
    lb, rb = bursts(600 * 1152, 0x5EED0005)
    out = M.encode_streams(2, 44100, 128, [lb], [rb])[0]
    ref, _, tr = oracle.encode_stream(2, 44100, 128, lb, rb, trace_frames=700)
    assert out == ref
    assert set(np.unique(tr["blocktype"])) == {0, 1, 2, 3}      # START/SHORT/STOP all exercised


def test_batched_live_encoders_one_launch_per_call(M, oracle):
    """SURVEY 8(b) batch row: N live Mp3Encoder objects fed different chunk sizes through mp3b200_encode_batch /
    mp3b200_flush_batch -- every per-call byte string equals what lamejs' encodeBuffer / flush returns for that
    stream (oracle), including calls that complete no frame and encoders that receive nothing in a call."""
    sigs = [make_signal(k, n, 44100, 40 + i) for i, (k, n) in enumerate([("noise", 9000), ("burst", 14000), ("sweep", 5000), ("white", 1)])]
    encs = [M.Mp3Encoder(2, 44100, 128) for _ in sigs]
    refs = [oracle.OracleEncoder(2, 44100, 128) for _ in sigs]
    pos = [0] * len(sigs)
    chunks = [700, 2500, 1152, 1]
    for rnd in range(8):
        ls, rs = [], []
        for i, (l, r) in enumerate(sigs):
            n = 0 if (rnd + i) % 5 == 4 else chunks[i]
            ls.append(l[pos[i]:pos[i] + n]); rs.append(r[pos[i]:pos[i] + n]); pos[i] += len(ls[-1])
        got = M.encode_batch(encs, ls, rs)
        for i in range(len(sigs)):
            want = refs[i].encode_buffer(ls[i], rs[i]) if len(ls[i]) else b""
            assert got[i] == want, (rnd, i)
    got = M.flush_batch(encs)
    for i in range(len(sigs)):
        assert got[i] == refs[i].flush(), i
    assert M.flush_batch(encs) == [b""] * len(sigs)
    for e, r in zip(encs, refs):
        e.close(); r.close()


@pytest.mark.parametrize("sr", oracle_inputs.CONFIG_MATRIX_RATES)
def test_config_matrix(M, oracle, sr):
    """Every bitrate of the rate's MPEG version (and an off-ladder one that lamejs snaps, worker-realtime.js passes 123) x
    mono/stereo at each sample rate: short noisy + transient streams, byte-exact against the oracle.  The C ABI must reject
    exactly the configurations in which lamejs resamples (oracle.out_samplerate != sr)."""
    (l, r), (l2, r2) = oracle_inputs.config_matrix_signals(sr)
    tried = 0
    for kbps in oracle_inputs.CONFIG_MATRIX_KBPS:
        for ch in (1, 2):
            native = oracle.out_samplerate(ch, sr, kbps) == sr
            try:
                outs = M.encode_streams(ch, sr, kbps, [l, l2], [r, r2] if ch == 2 else None)
            except M.Mp3B200Error:
                assert not native, (ch, sr, kbps)
                continue
            assert native, (ch, sr, kbps)
            tried += 1
            assert outs[0] == oracle.encode_stream(ch, sr, kbps, l, r if ch == 2 else None)[0], (ch, sr, kbps)
            assert outs[1] == oracle.encode_stream(ch, sr, kbps, l2, r2 if ch == 2 else None)[0], (ch, sr, kbps)
    assert tried >= 8


@pytest.mark.gpu
def test_four_host_threads_with_own_handles(oracle):
    """SURVEY 8(b) threading row: distinct handles are usable concurrently from distinct host threads (each thread drives
    its own CUDA stream); every stream's bytes equal the oracle's."""
    import threading

    import lamejs_b200 as M

    cfgs = [(2, 44100, 128, "burst"), (1, 44100, 128, "octave"), (2, 48000, 320, "white"), (2, 32000, 192, "noise")]
    res, err = [None] * 4, []

    def work(i):
        try:
            ch, sr, kbps, kind = cfgs[i]
            l, r = make_signal(kind, 40 * 1152 + 37 * i, sr, 300 + i)
            enc = M.Mp3Encoder(ch, sr, kbps)
            out = bytearray()
            for k in range(0, len(l), 1152):
                out += enc.encodeBuffer(l[k:k + 1152], r[k:k + 1152] if ch == 2 else None)
            out += enc.flush()
            enc.close()
            res[i] = bytes(out)
        except Exception as e:   # noqa: BLE001
            err.append((i, repr(e)))

    ths = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not err, err
    for i, (ch, sr, kbps, kind) in enumerate(cfgs):
        l, r = make_signal(kind, 40 * 1152 + 37 * i, sr, 300 + i)
        ref, _, _ = oracle.encode_stream(ch, sr, kbps, l, r if ch == 2 else None, chunk=1152)
        assert res[i] == ref, i


@pytest.mark.gpu
def test_empty_batch_and_error_paths_keep_the_stream_intact(oracle):
    import ctypes

    import lamejs_b200 as M

    assert M.encode_streams(2, 44100, 128, [], []) == []
    L = M.lib()
    # a too-small output buffer fails the call but not the stream: the next call delivers the backlog
    l, r = make_signal("noise", 6 * 1152, 44100, 41)
    ref, _, _ = oracle.encode_stream(2, 44100, 128, l, r)
    h = ctypes.c_void_p()
    assert L.mp3b200_create(2, 44100, 128, ctypes.byref(h)) == 0
    small = np.empty(100, dtype=np.uint8)
    big = np.empty(20000, dtype=np.uint8)
    rc = L.mp3b200_encode(h, l.ctypes.data, r.ctypes.data, len(l), small.ctypes.data, len(small))
    assert rc < 0
    got = bytearray()
    rc = L.mp3b200_encode(h, l.ctypes.data, r.ctypes.data, 0, big.ctypes.data, len(big))
    assert rc > 0
    got += big[:rc].tobytes()
    rc = L.mp3b200_flush(h, big.ctypes.data, len(big))
    assert rc > 0
    got += big[:rc].tobytes()
    L.mp3b200_destroy(h)
    assert bytes(got) == ref


@pytest.mark.parametrize("kind,ch,sr,kbps,frames", oracle_inputs.LSF_STAGE_PARITY_CASES)
def test_stage_parity_lsf(M, oracle, kind, ch, sr, kbps, frames):
    """MPEG-2 / MPEG-2.5 (one granule per frame, 576-sample frames, scale_bitcount_lsf, 9/17-byte side info): every stage
    tap bit-equal to the oracle, which is byte-identical to real lamejs on these configurations (test_lamejs_pin)."""
    l, r = oracle_inputs.lsf_stage_parity_signal((kind, ch, sr, kbps, frames))
    assert M.granules_per_frame(ch, sr, kbps) == 1
    F = M.stream_frames(len(l), ch, sr, kbps)
    ref, _, tr = oracle.encode_stream(ch, sr, kbps, l, r, trace_frames=F + 2)
    assert len(tr) == F
    g = M.debug_stages(ch, sr, kbps, l, r, want=stage_taps.ALL_TAPS)
    stage_taps.compare(g, tr, ref, 1, ch)


def test_lsf_batches_and_handles(M, oracle):
    """LSF through the batch API (ragged streams) and through live handles with odd chunkings (flush completes two 576-sample
    frames from one 1152-sample zero bunch, Lame.js:1416-1443)."""
    for ch, sr, kbps in [(2, 22050, 64), (1, 16000, 24), (2, 8000, 16)]:
        lens = [0, 1, 575, 576, 800, 1329, 5000, 576 * 40 + 3]
        sigs = [make_signal("burst" if i % 2 else "noise", n, sr, 70 + i) for i, n in enumerate(lens)]
        outs = M.encode_streams(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None)
        for n, s, o in zip(lens, sigs, outs):
            assert o == oracle.encode_stream(ch, sr, kbps, s[0], s[1] if ch == 2 else None)[0], (ch, sr, kbps, n)
        l, r = make_signal("burst", 576 * 50 + 77, sr, 9)
        for chunk in (576, 1152, 777, 5000):
            enc = M.Mp3Encoder(ch, sr, kbps)
            ref = oracle.OracleEncoder(ch, sr, kbps)
            for i in range(0, len(l), chunk):
                assert enc.encodeBuffer(l[i:i + chunk], r[i:i + chunk] if ch == 2 else None) == ref.encode_buffer(l[i:i + chunk], r[i:i + chunk]), (chunk, i)
            assert enc.flush() == ref.flush()
            assert enc.flush() == b"" == ref.flush()
            enc.close(); ref.close()
