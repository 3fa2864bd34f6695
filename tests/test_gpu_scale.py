"""BASELINE.json configs #3/#4/#5 at (or near) their stated sizes, EVERY stream compared byte for byte with the CPU oracle
(thread pool over the host cores; ctypes releases the GIL), plus a randomised soak of >= 30 k frames.  The speculate /
verify / re-validate machinery of the quantizer (cross-frame OldValue recurrence) is exactly the kind of logic whose
rare failure only shows up at scale."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from synth import bursts, make_signal, octave_hold, white

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import lamejs_b200 as m
    return m


def _check_all(M, oracle, ch, sr, kbps, ls, rs):
    oracle.lib()
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        futs = [ex.submit(lambda j=j: oracle.encode_stream(ch, sr, kbps, ls[j], rs[j] if ch == 2 else None)[0]) for j in range(len(ls))]
        outs = M.encode_streams(ch, sr, kbps, ls, rs if ch == 2 else None)
        bad = [j for j, f in enumerate(futs) if outs[j] != f.result()]
    assert not bad, "streams differing from the oracle: %s" % bad[:10]
    return outs


def test_c3_full_size_white_noise_320k(M, oracle):
    """config #3: stereo 48 kHz 320 kbps, 100 streams x 1000 white-noise frames (stream j uses counter offset j * 2^32)."""
    S, n = 100, 1000 * 1152
    ls, rs = zip(*[white(n, 0x5EED0003, offset=j << 32) for j in range(S)])
    outs = _check_all(M, oracle, 2, 48000, 320, list(ls), list(rs))
    assert all(len(o) == 1001 * 960 for o in outs)


def test_c4_mono_octave_200_streams(M, oracle):
    """config #4 shape: mono 44.1 kHz 128 kbps octave-hold noise, 200 streams x 1000 frames (the 1000-stream run is a bench config)."""
    S, n = 200, 1000 * 1152
    ls = [octave_hold(n, 0x5EED0004 + 16 * j) for j in range(S)]
    _check_all(M, oracle, 1, 44100, 128, ls, ls)


def test_c5_full_size_bursts(M, oracle):
    """config #5 input (transient bursts -> START/SHORT/STOP switching) under CBR 128k: 100 streams x 1000 frames."""
    S, n = 100, 1000 * 1152
    ls, rs = zip(*[bursts(n, 0x5EED0005 + 64 * j) for j in range(S)])
    _check_all(M, oracle, 2, 44100, 128, list(ls), list(rs))


def _distinct_short_signals(k, sr):
    """k different short mono signals (lengths 1..~3 frames of MPEG-2.5 and their ragged tails, several kinds)."""
    kinds = ["noise", "burst", "white", "sine", "octave"]
    return [make_signal(kinds[i % 5], 300 + 37 * i, sr, 500 + i)[0] for i in range(k)]


def test_70000_short_mono_8k_streams(M, oracle):
    """More streams than a grid dimension holds (65535; the stream index is a grid y / z coordinate): the batch runs as
    consecutive launches and every stream equals the oracle.  97 distinct signals (prime, not a divisor of 65535) are dealt
    out round robin, so a stream of the second launch reading the first launch's data would show."""
    S, K = 70000, 97
    sigs = _distinct_short_signals(K, 8000)
    refs = [oracle.encode_stream(1, 8000, 16, s, None)[0] for s in sigs]
    outs = M.encode_streams(1, 8000, 16, [sigs[j % K] for j in range(S)])
    bad = [j for j in range(S) if outs[j] != refs[j % K]]
    assert not bad, "streams differing from the oracle: %s" % bad[:10]


def test_70000_live_handles_in_one_batch_call(M, oracle):
    """The handle batch path with more live handles than one launch holds."""
    S, K = 70000, 97
    sigs = _distinct_short_signals(K, 8000)
    want = []
    for s in sigs:
        ref = oracle.OracleEncoder(1, 8000, 16)
        want.append((ref.encode_buffer(s), ref.flush()))
        ref.close()
    encs = [M.Mp3Encoder(1, 8000, 16) for _ in range(S)]
    try:
        got = M.encode_batch(encs, [sigs[j % K] for j in range(S)])
        assert not [j for j in range(S) if got[j] != want[j % K][0]]
        got = M.flush_batch(encs)
        assert not [j for j in range(S) if got[j] != want[j % K][1]]
    finally:
        for e in encs:
            e.close()


def _quiet_across_chunk_1024(l, r, framesize):
    """Silence over frames 16376..16407: the passage spans chunk 1024 of the block-type / ATH scan (16 frames per chunk,
    1024 scan threads: past frame 16384 each scan thread owns a second chunk)."""
    a, b = 16376 * framesize, 16408 * framesize
    l[a:b] = 0
    r[a:b] = 0
    return l, r


@pytest.mark.parametrize("ch,sr,kbps", [(2, 44100, 128), (1, 22050, 48)])
def test_stream_longer_than_16384_frames(M, oracle, ch, sr, kbps):
    framesize = 1152 if sr >= 32000 else 576
    n = 17200 * framesize + 333
    l, r = bursts(n, 0x5EED0051 + ch)
    l, r = _quiet_across_chunk_1024(l, r, framesize)
    assert M.stream_frames(n, ch, sr, kbps) > 17000
    out = M.encode_streams(ch, sr, kbps, [l], [r] if ch == 2 else None)[0]
    assert out == oracle.encode_stream(ch, sr, kbps, l, r if ch == 2 else None)[0]


def test_device_entry_with_gapped_out_of_order_offsets(M, oracle):
    """encode_streams_device with caller-chosen offsets: streams stored in reverse order, at odd offsets, with gaps, in both
    the PCM and the output buffer.  Bytes equal encode_streams; the PCM buffer and every output byte outside the streams
    keep their sentinel values."""
    import torch

    ch, sr, kbps = 2, 44100, 128
    sigs = [make_signal(k, n, sr, 70 + i) for i, (k, n) in enumerate([("burst", 20000), ("noise", 1), ("white", 7001),
                                                                     ("sweep", 1152 * 40 + 3), ("octave", 0), ("noise", 5000)])]
    ns = [len(l) for l, _ in sigs]
    nb = [M.stream_bytes(ch, sr, kbps, n) for n in ns]
    pcm = np.full(sum(ns) * ch + 1000, 0x5A5A, dtype=np.int16)
    out_size = sum(nb) + 777
    pcm_off, out_off = [0] * len(sigs), [0] * len(sigs)
    p, o = 13, 101
    for i in reversed(range(len(sigs))):                 # last stream first, odd gaps between them
        pcm_off[i], out_off[i] = p, o
        l, r = sigs[i]
        pcm[p:p + ns[i]] = l
        pcm[p + ns[i]:p + 2 * ns[i]] = r
        p += 2 * ns[i] + 2 * i + 1
        o += nb[i] + 3 * i + 5
    assert p <= len(pcm) and o <= out_size
    d_pcm = torch.from_numpy(pcm.copy()).cuda()
    d_out = torch.full((out_size,), 0xA5, dtype=torch.uint8, device="cuda")
    tm = M.encode_streams_device(ch, sr, kbps, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off)
    assert tm[7] >= 2
    out = d_out.cpu().numpy()
    assert np.array_equal(d_pcm.cpu().numpy(), pcm)
    want = M.encode_streams(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs])
    touched = np.zeros(out_size, dtype=bool)
    for i in range(len(sigs)):
        assert out[out_off[i]:out_off[i] + nb[i]].tobytes() == want[i], i
        touched[out_off[i]:out_off[i] + nb[i]] = True
    assert (out[~touched] == 0xA5).all()
    for i in (0, 3):
        assert want[i] == oracle.encode_stream(ch, sr, kbps, sigs[i][0], sigs[i][1])[0]


def test_random_soak_30k_frames(M, oracle):
    rng = np.random.default_rng(20260924)
    kinds = ["noise", "burst", "sweep", "white", "sine", "octave", "silence"]
    configs = [(ch, sr, kbps) for sr in (32000, 44100, 48000) for kbps in (64, 96, 112, 128, 160, 192, 256, 320) for ch in (1, 2)
               if M.stream_bytes(ch, sr, kbps, 1152) > 0]
    by_cfg, frames = {}, 0
    for i in range(150):
        cfg = configs[rng.integers(len(configs))]
        kind = kinds[rng.integers(len(kinds))]
        n = int(rng.integers(1, 420 * 1152))
        by_cfg.setdefault(cfg, []).append(make_signal(kind, n, cfg[1], int(rng.integers(1 << 30))))
        frames += M.stream_frames(n)
    assert frames >= 30000
    for (ch, sr, kbps), sigs in by_cfg.items():
        _check_all(M, oracle, ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs])
