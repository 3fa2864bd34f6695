"""Tagged whole streams on device buffers (mp3b200_encode_streams_tagged_device / _f32, encode_streams_device_tagged): the
same files, out_bytes and gains as the host tagged path, the streams' layout in one device buffer, the lamejs fixtures whose
schedule is one whole encodeBuffer call and a flush, batches past 65535 streams, refusals and ordering behind torch work."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import float_signals as FS
from synth import make_signal

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 0xA5
FRACTIONAL = (44100, 22050, 11025)     # lamejs's own tagged stream differs from the oracle's there (tests/test_tag_oracle.py)


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def _rs(M, ch, sr, kb):
    return M.out_samplerate(ch, sr, kb) != sr


def _device_pcm(ch, lefts, rights, f32):
    """one device tensor holding every stream's rows (left, then right), each stream behind a few samples of gap"""
    import torch
    dt = np.float32 if f32 else np.int16
    parts, offs, at = [], [], 0
    for i, l in enumerate(lefts):
        gap = np.full(3 + i % 5, 7, dtype=dt)
        parts.append(gap)
        at += len(gap)
        offs.append(at)
        rows = [np.asarray(l, dtype=dt)] + ([np.asarray(rights[i], dtype=dt)] if ch == 2 else [])
        parts += rows
        at += sum(len(x) for x in rows)
    return torch.from_numpy(np.concatenate(parts + [np.zeros(8, dtype=dt)])).cuda(), offs


def _layout(room):
    """odd, non-contiguous offsets, the streams in reverse order: (offsets, buffer size)"""
    offs, at = [0] * len(room), 5
    for s in reversed(range(len(room))):
        at += 2 * (s % 3) + 1
        at += 1 - at % 2
        offs[s] = at
        at += room[s]
    return offs, at + 11


def device_tagged(M, ch, sr, kb, lefts, rights, f32=False, rg=False):
    """the streams through encode_streams_device_tagged, laid out by _layout in a sentinel-filled buffer; checks that
    nothing outside the files was written.  Returns (files, title_db, album_db, files' audio as encode_streams_device wrote
    it untagged for the same PCM)"""
    import torch
    rs = _rs(M, ch, sr, kb)
    tfs = M.lametag_size(ch, sr, kb, resample=rs)
    audio = [M.stream_bytes(ch, sr, kb, len(l), resample=rs) for l in lefts]
    room = [a + tfs for a in audio]
    d_pcm, pcm_off = _device_pcm(ch, lefts, rights, f32)
    offs, size = _layout(room)
    d_out = torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda")
    out_bytes, title, album = M.encode_streams_device_tagged(ch, sr, kb, d_pcm.data_ptr(), pcm_off, [len(l) for l in lefts],
                                                             d_out.data_ptr(), offs, resample=rs, float32=f32, find_replay_gain=rg)
    assert out_bytes == room
    buf = d_out.cpu().numpy()
    files = [buf[o:o + n].tobytes() for o, n in zip(offs, out_bytes)]
    outside = np.ones(size, dtype=bool)
    for o, n in zip(offs, out_bytes):
        outside[o:o + n] = False
    assert (buf[outside] == SENTINEL).all()
    plain = torch.full((sum(audio) + 8,), SENTINEL, dtype=torch.uint8, device="cuda")
    M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, [len(l) for l in lefts], plain.data_ptr(),
                            np.cumsum([0] + audio[:-1]), resample=rs, float32=f32)
    p = plain.cpu().numpy().tobytes()
    untagged = [p[o:o + a] for o, a in zip(np.cumsum([0] + audio[:-1]), audio)]
    return files, title, album, untagged


def _ragged(ch, sr, f32):
    lens = [0, 37, 1152, 5 * 1152 + 1, sr // 2, 2 * sr + 999, 7000]
    kinds = ["noise", "silence", "sweep", "white", "noise", "octave", "burst"]
    sig = [make_signal(k, n, sr, seed=i + 5) for i, (k, n) in enumerate(zip(kinds, lens))]
    lefts, rights = [s[0] for s in sig], [s[1] for s in sig]
    if f32:       # fractions, so that the Float32 path is the one that runs
        lefts = [(x * 0.61 + 0.37).astype(np.float32) for x in lefts]
        rights = [(x * -0.83 + 0.11).astype(np.float32) for x in rights]
    return lefts, rights if ch == 2 else None


@pytest.mark.parametrize("rg", [False, True], ids=["tag", "replaygain"])
@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 8000, 24), (2, 22050, 64), (2, 48000, 64), (2, 32000, 24), (1, 8000, 8)])
def test_equals_host_tagged_path(M, ch, sr, kb, f32, rg):
    """every stream's file, out_bytes and both gains equal the host tagged path's; behind the tag the bytes are those of the
    untagged device path; (1, 8000, 8): the tag does not fit, nothing is tagged or analysed"""
    rs = _rs(M, ch, sr, kb)
    lefts, rights = _ragged(ch, sr, f32)
    host, h_title, h_album = M.encode_streams_replaygain(ch, sr, kb, lefts, rights, resample=rs, find_replay_gain=rg)
    files, title, album, untagged = device_tagged(M, ch, sr, kb, lefts, rights, f32=f32, rg=rg)
    assert files == host
    assert title == h_title and album == h_album
    tfs = M.lametag_size(ch, sr, kb, resample=rs)
    assert [f[tfs:] for f in files] == untagged
    if tfs == 0 or not rg:
        assert title == [M.GAIN_NOT_ENOUGH_SAMPLES] * len(lefts) and album == M.GAIN_NOT_ENOUGH_SAMPLES
    if tfs == 0:
        assert files == untagged


def _at(ch, out_sr):
    """offset of the tag's Radio Replay Gain field"""
    return 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19


def _placeholder(M, ch, sr, kb, rs):
    e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs)
    b = e.flush()[:M.lametag_size(ch, sr, kb, resample=rs)]
    e.close()
    return b


def _check_fixture(M, name, c, l, r, f32):
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    rs = _rs(M, ch, sr, kb)
    out_sr = M.out_samplerate(ch, sr, kb)
    files, title, _, _ = device_tagged(M, ch, sr, kb, [l], None if r is None else [r], f32=f32, rg=True)
    at = _at(ch, out_sr)
    assert M.radio_gain(title[0]) == c["radio_gain"][-1], name
    assert files[0][at:at + 2] == bytes.fromhex(c["tag"])[at:at + 2], name
    if out_sr not in FRACTIONAL:
        ph = _placeholder(M, ch, sr, kb, rs)
        assert hashlib.sha256(ph + files[0][len(ph):]).hexdigest() == c["sha256"], name


RG_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_replaygain_golden.json")))
FLOAT_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))


@pytest.mark.parametrize("name", sorted(n for n, c in RG_GOLDEN.items() if len(c["schedule"]) == 2 and c["schedule"][1] == -1))
def test_replaygain_fixture(M, name):
    """lamejs's ReplayGain fixtures of one encodeBuffer call and a flush, Int16 rows"""
    c = RG_GOLDEN[name]
    assert c["schedule"][0] == c["samples"]
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], seed=c["seed"])
    _check_fixture(M, name, c, l, r if c["channels"] == 2 else None, False)


@pytest.mark.parametrize("name", sorted(n for n, c in FLOAT_GOLDEN.items()
                                        if c["rg"] and len(c["schedule"]) == 2 and c["schedule"][0][1] == "f"))
def test_float_replaygain_fixture(M, name):
    """lamejs's Float32 ReplayGain fixtures of one encodeBuffer call and a flush"""
    c = FLOAT_GOLDEN[name]
    l, r, _ = FS.case_signal(c)
    _check_fixture(M, name, c, l.astype(np.float32), None if r is None else r.astype(np.float32), True)


def test_c2_length_with_replaygain(M):
    """one C2-length stream (10000 frames of a sweep, 44.1 kHz stereo) with the analysis, against the host path"""
    l, r = make_signal("sweep", 10000 * 1152, 44100, seed=1)
    host, h_title, h_album = M.encode_streams_replaygain(2, 44100, 128, [l], [r])
    files, title, album, untagged = device_tagged(M, 2, 44100, 128, [l], [r], rg=True)
    assert files == host and title == h_title and album == h_album
    assert files[0][M.lametag_size(2, 44100, 128):] == untagged[0]


def test_more_than_65535_streams(M):
    """65635 tiny streams: two launch groups and two k_music_crc groups, the same files as the host path; with the analysis
    the batch is refused as the host path refuses it"""
    import torch
    S = 65535 + 100
    rng = np.random.default_rng(3)
    lefts = [rng.integers(-3000, 3000, size=int(n), dtype=np.int16) for n in rng.integers(0, 700, size=S)]
    host = M.encode_streams_tagged(1, 8000, 24, lefts)
    tfs = M.lametag_size(1, 8000, 24)
    room = [M.stream_bytes(1, 8000, 24, len(l)) + tfs for l in lefts]
    out_off = np.cumsum([0] + room[:-1])
    d_pcm = torch.from_numpy(np.concatenate(lefts + [np.zeros(8, np.int16)])).cuda()
    pcm_off = np.cumsum([0] + [len(l) for l in lefts[:-1]])
    ns = [len(l) for l in lefts]
    d_out = torch.full((sum(room),), SENTINEL, dtype=torch.uint8, device="cuda")
    out_bytes, _, _ = M.encode_streams_device_tagged(1, 8000, 24, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off)
    assert out_bytes == room
    buf = d_out.cpu().numpy().tobytes()
    assert [buf[o:o + n] for o, n in zip(out_off, out_bytes)] == host
    with pytest.raises(M.Mp3B200Error, match="error -3: ReplayGain batches hold at most 65535 streams"):
        M.encode_streams_replaygain(1, 8000, 24, lefts)
    with pytest.raises(M.Mp3B200Error, match="error -3: ReplayGain batches hold at most 65535 streams"):
        M.encode_streams_device_tagged(1, 8000, 24, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off, find_replay_gain=True)


def test_unknown_flag_is_refused(M):
    import torch
    L = M.lib()
    d_pcm = torch.zeros(5000, dtype=torch.int16, device="cuda")
    d_f32 = torch.zeros(5000, dtype=torch.float32, device="cuda")
    d_out = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    i64 = lambda v: np.array(v, dtype=np.int64)     # noqa: E731
    pcm_off, ns, out_off, got = i64([0]), i64([5000]), i64([0]), i64([0])
    for fn, p in ((L.mp3b200_encode_streams_tagged_device, d_pcm), (L.mp3b200_encode_streams_tagged_device_f32, d_f32)):
        for flags in (4, 8, 1 << 30, 4 | M.REPLAYGAIN):
            rc = fn(1, 44100, 128, flags, 1, p.data_ptr(), pcm_off.ctypes.data, ns.ctypes.data, d_out.data_ptr(), out_off.ctypes.data,
                    got.ctypes.data, None, None)
            assert rc == -1 and L.mp3b200_last_error() == b"unknown flags", (fn, flags)


def test_non_finite_float_is_refused_and_the_next_call_works(M):
    import torch
    l, r = make_signal("noise", 20000, 44100, seed=8)
    lf, rf = (l * 0.5).astype(np.float32), (r * 0.25).astype(np.float32)
    tfs = M.lametag_size(2, 44100, 128)
    room = M.stream_bytes(2, 44100, 128, len(lf)) + tfs
    for bad in (np.nan, np.inf, 3e38):
        x = rf.copy()
        x[12345] = bad
        d_pcm = torch.from_numpy(np.concatenate([lf, x])).cuda()
        d_out = torch.full((room,), SENTINEL, dtype=torch.uint8, device="cuda")
        with pytest.raises(M.Mp3B200Error, match="error -1: non-finite"):
            M.encode_streams_device_tagged(2, 44100, 128, d_pcm.data_ptr(), [0], [len(lf)], d_out.data_ptr(), [0], float32=True,
                                           find_replay_gain=True)
        assert (d_out[:tfs].cpu().numpy() == SENTINEL).all()          # no tag frame placed
        files, title, album, _ = device_tagged(M, 2, 44100, 128, [lf], [rf], f32=True, rg=True)
        host, h_title, h_album = M.encode_streams_replaygain(2, 44100, 128, [lf], [rf])
        assert files == host and title == h_title and album == h_album


@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_waits_for_torch_work_on_the_default_stream(M, f32):
    """PCM and the output's fill written by torch kernels just before the call, without a synchronise, behind a long kernel:
    the call encodes that PCM into that buffer, and the ReplayGain analysis reads that PCM (Int16 rows are analysed where the
    caller left them)"""
    import torch
    n = 3 * 44100
    t = torch.arange(2 * n, device="cuda", dtype=torch.float64)
    d_out = torch.empty(M.stream_bytes(2, 44100, 128, n) + M.lametag_size(2, 44100, 128), dtype=torch.uint8, device="cuda")

    def write_pcm(dst):
        x = torch.sin(t * 0.031) * 12000 + torch.sin(t * 0.0007) * 9000
        dst.copy_(x if f32 else x.round())

    def call():
        return M.encode_streams_device_tagged(2, 44100, 128, d_pcm.data_ptr(), [0], [n], d_out.data_ptr(), [0], float32=f32,
                                              find_replay_gain=True)

    # everything once with the same shapes: no torch kernel loads a module and no library buffer grows (cudaFree and
    # cudaMalloc synchronise the device) in the part below, so the spin kernel is still running when the call is made
    d_pcm = torch.zeros(2 * n, dtype=torch.float32 if f32 else torch.int16, device="cuda")
    write_pcm(d_pcm)
    d_out.fill_(0)
    torch.cuda._sleep(1000)
    call()
    torch.cuda.synchronize()
    d_pcm.zero_()
    d_out.fill_(SENTINEL)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)         # spins well beyond the library's host work before the call queues anything
    write_pcm(d_pcm)
    d_out.fill_(0)
    out_bytes, title, album = call()
    got =d_out.cpu().numpy().tobytes()[:out_bytes[0]]
    pcm = d_pcm.cpu().numpy()
    host, h_title, h_album = M.encode_streams_replaygain(2, 44100, 128, [pcm[:n]], [pcm[n:]])
    assert got == host[0] and title == h_title and album == h_album
    assert h_title[0] != M.GAIN_NOT_ENOUGH_SAMPLES
