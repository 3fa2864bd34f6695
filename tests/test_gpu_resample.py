"""Integer-ratio resampling on the GPU (MP3B200_RESAMPLE): k_resample against the oracle's resampler, every stage tap behind
it against the oracle's traces, the bytes of every entry point against the oracle and real lamejs, the handle API on
resampled handles, and that nothing else moved."""
import hashlib
import json
import os

import numpy as np
import pytest

import resample_tap as T
from synth import make_signal

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
INT = T.resampled_configs(integer=True)
FRAC = T.resampled_configs(integer=False)
IDS = ["%d_%d_%d" % c for c in INT]


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    lamejs_b200.lib()
    return lamejs_b200


def stereo(kind, n, sr, seed):
    l, r = make_signal(kind, n, sr, seed)
    return l, np.roll(r, 7)                      # L != R even for kinds that repeat one channel


def handle_encode(M, cfg, l, r, chunk, **kw):
    ch, sr, kb = cfg
    enc = M.Mp3Encoder(ch, sr, kb, resample=True, **kw)
    out, sizes = bytearray(), []
    step = chunk or max(len(l), 1)
    for i in range(0, len(l), step):
        b = enc.encodeBuffer(l[i:i + step], r[i:i + step])
        sizes.append(len(b))
        out += b
    b = enc.flush()
    sizes.append(len(b))
    out += b
    return bytes(out), sizes, enc


def _lamejs_fixtures():
    import oracle_lib as O

    gold = json.load(open(os.path.join(HERE, "golden", "lamejs_golden.json")))["cases"]
    out = []
    for k, c in sorted(gold.items()):
        if "error" in c:
            continue
        o = O.out_samplerate(c["channels"], c["samplerate"], c["kbps"])
        if o != c["samplerate"] and T.is_integer_ratio(c["samplerate"], o):
            out.append(k)
    return gold, out


GOLD, GOLD_NAMES = _lamejs_fixtures()


def test_lamejs_fixture_inventory():
    assert len(GOLD_NAMES) == 17, GOLD_NAMES


@pytest.mark.parametrize("name", GOLD_NAMES)
def test_pinned_to_lamejs(M, name):
    """Fixtures real lamejs encoded in integer-ratio configurations, in their recorded chunking: same bytes and per-call
    sizes through Mp3Encoder(..., resample=True)."""
    c = GOLD[name]
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], c["seed"])
    data, sizes, _ = handle_encode(M, (c["channels"], c["samplerate"], c["kbps"]), l, r if c["channels"] == 2 else l, c["chunk"])
    assert hashlib.sha256(data).hexdigest() == c["sha256"]
    assert len(sizes) == c["calls"]
    assert hashlib.sha256(json.dumps([int(s) for s in sizes]).encode()).hexdigest() == c["sizes_sha256"]


@pytest.mark.parametrize("cfg", INT, ids=IDS)
def test_resampler_tap_equals_oracle(M, cfg):
    """k_resample's output is, bit for bit, every value the oracle's resampler wrote (flush included)."""
    ch, sr, kb = cfg
    n = 9 * 1152 + 77
    l, r = stereo("burst", n, sr, 3)
    y, _, _, _ = T.record(ch, sr, kb, l, r, [1152] * (n // 1152) + [n % 1152])
    got = M.debug_resample(ch, sr, kb, l, r, ny=y.shape[1])
    assert got.shape == y.shape
    assert np.array_equal(got.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("cfg", INT, ids=IDS)
def test_stage_parity(M, oracle, cfg):
    """Every stage tap after k_resample -- MDCT spectrum, block types, masking, ATH adjust, quantized lines, side info,
    scalefactors, xmin, and the OldValue / CurrentStep chain -- bit-equal to the oracle's frame and quantizer traces, for two
    signals of about 20 output frames plus a ragged tail (L != R)."""
    import stage_taps

    ch, sr, kb = cfg
    r = sr // M.out_samplerate(ch, sr, kb)
    G = M.granules_per_frame(ch, sr, kb, resample=True)
    n = r * (20 * 576 * G + 211) + 5
    for kind, seed in (("burst", 21), ("noise", 22)):
        l, rt = stereo(kind, n, sr, seed)
        rr = rt if ch == 2 else None
        F = M.stream_frames(n, ch, sr, kb, resample=True)
        ref, _, tr = oracle.encode_stream(ch, sr, kb, l, rr, trace_frames=F + 2)
        assert len(tr) == F and F >= 20
        g = M.debug_stages(ch, sr, kb, l, rr, want=stage_taps.ALL_TAPS, resample=True)
        stage_taps.compare(g, tr, ref, G, ch, "%s %d/%d/%d" % (kind, ch, sr, kb))


def test_stage_taps_flag_on_native_configurations(M):
    """debug_stages(..., resample=True) on configurations that encode at their input rate returns the unflagged taps; without
    the flag a resampled configuration is refused."""
    import stage_taps

    l, r = stereo("burst", 9 * 1152 + 300, 44100, 31)
    for ch, sr, kb in ((2, 44100, 128), (1, 22050, 32), (2, 8000, 16)):
        rr = r if ch == 2 else None
        plain = M.debug_stages(ch, sr, kb, l, rr, want=stage_taps.ALL_TAPS)
        flagged = M.debug_stages(ch, sr, kb, l, rr, want=stage_taps.ALL_TAPS, resample=True)
        assert plain.keys() == flagged.keys()
        for k in plain:
            assert plain[k].shape == flagged[k].shape and plain[k].tobytes() == flagged[k].tobytes(), (ch, sr, kb, k)
    with pytest.raises(M.Mp3B200Error):
        M.debug_stages(2, 48000, 64, l, r, want=("xr",))


@pytest.mark.parametrize("cfg", INT, ids=IDS)
def test_handles_match_oracle(M, oracle, cfg):
    """Three signals x four chunkings through handles: bytes and per-call sizes equal the oracle's."""
    ch, sr, kb = cfg
    n = 14000 + 77
    for kind in ("burst", "noise", "sweep"):
        l, r = stereo(kind, n, sr, 11)
        rr = r if ch == 2 else None
        for chunk in (None, 1152, 577, 4099):
            want, wsizes, _ = oracle.encode_stream(ch, sr, kb, l, rr, chunk=chunk)
            got, sizes, enc = handle_encode(M, cfg, l, r if ch == 2 else l, chunk)
            enc.close()
            assert got == want, (kind, chunk)
            assert sizes == wsizes, (kind, chunk)


@pytest.mark.parametrize("cfg", [(2, 48000, 64), (1, 44100, 32), (2, 48000, 8), (1, 32000, 24)], ids=lambda c: "%d_%d_%d" % c)
def test_ragged_batch_matches_oracle(M, oracle, cfg):
    """encode_streams(resample=True) on a ragged batch: 0, 1, 16, 17, 18 samples, frame edges in input units, and a stream
    of over 2000 frames."""
    ch, sr, kb = cfg
    r = sr // M.out_samplerate(ch, sr, kb)
    lens = [0, 1, 16, 17, 18, 19, r * 576, r * 576 + 16, r * 576 + 17, r * (576 + 752 - 528) + 16, r * (2 * 576 - 1104 + 752) + 17,
            r * 576 * 2001 + 123]
    sigs = [stereo("burst" if i % 2 else "noise", n, sr, 40 + i) for i, n in enumerate(lens)]
    got = M.encode_streams(ch, sr, kb, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None, resample=True)
    for (l, rt), g in zip(sigs, got):
        assert g == oracle.encode_stream(ch, sr, kb, l, rt if ch == 2 else None)[0], len(l)
        assert len(g) == M.stream_bytes(ch, sr, kb, len(l), resample=True)


def test_device_entry_gapped_offsets(M, oracle):
    """encode_streams_device(resample=True) with reversed, gapped offsets: bytes equal the oracle's, the sentinels around the
    streams stay, and slot 14 holds the resampler's time."""
    import torch

    ch, sr, kb = 2, 48000, 64
    sigs = [stereo(k, n, sr, 80 + i) for i, (k, n) in enumerate([("burst", 30000), ("noise", 1), ("sweep", 7001), ("noise", 0),
                                                                 ("burst", 12345)])]
    ns = [len(l) for l, _ in sigs]
    nb = [M.stream_bytes(ch, sr, kb, n, resample=True) for n in ns]
    pcm = np.full(sum(ns) * ch + 1000, 0x5A5A, dtype=np.int16)
    out_size = sum(nb) + 777
    pcm_off, out_off = [0] * len(sigs), [0] * len(sigs)
    p, o = 13, 101
    for i in reversed(range(len(sigs))):
        pcm_off[i], out_off[i] = p, o
        l, r = sigs[i]
        pcm[p:p + ns[i]] = l
        pcm[p + ns[i]:p + 2 * ns[i]] = r
        p += 2 * ns[i] + 2 * i + 1
        o += nb[i] + 3 * i + 5
    d_pcm = torch.from_numpy(pcm.copy()).cuda()
    d_out = torch.full((out_size,), 0xA5, dtype=torch.uint8, device="cuda")
    tm = M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off, resample=True)
    assert tm[14] > 0
    out = d_out.cpu().numpy()
    assert np.array_equal(d_pcm.cpu().numpy(), pcm)
    touched = np.zeros(out_size, dtype=bool)
    for i, (l, r) in enumerate(sigs):
        assert out[out_off[i]:out_off[i] + nb[i]].tobytes() == oracle.encode_stream(ch, sr, kb, l, r)[0], i
        touched[out_off[i]:out_off[i] + nb[i]] = True
    assert (out[~touched] == 0xA5).all()
    native = M.encode_streams_device(2, 24000, 64, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off)
    assert native[14] == 0


def test_handle_api(M, oracle):
    """Repeated handle in a batch, export -> import hand-over, equal blobs from three chunkings, a blob of another rate pair
    refused, seek refused with -2 -- all checked against the oracle."""
    cfg = ch, sr, kb = (2, 48000, 64)
    n = 40000
    l, r = stereo("burst", n, sr, 5)
    want, _, _ = oracle.encode_stream(ch, sr, kb, l, r)
    # a batch listing one handle twice runs its entries in order
    a, b = M.Mp3Encoder(*cfg, resample=True), M.Mp3Encoder(*cfg, resample=True)
    cut = [0, 5000, 17001, 17017, 29999, n]
    got_a, got_b = bytearray(), bytearray()
    for i in range(0, len(cut) - 2, 2):
        outs = M.encode_batch([a, b, a], [l[cut[i]:cut[i + 1]], l[cut[i]:cut[i + 2]], l[cut[i + 1]:cut[i + 2]]],
                              [r[cut[i]:cut[i + 1]], r[cut[i]:cut[i + 2]], r[cut[i + 1]:cut[i + 2]]])
        got_a += outs[0] + outs[2]
        got_b += outs[1]
    tail = M.encode_batch([a, b], [l[cut[-2]:], l[cut[-2]:]], [r[cut[-2]:], r[cut[-2]:]])
    got_a += tail[0]
    got_b += tail[1]
    fl = M.flush_batch([a, b, a])
    assert fl[2] == b""
    assert bytes(got_a + fl[0]) == want and bytes(got_b + fl[1]) == want
    # hand-over mid-stream, and equal blobs from three chunkings
    blobs = []
    for chunk in (1152, 577, 30001):
        e = M.Mp3Encoder(*cfg, resample=True)
        head = bytearray()
        for i in range(0, 30001, chunk):
            head += e.encodeBuffer(l[i:min(i + chunk, 30001)], r[i:min(i + chunk, 30001)])
        blobs.append((e.export_state(), bytes(head)))
        e.close()
    assert blobs[0][0] == blobs[1][0] == blobs[2][0]
    f = M.Mp3Encoder(*cfg, resample=True)
    f.import_state(blobs[0][0])
    rest = f.encodeBuffer(l[30001:], r[30001:]) + f.flush()
    assert blobs[0][1] + rest == want
    # another rate pair, another magic: refused
    for other in (M.Mp3Encoder(2, 44100, 48, resample=True), M.Mp3Encoder(2, 24000, 64), M.Mp3Encoder(1, 48000, 40, resample=True)):
        with pytest.raises(M.Mp3B200Error):
            other.import_state(blobs[0][0])
    native = M.Mp3Encoder(2, 24000, 64)
    native.encodeBuffer(l[:5000], r[:5000])
    with pytest.raises(M.Mp3B200Error):
        f.import_state(native.export_state())
    # seek: not supported
    g = M.Mp3Encoder(*cfg, resample=True)
    h = np.zeros(1104 + 224 + 576, dtype=np.int16)
    assert M.lib().mp3b200_seek(g._h, 2, h.ctypes.data, h.ctypes.data, len(h)) == -2


@pytest.mark.parametrize("cfg,chunk", [((2, 48000, 64), 1152), ((1, 44100, 32), None), ((2, 48000, 8), 4099), ((2, 32000, 40), 577)],
                         ids=["48k_st64", "44k1_mono32", "48k_st8", "32k_st40"])
def test_tagged_handle(M, oracle, cfg, chunk):
    """A tagged resampled handle: bytes, tag frame, music CRC, bytes written and encoder padding equal the oracle's."""
    ch, sr, kb = cfg
    l, r = stereo("sweep", 25000, sr, 9)
    want, wsizes, info = oracle.encode_stream_tagged(ch, sr, kb, l, r if ch == 2 else None, chunk=chunk)
    got, sizes, enc = handle_encode(M, cfg, l, r if ch == 2 else l, chunk, write_vbr_tag=True)
    assert enc.tag_on == info["tag_on"]
    assert got == want and sizes == wsizes
    tag = enc.lametag_frame()
    assert tag == info["tag"]
    if info["tag_on"]:
        assert enc.music_crc() == info["music_crc"] and enc.bytes_written() == info["bytes_written"]
        assert M.get_vbr_tag(tag)["enc_padding"] == info["encoder_padding"]


def test_nothing_else_moved(M, oracle):
    """Native configurations give the same bytes with and without the flag; fractional ratios stay rejected with it; the
    unflagged size of a resampling configuration stays -1 after a resampled handle of it exists."""
    l, r = stereo("noise", 20000, 44100, 2)
    for cfg in [(2, 44100, 128), (1, 22050, 32), (2, 8000, 16), (1, 48000, 320)]:
        ch, sr, kb = cfg
        plain = M.encode_streams(ch, sr, kb, [l], [r] if ch == 2 else None)[0]
        assert M.encode_streams(ch, sr, kb, [l], [r] if ch == 2 else None, resample=True)[0] == plain
        assert handle_encode(M, cfg, l, r if ch == 2 else l, 1152)[0] == oracle.encode_stream(ch, sr, kb, l, r if ch == 2 else None, chunk=1152)[0]
    for ch, sr, kb in FRAC:
        with pytest.raises(M.Mp3B200Error):
            M.Mp3Encoder(ch, sr, kb, resample=True)
        assert M.stream_bytes(ch, sr, kb, 1000, resample=True) == -1
    keep = M.Mp3Encoder(2, 48000, 64, resample=True)
    assert M.stream_bytes(2, 48000, 64, 1000) == -1
    with pytest.raises(M.Mp3B200Error):
        M.Mp3Encoder(2, 48000, 64)
    keep.close()
