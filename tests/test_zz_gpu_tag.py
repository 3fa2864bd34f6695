"""SURVEY.md 8(f3) on the GPU: the music CRC kernel (k_music_crc) and the tag-writing entry points of the C-ABI against the
CPU oracle, which is pinned to lamejs for this row by tests/test_tag_oracle.py.  (File name: runs after the other GPU suites.)"""
import numpy as np
import pytest

from synth import make_signal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    assert torch.cuda.is_available()
    return torch


def test_crc_kernel_on_device_buffers(M, oracle, torch_cuda):
    """ragged ranges incl. empty, sub-lane, piece-boundary and multi-megabyte ones, at odd offsets"""
    torch = torch_cuda
    rng = np.random.default_rng(3)
    lens = [0, 1, 15, 16, 17, 511, 512, 513, 417, 418, 1440, 100003, 4180009, 33]
    offs, pos = [], 5
    for n in lens:
        offs.append(pos)
        pos += n + int(rng.integers(0, 7))
    host = rng.integers(0, 256, pos + 16).astype(np.uint8)
    dev = torch.from_numpy(host).cuda()
    got = M.debug_music_crc(dev.data_ptr(), offs, lens)
    want = [oracle.crc16(host[o:o + n].tobytes()) for o, n in zip(offs, lens)]
    assert got == want
    got2, ms = M.debug_music_crc(dev.data_ptr(), offs, lens, timed=True)
    assert got2 == want and ms > 0


@pytest.mark.parametrize("kind,ch,sr,kbps,frames,chunk", [
    ("noise", 2, 44100, 128, 40, 1152), ("burst", 2, 48000, 320, 30, 0), ("octave", 1, 32000, 64, 25, 777),
    ("noise", 2, 24000, 64, 50, 1152), ("noise", 1, 8000, 24, 40, 576), ("sweep", 2, 44100, 192, 450, 5000),
    # off the bitrate ladder: the tag's low-pass comes from the rate as given, the frames from the snapped one
    ("noise", 1, 44100, 72, 30, 1152), ("octave", 1, 32000, 52, 25, 777), ("noise", 2, 12000, 36, 40, 576),
    ("sweep", 2, 8000, 28, 40, 0), ("burst", 2, 44100, 104, 30, 5000)])
def test_tagged_handle_matches_oracle(M, oracle, kind, ch, sr, kbps, frames, chunk):
    fs = 1152 if sr >= 32000 else 576
    l, r = make_signal(kind, frames * fs + 77, sr, seed=9)
    r = r if ch == 2 else None
    ref, ref_sizes, info = oracle.encode_stream_tagged(ch, sr, kbps, l, r, chunk=chunk or None)
    assert info["tag_on"]
    enc = M.Mp3Encoder(ch, sr, kbps, write_vbr_tag=True)
    assert enc.tag_on
    out, sizes = bytearray(), []
    step = chunk or len(l)
    for i in range(0, len(l), step):
        b = enc.encodeBuffer(l[i:i + step], None if r is None else r[i:i + step])
        sizes.append(len(b))
        out += b
    assert enc.lametag_frame() != b"" or enc.bytes_written() == 0
    b = enc.flush()
    sizes.append(len(b))
    out += b
    assert bytes(out) == ref and sizes == ref_sizes
    assert enc.music_crc() == info["music_crc"] and enc.bytes_written() == info["bytes_written"]
    tag = enc.lametag_frame()
    assert tag == info["tag"]
    assert enc.flush() == b"" and enc.lametag_frame() == tag
    enc.close()
    # the finished file: the tag frame over the placeholder
    final = tag + bytes(out[len(tag):])
    assert final[len(tag):] == oracle.encode_stream(ch, sr, kbps, l, r, chunk=chunk or None)[0]


def test_tag_refused_and_tag_off(M, oracle):
    # 72- and 52-byte frames: InitVbrTag switches the tag off (at 12 kbps the snapped 8 kbps alone would make lamejs resample)
    for sr, kbps in ((8000, 8), (11025, 12)):
        l, _ = make_signal("noise", 20 * 576, sr, seed=4)
        enc = M.Mp3Encoder(1, sr, kbps, write_vbr_tag=True)
        assert not enc.tag_on
        got = enc.encodeBuffer(l) + enc.flush()
        assert got == oracle.encode_stream(1, sr, kbps, l, None)[0] and enc.lametag_frame() == b"" and enc.music_crc() == -1
        enc.close()
    e2 = M.Mp3Encoder(2, 44100, 128)                              # ordinary encoder: accumulators idle, nothing prefixed
    l, r = make_signal("noise", 5 * 1152, 44100, seed=5)
    assert e2.encodeBuffer(l, r) + e2.flush() == oracle.encode_stream(2, 44100, 128, l, r)[0]
    assert e2.lametag_frame() == b"" and e2.bytes_written() == -1
    L = M.lib()
    assert L.mp3b200_set_write_vbr_tag(e2._h, 1) < 0               # too late: samples were fed
    e2.close()


def test_tagged_and_plain_handles_in_one_batch(M, oracle):
    cfg = (2, 44100, 128)
    sigs = [make_signal("noise", 1152 * 6 + 10 * i, 44100, seed=20 + i) for i in range(4)]
    encs = [M.Mp3Encoder(*cfg, write_vbr_tag=(i % 2 == 0)) for i in range(4)]
    outs = [bytearray() for _ in encs]
    for lo in range(0, 1152 * 6, 1152 * 2):
        parts = M.encode_batch(encs, [s[0][lo:lo + 1152 * 2] for s in sigs], [s[1][lo:lo + 1152 * 2] for s in sigs])
        for o, p in zip(outs, parts):
            o += p
    parts = M.encode_batch(encs, [s[0][1152 * 6:] for s in sigs], [s[1][1152 * 6:] for s in sigs])
    for o, p in zip(outs, parts):
        o += p
    for o, p in zip(outs, M.flush_batch(encs)):
        o += p
    for i, (e, (l, r)) in enumerate(zip(encs, sigs)):
        if i % 2 == 0:
            ref, _, info = oracle.encode_stream_tagged(*cfg, l, r, chunk=1152 * 2)
            assert bytes(outs[i]) == ref and e.lametag_frame() == info["tag"] and e.music_crc() == info["music_crc"]
        else:
            assert bytes(outs[i]) == oracle.encode_stream(*cfg, l, r, chunk=1152 * 2)[0] and e.lametag_frame() == b""
        e.close()


def test_encode_streams_tagged(M, oracle):
    """whole-file batch: out[s] = finished tag frame ++ audio; one CRC launch for all streams"""
    for ch, sr, kbps in [(2, 44100, 128), (1, 48000, 96), (2, 22050, 64)]:
        fs = 1152 if sr >= 32000 else 576
        lens = [0, 1, 700, fs * 7, fs * 31 + 5, fs * 64, fs * 401]
        sigs = [make_signal("noise", n, sr, seed=30 + i) for i, n in enumerate(lens)]
        got = M.encode_streams_tagged(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None)
        plain = M.encode_streams(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None)
        for (l, r), g, p in zip(sigs, got, plain):
            ref, _, info = oracle.encode_stream_tagged(ch, sr, kbps, l, r if ch == 2 else None)
            tag = info["tag"]
            assert g == tag + ref[len(tag):] and g[len(tag):] == p
    # a configuration without room for the tag: the plain streams
    l, _ = make_signal("noise", 30 * 576, 16000, seed=1)
    assert M.encode_streams_tagged(1, 16000, 32, [l]) == M.encode_streams(1, 16000, 32, [l])


def test_c2_stream_crc_and_tag(M, oracle):
    """BASELINE config #2 (10 001 frames): CRC field of the tag == serial CRC of the 4.18 MB the GPU produced"""
    l, r = make_signal("sweep", 10000 * 1152, 44100, seed=0)
    g = M.encode_streams_tagged(2, 44100, 128, [l], [r])[0]
    tag, audio = g[:417], g[417:]
    assert len(audio) == M.stream_bytes(2, 44100, 128, len(l))
    x = 36
    assert tag[x:x + 4] == b"Info" and int.from_bytes(tag[x + 8:x + 12], "big") == 10001 and int.from_bytes(tag[x + 12:x + 16], "big") == len(g)
    assert int.from_bytes(tag[x + 152:x + 154], "big") == oracle.crc16(audio)
    assert int.from_bytes(tag[x + 154:x + 156], "big") == oracle.crc16(tag[:x + 154])
    assert tag == M.lametag_build(2, 44100, 128, 10001, len(audio), oracle.crc16(audio), int.from_bytes(tag[x + 142:x + 144], "big") & 0xFFF)


def test_put_vbr_tag_in_memory(M, oracle):
    """putVbrTag: the finished frame lands over the placeholder -- at offset 0, or behind an ID3v2 tag"""
    l, r = make_signal("octave", 20 * 1152, 48000, seed=12)
    for head in (b"", M.id3v2_tag(flags=M.ID3_ADD_V2, title="put", artist="vbr", num_samples=len(l), samplerate=48000)):
        enc = M.Mp3Encoder(2, 48000, 160, write_vbr_tag=True)
        stream = bytearray(head + enc.encodeBuffer(l, r) + enc.flush())
        tag = enc.lametag_frame()
        assert enc.put_vbr_tag(stream) == 0
        assert bytes(stream[:len(head)]) == head and bytes(stream[len(head):len(head) + len(tag)]) == tag
        d = M.get_vbr_tag(stream[len(head):len(head) + len(tag)])
        assert d["frames"] == M.stream_frames(len(l), 2, 48000, 160) and d["bytes"] == len(stream) - len(head)
        assert bytes(stream[len(head) + len(tag):]) == oracle.encode_stream(2, 48000, 160, l, r)[0]
        enc.close()
    e = M.Mp3Encoder(2, 48000, 160, write_vbr_tag=True)
    assert e.put_vbr_tag(bytearray(1000)) == -1          # nothing encoded yet
    e.close()
