import ctypes
import os

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


class Mp3B200Error(RuntimeError):
    pass


class DebugTaps(ctypes.Structure):
    """mp3b200_debug_taps (include/mp3b200.h)"""
    _vp = ctypes.c_void_p
    _fields_ = [("size", ctypes.c_int32), ("channels", ctypes.c_int32), ("samplerate", ctypes.c_int32), ("kbps", ctypes.c_int32),
                ("left", _vp), ("right", _vp), ("nsamples", ctypes.c_int64), ("force_blocktype", _vp),
                ("xr", _vp), ("blocktype", _vp), ("en_l", _vp), ("thm_l", _vp), ("en_s", _vp), ("thm_s", _vp), ("ath_adjust", _vp),
                ("l3_enc", _vp), ("ginfo", _vp), ("bytes_out", _vp), ("bytes_cap", ctypes.c_int64),
                ("scalefac", _vp), ("subblock_gain", _vp), ("xmin", _vp), ("max_nonzero_coeff", _vp), ("xrpow_max", _vp),
                ("scfsi", _vp), ("old_value", _vp), ("cur_step", _vp)]


def lib():
    """Load (building if needed) libmp3b200.so and declare the C-ABI of include/mp3b200.h."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("MP3B200_LIB")          # tuning experiments: a variant built by tools/build_variants.py
    if not path:
        path = _build.LIB
        if not os.path.exists(path):
            _build.build()
    L = ctypes.CDLL(path)
    c_int, c_i64, vp = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    L.mp3b200_last_error.restype = ctypes.c_char_p
    L.mp3b200_launch_count.restype = c_i64
    L.mp3b200_set_device.argtypes = [c_int]
    L.mp3b200_create.argtypes = [c_int, c_int, c_int, ctypes.POINTER(vp)]
    L.mp3b200_encode.argtypes = [vp, vp, vp, c_int, vp, c_int]
    L.mp3b200_flush.argtypes = [vp, vp, c_int]
    L.mp3b200_destroy.argtypes = [vp]
    L.mp3b200_encode_batch.argtypes = [vp, vp, vp, vp, vp, vp, c_int, vp]
    L.mp3b200_flush_batch.argtypes = [vp, vp, vp, c_int, vp]
    L.mp3b200_destroy.restype = None
    L.mp3b200_export_state.argtypes = [vp, vp, c_int]
    L.mp3b200_import_state.argtypes = [vp, vp, c_int]
    L.mp3b200_seek.argtypes = [vp, c_i64, vp, vp, c_int]
    L.mp3b200_stream_bytes.restype = c_i64
    L.mp3b200_stream_bytes.argtypes = [c_int, c_int, c_int, c_i64]
    L.mp3b200_stream_frames.restype = c_i64
    L.mp3b200_stream_frames.argtypes = [c_i64]
    L.mp3b200_stream_frames_cfg.restype = c_i64
    L.mp3b200_stream_frames_cfg.argtypes = [c_int, c_int, c_int, c_i64]
    L.mp3b200_granules_per_frame.argtypes = [c_int, c_int, c_int]
    L.mp3b200_encode_streams.argtypes = [c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_device.argtypes = [c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_set_write_vbr_tag.argtypes = [vp, c_int]
    L.mp3b200_get_lametag_frame.argtypes = [vp, vp, c_int]
    L.mp3b200_music_crc.argtypes = [vp]
    L.mp3b200_bytes_written.argtypes = [vp]
    L.mp3b200_bytes_written.restype = c_i64
    L.mp3b200_lametag_size.argtypes = [c_int, c_int, c_int]
    L.mp3b200_lametag_build.argtypes = [c_int, c_int, c_int, c_i64, c_i64, c_int, c_int, vp, c_int]
    L.mp3b200_encode_streams_tagged.argtypes = [c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_wav_read_header.argtypes = [vp, c_i64, vp]
    L.mp3b200_debug_music_crc.argtypes = [vp, vp, vp, c_int, vp, vp]
    L.mp3b200_debug_stages.argtypes = [c_int, c_int, c_int, vp, vp, c_i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, c_i64]
    L.mp3b200_debug_stages_ex.argtypes = [ctypes.POINTER(DebugTaps)]
    _lib = L
    return L


def _check(rc):
    if rc < 0:
        raise Mp3B200Error("libmp3b200 error %d: %s" % (rc, lib().mp3b200_last_error().decode()))
    return rc


def stream_frames(nsamples, channels=None, samplerate=None, kbps=None):
    """Frames encodeBuffer(nsamples) + flush() produce.  Without a configuration: MPEG-1 (1152-sample frames)."""
    if samplerate is None:
        return int(lib().mp3b200_stream_frames(int(nsamples)))
    return int(lib().mp3b200_stream_frames_cfg(channels, samplerate, kbps, int(nsamples)))


def granules_per_frame(channels, samplerate, kbps):
    """2 for MPEG-1 (32/44.1/48 kHz), 1 for MPEG-2 / 2.5 (8..24 kHz); -1 for configurations the library rejects."""
    return int(lib().mp3b200_granules_per_frame(channels, samplerate, kbps))


def stream_bytes(channels, samplerate, kbps, nsamples):
    return int(lib().mp3b200_stream_bytes(channels, samplerate, kbps, int(nsamples)))


class WavHeader:
    """lamejs.WavHeader (src/js/index.js:138-193): dataOffset, dataLen, channels, sampleRate."""

    def __init__(self):
        self.dataOffset = self.dataLen = self.channels = self.sampleRate = 0

    class _C(ctypes.Structure):
        _fields_ = [("data_offset", ctypes.c_int64), ("data_len", ctypes.c_int64), ("channels", ctypes.c_int32), ("sample_rate", ctypes.c_uint32)]

    @staticmethod
    def readHeader(data):
        """WavHeader.readHeader(dataView): a WavHeader, None where the reference returns undefined; raises ValueError where it
        throws 'extended fmt chunk not implemented', IndexError where its DataView read leaves the buffer (RangeError)."""
        a = np.frombuffer(bytes(data), dtype=np.uint8)
        c = WavHeader._C()
        rc = lib().mp3b200_wav_read_header(a.ctypes.data if len(a) else None, len(a), ctypes.byref(c))
        if rc == 0:
            return None
        if rc == -1:
            raise ValueError("extended fmt chunk not implemented")
        if rc != 1:
            raise IndexError("read past the end of the buffer")
        w = WavHeader()
        w.dataOffset, w.dataLen, w.channels, w.sampleRate = c.data_offset, c.data_len, c.channels, c.sample_rate
        return w


class _Id3C(ctypes.Structure):
    _fields_ = [(k, ctypes.c_char_p) for k in ("title", "artist", "album", "year", "comment", "track", "genre")] + \
               [("flags", ctypes.c_int), ("padding", ctypes.c_int), ("num_samples", ctypes.c_int64), ("samplerate", ctypes.c_int)]


ID3_ADD_V2, ID3_V1_ONLY, ID3_V2_ONLY, ID3_SPACE_V1, ID3_PAD_V2 = 2, 4, 8, 16, 32


def _id3_struct(fields, flags, padding, num_samples, samplerate):
    c = _Id3C()
    for k in ("title", "artist", "album", "year", "comment", "track", "genre"):
        v = fields.get(k)
        setattr(c, k, None if v is None else str(v).encode("latin-1"))
    c.flags, c.padding, c.num_samples, c.samplerate = flags, padding, num_samples, samplerate
    return c


def id3v2_tag(flags=0, padding=0, num_samples=-1, samplerate=0, **fields):
    """ID3v2.3 tag (ID3Tag.java lame_get_id3v2_tag): title / artist / album / year / comment / track / genre as Latin-1 text;
    b'' when the reference would write none."""
    L = lib()
    L.mp3b200_id3v2_tag.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    c = _id3_struct(fields, flags, padding, num_samples, samplerate)
    n = _check(L.mp3b200_id3v2_tag(ctypes.byref(c), None, 0))
    buf = np.zeros(max(n, 1), dtype=np.uint8)
    n = _check(L.mp3b200_id3v2_tag(ctypes.byref(c), buf.ctypes.data, n))
    return buf[:n].tobytes()


def id3v1_tag(flags=0, **fields):
    """ID3v1 / v1.1 tag (ID3Tag.java lame_get_id3v1_tag): 128 bytes, or b'' when nothing is set."""
    L = lib()
    L.mp3b200_id3v1_tag.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    c = _id3_struct(fields, flags, 0, -1, 0)
    buf = np.zeros(128, dtype=np.uint8)
    n = _check(L.mp3b200_id3v1_tag(ctypes.byref(c), buf.ctypes.data, 128))
    return buf[:n].tobytes()


class _VbrTagC(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ("h_id", "samprate", "flags", "frames", "bytes", "vbr_scale", "headersize", "enc_delay", "enc_padding")] + \
               [("toc", ctypes.c_uint8 * 100)]


def get_vbr_tag(frame):
    """VBRTag.getVbrTag: dict of the Xing / Info tag fields in the first frame of a stream, or None when there is no tag."""
    a = np.frombuffer(bytes(frame), dtype=np.uint8)
    c = _VbrTagC()
    L = lib()
    L.mp3b200_get_vbr_tag.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    rc = L.mp3b200_get_vbr_tag(a.ctypes.data if len(a) else None, len(a), ctypes.byref(c))
    if rc == 0:
        return None
    if rc != 1:
        raise IndexError("frame too short")
    d = {k: int(getattr(c, k)) for k, _ in _VbrTagC._fields_[:-1]}
    d["toc"] = bytes(c.toc)
    return d


def crc16_combine(crc_a, crc_b, len_b):
    """CRC-16 of A || B from crc(A), crc(B), len(B) (VBRTag.js:547-556 is linear over GF(2))."""
    L = lib()
    L.mp3b200_crc16_combine.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64]
    return _check(L.mp3b200_crc16_combine(int(crc_a), int(crc_b), int(len_b)))


def lametag_size(channels, samplerate, kbps):
    """Size of the Xing / Info / LAME tag frame of a configuration (0: InitVbrTag would switch the tag off)."""
    return _check(lib().mp3b200_lametag_size(channels, samplerate, kbps))


def lametag_build(channels, samplerate, kbps, nframes, music_bytes, music_crc, encoder_padding):
    """The tag frame from numbers (no device needed): VBRTag.getLameTagFrame for a CBR stream of `nframes` frames."""
    buf = np.zeros(2880, dtype=np.uint8)
    n = _check(lib().mp3b200_lametag_build(channels, samplerate, kbps, int(nframes), int(music_bytes), int(music_crc), int(encoder_padding),
                                           buf.ctypes.data, 2880))
    return buf[:n].tobytes()


class Mp3Encoder:
    """Drop-in for lamejs.Mp3Encoder(channels, samplerate, kbps) (src/js/index.js:66-136).  `write_vbr_tag=True` is
    gfp.bWriteVbrTag (index.js:107 sets it false): the stream then starts with a placeholder frame, and `lametag_frame()`
    after flush() returns the finished Info / LAME tag frame to write over it."""

    def __init__(self, channels=1, samplerate=44100, kbps=128, write_vbr_tag=False):
        self._L = lib()
        self._h = ctypes.c_void_p()
        self.channels = channels
        rc = self._L.mp3b200_create(channels, samplerate, kbps, ctypes.byref(self._h))
        _check(rc)
        self.tag_on = bool(write_vbr_tag) and _check(self._L.mp3b200_set_write_vbr_tag(self._h, 1)) == 1
        self._tag_room = lametag_size(channels, samplerate, kbps) if self.tag_on else 0

    def lametag_frame(self):
        buf = np.zeros(2880, dtype=np.uint8)
        n = _check(self._L.mp3b200_get_lametag_frame(self._h, buf.ctypes.data, 2880))
        return buf[:n].tobytes()

    def music_crc(self):
        return int(self._L.mp3b200_music_crc(self._h))

    def put_vbr_tag(self, stream):
        """VBRTag.putVbrTag on a stream held in a bytearray / writable uint8 array: the finished frame over the placeholder
        (behind an ID3v2 tag if the stream starts with one).  Returns 0, or -1 like the reference."""
        a = np.frombuffer(stream, dtype=np.uint8)
        self._L.mp3b200_put_vbr_tag.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
        return int(self._L.mp3b200_put_vbr_tag(self._h, a.ctypes.data if len(a) else None, len(a)))

    def bytes_written(self):
        return int(self._L.mp3b200_bytes_written(self._h))

    def encodeBuffer(self, left, right=None):
        left = np.ascontiguousarray(left, dtype=np.int16)
        if self.channels == 1 or right is None:
            right = left
        right = np.ascontiguousarray(right, dtype=np.int16)
        assert len(left) == len(right)
        cap = int(1.25 * len(left) + 7200) + self._tag_room     # index.js:114,124
        buf = np.empty(cap, dtype=np.uint8)
        n = _check(self._L.mp3b200_encode(self._h, left.ctypes.data, right.ctypes.data, len(left), buf.ctypes.data, cap))
        return buf[:n].tobytes()

    def flush(self):
        cap = 7200 + 8 * 1441 + self._tag_room
        buf = np.empty(cap, dtype=np.uint8)
        n = _check(self._L.mp3b200_flush(self._h, buf.ctypes.data, cap))
        return buf[:n].tobytes()

    # pythonic aliases
    encode_buffer = encodeBuffer

    # ---- state: checkpoint / resume and segment encoding (include/mp3b200.h "encoder state") ----
    def export_state(self):
        n = _check(self._L.mp3b200_export_state(self._h, None, 0))
        buf = np.empty(n, dtype=np.uint8)
        n = _check(self._L.mp3b200_export_state(self._h, buf.ctypes.data, n))
        return buf[:n].tobytes()

    def import_state(self, blob):
        buf = np.frombuffer(blob, dtype=np.uint8)
        _check(self._L.mp3b200_import_state(self._h, buf.ctypes.data, len(buf)))

    def seek(self, frame, left_hist, right_hist=None):
        """fresh encoder -> frame `frame` of a stream with start-of-stream sequential state; *_hist = samples
        [max(0, frame*framesize-1104), frame*framesize+224)"""
        left_hist = np.ascontiguousarray(left_hist, dtype=np.int16)
        right_hist = left_hist if (self.channels == 1 or right_hist is None) else np.ascontiguousarray(right_hist, dtype=np.int16)
        _check(self._L.mp3b200_seek(self._h, int(frame), left_hist.ctypes.data, right_hist.ctypes.data, len(left_hist)))

    def close(self):
        if self._h:
            self._L.mp3b200_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def encode_batch(encoders, lefts, rights=None):
    """encodeBuffer on many live Mp3Encoder objects of one configuration in ONE pipeline launch (SURVEY 8(b) batch row):
    returns [enc.encodeBuffer(l, r) for ...] byte strings."""
    L = lib()
    S = len(encoders)
    lefts = [np.ascontiguousarray(x, dtype=np.int16) for x in lefts]
    rights = lefts if rights is None else [np.ascontiguousarray(x if x is not None else l, dtype=np.int16) for x, l in zip(rights, lefts)]
    ns = np.array([len(x) for x in lefts], dtype=np.int32)
    caps = np.array([int(1.25 * n + 7200) for n in ns], dtype=np.int32)
    outs = [np.empty(int(c), dtype=np.uint8) for c in caps]
    hp = (ctypes.c_void_p * S)(*[e._h for e in encoders])
    lp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in lefts])
    rp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in rights])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    got = np.zeros(S, dtype=np.int32)
    _check(L.mp3b200_encode_batch(hp, lp, rp, ns.ctypes.data, op, caps.ctypes.data, S, got.ctypes.data))
    for g in got:
        _check(int(g))
    return [o[: int(g)].tobytes() for o, g in zip(outs, got)]


def flush_batch(encoders):
    """flush() on many live Mp3Encoder objects in one pipeline launch."""
    L = lib()
    S = len(encoders)
    cap = 7200 + 8 * 1441
    outs = [np.empty(cap, dtype=np.uint8) for _ in range(S)]
    hp = (ctypes.c_void_p * S)(*[e._h for e in encoders])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    caps = np.full(S, cap, dtype=np.int32)
    got = np.zeros(S, dtype=np.int32)
    _check(L.mp3b200_flush_batch(hp, op, caps.ctypes.data, S, got.ctypes.data))
    for g in got:
        _check(int(g))
    return [o[: int(g)].tobytes() for o, g in zip(outs, got)]


def encode_streams(channels, samplerate, kbps, lefts, rights=None):
    """Batch extension: encodeBuffer(whole stream) + flush() for many independent streams in one launch sequence.
    Host buffers in, list of bytes out."""
    L = lib()
    S = len(lefts)
    if S == 0:
        return []
    lefts = [np.ascontiguousarray(x, dtype=np.int16) for x in lefts]
    rights = lefts if (rights is None or channels == 1) else [np.ascontiguousarray(x, dtype=np.int16) for x in rights]
    ns = np.array([len(x) for x in lefts], dtype=np.int64)
    nb = [stream_bytes(channels, samplerate, kbps, int(n)) for n in ns]
    if any(b < 0 for b in nb):
        raise Mp3B200Error("unsupported configuration: channels=%d samplerate=%d kbps=%d (lame_init_params would resample)" % (channels, samplerate, kbps))
    outs = [np.empty(b, dtype=np.uint8) for b in nb]
    lp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in lefts])
    rp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in rights])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    caps = np.array(nb, dtype=np.int64)
    got = np.zeros(S, dtype=np.int64)
    _check(L.mp3b200_encode_streams(channels, samplerate, kbps, S, lp, rp, ns.ctypes.data, op, caps.ctypes.data, got.ctypes.data))
    return [o[: int(g)].tobytes() for o, g in zip(outs, got)]


def encode_streams_tagged(channels, samplerate, kbps, lefts, rights=None):
    """encode_streams with gfp.bWriteVbrTag on: every returned stream starts with its finished Info / LAME tag frame (frame
    and byte counts, seek table, encoder delay / padding, CRC-16 of the audio bytes computed on the GPU)."""
    L = lib()
    S = len(lefts)
    if S == 0:
        return []
    lefts = [np.ascontiguousarray(x, dtype=np.int16) for x in lefts]
    rights = lefts if (rights is None or channels == 1) else [np.ascontiguousarray(x, dtype=np.int16) for x in rights]
    ns = np.array([len(x) for x in lefts], dtype=np.int64)
    room = lametag_size(channels, samplerate, kbps)
    nb = [stream_bytes(channels, samplerate, kbps, int(n)) + room for n in ns]
    outs = [np.empty(b, dtype=np.uint8) for b in nb]
    lp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in lefts])
    rp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in rights])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    caps = np.array(nb, dtype=np.int64)
    got = np.zeros(S, dtype=np.int64)
    _check(L.mp3b200_encode_streams_tagged(channels, samplerate, kbps, S, lp, rp, ns.ctypes.data, op, caps.ctypes.data, got.ctypes.data))
    return [o[: int(g)].tobytes() for o, g in zip(outs, got)]


def debug_music_crc(d_buf_ptr, offsets, lengths, timed=False):
    """k_music_crc on byte ranges of a device buffer (raw pointer as int): list of CRC-16 values (+ ms if `timed`)."""
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    ln = np.ascontiguousarray(lengths, dtype=np.int64)
    crc = np.zeros(len(off), dtype=np.uint32)
    ms = ctypes.c_float(0)
    _check(lib().mp3b200_debug_music_crc(d_buf_ptr, off.ctypes.data, ln.ctypes.data, len(off), crc.ctypes.data, ctypes.byref(ms) if timed else None))
    return ([int(c) for c in crc], float(ms.value)) if timed else [int(c) for c in crc]


def encode_streams_device(channels, samplerate, kbps, d_pcm_ptr, pcm_off, nsamples, d_out_ptr, out_off):
    """Device-resident batch (raw device pointers as ints).  Returns the 16 timing slots of include/mp3b200.h (ms)."""
    L = lib()
    pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
    nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
    out_off = np.ascontiguousarray(out_off, dtype=np.int64)
    tm = np.zeros(16, dtype=np.float32)
    _check(L.mp3b200_encode_streams_device(channels, samplerate, kbps, len(nsamples), d_pcm_ptr, pcm_off.ctypes.data,
                                           nsamples.ctypes.data, d_out_ptr, out_off.ctypes.data, tm.ctypes.data))
    return tm


def debug_stages(channels, samplerate, kbps, left, right=None, force_blocktype=None, want=("xr",)):
    """Stage taps for parity tests: returns a dict of numpy arrays (see include/mp3b200.h).  `want` names any of xr,
    blocktype, en_l, thm_l, en_s, thm_s, ath_adjust, l3_enc, ginfo, bytes, scalefac, subblock_gain, xmin, max_nonzero_coeff,
    xrpow_max, scfsi, old_value and cur_step (the last two [F][3][nch]: frame start, after gr0, frame end)."""
    L = lib()
    left = np.ascontiguousarray(left, dtype=np.int16)
    right = left if (right is None or channels == 1) else np.ascontiguousarray(right, dtype=np.int16)
    n = len(left)
    F = stream_frames(n, channels, samplerate, kbps)
    G = granules_per_frame(channels, samplerate, kbps)
    if F < 0 or G < 0:
        raise Mp3B200Error("unsupported configuration: channels=%d samplerate=%d kbps=%d" % (channels, samplerate, kbps))
    nch = channels
    res = {}

    def alloc(name, shape, dt):
        if name in want:
            res[name] = np.zeros(shape, dtype=dt)
            return res[name].ctypes.data
        return None

    fb = None
    if force_blocktype is not None:
        fb = np.ascontiguousarray(force_blocktype, dtype=np.int32)
        assert fb.shape == (F, G, nch)
    p_xr = alloc("xr", (F, G, nch, 576), np.float32)
    p_bt = alloc("blocktype", (F, G, nch), np.int32)
    p_enl = alloc("en_l", (F, G, nch, 22), np.float32)
    p_thl = alloc("thm_l", (F, G, nch, 22), np.float32)
    p_ens = alloc("en_s", (F, G, nch, 13, 3), np.float32)
    p_ths = alloc("thm_s", (F, G, nch, 13, 3), np.float32)
    p_ath = alloc("ath_adjust", (F,), np.float64)
    p_l3 = alloc("l3_enc", (F, G, nch, 576), np.int32)
    p_gi = alloc("ginfo", (F, G, nch, 16), np.int32)
    nb = stream_bytes(channels, samplerate, kbps, n)
    if nb < 0:
        raise Mp3B200Error("unsupported configuration: channels=%d samplerate=%d kbps=%d" % (channels, samplerate, kbps))
    p_by = alloc("bytes", (nb,), np.uint8)
    t = DebugTaps(size=ctypes.sizeof(DebugTaps), channels=channels, samplerate=samplerate, kbps=kbps, left=left.ctypes.data,
                  right=right.ctypes.data, nsamples=n, force_blocktype=fb.ctypes.data if fb is not None else None,
                  xr=p_xr, blocktype=p_bt, en_l=p_enl, thm_l=p_thl, en_s=p_ens, thm_s=p_ths, ath_adjust=p_ath,
                  l3_enc=p_l3, ginfo=p_gi, bytes_out=p_by, bytes_cap=nb,
                  scalefac=alloc("scalefac", (F, G, nch, 39), np.int32), subblock_gain=alloc("subblock_gain", (F, G, nch, 3), np.int32),
                  xmin=alloc("xmin", (F, G, nch, 39), np.float32), max_nonzero_coeff=alloc("max_nonzero_coeff", (F, G, nch), np.int32),
                  xrpow_max=alloc("xrpow_max", (F, G, nch), np.float64), scfsi=alloc("scfsi", (F, nch, 4), np.int32),
                  old_value=alloc("old_value", (F, 3, nch), np.int32), cur_step=alloc("cur_step", (F, 3, nch), np.int32))
    _check(L.mp3b200_debug_stages_ex(ctypes.byref(t)))
    return res
