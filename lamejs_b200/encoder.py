import contextlib
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
                ("scfsi", _vp), ("old_value", _vp), ("cur_step", _vp), ("flags", ctypes.c_int32)]


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
    L.mp3b200_stream_frames_ex.restype = c_i64
    L.mp3b200_stream_frames_ex.argtypes = [c_int, c_int, c_int, c_int, c_i64]
    L.mp3b200_granules_per_frame_ex.argtypes = [c_int, c_int, c_int, c_int]
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
    L.mp3b200_encode_streams_tagged_ex.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_lametag_build_ex.argtypes = [c_int, c_int, c_int, c_int, c_i64, c_i64, c_int, c_int, c_int, vp, c_int]
    L.mp3b200_set_find_replay_gain.argtypes = [vp, c_int]
    L.mp3b200_get_replay_gain.argtypes = [vp, vp, vp]
    L.mp3b200_album_gain.argtypes = [vp, c_int, vp]
    L.mp3b200_debug_replaygain.argtypes = [c_int, c_int, c_int, c_int, vp, vp, c_i64, vp, vp, c_i64, vp, vp, vp]
    L.mp3b200_wav_read_header.argtypes = [vp, c_i64, vp]
    L.mp3b200_debug_music_crc.argtypes = [vp, vp, vp, c_int, vp, vp]
    L.mp3b200_debug_stages.argtypes = [c_int, c_int, c_int, vp, vp, c_i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, c_i64]
    L.mp3b200_debug_stages_ex.argtypes = [ctypes.POINTER(DebugTaps)]
    L.mp3b200_create_ex.argtypes = [c_int, c_int, c_int, c_int, ctypes.POINTER(vp)]
    L.mp3b200_out_samplerate.argtypes = [c_int, c_int, c_int]
    L.mp3b200_stream_bytes_ex.restype = c_i64
    L.mp3b200_stream_bytes_ex.argtypes = [c_int, c_int, c_int, c_int, c_i64]
    L.mp3b200_encode_streams_ex.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_device_ex.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_lametag_size_ex.argtypes = [c_int, c_int, c_int, c_int]
    L.mp3b200_debug_resample.argtypes = [c_int, c_int, c_int, vp, vp, c_i64, vp, c_i64]
    L.mp3b200_encode_f32.argtypes = [vp, vp, vp, c_int, vp, c_int]
    L.mp3b200_encode_batch_f32.argtypes = [vp, vp, vp, vp, vp, vp, c_int, vp]
    L.mp3b200_seek_f32.argtypes = [vp, c_i64, vp, vp, c_int]
    L.mp3b200_encode_streams_f32.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_tagged_f32.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_device_f32.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_tagged_device.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_tagged_device_f32.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_debug_stages_f32.argtypes = [ctypes.POINTER(DebugTaps), vp, vp]
    L.mp3b200_debug_resample_f32.argtypes = [c_int, c_int, c_int, vp, vp, c_i64, vp, c_i64]
    L.mp3b200_debug_replaygain_f32.argtypes = [c_int, c_int, c_int, c_int, vp, vp, c_i64, vp, vp, c_i64, vp, vp, vp]
    L.mp3b200_encode_device.argtypes = [vp, vp, vp, c_int, vp, c_int]
    L.mp3b200_encode_device_f32.argtypes = [vp, vp, vp, c_int, vp, c_int]
    L.mp3b200_encode_batch_device.argtypes = [vp, vp, vp, vp, vp, vp, c_int, vp]
    L.mp3b200_encode_batch_device_f32.argtypes = [vp, vp, vp, vp, vp, vp, c_int, vp]
    L.mp3b200_encoder_device.argtypes = [vp]
    L.mp3b200_session_create.argtypes = [vp, ctypes.POINTER(vp)]
    L.mp3b200_session_destroy.argtypes = [vp]
    L.mp3b200_encode_streams_async.argtypes = [vp, c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_async_f32.argtypes = [vp, c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_check_status.argtypes = [vp]
    L.mp3b200_encode_streams_tagged_async.argtypes = [vp, c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_streams_tagged_async_f32.argtypes = [vp, c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_session_encode_batch.argtypes = [vp, vp, vp, vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_encode_batch_f32.argtypes = [vp, vp, vp, vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_flush_batch.argtypes = [vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_encode_bytes.argtypes = [vp, c_int]
    L.mp3b200_session_release.argtypes = [vp, vp, c_int]
    L.mp3b200_session_tail_capacity.argtypes = [c_int, c_int, c_int, c_int]
    L.mp3b200_session_encode_batch_tagged.argtypes = [vp, vp, vp, vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_encode_batch_tagged_f32.argtypes = [vp, vp, vp, vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_flush_batch_tagged.argtypes = [vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_lametag_frames.argtypes = [vp, vp, c_int, vp, vp, vp, vp]
    L.mp3b200_session_album_gain.argtypes = [vp, vp, c_int, vp, vp]
    L.mp3b200_session_graph_instantiations.argtypes = [vp]
    L.mp3b200_encode_bytes_schedule.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, c_int, vp]
    L.mp3b200_session_graph_instantiations.restype = c_i64
    for name in ("mp3b200_replaygain_streams", "mp3b200_replaygain_streams_f32", "mp3b200_replaygain_streams_device",
                 "mp3b200_replaygain_streams_device_f32"):
        getattr(L, name).argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp]
    L.mp3b200_finish_tags_device.argtypes = [c_int, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp]
    L.mp3b200_session_tail_capacity.restype = c_i64
    L.mp3b200_wav_plan.argtypes = [c_int, c_int, c_int, vp, vp, vp]
    L.mp3b200_encode_wav.argtypes = [c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]
    L.mp3b200_encode_wav_tagged.argtypes = [c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mp3b200_debug_stage_wav.argtypes = [c_int, c_int, c_int, vp, vp, vp, c_i64, vp]
    _lib = L
    return L


def _rows(lefts, rights=None):
    """One call's sample rows as the C entry points take them: (lefts, rights, f32).  When any row holds floating-point
    values all become Float32, rounded once from the caller's values (Math.fround), for the _f32 entry points, which take
    them as lamejs's Float32Array store does; otherwise contiguous Int16.  A missing right row (rights None, or an entry
    None) is its left row."""
    rights = [None] * len(lefts) if rights is None else list(rights)
    f32 = any(a is not None and np.asarray(a).dtype.kind in "fc" for a in (*lefts, *rights))
    dt = np.float32 if f32 else np.int16
    lefts = [np.ascontiguousarray(x, dtype=dt) for x in lefts]
    return lefts, [l if r is None else np.ascontiguousarray(r, dtype=dt) for l, r in zip(lefts, rights)], f32


def _on_cuda(x):
    """True for a torch tensor in CUDA memory"""
    return bool(getattr(x, "is_cuda", False))


def _device_rows(lefts, rights, device):
    """_rows for CUDA tensors: contiguous Float32 (floating dtypes, rounded once) or Int16 tensors on `device`, the encoders'
    CUDA device index.  Raises ValueError for a row in host memory or on another device.  Makes torch's default stream wait
    for the current one, as the library's calls wait for the default stream: rows produced on a side stream are ordered."""
    import torch
    rights = [None] * len(lefts) if rights is None else list(rights)
    rows = [x for x in (*lefts, *rights) if x is not None]
    if not all(_on_cuda(x) for x in rows):
        raise ValueError("one call takes rows either all in host memory or all in CUDA memory")
    if any(x.device.index != device for x in rows):
        raise ValueError("CUDA rows must be on the encoders' device (cuda:%d)" % device)
    f32 = any(x.dtype.is_floating_point or x.dtype.is_complex for x in rows)
    dt = torch.float32 if f32 else torch.int16
    lefts = [x.to(dt).contiguous() for x in lefts]
    rights = [l if r is None else r.to(dt).contiguous() for l, r in zip(lefts, rights)]
    torch.cuda.default_stream(device).wait_stream(torch.cuda.current_stream(device))
    return lefts, rights, f32


# each Int16 entry point and its Float32 twin, which takes the same arguments with Float32 rows
_F32_TWIN = {
    "mp3b200_encode": "mp3b200_encode_f32",
    "mp3b200_encode_batch": "mp3b200_encode_batch_f32",
    "mp3b200_encode_device": "mp3b200_encode_device_f32",
    "mp3b200_encode_batch_device": "mp3b200_encode_batch_device_f32",
    "mp3b200_seek": "mp3b200_seek_f32",
    "mp3b200_encode_streams_ex": "mp3b200_encode_streams_f32",
    "mp3b200_encode_streams_tagged_ex": "mp3b200_encode_streams_tagged_f32",
    "mp3b200_encode_streams_device_ex": "mp3b200_encode_streams_device_f32",
    "mp3b200_encode_streams_tagged_device": "mp3b200_encode_streams_tagged_device_f32",
    "mp3b200_encode_streams_tagged_async": "mp3b200_encode_streams_tagged_async_f32",
    "mp3b200_session_encode_batch": "mp3b200_session_encode_batch_f32",
    "mp3b200_session_encode_batch_tagged": "mp3b200_session_encode_batch_tagged_f32",
    "mp3b200_debug_resample": "mp3b200_debug_resample_f32",
    "mp3b200_debug_replaygain": "mp3b200_debug_replaygain_f32",
    "mp3b200_replaygain_streams": "mp3b200_replaygain_streams_f32",
    "mp3b200_replaygain_streams_device": "mp3b200_replaygain_streams_device_f32",
}


def _entry(name, f32):
    """the entry point `name`, or its Float32 twin"""
    return getattr(lib(), _F32_TWIN[name] if f32 else name)


def _check(rc):
    if rc < 0:
        raise Mp3B200Error("libmp3b200 error %d: %s" % (rc, lib().mp3b200_last_error().decode()))
    return rc


RESAMPLE = 1     # MP3B200_RESAMPLE
REPLAYGAIN = 2   # MP3B200_REPLAYGAIN


def stream_frames(nsamples, channels=None, samplerate=None, kbps=None, resample=False):
    """Frames encodeBuffer(nsamples) + flush() produce, -1 for a rejected configuration.  Without a configuration: MPEG-1
    (1152-sample frames).  resample=True: see stream_bytes."""
    if samplerate is None:
        return int(lib().mp3b200_stream_frames(int(nsamples)))
    return int(lib().mp3b200_stream_frames_ex(channels, samplerate, kbps, RESAMPLE if resample else 0, int(nsamples)))


def granules_per_frame(channels, samplerate, kbps, resample=False):
    """2 for MPEG-1 (32/44.1/48 kHz), 1 for MPEG-2 / 2.5 (8..24 kHz); -1 for configurations the library rejects.  With
    resample=True a configuration lamejs resamples gets the value of the rate it encodes at."""
    return int(lib().mp3b200_granules_per_frame_ex(channels, samplerate, kbps, RESAMPLE if resample else 0))


def stream_bytes(channels, samplerate, kbps, nsamples, resample=False):
    """Bytes encodeBuffer(nsamples) + flush() produce, -1 for a rejected configuration.  resample=True also accepts the
    configurations lamejs resamples by an integer ratio (nsamples at the input rate)."""
    if resample:
        return int(lib().mp3b200_stream_bytes_ex(channels, samplerate, kbps, RESAMPLE, int(nsamples)))
    return int(lib().mp3b200_stream_bytes(channels, samplerate, kbps, int(nsamples)))


def out_samplerate(channels, samplerate, kbps):
    """The rate lamejs encodes (channels, samplerate, kbps) at (!= samplerate: it resamples); 0 for a bad channel count."""
    return int(lib().mp3b200_out_samplerate(channels, samplerate, kbps))


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


def lametag_size(channels, samplerate, kbps, resample=False):
    """Size of the Xing / Info / LAME tag frame of a configuration (0: InitVbrTag would switch the tag off).  resample=True:
    see Mp3Encoder."""
    return _check(lib().mp3b200_lametag_size_ex(channels, samplerate, kbps, RESAMPLE if resample else 0))


def lametag_build(channels, samplerate, kbps, nframes, music_bytes, music_crc, encoder_padding):
    """The tag frame from numbers (no device needed): VBRTag.getLameTagFrame for a CBR stream of `nframes` frames."""
    buf = np.zeros(2880, dtype=np.uint8)
    n = _check(lib().mp3b200_lametag_build(channels, samplerate, kbps, int(nframes), int(music_bytes), int(music_crc), int(encoder_padding),
                                           buf.ctypes.data, 2880))
    return buf[:n].tobytes()


class Mp3Encoder:
    """Drop-in for lamejs.Mp3Encoder(channels, samplerate, kbps) (src/js/index.js:66-136).  `write_vbr_tag=True` is
    gfp.bWriteVbrTag (index.js:107 sets it false): the stream then starts with a placeholder frame, and `lametag_frame()`
    after flush() returns the finished Info / LAME tag frame to write over it.  `resample=True` also accepts the
    configurations lamejs resamples by an integer ratio, e.g. Mp3Encoder(2, 48000, 64), which encodes at 24 kHz: samples
    are fed at the input rate and resampled on the GPU (seek() is not supported then).  `find_replay_gain=True` is
    gfp.findReplayGain (it needs the tag: without write_vbr_tag, or where the tag does not fit, it stays off): every
    sample is analysed on the GPU, each flush() ends a title, `replay_gain` is then the last title's (gain in dB,
    gfc.RadioGain) and the tag carries it; album_gain(encoders) combines titles.  State export / import and seek() are not
    supported then."""

    def __init__(self, channels=1, samplerate=44100, kbps=128, write_vbr_tag=False, resample=False, find_replay_gain=False):
        self._L = lib()
        self._h = ctypes.c_void_p()
        self.channels = channels
        flags = RESAMPLE if resample else 0
        rc = self._L.mp3b200_create_ex(channels, samplerate, kbps, flags, ctypes.byref(self._h))
        _check(rc)
        self.device = _check(self._L.mp3b200_encoder_device(self._h))     # CUDA tensors fed to it must live there
        self.tag_on = bool(write_vbr_tag) and _check(self._L.mp3b200_set_write_vbr_tag(self._h, 1)) == 1
        self._tag_room = _check(self._L.mp3b200_lametag_size_ex(channels, samplerate, kbps, flags)) if self.tag_on else 0
        self.replay_gain_on = bool(find_replay_gain) and _check(self._L.mp3b200_set_find_replay_gain(self._h, 1)) == 1

    @property
    def replay_gain(self):
        """(title gain in dB, gfc.RadioGain) of the title the last flush() ended; None before it or with the analysis off"""
        db, radio = ctypes.c_double(0.0), ctypes.c_int(0)
        if _check(self._L.mp3b200_get_replay_gain(self._h, ctypes.byref(db), ctypes.byref(radio))) != 1:
            return None
        return float(db.value), int(radio.value)

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
        """Int16 samples, or floating-point samples (Float32Array / plain Array in lamejs: rounded to Float32 once and
        scaled like lamejs scales them; non-finite values are refused).  CUDA torch tensors are encoded from device memory
        (mp3b200_encode_device): the same bytes, without a copy of the samples to the host."""
        right = None if self.channels == 1 else right
        if _on_cuda(left) or _on_cuda(right):
            (left,), (right,), f32 = _device_rows([left], [right], self.device)
            name, ptr = "mp3b200_encode_device", (lambda x: x.data_ptr())
        else:
            (left,), (right,), f32 = _rows([left], [right])
            name, ptr = "mp3b200_encode", (lambda x: x.ctypes.data)
        assert len(left) == len(right)
        cap = int(1.25 * len(left) + 7200) + self._tag_room     # index.js:114,124
        buf = np.empty(cap, dtype=np.uint8)
        n = _check(_entry(name, f32)(self._h, ptr(left), ptr(right), len(left), buf.ctypes.data, cap))
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
        [max(0, frame*framesize-1104), frame*framesize+224) (CUDA tensors are copied to the host: at most 1328 samples)"""
        left_hist, right_hist = [x.cpu() if _on_cuda(x) else x for x in (left_hist, right_hist)]
        (left_hist,), (right_hist,), f32 = _rows([left_hist], [None if self.channels == 1 else right_hist])
        _check(_entry("mp3b200_seek", f32)(self._h, int(frame), left_hist.ctypes.data, right_hist.ctypes.data, len(left_hist)))

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
    returns [enc.encodeBuffer(l, r) for ...] byte strings.  CUDA torch tensors are encoded from device memory
    (mp3b200_encode_batch_device); one call takes rows all in host memory or all on the encoders' CUDA device."""
    S = len(encoders)
    if any(_on_cuda(x) for x in (*lefts, *(() if rights is None else rights))):
        devs = {e.device for e in encoders}
        if len(devs) != 1:
            raise ValueError("CUDA rows need encoders of one device")
        lefts, rights, f32 = _device_rows(lefts, rights, devs.pop())
        name, ptr = "mp3b200_encode_batch_device", (lambda x: x.data_ptr())
    else:
        lefts, rights, f32 = _rows(lefts, rights)
        name, ptr = "mp3b200_encode_batch", (lambda x: x.ctypes.data)
    ns = np.array([len(x) for x in lefts], dtype=np.int32)
    caps = np.array([int(1.25 * n + 7200) for n in ns], dtype=np.int32)
    outs = [np.empty(int(c), dtype=np.uint8) for c in caps]
    hp = (ctypes.c_void_p * S)(*[e._h for e in encoders])
    lp = (ctypes.c_void_p * S)(*[ptr(x) for x in lefts])
    rp = (ctypes.c_void_p * S)(*[ptr(x) for x in rights])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    got = np.zeros(S, dtype=np.int32)
    _check(_entry(name, f32)(hp, lp, rp, ns.ctypes.data, op, caps.ctypes.data, S, got.ctypes.data))
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


def _encode_host_streams(name, flags, channels, samplerate, kbps, lefts, rights, room, resample, *tail):
    """Marshalling of the whole-stream host calls `name` (an _ex entry point) and its Float32 twin: out[s] has room for
    the stream's bytes plus `room`; `tail` are the arguments after out_bytes."""
    S = len(lefts)
    if S == 0:
        return []
    lefts, rights, f32 = _rows(lefts, None if channels == 1 else rights)
    ns = np.array([len(x) for x in lefts], dtype=np.int64)
    nb = [stream_bytes(channels, samplerate, kbps, int(n), resample) for n in ns]
    if any(b < 0 for b in nb):
        raise Mp3B200Error("unsupported configuration: channels=%d samplerate=%d kbps=%d (lame_init_params would resample)" % (channels, samplerate, kbps))
    nb = [b + room for b in nb]
    outs = [np.empty(b, dtype=np.uint8) for b in nb]
    lp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in lefts])
    rp = (ctypes.c_void_p * S)(*[x.ctypes.data for x in rights])
    op = (ctypes.c_void_p * S)(*[x.ctypes.data for x in outs])
    caps = np.array(nb, dtype=np.int64)
    got = np.zeros(S, dtype=np.int64)
    _check(_entry(name, f32)(channels, samplerate, kbps, flags, S, lp, rp, ns.ctypes.data, op, caps.ctypes.data, got.ctypes.data,
                             *tail))
    return [o[: int(g)].tobytes() for o, g in zip(outs, got)]


def encode_streams(channels, samplerate, kbps, lefts, rights=None, resample=False):
    """Batch extension: encodeBuffer(whole stream) + flush() for many independent streams in one launch sequence.
    Host buffers in, list of bytes out.  resample=True: see Mp3Encoder."""
    return _encode_host_streams("mp3b200_encode_streams_ex", RESAMPLE if resample else 0, channels, samplerate, kbps, lefts,
                                rights, 0, resample)


def encode_streams_tagged(channels, samplerate, kbps, lefts, rights=None, resample=False):
    """encode_streams with gfp.bWriteVbrTag on: every returned stream starts with its finished Info / LAME tag frame (frame
    and byte counts, seek table, encoder delay / padding, CRC-16 of the audio bytes computed on the GPU).  resample=True:
    see Mp3Encoder."""
    if not resample:
        return _encode_host_streams("mp3b200_encode_streams_tagged_ex", 0, channels, samplerate, kbps, lefts, rights,
                                    lametag_size(channels, samplerate, kbps), False, None, None)
    return encode_streams_replaygain(channels, samplerate, kbps, lefts, rights, resample=True, find_replay_gain=False)[0]


def encode_streams_replaygain(channels, samplerate, kbps, lefts, rights=None, resample=False, find_replay_gain=True):
    """encode_streams_tagged with gfp.findReplayGain: every stream's ReplayGain is analysed on the GPU and written into its
    tag, as lamejs does.  Returns (streams, title_db, album_db): the list of bytes, GetTitleGain of each stream in dB and
    GetAlbumGain of the batch (-24601: less than one RMS window, or the tag does not fit and nothing was analysed)."""
    flags = (REPLAYGAIN if find_replay_gain else 0) | (RESAMPLE if resample else 0)
    title = np.zeros(max(len(lefts), 1), dtype=np.float64)
    album = ctypes.c_double(0.0)
    room = lib().mp3b200_lametag_size_ex(channels, samplerate, kbps, RESAMPLE if resample else 0)
    out = _encode_host_streams("mp3b200_encode_streams_tagged_ex", flags, channels, samplerate, kbps, lefts, rights, max(room, 0),
                               resample, title.ctypes.data, ctypes.byref(album))
    return out, [float(t) for t in title[:len(lefts)]], float(album.value) if lefts else float(GAIN_NOT_ENOUGH_SAMPLES)


def replay_gain_streams(channels, samplerate, kbps, lefts, rights=None, resample=False):
    """The ReplayGain analysis of encode_streams_replaygain without the encoder (mp3b200_replaygain_streams): returns
    (title_db list, album_db), bit-identical to its gains wherever the tag fits; where it does not, the encode analyses
    nothing (-24601) and this still analyses.  Host rows with the dtype rules of encode_streams."""
    S = len(lefts)
    lefts, rights, f32 = _rows(lefts, None if channels == 1 else rights)
    ns = np.array([len(x) for x in lefts] or [0], dtype=np.int64)
    lp = (ctypes.c_void_p * max(S, 1))(*[x.ctypes.data for x in lefts])
    rp = (ctypes.c_void_p * max(S, 1))(*[x.ctypes.data for x in rights])
    title = np.zeros(max(S, 1), dtype=np.float64)
    album = ctypes.c_double(0.0)
    _check(_entry("mp3b200_replaygain_streams", f32)(channels, samplerate, kbps, RESAMPLE if resample else 0, S, lp, rp,
                                                     ns.ctypes.data, title.ctypes.data, ctypes.byref(album)))
    return [float(t) for t in title[:S]], float(album.value)


def replay_gain_streams_device(channels, samplerate, kbps, d_pcm_ptr, pcm_off, nsamples, resample=False, float32=False):
    """replay_gain_streams on device rows (raw device pointer as int), laid out as encode_streams_device reads them:
    returns (title_db list, album_db).  float32=True: d_pcm holds Float32 samples; a non-finite one raises Mp3B200Error."""
    pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
    nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
    S = len(nsamples)
    title = np.zeros(max(S, 1), dtype=np.float64)
    album = ctypes.c_double(0.0)
    _check(_entry("mp3b200_replaygain_streams_device", float32)(channels, samplerate, kbps, RESAMPLE if resample else 0, S, d_pcm_ptr,
                                                                pcm_off.ctypes.data, nsamples.ctypes.data, title.ctypes.data,
                                                                ctypes.byref(album)))
    return [float(t) for t in title[:S]], float(album.value)


def finish_tags_device(channels, samplerate, kbps, d_files_ptr, file_off, nsamples, title_db=None, resample=False):
    """The tag step of encode_streams_device_tagged on audio already in device memory (mp3b200_finish_tags_device): file s
    at d_files + file_off[s] is lametag_size(...) bytes of room followed by the stream_bytes(..., nsamples[s]) audio bytes
    of a whole encodeBuffer + flush; the finished tag frame is written into the room, its Radio Replay Gain field from
    title_db[s] (None: 0).  Returns each file's length."""
    file_off = np.ascontiguousarray(file_off, dtype=np.int64)
    nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
    S = len(nsamples)
    got = np.zeros(max(S, 1), dtype=np.int64)
    gains = None if title_db is None else np.ascontiguousarray(title_db, dtype=np.float64)
    if gains is not None and len(gains) != S:
        raise ValueError("title_db needs one gain per stream")
    _check(lib().mp3b200_finish_tags_device(channels, samplerate, kbps, RESAMPLE if resample else 0, S, d_files_ptr,
                                            file_off.ctypes.data, nsamples.ctypes.data,
                                            None if gains is None else gains.ctypes.data, got.ctypes.data))
    return [int(g) for g in got[:S]]


def album_gain(encoders):
    """GetAlbumGain over the titles the Mp3Encoders (find_replay_gain=True) have ended with flush()"""
    hs = (ctypes.c_void_p * max(len(encoders), 1))(*[e._h.value for e in encoders])
    out = ctypes.c_double(0.0)
    _check(lib().mp3b200_album_gain(hs, len(encoders), ctypes.byref(out)))
    return float(out.value)


GAIN_NOT_ENOUGH_SAMPLES = -24601

# the status of a file in encode_wav_files / wav_plan (MP3B200_WAV_*, include/mp3b200.h)
WAV_ENCODED, WAV_NOT_WAV, WAV_EXTENDED_FMT, WAV_RANGE_ERROR, WAV_NOT_PCM16, WAV_UNSUPPORTED = range(6)
WAV_TAG = 4      # MP3B200_WAV_TAG


class WavPlanEntry(ctypes.Structure):
    """mp3b200_wav_plan_entry (include/mp3b200.h)"""
    _fields_ = [("status", ctypes.c_int32), ("channels", ctypes.c_int32), ("sample_rate", ctypes.c_int32),
                ("out_samplerate", ctypes.c_int32), ("data_offset", ctypes.c_int64), ("nsamples", ctypes.c_int64),
                ("out_bytes", ctypes.c_int64)]


def _wav_files(files):
    """the files as contiguous uint8 arrays (bytes, bytearray, or uint8 arrays), their pointer and length arrays"""
    arrs = [np.frombuffer(f, dtype=np.uint8) if isinstance(f, (bytes, bytearray, memoryview)) else np.ascontiguousarray(f, dtype=np.uint8)
            for f in files]
    empty = np.zeros(1, dtype=np.uint8)              # a file of no bytes still needs a pointer
    ptrs = (ctypes.c_void_p * max(len(arrs), 1))(*[(a if len(a) else empty).ctypes.data for a in arrs])
    lens = np.array([len(a) for a in arrs] or [0], dtype=np.int64)
    return arrs, ptrs, lens


def wav_plan(files, kbps, resample=False, write_vbr_tag=False):
    """What encode_wav_files does with each file, from its bytes alone (mp3b200_wav_plan, no device): a list of dicts with
    status (WAV_*), channels, sample_rate, out_samplerate, data_offset, nsamples (per channel) and out_bytes (the MP3 file's
    exact size; with write_vbr_tag its tag frame included)."""
    arrs, ptrs, lens = _wav_files(files)
    plan = (WavPlanEntry * max(len(arrs), 1))()
    flags = (RESAMPLE if resample else 0) | (WAV_TAG if write_vbr_tag else 0)
    _check(lib().mp3b200_wav_plan(int(kbps), flags, len(arrs), ptrs, lens.ctypes.data, plan))
    return [{k: getattr(p, k) for k, _ in WavPlanEntry._fields_} for p in plan[:len(arrs)]]


def encode_wav_files(files, kbps, resample=False, write_vbr_tag=False, find_replay_gain=False):
    """WAV files in, MP3 files out: each file encoded as lamejs's worker-example does it with the whole file in one
    encodeBuffer + flush (WavHeader.readHeader, the Int16 view of the data chunk, new Mp3Encoder(channels, sampleRate, kbps)).
    `files` are bytes, bytearray or uint8 arrays of whole WAV files.  Returns (mp3s, status): mp3s[s] is the file's MP3
    bytes, or None when status[s] != WAV_ENCODED.  write_vbr_tag: every file starts with its Info / LAME tag frame, as from
    encode_streams_tagged.  find_replay_gain (implies the tag): returns (mp3s, status, title_db, album_db) with the gains of
    encode_streams_replaygain; the album covers every analysed file, whatever its configuration."""
    tagged = write_vbr_tag or find_replay_gain
    plan = wav_plan(files, kbps, resample, tagged)
    arrs, ptrs, lens = _wav_files(files)
    S = len(arrs)
    outs = [np.empty(max(p["out_bytes"], 1), dtype=np.uint8) for p in plan]
    op = (ctypes.c_void_p * max(S, 1))(*[o.ctypes.data for o in outs])
    caps = np.array([p["out_bytes"] for p in plan] or [0], dtype=np.int64)
    got = np.zeros(max(S, 1), dtype=np.int64)
    status = np.zeros(max(S, 1), dtype=np.int32)
    flags = RESAMPLE if resample else 0
    if tagged:
        title = np.zeros(max(S, 1), dtype=np.float64)
        album = ctypes.c_double(0.0)
        flags |= REPLAYGAIN if find_replay_gain else 0
        _check(lib().mp3b200_encode_wav_tagged(int(kbps), flags, S, ptrs, lens.ctypes.data, op, caps.ctypes.data, got.ctypes.data,
                                               status.ctypes.data, title.ctypes.data, ctypes.byref(album)))
    else:
        _check(lib().mp3b200_encode_wav(int(kbps), flags, S, ptrs, lens.ctypes.data, op, caps.ctypes.data, got.ctypes.data,
                                        status.ctypes.data))
    mp3s = [o[: int(g)].tobytes() if st == WAV_ENCODED else None for o, g, st in zip(outs, got, status)]
    st = [int(x) for x in status[:S]]
    if find_replay_gain:
        return mp3s, st, [float(t) for t in title[:S]], float(album.value)
    return mp3s, st


def radio_gain(title_db):
    """gfc.RadioGain, the value the tag stores (tenths of a dB): Math.floor(title_db * 10 + 0.5)"""
    return int(np.floor(title_db * 10.0 + 0.5))


def lametag_build_ex(channels, samplerate, kbps, nframes, music_bytes, music_crc, encoder_padding, radio_gain, resample=False):
    """mp3b200_lametag_build with the Radio Replay Gain field (gfc.RadioGain of a stream the caller analysed)"""
    buf = np.zeros(2880, dtype=np.uint8)
    n = lib().mp3b200_lametag_build_ex(channels, samplerate, kbps, RESAMPLE if resample else 0, nframes, music_bytes, music_crc,
                                       encoder_padding, radio_gain, buf.ctypes.data, len(buf))
    _check(min(n, 0))
    return buf[:n].tobytes()


def debug_replaygain(channels, samplerate, kbps, left, right=None, resample=False):
    """The ReplayGain analysis of one whole stream (encodeBuffer(all) + flush()) as the GPU ran it: dict with `sums`
    (float64 [windows][2]: lsum, rsum), `idx` (int32 [windows]), `hist` (int32 [12000]), `title_db`, `passes` (repair
    passes), `reruns` (chunks run again) and `ms` (the analysis's CUDA-event time)."""
    (left,), (right,), f32 = _rows([left], [None if channels == 1 else right])
    cap = len(left) // 400 + 64
    sums = np.zeros((cap, 2), dtype=np.float64)
    idx = np.zeros(cap, dtype=np.int32)
    hist = np.zeros(12000, dtype=np.int32)
    title = ctypes.c_double(0.0)
    stats = np.zeros(4, dtype=np.int32)
    _check(_entry("mp3b200_debug_replaygain", f32)(channels, samplerate, kbps, RESAMPLE if resample else 0, left.ctypes.data,
                                                   right.ctypes.data, len(left), sums.ctypes.data, idx.ctypes.data, cap,
                                                   hist.ctypes.data, ctypes.byref(title), stats.ctypes.data))
    n = int(stats[0])
    assert n <= cap
    return {"sums": sums[:n].copy(), "idx": idx[:n].copy(), "hist": hist, "title_db": float(title.value), "passes": int(stats[1]),
            "reruns": int(stats[2]), "ms": float(stats[3:4].view(np.float32)[0])}


DOMAIN_SITES = ("trunc_mask_idx", "trunc_log16", "trunc_quant", "trunc_noise", "dmax", "dmin", "pack_search", "pack_outer",
                "region_mx", "bitsum_field", "log16_table", "f32_overflow")     # DomainSite (mp3_device.cuh)


def debug_domain_hits():
    """A library built with -DMP3_DOMAIN_CHECK only: per DomainSite, how many arguments fell outside the domain the site is
    exact on since the last call (the counters are cleared).  int64 array indexed like DOMAIN_SITES."""
    fn = getattr(lib(), "mp3b200_debug_domain_hits", None)
    if fn is None:
        raise Mp3B200Error("the library was built without MP3_DOMAIN_CHECK")
    out = np.zeros(len(DOMAIN_SITES), dtype=np.uint64)
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int]
    n = _check(fn(out.ctypes.data, len(out)))
    assert n == len(DOMAIN_SITES), n
    return out.astype(np.int64)


def debug_music_crc(d_buf_ptr, offsets, lengths, timed=False):
    """k_music_crc on byte ranges of a device buffer (raw pointer as int): list of CRC-16 values (+ ms if `timed`)."""
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    ln = np.ascontiguousarray(lengths, dtype=np.int64)
    crc = np.zeros(len(off), dtype=np.uint32)
    ms = ctypes.c_float(0)
    _check(lib().mp3b200_debug_music_crc(d_buf_ptr, off.ctypes.data, ln.ctypes.data, len(off), crc.ctypes.data, ctypes.byref(ms) if timed else None))
    return ([int(c) for c in crc], float(ms.value)) if timed else [int(c) for c in crc]


def encode_streams_device(channels, samplerate, kbps, d_pcm_ptr, pcm_off, nsamples, d_out_ptr, out_off, resample=False, float32=False):
    """Device-resident batch (raw device pointers as ints).  Returns the 16 timing slots of include/mp3b200.h (ms); with
    resample=True slot 14 is the resampler's time.  float32=True: d_pcm holds Float32 samples (a float32 torch tensor),
    encoded as lamejs encodes a Float32Array; a non-finite sample raises Mp3B200Error."""
    pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
    nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
    out_off = np.ascontiguousarray(out_off, dtype=np.int64)
    tm = np.zeros(16, dtype=np.float32)
    _check(_entry("mp3b200_encode_streams_device_ex", float32)(channels, samplerate, kbps, RESAMPLE if resample else 0, len(nsamples),
                                                                d_pcm_ptr, pcm_off.ctypes.data, nsamples.ctypes.data, d_out_ptr,
                                                                out_off.ctypes.data, tm.ctypes.data))
    return tm


def encode_streams_device_tagged(channels, samplerate, kbps, d_pcm_ptr, pcm_off, nsamples, d_out_ptr, out_off, resample=False,
                                 float32=False, find_replay_gain=False):
    """encode_streams_device with the tag on (and, with find_replay_gain=True, the ReplayGain analysis): stream s is written
    as one finished file at d_out + out_off[s], its Info / LAME tag frame followed by its audio, byte-identical to what
    encode_streams_replaygain returns for the same samples.  Stream s needs stream_bytes(...) + lametag_size(...) bytes of
    room (with the same `resample`).  Returns (out_bytes, title_db, album_db): the
    length of each file, GetTitleGain of each stream in dB and GetAlbumGain of the batch (-24601: less than one RMS window,
    or nothing was analysed)."""
    pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
    nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
    out_off = np.ascontiguousarray(out_off, dtype=np.int64)
    S = len(nsamples)
    got = np.zeros(max(S, 1), dtype=np.int64)
    title = np.zeros(max(S, 1), dtype=np.float64)
    album = ctypes.c_double(0.0)
    flags = (REPLAYGAIN if find_replay_gain else 0) | (RESAMPLE if resample else 0)
    _check(_entry("mp3b200_encode_streams_tagged_device", float32)(channels, samplerate, kbps, flags, S, d_pcm_ptr, pcm_off.ctypes.data,
                                                                    nsamples.ctypes.data, d_out_ptr, out_off.ctypes.data,
                                                                    got.ctypes.data, title.ctypes.data, ctypes.byref(album)))
    return ([int(g) for g in got[:S]], [float(t) for t in title[:S]],
            float(album.value) if S else float(GAIN_NOT_ENOUGH_SAMPLES))


class EncodeSession:
    """Whole device-resident streams encoded on one CUDA stream without blocking the calling thread (mp3b200_session,
    DESIGN.md 14).  `stream` is a torch.cuda.Stream (None: torch.cuda.current_stream() now).  encode_streams queues the
    encode behind everything already queued on that stream and returns; later work on the stream sees `out` and the
    returned status.  A session must not be used from two threads at once; separate sessions share nothing."""

    def __init__(self, stream=None):
        import torch
        self.stream = torch.cuda.current_stream() if stream is None else stream
        self.device = self.stream.device
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _check(lib().mp3b200_session_create(ctypes.c_void_p(self.stream.cuda_stream or None), ctypes.byref(h)))
        self._h = h

    def _checked(self, channels, samplerate, kbps, pcm, pcm_off, nsamples, out, out_off, resample, tag_bytes):
        """the tensor and layout checks of a call; tag_bytes: room of a stream's tag frame.  Returns the three int64 arrays."""
        import torch
        if self._h is None:
            raise ValueError("the session is closed")
        if pcm.dtype not in (torch.int16, torch.float32):
            raise TypeError("pcm must be int16 or float32, not %s" % pcm.dtype)
        if out.dtype != torch.uint8:
            raise TypeError("out must be uint8, not %s" % out.dtype)
        for name, t in (("pcm", pcm), ("out", out)):
            if not _on_cuda(t) or t.device != self.device:
                raise ValueError("%s must be a CUDA tensor on the session's device (%s)" % (name, self.device))
            if t.dim() != 1 or not t.is_contiguous():
                raise ValueError("%s must be a contiguous 1-D tensor" % name)
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        nsamples = np.ascontiguousarray(nsamples, dtype=np.int64)
        out_off = np.ascontiguousarray(out_off, dtype=np.int64)
        S = len(nsamples)
        if len(pcm_off) != S or len(out_off) != S:
            raise ValueError("pcm_off, nsamples and out_off must have one entry per stream")
        if S:
            nb = {int(n): stream_bytes(channels, samplerate, kbps, int(n), resample) for n in np.unique(nsamples) if n >= 0}
            if all(b >= 0 for b in nb.values()) and (nsamples >= 0).all():
                room = np.array([nb[int(n)] + tag_bytes for n in nsamples], dtype=np.int64)
                if ((pcm_off < 0) | (pcm_off + nsamples * channels > pcm.numel()) | (out_off < 0) |
                        (out_off + room > out.numel())).any():
                    raise ValueError("a stream lies outside pcm or out")
        return pcm_off, nsamples, out_off

    def encode_streams(self, channels, samplerate, kbps, pcm, pcm_off, nsamples, out, out_off, resample=False):
        """encode_streams_device on tensors, queued: `pcm` is a 1-D CUDA tensor of int16 or float32 samples (float32 is
        encoded as lamejs encodes a Float32Array), laid out as encode_streams_device reads d_pcm; `out` a uint8 CUDA tensor,
        stream s written at out_off[s].  pcm_off, nsamples and out_off are host sequences.  Returns the int32[4] status
        tensor the call fills on the session's stream (check_status reads it)."""
        import torch
        pcm_off, nsamples, out_off = self._checked(channels, samplerate, kbps, pcm, pcm_off, nsamples, out, out_off, resample, 0)
        with torch.cuda.stream(self.stream):
            status = torch.empty(4, dtype=torch.int32, device=self.device)
        fn = lib().mp3b200_encode_streams_async_f32 if pcm.dtype == torch.float32 else lib().mp3b200_encode_streams_async
        _check(fn(self._h, channels, samplerate, kbps, RESAMPLE if resample else 0, len(nsamples), pcm.data_ptr(), pcm_off.ctypes.data,
                  nsamples.ctypes.data, out.data_ptr(), out_off.ctypes.data, status.data_ptr()))
        for t in (pcm, out, status):
            t.record_stream(self.stream)
        return status

    def encode_streams_tagged(self, channels, samplerate, kbps, pcm, pcm_off, nsamples, out, out_off, resample=False,
                              find_replay_gain=False):
        """encode_streams_device_tagged on tensors, queued (DESIGN.md 15): stream s becomes one finished file at
        out[out_off[s]:], its Info / LAME tag frame and then its audio, and needs stream_bytes(...) + lametag_size(...) bytes
        of room.  Returns (out_bytes, gains, status): the files' lengths, a host list known at once; with find_replay_gain a
        float64 CUDA tensor of the title gains and, last, the album gain in dB (-24601: nothing to analyse), else None; and
        the int32[8] status tensor (check_status reads it; [4] and [5] are the analysis's passes and reruns).  Tensors and
        status are filled on the session's stream."""
        import torch
        tfs = lametag_size(channels, samplerate, kbps, resample)
        pcm_off, nsamples, out_off = self._checked(channels, samplerate, kbps, pcm, pcm_off, nsamples, out, out_off, resample,
                                                   max(tfs, 0))
        S = len(nsamples)
        got = np.zeros(max(S, 1), dtype=np.int64)
        with torch.cuda.stream(self.stream):
            status = torch.empty(8, dtype=torch.int32, device=self.device)
            gains = torch.empty(S + 1, dtype=torch.float64, device=self.device) if find_replay_gain else None
        flags = (REPLAYGAIN if find_replay_gain else 0) | (RESAMPLE if resample else 0)
        fn = _entry("mp3b200_encode_streams_tagged_async", pcm.dtype == torch.float32)
        _check(fn(self._h, channels, samplerate, kbps, flags, S, pcm.data_ptr(), pcm_off.ctypes.data, nsamples.ctypes.data,
                  out.data_ptr(), out_off.ctypes.data, got.ctypes.data, gains.data_ptr() if find_replay_gain else None,
                  status.data_ptr()))
        for t in (pcm, out, status) + ((gains,) if find_replay_gain else ()):
            t.record_stream(self.stream)
        return [int(g) for g in got[:S]], gains, status

    def _handles(self, encoders):
        if self._h is None:
            raise ValueError("the session is closed")
        if any(not isinstance(e, Mp3Encoder) or not e._h for e in encoders):
            raise ValueError("encoders must be open Mp3Encoder objects")
        if len({id(e) for e in encoders}) != len(encoders):
            raise ValueError("a session call names each encoder once (make two calls instead)")
        return (ctypes.c_void_p * max(len(encoders), 1))(*[e._h for e in encoders])

    def _queue(self, encoders, lengths, call, *tensors, status_words=4):
        """allocates `out` for the calls' exact lengths on the session's stream and runs call(hp, out, offsets, got, status)"""
        import torch
        S = len(encoders)
        hp = self._handles(encoders)
        lengths = [_check(int(lib().mp3b200_encode_bytes(e._h, n))) for e, n in zip(encoders, lengths)]
        offsets = np.zeros(max(S, 1), dtype=np.int64)
        if S > 1:
            offsets[1:S] = np.cumsum(lengths[:-1])
        with torch.cuda.stream(self.stream):
            out = torch.empty(max(sum(lengths), 1), dtype=torch.uint8, device=self.device)
            status = torch.empty(status_words, dtype=torch.int32, device=self.device)
        got = np.zeros(max(S, 1), dtype=np.int32)
        _check(call(hp, out.data_ptr(), offsets.ctypes.data, got.ctypes.data, status.data_ptr()))
        for t in (out, status) + tensors:
            t.record_stream(self.stream)
        assert [int(g) for g in got[:S]] == lengths
        return out, [int(o) for o in offsets[:S]], lengths, status

    def encode_batch(self, encoders, lefts, rights=None):
        """encodeBuffer on live Mp3Encoder objects of one configuration, queued on the session's stream (DESIGN.md 16):
        `lefts` / `rights` are CUDA tensors on the session's device (floating dtypes are encoded as Float32, like
        Mp3Encoder.encodeBuffer).  Each encoder's first session call binds it to the session: until release() its host
        calls raise Mp3B200Error.  Returns (out, offsets, lengths, status): a uint8 CUDA tensor filled on the stream, encoder
        i's bytes at out[offsets[i]:offsets[i] + lengths[i]] (host lists, known at once), and the int32[4] status tensor
        check_status reads.  Nothing here orders the rows: produce them on the session's stream, or make it wait."""
        return self._encode(encoders, lefts, rights, False)

    def encode_batch_tagged(self, encoders, lefts, rights=None):
        """encode_batch for encoders in any mix of plain, write_vbr_tag and find_replay_gain (DESIGN.md 17), queued on the
        session's stream: the same rows, the same (out, offsets, lengths, status), where a tagged encoder's first feeding
        call hands out the all-zero placeholder frame first, and status is int32[8] ([4] and [5]: the analysis's passes and
        reruns).  The music CRC and ReplayGain stay on the device until release(); lametag_frames and album_gain read them
        there, ordered behind this call by the session's stream."""
        return self._encode(encoders, lefts, rights, True)

    def _encode(self, encoders, lefts, rights, tagged):
        import torch
        if self._h is None:
            raise ValueError("the session is closed")
        S = len(encoders)
        if len(lefts) != S or (rights is not None and len(rights) != S):
            raise ValueError("one row (pair) per encoder")
        rights = [None] * S if rights is None else list(rights)
        rows = [x for x in (*lefts, *rights) if x is not None]
        if not all(_on_cuda(x) and x.device == self.device for x in rows):
            raise ValueError("rows must be CUDA tensors on the session's device (%s)" % self.device)
        if any(x.dim() != 1 for x in rows):
            raise ValueError("rows must be 1-D")
        f32 = any(x.dtype.is_floating_point for x in rows)
        dt = torch.float32 if f32 else torch.int16
        with torch.cuda.stream(self.stream):
            lefts = [x.to(dt).contiguous() for x in lefts]
            rights = [l if (r is None or e.channels == 1) else r.to(dt).contiguous() for e, l, r in zip(encoders, lefts, rights)]
        if any(len(l) != len(r) for l, r in zip(lefts, rights)):
            raise ValueError("left and right rows differ in length")
        ns = np.array([len(x) for x in lefts] or [0], dtype=np.int32)
        lp = (ctypes.c_void_p * max(S, 1))(*[x.data_ptr() for x in lefts])
        rp = (ctypes.c_void_p * max(S, 1))(*[x.data_ptr() for x in rights])
        fn = _entry("mp3b200_session_encode_batch_tagged" if tagged else "mp3b200_session_encode_batch", f32)
        return self._queue(encoders, [int(n) for n in ns[:S]],
                           lambda hp, o, off, got, st: fn(self._h, hp, lp, rp, ns.ctypes.data, S, o, off, got, st),
                           *lefts, *rights, status_words=8 if tagged else 4)

    def flush_batch(self, encoders):
        """flush() on live Mp3Encoder objects, queued on the session's stream; returns what encode_batch returns"""
        S = len(encoders)
        return self._queue(encoders, [-1] * S,
                           lambda hp, o, off, got, st: lib().mp3b200_session_flush_batch(self._h, hp, S, o, off, got, st))

    def flush_batch_tagged(self, encoders):
        """flush() on encoders in any mix of plain, tagged and ReplayGain, queued on the session's stream; returns what
        encode_batch_tagged returns.  Each flush ends a ReplayGain title on the device, ordered by the session's stream."""
        S = len(encoders)
        return self._queue(encoders, [-1] * S,
                           lambda hp, o, off, got, st: lib().mp3b200_session_flush_batch_tagged(self._h, hp, S, o, off, got, st),
                           status_words=8)

    def lametag_frames(self, encoders):
        """The frame lametag_frame() would return for each encoder (one configuration) at this point of its stream, written
        on the session's stream behind every call queued before: (out, offsets, lengths, status) as encode_batch returns
        them, a length 0 where the tag is off or no frame has been encoded; status int32[4] (check_status raises where an
        encoder was refused by an earlier call).  Binds the encoders that are not bound yet."""
        import torch
        S = len(encoders)
        hp = self._handles(encoders)
        room = [e._tag_room if e.tag_on else 0 for e in encoders]     # the call says which frames exist
        offsets = np.zeros(max(S, 1), dtype=np.int64)
        if S > 1:
            offsets[1:S] = np.cumsum(room[:-1])
        with torch.cuda.stream(self.stream):
            out = torch.empty(max(sum(room), 1), dtype=torch.uint8, device=self.device)
            status = torch.empty(4, dtype=torch.int32, device=self.device)
        got = np.zeros(max(S, 1), dtype=np.int32)
        _check(lib().mp3b200_session_lametag_frames(self._h, hp, S, out.data_ptr(), offsets.ctypes.data, got.ctypes.data,
                                                    status.data_ptr()))
        for t in (out, status):
            t.record_stream(self.stream)
        return out, [int(o) for o in offsets[:S]], [int(g) for g in got[:S]], status

    def album_gain(self, encoders):
        """album_gain(encoders) on the session's stream, behind every call queued before: a float64 CUDA tensor of one
        element (-24601: nothing analysed) and an int32[4] status (check_status raises where an encoder was refused).
        Binds the encoders that are not bound yet."""
        import torch
        hp = self._handles(encoders)
        with torch.cuda.stream(self.stream):
            album = torch.empty(1, dtype=torch.float64, device=self.device)
            status = torch.empty(4, dtype=torch.int32, device=self.device)
        _check(lib().mp3b200_session_album_gain(self._h, hp, len(encoders), album.data_ptr(), status.data_ptr()))
        for t in (album, status):
            t.record_stream(self.stream)
        return album, status

    def graph_instantiations(self):
        """loop graphs the session has instantiated so far (constant once a steady workload's shapes are warm)"""
        if self._h is None:
            raise ValueError("the session is closed")
        return int(lib().mp3b200_session_graph_instantiations(self._h))

    def release(self, encoders):
        """Waits for the session's work on `encoders` and gives them back to their host calls: each continues its stream
        exactly where it stands (a handle of a refused call: where it stood before that call)."""
        hp = self._handles(encoders)
        _check(lib().mp3b200_session_release(self._h, hp, len(encoders)))

    def close(self):
        """Waits for the session's queued work and frees it."""
        if self._h is not None:
            h, self._h = self._h, None
            _check(lib().mp3b200_session_destroy(h))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def check_status(status):
    """Synchronises the device, then raises Mp3B200Error as encode_streams_device would have for the call that filled
    `status` (a refused Float32 sample, a frame over its bit budget, an internal fault).  Returns the quantizer pass count."""
    import torch
    torch.cuda.synchronize(status.device)
    words = np.ascontiguousarray(status.cpu().numpy(), dtype=np.int32)
    _check(lib().mp3b200_check_status(words.ctypes.data))
    return int(words[2])


def debug_resample(channels, samplerate, kbps, left, right=None, ny=None):
    """k_resample's output for an input extended with zeros on both sides: float32 array [nch][ny] (default ny: every output
    the input reaches)."""
    (left,), (right,), f32 = _rows([left], [None if channels == 1 else right])
    r = samplerate // out_samplerate(channels, samplerate, kbps)
    if ny is None:
        ny = (len(left) + 15) // r + 1
    y = np.zeros((channels, ny), dtype=np.float32)
    _check(_entry("mp3b200_debug_resample", f32)(channels, samplerate, kbps, left.ctypes.data, right.ctypes.data, len(left),
                                                 y.ctypes.data, ny))
    return y


# the rows mp3b200_debug_psy_take hands out (include/mp3b200.h)
PSY_UNIT_DTYPE = np.dtype({"names": ["eb_l", "peaks", "loudness", "mask_idx", "attack"],
                           "formats": [(np.float32, 64), (np.float32, 9), np.float32, (np.uint8, 64), (np.uint8, 4)],
                           "offsets": [0, 256, 292, 296, 360], "itemsize": 368})
PSY_SHORT_DTYPE = np.dtype({"names": ["ecb_s", "eb_s"], "formats": [(np.float64, (3, 64)), (np.float32, (3, 64))],
                            "offsets": [0, 1536], "itemsize": 2304})
PSY_RATIO_DTYPE = np.dtype([("en_l", np.float32, 22), ("thm_l", np.float32, 22), ("en_s", np.float32, (13, 3)),
                            ("thm_s", np.float32, (13, 3))])


class PsyCapture:
    """What debug_psy_capture recorded: `launches`, one dict per pipeline launch in launch order, filled when the block ends:
    "streams": per stream of the launch {"z", "frame0", "nframes", "rows"} with rows PSY_UNIT_DTYPE[G nframes + 1][nch] for
    u = -1 .. G nframes - 1, and the rows after the MDCT: "bt" and "bt_prev" int8[G nframes][nch] (the final block type and
    the one the unit's psy call saw), "ath_psy" and "ath_q" float64[nframes], "ratio" PSY_RATIO_DTYPE[G nframes + 1][nch]
    for u = -1 .. G nframes - 1 (row u is the masking granule u + 1 uses) and "xr" float32[G nframes][nch][576]; "short": the
    short list as an int array [count][3] of (stream, u, channel) in list order; "short_rows": PSY_SHORT_DTYPE[count];
    "k2_launches": how many k_psy_analysis launches the pipeline made."""

    def __init__(self):
        self.launches = []

    def _parse(self, raw):
        by, front = {}, {}
        off = 0
        while off < len(raw):
            h = np.frombuffer(raw, dtype=np.int32, count=8, offset=off)
            off += 32
            kind, launch = int(h[0]), int(h[1])
            rec = by.setdefault(launch, {"streams": [], "short": None, "short_rows": None, "k2_launches": None})
            if kind == 1:
                z, frame0, nframes, nch, G, rb = (int(v) for v in h[2:])
                assert rb == PSY_UNIT_DTYPE.itemsize, rb
                n = (G * nframes + 1) * nch
                rows = np.frombuffer(raw, dtype=PSY_UNIT_DTYPE, count=n, offset=off).reshape(-1, nch).copy()
                off += n * rb
                rec["streams"].append({"z": z, "frame0": frame0, "nframes": nframes, "G": G, "rows": rows})
            elif kind == 3:
                z, frame0, nframes, nch, G, rb = (int(v) for v in h[2:])
                assert rb == PSY_RATIO_DTYPE.itemsize, rb
                n = G * nframes
                s = {}
                for k in ("ath_psy", "ath_q"):
                    s[k] = np.frombuffer(raw, dtype=np.float64, count=nframes, offset=off).copy()
                    off += 8 * nframes
                s["ratio"] = np.frombuffer(raw, dtype=PSY_RATIO_DTYPE, count=(n + 1) * nch, offset=off).reshape(-1, nch).copy()
                off += (n + 1) * nch * rb
                s["xr"] = np.frombuffer(raw, dtype=np.float32, count=n * nch * 576, offset=off).reshape(n, nch, 576).copy()
                off += 4 * n * nch * 576
                for k in ("bt", "bt_prev"):
                    s[k] = np.frombuffer(raw, dtype=np.int8, count=2 * n, offset=off).reshape(n, 2)[:, :nch].copy()
                    off += 2 * n
                off += -(4 * n) % 8
                front.setdefault(launch, {})[z] = s
            else:
                assert kind == 2, kind
                count, nch, G, k2, _, rb = (int(v) for v in h[2:])
                assert rb == PSY_SHORT_DTYPE.itemsize, rb
                pairs = np.frombuffer(raw, dtype=np.int32, count=2 * count, offset=off).reshape(-1, 2)
                off += 8 * count
                rec["short"] = np.stack([pairs[:, 0], (pairs[:, 1] >> 1) - 1, pairs[:, 1] & 1], axis=1) if count else np.zeros((0, 3), np.int64)
                rec["short_rows"] = np.frombuffer(raw, dtype=PSY_SHORT_DTYPE, count=count, offset=off).copy()
                off += count * rb
                rec["k2_launches"] = k2
        for k in sorted(by):
            by[k]["streams"].sort(key=lambda s: s["z"])
            for s in by[k]["streams"]:
                s.update(front.get(k, {}).get(s["z"], {}))
            self.launches.append(by[k])


@contextlib.contextmanager
def debug_psy_capture():
    """Debug only: while the block runs, every pipeline launch (any thread, any session) poisons its front-end rows before
    the long-block analysis (psy rows, short rows, subband slabs, masking, xr, ATH adjustments, block types) and records them
    after the attack pre-pass, the short-block analysis and the MDCT (mp3b200_debug_psy_capture; each launch synchronises
    its stream at those points).  Yields a PsyCapture, filled when the block ends."""
    L = lib()
    L.mp3b200_debug_psy_capture.argtypes = [ctypes.c_int]
    L.mp3b200_debug_psy_take.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    L.mp3b200_debug_psy_take.restype = ctypes.c_int64
    cap = PsyCapture()
    _check(L.mp3b200_debug_psy_capture(1))
    try:
        yield cap
    finally:
        L.mp3b200_debug_psy_capture(0)
        while True:
            n = L.mp3b200_debug_psy_take(None, 0)
            buf = np.empty(n, dtype=np.uint8)
            if L.mp3b200_debug_psy_take(buf.ctypes.data, n) == n:
                break
        cap._parse(buf.tobytes())


def debug_stages(channels, samplerate, kbps, left, right=None, force_blocktype=None, want=("xr",), resample=False):
    """Stage taps for parity tests: returns a dict of numpy arrays (see include/mp3b200.h).  `want` names any of xr,
    blocktype, en_l, thm_l, en_s, thm_s, ath_adjust, l3_enc, ginfo, bytes, scalefac, subblock_gain, xmin, max_nonzero_coeff,
    xrpow_max, scfsi, old_value and cur_step (the last two [F][3][nch]: frame start, after gr0, frame end).  resample=True
    also accepts the configurations lamejs resamples by an integer ratio: left / right are input samples, the taps are
    those of the output rate, after k_resample."""
    L = lib()
    (left,), (right,), f32 = _rows([left], [None if channels == 1 else right])
    n = len(left)
    F = stream_frames(n, channels, samplerate, kbps, resample)
    G = granules_per_frame(channels, samplerate, kbps, resample)
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
    nb = stream_bytes(channels, samplerate, kbps, n, resample)
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
                  old_value=alloc("old_value", (F, 3, nch), np.int32), cur_step=alloc("cur_step", (F, 3, nch), np.int32),
                  flags=RESAMPLE if resample else 0)
    if f32:
        _check(L.mp3b200_debug_stages_f32(ctypes.byref(t), left.ctypes.data, right.ctypes.data))
    else:
        _check(L.mp3b200_debug_stages_ex(ctypes.byref(t)))
    return res
