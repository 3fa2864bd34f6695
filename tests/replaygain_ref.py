"""ReplayGain as lamejs computes it with gfp.findReplayGain = true (tests/replaygain_ref.cpp), driven with the pieces lamejs
hands to AnalyzeSamples.  Test infrastructure only.

lame_encode_buffer_sample (Lame.js:1592-1663) calls AnalyzeSamples once per fill_buffer step, on the n_out samples that
step wrote at mf_size: up to one frame of samples at the encoding rate, so a call of n samples is analysed as pieces of
framesize and a last, shorter piece; lame_encode_flush feeds zero bunches the same way.  With resampling the pieces count
the resampler's outputs.  The filters run on continuously, but the sums do not: a piece's first MAX_ORDER samples and every
RMS window end start a new run of `% 8` single adds and groups of eight, so the sum bits depend on the pieces.

A schedule is a list of ("enc", n) and ("flush",) steps; each flush ends a title (GetTitleGain in flush_bitstream)."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import resample_tap

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HIST = 12000
GAIN_NOT_ENOUGH_SAMPLES = -24601
RATES = (48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000)

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(HERE, "replaygain_ref.cpp"), os.path.join(ROOT, "oracle", "js_math.h")]
    h = hashlib.sha256()
    for p in srcs:
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "mp3b200_replaygain_ref_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "librg.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = os.path.join(d, "librg.%d.so" % os.getpid())
        subprocess.check_call(["g++"] + resample_tap.CXXFLAGS + ["-shared", "-o", tmp, srcs[0], "-lm"])
        os.replace(tmp, so)
    L = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    L.rg_create.restype = vp
    L.rg_create.argtypes = [ctypes.c_int]
    L.rg_destroy.argtypes = [vp]
    L.rg_sample_window.argtypes = [vp]
    L.rg_analyze.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int]
    L.rg_title_gain.argtypes = [vp]
    L.rg_title_gain.restype = ctypes.c_double
    L.rg_album_gain.argtypes = [vp]
    L.rg_album_gain.restype = ctypes.c_double
    L.rg_analyze_result.argtypes = [vp]
    L.rg_analyze_result.restype = ctypes.c_double
    L.rg_trace.argtypes = [vp, vp, ctypes.c_longlong]
    L.rg_trace.restype = ctypes.c_longlong
    L.rg_hist.argtypes = [vp, vp, vp]
    _lib = L
    return L


def sample_window(sr):
    return (sr + 19) // 20


class Fifo:
    """lamejs's input FIFO counted without samples (the model of lamejs_b200's LameFifo), listing the pieces."""

    def __init__(self, mode_gr, ratio=1):
        self.framesize = 576 * mode_gr
        self.mf_size = 576 - 48
        self.to_encode = 576 + 1152
        self.ratio = ratio
        self.in_fed = 0

    def outputs(self, p):
        if self.ratio == 1:
            return p
        return (p - resample_tap.HALF + self.ratio - 1) // self.ratio if p > resample_tap.HALF else 0

    def feed(self, n):
        """pieces (output counts) of one lame_encode_buffer call of n input samples"""
        self.frames = 0
        if n <= 0:
            return []
        k = self.outputs(self.in_fed + n) - self.outputs(self.in_fed)
        self.in_fed += n
        need = self.framesize + 752
        frames = (self.mf_size + k - need) // self.framesize + 1 if self.mf_size + k >= need else 0
        if self.to_encode < 1:
            self.to_encode = 576 + 1152
        self.frames = frames
        self.mf_size += k - frames * self.framesize
        self.to_encode += k - frames * self.framesize
        return [min(self.framesize, k - i) for i in range(0, k, self.framesize)]

    def flush(self):
        """(pieces, zero input samples fed) of lame_encode_flush"""
        if self.to_encode < 1:
            return [], 0
        fs = self.framesize
        ste = float(self.to_encode - 1152)
        if self.ratio > 1:
            ste += 16. / self.ratio
        end_padding = fs - np.fmod(ste, float(fs))
        if end_padding < 576:
            end_padding += fs
        frames_left = (ste + end_padding) / fs
        pieces, zeros = [], 0
        while frames_left > 0:
            bunch = float(fs + 752 - self.mf_size) * self.ratio
            bunch = min(max(bunch, 1.0), 1152.0)
            pieces += self.feed(int(bunch))
            got = self.frames
            zeros += int(bunch)
            frames_left -= 1 if got > 0 else 0
        self.to_encode = 0
        return pieces, zeros


def schedule_of(n, chunk=None):
    """encodeBuffer over n samples in calls of `chunk` (None: one call; a list: those call sizes), then flush()"""
    if chunk is None:
        calls = [n] if n > 0 else []
    elif isinstance(chunk, (list, tuple)):
        calls = list(chunk)
        assert sum(calls) == n
    else:
        calls = [min(chunk, n - i) for i in range(0, n, chunk)]
    return [("enc", c) for c in calls] + [("flush",)]


def _scale(channels, samplerate, kbps):
    L = resample_tap.lib()
    e = L.lj_create(channels, samplerate, kbps)
    assert e, (channels, samplerate, kbps)
    s = L.tap_scale(e)
    L.lj_destroy(e)
    return s


def analysed(channels, samplerate, kbps, left, right, schedule):
    """(rows float32 [nch][m], out rate, piece lists per title): every sample AnalyzeSamples sees, in order, and the pieces
    it sees them in.  Native rates: Float32(x * gfp.scale) (x when the scale is 0 or 1), the flush's zeros in place;
    resampled rates: what the oracle's resampler wrote (tests/resample_tap.py), which needs a single flush at the end."""
    import oracle_lib
    out_sr = oracle_lib.out_samplerate(channels, samplerate, kbps)
    ratio = samplerate // out_sr
    mode_gr = 2 if out_sr >= 32000 else 1
    left = np.asarray(left, dtype=np.int16)
    right = left if (right is None or channels == 1) else np.asarray(right, dtype=np.int16)
    fifo = Fifo(mode_gr, ratio)
    titles, cur, rows, pos = [], [], [[] for _ in range(channels)], 0
    for step in schedule:
        if step[0] == "enc":
            n = step[1]
            cur += fifo.feed(n)
            for c, x in enumerate((left, right)[:channels]):
                rows[c].append(x[pos:pos + n])
            pos += n
        else:
            if fifo.to_encode < 1:             # flush() again: lamejs returns at once (no flush_bitstream, no GetTitleGain)
                continue
            p, z = fifo.flush()
            cur += p
            for c in range(channels):
                rows[c].append(np.zeros(z, dtype=np.int16))
            titles.append(cur)
            cur = []
    if cur:
        titles.append(cur)
    assert pos == len(left)
    if ratio > 1:
        total = sum(sum(t) for t in titles)
        flushes = [i for i, s in enumerate(schedule) if s[0] == "flush"]
        if flushes == [len(schedule) - 1]:
            calls = [s[1] for s in schedule if s[0] == "enc"]
            y, _, _, _ = resample_tap.record(channels, samplerate, kbps, left, right, calls=calls or [0])
        else:
            # flush then more samples: the resampler runs on through the flush's zeros (they are input samples to it), so
            # its outputs are the integer-ratio FIR model (equal to the oracle's, tests/test_resample_cpu.py) of the input
            # with the zeros in place
            _, h, scale, _ = resample_tap.record(channels, samplerate, kbps, left[:4096], right[:4096])
            y = np.stack([resample_tap.fir(np.concatenate(rows[c]), h, scale, ratio, total) for c in range(channels)])
        assert y.shape[1] >= total
        return np.ascontiguousarray(y[:, :total]), out_sr, titles
    scale = _scale(channels, samplerate, kbps)
    out = []
    for c in range(channels):
        x = np.concatenate(rows[c]).astype(np.float64) if rows[c] else np.zeros(0)
        xs = x if scale in (0.0, 1.0) else x * scale
        out.append(xs.astype(np.float32))
    return np.ascontiguousarray(np.stack(out)), out_sr, titles


class Result:
    def __init__(self):
        self.title_db, self.radio, self.windows, self.hist = [], [], [], []
        self.album_db = None


def radio_gain(title_db):
    """gfc.RadioGain = Math.floor(RadioGain * 10.0 + 0.5) | 0 (BitStream.js:785)"""
    return int(np.floor(title_db * 10.0 + 0.5))


def run(rows, out_sr, titles):
    """AnalyzeSamples on every piece, GetTitleGain after every title.  Returns a Result: per title the gain in dB,
    gfc.RadioGain, the windows (uint64 [k][3]: lsum bits, rsum bits, histogram index) and the histogram A; album_db is
    GetAlbumGain over all titles."""
    L = lib()
    nch = rows.shape[0]
    h = L.rg_create(out_sr)
    assert h
    r = Result()
    pos = 0
    done = 0
    try:
        for pieces in titles:
            for p in pieces:
                seg = [np.ascontiguousarray(rows[c, pos:pos + p]) for c in range(nch)]
                assert L.rg_analyze(h, seg[0].ctypes.data, seg[-1].ctypes.data, p, nch) == 1
                pos += p
            k = L.rg_trace(h, None, 0)
            tr = np.zeros((k, 3), dtype=np.uint64)
            L.rg_trace(h, tr.ctypes.data, k)
            a = np.zeros(HIST, dtype=np.int32)
            L.rg_hist(h, a.ctypes.data, None)
            g = L.rg_title_gain(h)
            r.title_db.append(g)
            r.radio.append(radio_gain(g))
            r.windows.append(tr[done:])
            r.hist.append(a)
            done = k
        r.album_db = L.rg_album_gain(h)
    finally:
        L.rg_destroy(h)
    return r


def analyze_stream(channels, samplerate, kbps, left, right=None, chunk=None, schedule=None):
    """ReplayGain of encodeBuffer calls (see schedule_of) and flush(): a Result"""
    sched = schedule if schedule is not None else schedule_of(len(left), chunk)
    rows, out_sr, titles = analysed(channels, samplerate, kbps, left, right, sched)
    return run(rows, out_sr, titles)


def analyze_result(hist):
    a = np.ascontiguousarray(hist, dtype=np.int32)
    assert a.shape == (HIST,)
    return lib().rg_analyze_result(a.ctypes.data)


def tag_field(radio):
    """the Radio Replay Gain field of the LAME tag (VBRTag.js:640-661): name code 1, originator 3 (automatic), sign, |gain|
    clamped to 0x1FE"""
    radio = max(-0x1FE, min(0x1FE, radio))
    v = 0x2000 | 0xC00
    return v | radio if radio >= 0 else v | 0x200 | -radio


def window_digest(windows):
    return hashlib.sha256(np.ascontiguousarray(windows, dtype="<u8").tobytes()).hexdigest()
