"""The oracle's resampler output, recorded (tests/resample_tap.cpp), and the FIR model of it for integer rate ratios.

Test infrastructure only.  The tap library is the oracle's own sources plus resample_tap.cpp, compiled once per process
into a temporary directory; the oracle's code and bytes are unchanged."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE = oracle_lib.ORACLE_DIR
SRCS = ["lj_mdct.cpp", "lj_psy.cpp", "lj_quant.cpp", "lj_bitstream.cpp", "lj_vbrtag.cpp"]
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fwrapv", "-w"]
FIFO_LEAD = 576 - 48          # zeros a fresh FIFO holds in front of the first output
HALF, TAPS = 16, 33

RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)
KBPS = (8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 123, 128, 144, 160, 192, 224, 256, 320)


def all_configs():
    """the 342 (channels, rate, kbps) combinations of the acceptance tests"""
    return [(ch, sr, kb) for sr in RATES for kb in KBPS for ch in (1, 2)]


def is_integer_ratio(sr, out):
    ratio = sr / out
    return abs(ratio - np.floor(.5 + ratio)) < 1e-4


def resampled_configs(integer=True):
    """configurations lamejs resamples, with an integer (or fractional) rate ratio"""
    out = []
    for ch, sr, kb in all_configs():
        o = oracle_lib.out_samplerate(ch, sr, kb)
        if o != sr and is_integer_ratio(sr, o) == integer:
            out.append((ch, sr, kb))
    return out


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(ORACLE, s) for s in ["lj_init.cpp"] + SRCS] + [os.path.join(HERE, "resample_tap.cpp")]
    h = hashlib.sha256()
    for p in srcs + [os.path.join(ORACLE, f) for f in os.listdir(ORACLE) if f.endswith(".h")]:
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "mp3b200_resample_tap_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "libtap.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = os.path.join(d, "libtap.%d.so" % os.getpid())
        init_o = os.path.join(d, "lj_init.%d.o" % os.getpid())
        subprocess.check_call(["g++"] + CXXFLAGS + ["-Dlj_psycho_anal_ns=tap_psycho_anal_ns", "-c", srcs[0], "-o", init_o])
        subprocess.check_call(["g++"] + CXXFLAGS + ["-shared", "-o", tmp, init_o] + srcs[1:] + ["-lm"])
        os.replace(tmp, so)
        os.remove(init_o)
    L = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    L.lj_create.restype = vp
    L.lj_create.argtypes = [ctypes.c_int] * 3
    L.lj_encode.argtypes = [vp, vp, vp, ctypes.c_int, vp, ctypes.c_int]
    L.lj_flush.argtypes = [vp, vp, ctypes.c_int]
    L.lj_destroy.argtypes = [vp]
    L.tap_begin.argtypes = [vp]
    L.tap_end.argtypes = [vp]
    L.tap_end.restype = ctypes.c_longlong
    L.tap_copy.argtypes = [ctypes.c_int, vp]
    L.tap_filter.argtypes = [vp, ctypes.c_int, vp]
    L.tap_bpc.argtypes = [vp]
    L.tap_scale.argtypes = [vp]
    L.tap_scale.restype = ctypes.c_double
    _lib = L
    return L


def record(channels, samplerate, kbps, left, right=None, calls=None, flush=True):
    """Runs the oracle like Mp3Encoder.encodeBuffer over `calls` (a list of call sizes; None: one call) and flush(), and
    returns (y, h, scale, out_bytes): y = float32 [nch][n], every value fill_buffer_resample wrote, per channel in stream
    order; h = the filter bank's middle row (float32, 33 taps); scale = gfp.scale; out_bytes = the encoded stream."""
    L = lib()
    left = np.ascontiguousarray(left, dtype=np.int16)
    right = left if (right is None or channels == 1) else np.ascontiguousarray(right, dtype=np.int16)
    e = L.lj_create(channels, samplerate, kbps)
    assert e, (channels, samplerate, kbps)
    L.tap_begin(e)
    out = bytearray()
    buf = np.empty(int(1.25 * max(len(left), 1) + 7200 + 8 * 1441), dtype=np.uint8)
    calls = [len(left)] if calls is None else calls
    assert sum(calls) == len(left)
    pos = 0
    for n in calls:
        lc, rc = np.ascontiguousarray(left[pos:pos + n]), np.ascontiguousarray(right[pos:pos + n])
        k = L.lj_encode(e, lc.ctypes.data, rc.ctypes.data, n, buf.ctypes.data, len(buf))
        assert k >= 0
        out += buf[:k].tobytes()
        pos += n
    if flush:
        k = L.lj_flush(e, buf.ctypes.data, len(buf))
        assert k >= 0
        out += buf[:k].tobytes()
    n = L.tap_end(e)
    nch = channels
    y = np.zeros((nch, n), dtype=np.float32)
    for c in range(nch):
        L.tap_copy(c, y[c].ctypes.data)
    h = np.zeros(TAPS, dtype=np.float32)
    have = L.tap_filter(e, L.tap_bpc(e), h.ctypes.data)
    scale = L.tap_scale(e)
    L.lj_destroy(e)
    assert have, "the encoder never resampled"
    assert not y[:, :FIFO_LEAD].any()
    return y[:, FIFO_LEAD:], h, scale, bytes(out)


def outputs_after(p, r):
    """outputs the resampler has made after p input samples (output m needs input r m + 16)"""
    return max(0, -(-(p - HALF) // r))


def fir(x, h, scale, r, ny):
    """The integer-ratio model: y[m] = Float32(sum_{i=0..32} (double)h[i] * xs[r m - 16 + i]), summed in double in tap order
    from 0.0, xs = Float32(x * scale) unless scale is 0 or 1, xs = 0 outside the input."""
    x = np.asarray(x, dtype=np.float64)
    xs = x if scale in (0.0, 1.0) else (x * scale).astype(np.float32).astype(np.float64)
    pad = np.zeros(HALF + len(xs) + r * ny + TAPS, dtype=np.float64)
    pad[HALF:HALF + len(xs)] = xs                      # pad[k + 16] = xs[k]
    idx = r * np.arange(ny)
    acc = np.zeros(ny, dtype=np.float64)
    for i in range(TAPS):
        acc = acc + np.float64(h[i]) * pad[idx + i]
    return acc.astype(np.float32)
