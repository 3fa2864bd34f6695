"""The oracle with Float32 input (tests/oracle_f32.cpp): lamejs's encodeBuffer given a Float32Array or a plain Array.

Test infrastructure only.  The library is the oracle's own sources plus oracle_f32.cpp, compiled once per process into a
temporary directory; the oracle's code is unchanged, and lj_encode (Int16) works in the same library, so one encoder can
mix Int16Array and Float32Array calls as a lamejs caller can."""
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


def _makefile_flags():
    """the oracle's own compiler flags (oracle/Makefile's CXXFLAGS), so that this build cannot drift from it"""
    for line in open(os.path.join(ORACLE, "Makefile")):
        if line.startswith("CXXFLAGS"):
            return [f for f in line.split("=", 1)[1].split() if not f.startswith("-W")] + ["-w"]
    raise RuntimeError("no CXXFLAGS in oracle/Makefile")


CXXFLAGS = _makefile_flags()

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(HERE, "oracle_f32.cpp")] + [os.path.join(ORACLE, s) for s in SRCS]
    h = hashlib.sha256()
    for p in srcs + [os.path.join(ORACLE, "lj_init.cpp"), os.path.join(ORACLE, "Makefile")] + [os.path.join(ORACLE, f) for f in sorted(os.listdir(ORACLE)) if f.endswith(".h")]:
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "mp3b200_oracle_f32_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "liboracle_f32.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = os.path.join(d, "liboracle_f32.%d.so" % os.getpid())
        subprocess.check_call(["g++"] + CXXFLAGS + ["-shared", "-o", tmp] + srcs + ["-lm"])
        os.replace(tmp, so)
    _lib = bind(so)
    return _lib


def bind(so):
    """the ctypes library of a build of oracle_f32.cpp with the oracle's sources (lib()'s, or another build of them)"""
    L = ctypes.CDLL(so)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.lj_create.restype = vp
    L.lj_create.argtypes = [ci] * 3
    L.lj_encode.argtypes = [vp, vp, vp, ci, vp, ci]
    L.lj_encode_f32.argtypes = [vp, vp, vp, ci, vp, ci]
    L.lj_flush.argtypes = [vp, vp, ci]
    L.lj_destroy.argtypes = [vp]
    L.lj_set_trace.argtypes = [vp, vp, ci]
    L.lj_set_quant_trace.argtypes = [vp, vp, ci]
    L.lj_trace_count.argtypes = [vp]
    L.lj_enable_vbr_tag.argtypes = [vp]
    L.lj_get_lametag_frame.argtypes = [vp, vp, ci]
    L.lj_get_scale.argtypes = [vp]
    L.lj_gain_clamps.argtypes = [vp]
    L.lj_get_scale.restype = ctypes.c_double
    L.lj_get_state.argtypes = [vp, vp]
    assert L.lj_trace_size() == oracle_lib.TRACE_DTYPE.itemsize
    assert L.lj_state_size() == oracle_lib.STATE_DTYPE.itemsize
    oracle_lib.bind_psy_trace(L)
    oracle_lib.bind_quant_row_trace(L)
    return L


def is_float(a):
    return a is not None and np.asarray(a).dtype.kind in "fc"


class Encoder:
    """Mp3Encoder of the oracle whose encode_buffer takes Int16 arrays (lj_encode) or floating arrays (lj_encode_f32: rounded
    to Float32 once, like lamejs's store)."""

    def __init__(self, channels, samplerate, kbps, trace_frames=0, write_vbr_tag=False, psy_trace=False):
        self.L = lib()
        self.h = self.L.lj_create(channels, samplerate, kbps)
        if not self.h:
            raise ValueError("unsupported configuration")
        self.channels = channels
        self.psy = oracle_lib.PsyTraceRows(self.L, self.h) if psy_trace else None
        self.tag_on = bool(write_vbr_tag) and self.L.lj_enable_vbr_tag(self.h) == 1
        self.trace, self.qtrace, self.qrtrace = oracle_lib.set_traces(self.L, self.h, trace_frames) if trace_frames else (None,) * 3

    def encode_buffer(self, left, right=None):
        if right is None or self.channels == 1:
            right = left
        f32 = is_float(left) or is_float(right)
        dt = np.float32 if f32 else np.int16
        left, right = np.ascontiguousarray(left, dtype=dt), np.ascontiguousarray(right, dtype=dt)
        cap = int(1.25 * len(left) + 7200) + 2880
        buf = np.empty(cap, dtype=np.uint8)
        if self.psy:
            self.psy.before_call(len(left) // 576 + 4)
        fn = self.L.lj_encode_f32 if f32 else self.L.lj_encode
        k = oracle_lib.check(fn(self.h, left.ctypes.data, right.ctypes.data, len(left), buf.ctypes.data, cap), "lj_encode")
        return buf[:k].tobytes()

    def flush(self):
        cap = 7200 + 4 * 1440 + 2880
        buf = np.empty(cap, dtype=np.uint8)
        if self.psy:
            self.psy.before_call(8)
        k = oracle_lib.check(self.L.lj_flush(self.h, buf.ctypes.data, cap), "lj_flush")
        return buf[:k].tobytes()

    def lametag_frame(self):
        buf = np.zeros(2880, dtype=np.uint8)
        k = self.L.lj_get_lametag_frame(self.h, buf.ctypes.data, 2880)
        return buf[:k].tobytes()

    def psy_traces(self):
        return self.psy.rows()

    def psy_block_traces(self):
        return self.psy.block_rows()

    def npart(self):
        return self.L.lj_psy_npart(self.h, 0), self.L.lj_psy_npart(self.h, 1)

    def state(self):
        """the state carried into the next call (oracle_lib.OracleEncoder.state)"""
        s = np.zeros((), dtype=oracle_lib.STATE_DTYPE)
        self.L.lj_get_state(self.h, s.ctypes.data)
        return s

    def traces(self):
        return oracle_lib.merged_traces(self.L, self.h, (self.trace, self.qtrace, self.qrtrace))

    def close(self):
        if self.h:
            self.L.lj_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def encode_calls(channels, samplerate, kbps, calls, trace_frames=0, write_vbr_tag=False):
    """encodeBuffer over `calls` (a list of (left, right) pairs, each Int16 or floating) + flush(); returns (bytes, per-call
    sizes, traces or None, tag frame)."""
    enc = Encoder(channels, samplerate, kbps, trace_frames, write_vbr_tag)
    out, sizes = bytearray(), []
    for left, right in calls:
        b = enc.encode_buffer(left, right)
        sizes.append(len(b))
        out += b
    b = enc.flush()
    sizes.append(len(b))
    out += b
    tr = enc.traces().copy() if trace_frames else None
    tag = enc.lametag_frame()
    enc.close()
    return bytes(out), sizes, tr, tag


def encode_stream(channels, samplerate, kbps, left, right=None, chunk=None, trace_frames=0):
    """encodeBuffer(whole stream or chunks of `chunk`) + flush(); returns (bytes, per-call sizes, traces)."""
    n = len(left)
    step = chunk or max(n, 1)
    calls = [(left[i:i + step], None if right is None else right[i:i + step]) for i in range(0, n, step)]
    b, sizes, tr, _ = encode_calls(channels, samplerate, kbps, calls, trace_frames)
    return b, sizes, tr
