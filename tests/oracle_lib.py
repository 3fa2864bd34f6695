"""ctypes binding of the CPU oracle (oracle/liblamejs_oracle.so).  Test infrastructure only:
imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg -- never by the product."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_SO = os.path.join(ORACLE_DIR, "liblamejs_oracle.so")
TABLES_H = os.path.join(ORACLE_DIR, "lj_tables.h")

SBMAX_l, SBMAX_s, SFBMAX = 22, 13, 39

TRACE_DTYPE = np.dtype(
    [
        ("xr", np.float32, (2, 2, 576)),
        ("en_l", np.float32, (2, 2, SBMAX_l)),
        ("thm_l", np.float32, (2, 2, SBMAX_l)),
        ("en_s", np.float32, (2, 2, SBMAX_s, 3)),
        ("thm_s", np.float32, (2, 2, SBMAX_s, 3)),
        ("blocktype", np.int32, (2, 2)),
        ("ath_adjust", np.float64),
        ("l3_enc", np.int32, (2, 2, 576)),
        ("global_gain", np.int32, (2, 2)),
        ("part2_3_length", np.int32, (2, 2)),
        ("part2_length", np.int32, (2, 2)),
        ("big_values", np.int32, (2, 2)),
        ("count1", np.int32, (2, 2)),
        ("scalefac", np.int32, (2, 2, SFBMAX)),
        ("scalefac_compress", np.int32, (2, 2)),
        ("table_select", np.int32, (2, 2, 3)),
        ("region0", np.int32, (2, 2)),
        ("region1", np.int32, (2, 2)),
        ("preflag", np.int32, (2, 2)),
        ("scalefac_scale", np.int32, (2, 2)),
        ("count1table", np.int32, (2, 2)),
        ("subblock_gain", np.int32, (2, 2, 3)),
        ("scfsi", np.int32, (2, 4)),
        ("frame_bytes", np.int32),
        ("padding", np.int32),
        ("old_value_in", np.int32, (2,)),
        ("old_value_out", np.int32, (2,)),
        ("cur_step_in", np.int32, (2,)),
        ("cur_step_out", np.int32, (2,)),
    ],
    align=True,
)

# lj_set_quant_trace: the quantizer's inputs, one row per TRACE_DTYPE row
QTRACE_DTYPE = np.dtype(
    [
        ("xmin", np.float32, (2, 2, SFBMAX)),             # calc_xmin's output as outer_loop receives it (psymax bands)
        ("max_nonzero_coeff", np.int32, (2, 2)),
        ("xrpow_max", np.float64, (2, 2)),                # after init_xrpow, before the rate loop
        ("old_value_mid", np.int32, (2,)),                # MPEG-1: the state gr1's search starts from (0 for LSF)
        ("cur_step_mid", np.int32, (2,)),
    ],
    align=True,
)

# lj_set_quant_row_trace: beside each QTRACE_DTYPE row, the rows lj_iteration_loop hands outer_loop
QROW_TRACE_DTYPE = np.dtype(
    [
        ("xrq", np.float32, (2, 2, 576)),                 # cod_info.xr as outer_loop receives it (short blocks reordered,
                                                          # analog silence zeroed)
        ("xrpow", np.float32, (2, 2, 576)),               # init_xrpow's rows
        ("have", np.int32, (2, 2)),                       # init_xrpow's result: the granule has energy
    ],
    align=True,
)

# lj_set_psy_trace: the psy model's per-granule analysis, one row per frame, [gr][ch] = psy call G k + gr of frame k; only the
# first npart_l / npart_s partitions are defined
PSY_TRACE_DTYPE = np.dtype(
    [
        ("eb_l", np.float32, (2, 2, 64)),                 # calc_energy
        ("peaks", np.float32, (2, 2, 9)),                 # en_subshort[3..11]: max(1, |high-pass|) per 64 samples
        ("loudness", np.float32, (2, 2)),                 # loudness_sq_save after the call
        ("eb_s", np.float32, (2, 2, 3, 64)),              # compute_masking_s per short block: partition energies
        ("ecb_s", np.float32, (2, 2, 3, 64)),             # ... and the spreading sum stored into nb_s1
        ("mask_idx_l", np.int32, (2, 2, 64)),             # calc_mask_index_l
        ("attack", np.int32, (2, 2, 4)),                  # ns_attacks after the ratio < 1.7 pass, before the lastAttacks rule
    ],
    align=True,
)

# lj_set_psy_block_trace: beside each psy row, blocktype_old as each psy call found it ([gr][ch]), before block_type_set
PSY_BLOCK_TRACE_DTYPE = np.dtype([("blocktype_old", np.int32, (2, 2))])

# what OracleEncoder.traces() returns: the fields of the three records
FULL_TRACE_DTYPE = np.dtype([(n, d.fields[n][0]) for d in (TRACE_DTYPE, QTRACE_DTYPE, QROW_TRACE_DTYPE) for n in d.names])

# lj_get_state: what an encoder carries from one call to the next
STATE_DTYPE = np.dtype(
    [
        ("ath_adjust", np.float64),
        ("ath_adjust_limit", np.float64),
        ("blocktype_old", np.int32, (2,)),
        ("last_attacks", np.int32, (2,)),
        ("old_value", np.int32, (2,)),
        ("current_step", np.int32, (2,)),
        ("frames_done", np.int32),
        ("mf_size", np.int32),
        ("mf_samples_to_encode", np.int32),
        ("pad_", np.int32),
        ("en_l", np.float32, (2, SBMAX_l)),               # gfc.en / gfc.thm: the masking handed to the next granule
        ("thm_l", np.float32, (2, SBMAX_l)),
        ("en_s", np.float32, (2, SBMAX_s, 3)),
        ("thm_s", np.float32, (2, SBMAX_s, 3)),
    ],
    align=True,
)

_lib = None


def build():
    import fcntl
    with open(os.path.join(ORACLE_DIR, ".build.lock"), "w") as lk:   # pytest-xdist workers build once, in turn
        fcntl.flock(lk, fcntl.LOCK_EX)
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_SO):
            build()
        L = ctypes.CDLL(ORACLE_SO)
        L.lj_create.restype = ctypes.c_void_p
        L.lj_create.argtypes = [ctypes.c_int] * 3
        L.lj_encode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.lj_flush.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.lj_destroy.argtypes = [ctypes.c_void_p]
        L.lj_set_trace.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.lj_trace_count.argtypes = [ctypes.c_void_p]
        L.lj_query_out_samplerate.argtypes = [ctypes.c_int] * 3
        L.lj_enable_vbr_tag.argtypes = [ctypes.c_void_p]
        L.lj_enable_reservoir.argtypes = [ctypes.c_void_p]
        L.lj_enable_joint_stereo.argtypes = [ctypes.c_void_p]
        L.lj_enable_reservoir_integer_bytes.argtypes = [ctypes.c_void_p]
        L.lj_music_crc.argtypes = [ctypes.c_void_p]
        L.lj_bytes_written.argtypes = [ctypes.c_void_p]
        L.lj_bytes_written.restype = ctypes.c_longlong
        L.lj_vbr_frames.argtypes = [ctypes.c_void_p]
        L.lj_encoder_padding.argtypes = [ctypes.c_void_p]
        L.lj_get_lametag_frame.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.lj_crc16.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int]
        L.lj_wav_read_header.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
        L.lj_get_state.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.lj_set_quant_trace.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        assert L.lj_trace_size() == TRACE_DTYPE.itemsize, (L.lj_trace_size(), TRACE_DTYPE.itemsize)
        assert L.lj_quant_trace_size() == QTRACE_DTYPE.itemsize, (L.lj_quant_trace_size(), QTRACE_DTYPE.itemsize)
        assert L.lj_state_size() == STATE_DTYPE.itemsize, (L.lj_state_size(), STATE_DTYPE.itemsize)
        bind_psy_trace(L)
        bind_quant_row_trace(L)
        _lib = L
    return _lib


def bind_quant_row_trace(L):
    """ctypes signature of the quantizer's row trace (the oracle's library or the Float32 build of its sources)"""
    L.lj_set_quant_row_trace.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    assert L.lj_quant_row_trace_size() == QROW_TRACE_DTYPE.itemsize, (L.lj_quant_row_trace_size(), QROW_TRACE_DTYPE.itemsize)


def set_traces(L, h, trace_frames):
    """the frame, quantizer and quantizer row traces of encoder h, trace_frames rows each (the three records of traces())"""
    recs = (np.zeros(trace_frames, dtype=TRACE_DTYPE), np.zeros(trace_frames, dtype=QTRACE_DTYPE),
            np.zeros(trace_frames, dtype=QROW_TRACE_DTYPE))
    L.lj_set_trace(h, recs[0].ctypes.data, trace_frames)
    L.lj_set_quant_trace(h, recs[1].ctypes.data, trace_frames)
    L.lj_set_quant_row_trace(h, recs[2].ctypes.data, trace_frames)
    return recs


def merged_traces(L, h, recs):
    """the traced frames so far: FULL_TRACE_DTYPE rows (the records of set_traces side by side)"""
    n = L.lj_trace_count(h)
    out = np.empty(n, dtype=FULL_TRACE_DTYPE)
    for rec in recs:
        for k in rec.dtype.names:
            out[k] = rec[k][:n]
    return out


def bind_psy_trace(L):
    """ctypes signatures of the psy trace (the oracle's library or the Float32 build of its sources)"""
    vp = ctypes.c_void_p
    L.lj_set_psy_trace.argtypes = [vp, vp, ctypes.c_int]
    L.lj_psy_trace_count.argtypes = [vp]
    L.lj_psy_attack_threshold.argtypes = [vp]
    L.lj_psy_attack_threshold.restype = ctypes.c_double
    L.lj_ath_aa_sensitivity.argtypes = [vp]
    L.lj_ath_aa_sensitivity.restype = ctypes.c_double
    L.lj_psy_npart.argtypes = [vp, ctypes.c_int]
    L.lj_set_psy_block_trace.argtypes = [vp, vp, ctypes.c_int]
    assert L.lj_psy_trace_size() == PSY_TRACE_DTYPE.itemsize, (L.lj_psy_trace_size(), PSY_TRACE_DTYPE.itemsize)
    assert L.lj_psy_block_trace_size() == PSY_BLOCK_TRACE_DTYPE.itemsize, (L.lj_psy_block_trace_size(), PSY_BLOCK_TRACE_DTYPE.itemsize)


class PsyTraceRows:
    """The psy trace of one encoder and the block types beside it, growing across its calls (lj_set_psy_trace,
    lj_set_psy_block_trace); shared by OracleEncoder and oracle_f32."""

    def __init__(self, L, h, cap=64):
        self.L, self.h = L, h
        self.done, self.bt_done = [], []
        self._set(cap)

    def _set(self, cap):
        self.buf = np.zeros(cap, dtype=PSY_TRACE_DTYPE)
        self.bt_buf = np.zeros(cap, dtype=PSY_BLOCK_TRACE_DTYPE)
        self.L.lj_set_psy_trace(self.h, self.buf.ctypes.data, cap)
        self.L.lj_set_psy_block_trace(self.h, self.bt_buf.ctypes.data, cap)

    def before_call(self, max_frames):
        """room for max_frames more rows: rows already written move to `done` and the buffers start over"""
        n = self.L.lj_psy_trace_count(self.h)
        if n + max_frames > len(self.buf):
            self.done.append(self.buf[:n].copy())
            self.bt_done.append(self.bt_buf[:n].copy())
            self._set(max(max_frames, 64))

    def rows(self):
        n = self.L.lj_psy_trace_count(self.h)
        return np.concatenate(self.done + [self.buf[:n]])

    def block_rows(self):
        """blocktype_old [frame][gr][ch] of every psy row"""
        n = self.L.lj_psy_trace_count(self.h)
        return np.concatenate(self.bt_done + [self.bt_buf[:n]])["blocktype_old"]


ERR_BITSTREAM = -10          # LJ_ERR_BITSTREAM (oracle/lj_encoder.h)


class LamejsThrows(RuntimeError):
    """The call in which lamejs throws, and every later one: format_bitstream's consistency check failed because a frame's
    bits do not fit its slot (BitStream.js:856-885 reports through System.err, which lamejs does not define)."""


def check(k, what):
    """k from lj_encode / lj_encode_f32 / lj_flush: raises on an error, else returns k"""
    if k == ERR_BITSTREAM:
        raise LamejsThrows("%s: frame over its bit budget (lamejs throws)" % what)
    if k < 0:
        raise RuntimeError("%s error %d" % (what, k))
    return k


def out_samplerate(channels, samplerate, kbps):
    """Output sample rate lame_init_params picks (Lame.js:285-364): != samplerate means lamejs resamples."""
    return lib().lj_query_out_samplerate(channels, samplerate, kbps)


class OracleEncoder:
    """Mirror of lamejs.Mp3Encoder (src/js/index.js:66-136) backed by the C++ restatement."""

    def __init__(self, channels, samplerate, kbps, trace_frames=0, write_vbr_tag=False, reservoir=False, joint_stereo=False,
                 psy_trace=False):
        self.L = lib()
        self.h = self.L.lj_create(channels, samplerate, kbps)
        if not self.h:
            raise ValueError("unsupported configuration")
        self.channels = channels
        self.psy = PsyTraceRows(self.L, self.h) if psy_trace else None
        if joint_stereo:                   # gfp.mode = JOINT_STEREO (SURVEY 8(f2); Mp3Encoder uses STEREO)
            assert self.L.lj_enable_joint_stereo(self.h) == 0
        if reservoir == "java":            # NOT lamejs: integer byte counts as in Reservoir.java (decodable streams)
            assert self.L.lj_enable_reservoir_integer_bytes(self.h) == 0
        elif reservoir:                    # gfp.disable_reservoir = false (SURVEY 8(f2); Mp3Encoder never does this)
            assert self.L.lj_enable_reservoir(self.h) == 0
        self.tag_on = bool(write_vbr_tag) and self.L.lj_enable_vbr_tag(self.h) == 1   # gfp.bWriteVbrTag (InitVbrTag may refuse)
        self.trace, self.qtrace, self.qrtrace = set_traces(self.L, self.h, trace_frames) if trace_frames else (None,) * 3

    def encode_buffer(self, left, right=None):
        left = np.ascontiguousarray(left, dtype=np.int16)
        right = left if (right is None or self.channels == 1) else np.ascontiguousarray(right, dtype=np.int16)
        assert len(left) == len(right)
        cap = int(1.25 * len(left) + 7200)
        buf = np.empty(cap, dtype=np.uint8)
        if self.psy:
            self.psy.before_call(len(left) // 576 + 4)
        k = check(self.L.lj_encode(self.h, left.ctypes.data, right.ctypes.data, len(left), buf.ctypes.data, cap), "lj_encode")
        return buf[:k].tobytes()

    def flush(self):
        cap = 7200 + 4 * 1440
        buf = np.empty(cap, dtype=np.uint8)
        if self.psy:
            self.psy.before_call(8)
        k = check(self.L.lj_flush(self.h, buf.ctypes.data, cap), "lj_flush")
        return buf[:k].tobytes()

    def traces(self):
        """the traced frames so far: FULL_TRACE_DTYPE rows (the frame trace and the quantizer traces side by side)"""
        return merged_traces(self.L, self.h, (self.trace, self.qtrace, self.qrtrace))

    def psy_traces(self):
        """every psy row since the encoder was made (PSY_TRACE_DTYPE, one per frame), across all calls"""
        return self.psy.rows()

    def psy_block_traces(self):
        """blocktype_old as each psy call found it, int32 [frame][gr][ch], beside psy_traces()"""
        return self.psy.block_rows()

    def attack_threshold(self):
        return self.L.lj_psy_attack_threshold(self.h)

    def ath_aa_sensitivity(self):
        return self.L.lj_ath_aa_sensitivity(self.h)

    def npart(self):
        """(npart_l, npart_s): the defined prefix of the psy trace's partition rows"""
        return self.L.lj_psy_npart(self.h, 0), self.L.lj_psy_npart(self.h, 1)

    def state(self):
        """The state carried into the next call: one STATE_DTYPE record (ATH adjust and its limit, blocktype_old,
        lastAttacks, OldValue, CurrentStep, frames done, the mfbuf fill level and samples to encode, and gfc.en / gfc.thm)."""
        s = np.zeros((), dtype=STATE_DTYPE)
        self.L.lj_get_state(self.h, s.ctypes.data)
        return s

    # gfc.nMusicCRC / VBR_seek_table.nBytesWritten: kept by copy_buffer on every call (BitStream.js:924-935)
    def music_crc(self):
        return self.L.lj_music_crc(self.h)

    def bytes_written(self):
        return self.L.lj_bytes_written(self.h)

    def vbr_frames(self):
        return self.L.lj_vbr_frames(self.h)

    def encoder_padding(self):
        return self.L.lj_encoder_padding(self.h)

    def lametag_frame(self):
        """VBRTag.getLameTagFrame: b'' when the tag is off."""
        buf = np.zeros(2880, dtype=np.uint8)
        k = self.L.lj_get_lametag_frame(self.h, buf.ctypes.data, 2880)
        return buf[:k].tobytes()

    def close(self):
        if self.h:
            self.L.lj_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def encode_stream(channels, samplerate, kbps, left, right=None, chunk=None, trace_frames=0):
    """encodeBuffer(whole stream or chunks) + flush(); returns (bytes, per-call sizes, traces)."""
    enc = OracleEncoder(channels, samplerate, kbps, trace_frames)
    out, sizes = bytearray(), []
    n = len(left)
    step = chunk or max(n, 1)
    for i in range(0, n, step):
        b = enc.encode_buffer(left[i : i + step], None if right is None else right[i : i + step])
        sizes.append(len(b))
        out += b
    b = enc.flush()
    sizes.append(len(b))
    out += b
    tr = enc.traces().copy() if trace_frames else None
    enc.close()
    return bytes(out), sizes, tr


def crc16(data, crc=0):
    """CRC-16 of VBRTag.js:547-556 (reflected 0xA001, start value `crc`)."""
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    return lib().lj_crc16(a.ctypes.data if len(a) else None, len(a), crc)


def wav_read_header(data):
    """WavHeader.readHeader (index.js:154-193): dict, None (`return undefined`), or raises like the reference throws."""
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    out = (ctypes.c_longlong * 4)()
    rc = lib().lj_wav_read_header(a.ctypes.data if len(a) else None, len(a), out)
    if rc == 0:
        return None
    if rc == -1:
        raise ValueError("extended fmt chunk not implemented")
    if rc == -2:
        raise IndexError("read past the end of the buffer")
    return {"dataOffset": out[0], "dataLen": out[1], "channels": out[2], "sampleRate": out[3]}


def encode_stream_tagged(channels, samplerate, kbps, left, right=None, chunk=None):
    """Like encode_stream with gfp.bWriteVbrTag = true: the first call's bytes start with the placeholder frame
    (InitVbrTag); returns (bytes, per-call sizes, info) with info = tag frame, music CRC, byte / frame counts, padding."""
    enc = OracleEncoder(channels, samplerate, kbps, write_vbr_tag=True)
    out, sizes = bytearray(), []
    n = len(left)
    step = chunk or max(n, 1)
    for i in range(0, n, step):
        b = enc.encode_buffer(left[i : i + step], None if right is None else right[i : i + step])
        sizes.append(len(b))
        out += b
    b = enc.flush()
    sizes.append(len(b))
    out += b
    info = {"tag_on": enc.tag_on, "tag": enc.lametag_frame(), "music_crc": enc.music_crc(), "bytes_written": enc.bytes_written(),
            "frames": enc.vbr_frames(), "encoder_padding": enc.encoder_padding()}
    enc.close()
    return bytes(out), sizes, info
