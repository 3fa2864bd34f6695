"""Seeded call schedules for the streaming handle API (mp3b200_encode / _flush / _encode_batch / _flush_batch / _export_state /
_import_state), their expected results from the oracle, and a runner that plays them on the library.

A schedule drives K logical streams of one configuration.  Its operations are single encode and flush calls, batch calls over
random subsets (a stream may occur more than once, NULL handles occur), export -> import into a fresh handle -> destroy of
the old one in the middle of a stream, and calls whose output buffer is deliberately one byte long.  Some streams carry the
Xing / Info tag.  The sizes of the calls are where the handle's bookkeeping turns: 0, 1 and 2 samples, around a granule
(575..577), a frame (1151..1153) and the first frame's fill level (1328, 1329), framesize * k +- 1, and up to 200 frames at
once.  The signals (click trains, loud/silent alternation, bursts, ...) put call boundaries inside short-block runs and ATH
decay.

The expected bytes of every call come from one OracleEncoder per logical stream that replays that stream's calls in order,
which is how include/mp3b200.h defines a batch call.  A call that fails for a too small buffer hands out nothing and keeps
its frames: the stream's next call returns them in front of its own.  After every operation the runner also compares the
state blob of each stream it named -- header and halo, including after hand-overs and flushes -- with that stream's
OracleEncoder.state().  tests/test_gpu_handle_soak.py and
tests/speculation_worker.py run schedules on the GPU; tests/test_handle_schedule_cpu.py checks what they reach."""
import ctypes
from collections import namedtuple

import numpy as np

import edge_signals
import oracle_lib
from synth import make_signal

ERR_BUFFER, ERR_HANDLE = -1, -3
START, SHORT = 1, 2

# the configurations of tests/test_gpu_handle_soak.py: MPEG-1 stereo / mono, MPEG-2 stereo, MPEG-2.5 mono
CONFIGS = [(2, 44100, 128), (1, 48000, 320), (2, 22050, 64), (1, 8000, 16)]

SMALL_SIZES = [0, 1, 2, 575, 576, 577, 1151, 1152, 1153, 1328, 1329]
EDGE_KINDS = ["clicks1", "clicks2", "clicks3", "clicks5", "click_pairs", "loud_silent", "square", "lsb_dither"]
SYNTH_KINDS = ["burst", "noise", "sweep", "octave", "sine", "silence", "white"]

# one entry of a call: logical stream s (None: a NULL handle), its samples [lo, hi) (encode only), and whether the call gets
# a one-byte output buffer
Call = namedtuple("Call", "s lo hi fail")


def framesize(sr):
    return 1152 if sr >= 32000 else 576


class Schedule:
    def __init__(self, cfg, signals, kinds, tagged, ops):
        self.cfg, self.signals, self.kinds, self.tagged, self.ops = cfg, signals, kinds, tagged, ops
        self.fs = framesize(cfg[1])

    @property
    def nstreams(self):
        return len(self.signals)


def make_schedule(cfg, nstreams, nops, seed, big=0.03, p_fail=0.06):
    """A seeded schedule of `nops` operations over `nstreams` logical streams, ended by a flush of every stream.  `big` is the
    share of calls that carry up to 200 frames at once; `p_fail` the share of calls on untagged streams given a one-byte
    buffer."""
    ch, sr, kbps = cfg
    fs = framesize(sr)
    rng = np.random.default_rng(seed)
    K = nstreams
    tagged = {s for s in range(K) if s % 8 == 5}
    flushable = [s for s in range(K) if s % 4 != 0]     # the others are flushed only at the end: one encodeBuffer stream each
    pos = [0] * K
    ops = []

    def size():
        u = rng.random()
        if u < 0.5:
            return int(rng.choice(SMALL_SIZES))
        if u < 1.0 - big:
            return fs * int(rng.integers(1, 17)) + int(rng.integers(-1, 2))
        return int(rng.integers(fs, 200 * fs + 1))

    def fail(s):
        return s not in tagged and rng.random() < p_fail

    def enc(s):
        n = size()
        c = Call(s, pos[s], pos[s] + n, fail(s))
        pos[s] += n
        return c

    def members(pool):
        """a random subset of `pool` in random order, some streams twice, sometimes a NULL handle"""
        sub = [int(s) for s in rng.choice(pool, min(int(rng.integers(2, 13)), len(pool)), replace=False)]
        sub += [s for s in sub if rng.random() < 0.2]
        if rng.random() < 0.15:
            sub.append(None)
        rng.shuffle(sub)
        return sub

    for _ in range(nops):
        u = rng.random()
        if u < 0.30:
            ops.append(("encode", [enc(int(rng.integers(K)))]))
        elif u < 0.72:
            ops.append(("encode_batch", [enc(s) if s is not None else Call(None, 0, 0, False) for s in members(list(range(K)))]))
        elif u < 0.80:
            s = int(rng.choice(flushable))
            ops.append(("flush", [Call(s, 0, 0, fail(s))]))
        elif u < 0.87:
            ops.append(("flush_batch", [Call(s, 0, 0, s is not None and fail(s)) for s in members(flushable)]))
        else:
            s = int(rng.integers(K))
            if s not in tagged:                   # the tag describes a whole stream and is not part of the state blob
                ops.append(("handover", [Call(s, 0, 0, False)]))
    last = list(range(K)) + [int(s) for s in rng.choice(K, 2, replace=False)]
    rng.shuffle(last)
    ops.append(("flush_batch", [Call(s, 0, 0, False) for s in last]))

    signals, kinds = [], []
    for s in range(K):
        n = max(pos[s], 1)
        kind = (EDGE_KINDS + SYNTH_KINDS)[(s + seed) % (len(EDGE_KINDS) + len(SYNTH_KINDS))]
        l, r = edge_signals.make(kind, n, sr, fs) if kind in EDGE_KINDS else make_signal(kind, n, sr, seed * 64 + s)
        signals.append((np.ascontiguousarray(l), np.ascontiguousarray(r) if ch == 2 else None))
        kinds.append(kind)
    return Schedule(cfg, signals, kinds, tagged, ops)


class Expected:
    """What a schedule must produce.  results[i][j]: bytes, or the negative error, of entry j of operation i (None for a
    hand-over).  raw[s]: the oracle's bytes of stream s call by call (including those a failed call held back).  epochs[s]:
    the sample ranges of stream s that a flush ended.  tags[s]: tag_on, tag frame, music CRC and bytes written after the last
    flush.  states[i]: {s: OracleEncoder.state()} after operation i for every stream it names.  With tracing, calls lists
    (s, frames the call completed, block types of its last granule) for every oracle call."""


def replay(sched, trace=False):
    ch, sr, kbps = sched.cfg
    K = sched.nstreams
    G = 2 if sr >= 32000 else 1
    nflush = [0] * K
    for _, entries in sched.ops:
        for c in entries:
            if c.s is not None:
                nflush[c.s] += 1
    encs = []
    for s in range(K):
        tf = len(sched.signals[s][0]) // sched.fs + 8 * nflush[s] + 16 if trace else 0
        encs.append(oracle_lib.OracleEncoder(ch, sr, kbps, trace_frames=tf, write_vbr_tag=s in sched.tagged))
    ex = Expected()
    ex.results, ex.calls = [], []
    ex.raw = [bytearray() for _ in range(K)]
    ex.epochs = [[] for _ in range(K)]
    epoch_lo = [0] * K
    backlog = [b""] * K

    def oracle_call(kind, c):
        e = encs[c.s]
        before = e.L.lj_trace_count(e.h) if trace else 0
        if kind.startswith("flush"):
            b = e.flush()
        else:
            l, r = sched.signals[c.s]
            b = e.encode_buffer(l[c.lo:c.hi], None if r is None else r[c.lo:c.hi]) if c.hi > c.lo else b""
        if trace:
            after = e.L.lj_trace_count(e.h)
            bt = tuple(int(x) for x in e.trace[after - 1]["blocktype"][G - 1][:ch]) if after > before else ()
            ex.calls.append((c.s, after - before, bt))
        ex.raw[c.s] += b
        return b

    pos = [0] * K
    ex.states = []
    for kind, entries in sched.ops:
        # what each stream the operation touches carries into its next call, after the operation
        ex.states.append({c.s: None for c in entries if c.s is not None})
        if kind == "handover":
            ex.results.append([None])
            ex.states[-1] = {s: encs[s].state() for s in ex.states[-1]}
            continue
        res = []
        for c in entries:
            if c.s is None:
                res.append(ERR_HANDLE)
                continue
            if kind.startswith("encode"):
                assert c.lo == pos[c.s]
                pos[c.s] = c.hi
            b = oracle_call(kind, c)
            if kind.startswith("flush"):
                ex.epochs[c.s].append((epoch_lo[c.s], pos[c.s]))
                epoch_lo[c.s] = pos[c.s]
            total = backlog[c.s] + b
            if c.fail and len(total) >= 2:
                res.append(ERR_BUFFER)
                backlog[c.s] = total
            else:
                res.append(total)
                backlog[c.s] = b""
        ex.results.append(res)
        ex.states[-1] = {s: encs[s].state() for s in ex.states[-1]}
    assert not any(backlog), "the schedule's last flush must deliver everything"
    ex.tags = [{"tag_on": e.tag_on, "tag": e.lametag_frame(), "music_crc": e.music_crc(), "bytes_written": e.bytes_written()}
               for e in encs]
    ex.raw = [bytes(b) for b in ex.raw]
    for e in encs:
        e.close()
    return ex


def reached(sched, ex):
    """Counts of the events a schedule exists to reach (needs replay(..., trace=True))."""
    frames = [f for _, f, _ in ex.calls]
    out = {
        "frames": int(sum(frames)),
        "calls": len(frames),
        "calls_0_frames": sum(f == 0 for f in frames),
        "calls_1_frame": sum(f == 1 for f in frames),
        "calls_16plus_frames": sum(f >= 16 for f in frames),
        "after_start": sum(f > 0 and START in bt for _, f, bt in ex.calls),
        "after_short": sum(f > 0 and SHORT in bt for _, f, bt in ex.calls),
        "handovers": sum(k == "handover" for k, _ in sched.ops),
        "repeated_batches": 0, "null_entries": 0, "injected_failures": 0, "flush_then_reuse": 0,
    }
    fed_after_flush = [False] * sched.nstreams
    for (kind, entries), res in zip(reversed(sched.ops), reversed(ex.results)):
        ss = [c.s for c in entries if c.s is not None]
        if kind.endswith("batch") and len(ss) != len(set(ss)):
            out["repeated_batches"] += 1
        out["null_entries"] += len(entries) - len(ss)
        out["injected_failures"] += sum(r == ERR_BUFFER for r in res)
        for c in entries:
            if c.s is None:
                continue
            if kind.startswith("encode") and c.hi > c.lo:
                fed_after_flush[c.s] = True
            elif kind.startswith("flush") and fed_after_flush[c.s]:
                out["flush_then_reuse"] += 1
                fed_after_flush[c.s] = False
    return out


# ---- the library side ----

# StateBlobHeader (lamejs_b200/csrc/mp3_handle.inc), followed by the halo (per channel the PsyRatioDev row en_l[22],
# thm_l[22], en_s[13][3], thm_s[13][3]) once a frame has been encoded, then the retained PCM
BLOB_HEADER = np.dtype([("magic", "<u4"), ("channels", "<i4"), ("samplerate", "<i4"), ("kbps", "<i4"),
                        ("frames_pending", "<i4"), ("mf_size", "<i4"), ("mf_samples_to_encode", "<i4"), ("halo_floats", "<i4"),
                        ("hist_base", "<i8"), ("fed", "<i8"), ("frames_done", "<i8"), ("pcm_samples", "<i8"),
                        ("ath_adjust", "<f8"), ("ath_adjust_limit", "<f8"), ("blocktype_old", "<i4", (2,)),
                        ("last_attacks", "<i4", (2,)), ("old_value", "<i4", (2,)), ("current_step", "<i4", (2,))])


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32) if a.dtype.kind == "f" else a


def blob_state_diff(blob, st, nch):
    """Names of the fields in which a handle's exported state blob differs from the oracle's state `st` (OracleEncoder.state())
    for the same stream after the same calls.  Floats are compared as bit patterns.  A handle whose last call failed still
    holds frames the oracle has encoded (frames_pending > 0): its fill level must agree, its sequential state is checked after
    the call that delivers them."""
    h = np.frombuffer(bytes(blob[:BLOB_HEADER.itemsize]), dtype=BLOB_HEADER)[0]
    bad = []
    if h["frames_done"] + h["frames_pending"] != st["frames_done"]:
        bad.append("frames_done")
    for k in ("mf_size", "mf_samples_to_encode"):
        if h[k] != st[k]:
            bad.append(k)
    if h["frames_pending"] > 0:
        return bad
    for k in ("ath_adjust", "ath_adjust_limit"):
        if _bits(h[k]) != _bits(st[k]):
            bad.append(k)
    for k in ("blocktype_old", "last_attacks", "old_value", "current_step"):
        if not np.array_equal(h[k][:nch], st[k][:nch]):
            bad.append(k)
    if h["frames_done"] > 0:
        if h["halo_floats"] != nch * 122:
            return bad + ["halo_floats"]
        halo = np.frombuffer(bytes(blob[BLOB_HEADER.itemsize:BLOB_HEADER.itemsize + 4 * nch * 122]), dtype="<f4").reshape(nch, 122)
        want = np.concatenate([st["en_l"][:nch], st["thm_l"][:nch], st["en_s"][:nch].reshape(nch, 39),
                               st["thm_s"][:nch].reshape(nch, 39)], axis=1)
        if not np.array_equal(_bits(halo), _bits(want)):
            bad.append("halo (en/thm handed to the next granule)")
    return bad


def export_blob(L, h):
    n = L.mp3b200_export_state(h, None, 0)
    blob = np.empty(n, dtype=np.uint8)
    assert L.mp3b200_export_state(h, blob.ctypes.data, n) == n
    return blob


SENTINEL = 0xA5
TAIL = 16               # sentinel bytes behind every output buffer


def _buffer(want):
    """(buffer, cap) for an entry expecting `want`: exactly the expected size, or one byte for an injected failure"""
    cap = 1 if not isinstance(want, bytes) else max(len(want), 1)
    return np.full(cap + TAIL, SENTINEL, dtype=np.uint8), cap


def _got(buf, cap, n, want):
    """the entry's bytes, or its error, checked for writes past the end of what it handed out"""
    if n < 0:
        if (buf != SENTINEL).any():
            return "wrote into the buffer of a failed call"
        return n
    if (buf[cap:] != SENTINEL).any():
        return "wrote past the end of its buffer"
    return buf[:n].tobytes()


def run(M, sched, ex):
    """Plays `sched` on the library through the C ABI; returns a list of what differed from `ex` (empty: all equal)."""
    L = M.lib()
    ch, sr, kbps = sched.cfg
    vp = ctypes.c_void_p
    fails = []

    def create(s):
        h = vp()
        assert L.mp3b200_create(ch, sr, kbps, ctypes.byref(h)) == 0
        if s in sched.tagged:
            assert L.mp3b200_set_write_vbr_tag(h, 1) == int(ex.tags[s]["tag_on"])
        return h

    hs = [create(s) for s in range(sched.nstreams)]

    def check_states(i, kind):
        """the state every stream named by operation i carries into its next call equals the oracle's"""
        for s, st in ex.states[i].items():
            bad = blob_state_diff(export_blob(L, hs[s]), st, ch)
            if bad:
                fails.append("op %d %s: state of stream %d differs in %s" % (i, kind, s, ", ".join(bad)))

    for i, ((kind, entries), want) in enumerate(zip(sched.ops, ex.results)):
        if kind == "handover":
            s = entries[0].s
            blob = export_blob(L, hs[s])
            h = create(s)
            if L.mp3b200_import_state(h, blob.ctypes.data, len(blob)) != 0:
                fails.append("op %d: import_state refused a blob of stream %d" % (i, s))
            L.mp3b200_destroy(hs[s])
            hs[s] = h
            check_states(i, kind)
            continue
        m = len(entries)
        bufs = [_buffer(w) for w in want]
        got = np.zeros(m, dtype=np.int32)
        ls, rs = [], []
        for c in entries:
            l, r = sched.signals[c.s] if c.s is not None else (None, None)
            ls.append(np.ascontiguousarray(l[c.lo:c.hi]) if c.s is not None and c.hi > c.lo else None)
            rs.append(np.ascontiguousarray(r[c.lo:c.hi]) if r is not None and c.hi > c.lo else None)
        ptr = lambda a: a.ctypes.data if a is not None else None     # noqa: E731
        if kind == "encode":
            c = entries[0]
            got[0] = L.mp3b200_encode(hs[c.s], ptr(ls[0]), ptr(rs[0]), c.hi - c.lo, bufs[0][0].ctypes.data, bufs[0][1])
        elif kind == "flush":
            got[0] = L.mp3b200_flush(hs[entries[0].s], bufs[0][0].ctypes.data, bufs[0][1])
        else:
            hp = (vp * m)(*[hs[c.s].value if c.s is not None else None for c in entries])
            op = (vp * m)(*[b.ctypes.data for b, _ in bufs])
            caps = np.array([cap for _, cap in bufs], dtype=np.int32)
            if kind == "encode_batch":
                lp = (vp * m)(*[ptr(a) for a in ls])
                rp = (vp * m)(*[ptr(a) for a in rs]) if ch == 2 else None
                ns = np.array([c.hi - c.lo for c in entries], dtype=np.int32)
                rc = L.mp3b200_encode_batch(hp, lp, rp, ns.ctypes.data, op, caps.ctypes.data, m, got.ctypes.data)
            else:
                rc = L.mp3b200_flush_batch(hp, op, caps.ctypes.data, m, got.ctypes.data)
            if rc != 0:
                fails.append("op %d %s: call returned %d (%s)" % (i, kind, rc, L.mp3b200_last_error().decode()))
                break
        for j, (c, w) in enumerate(zip(entries, want)):
            g = _got(bufs[j][0], bufs[j][1], int(got[j]), w)
            if g != w:
                what = g if isinstance(g, str) else ("%d bytes" % len(g) if isinstance(g, bytes) else "error %d" % g)
                wwhat = "%d bytes" % len(w) if isinstance(w, bytes) else "error %d" % w
                fails.append("op %d %s entry %d (stream %s, samples %d..%d): got %s, want %s" % (i, kind, j, c.s, c.lo, c.hi, what, wwhat))
        check_states(i, kind)
    for s, t in enumerate(ex.tags):
        if not t["tag_on"]:
            continue
        buf = np.zeros(2880, dtype=np.uint8)
        n = L.mp3b200_get_lametag_frame(hs[s], buf.ctypes.data, 2880)
        mine = {"tag_on": True, "tag": buf[:max(n, 0)].tobytes(), "music_crc": L.mp3b200_music_crc(hs[s]),
                "bytes_written": L.mp3b200_bytes_written(hs[s])}
        for k in mine:
            if mine[k] != t[k]:
                fails.append("stream %d: tag field %s differs" % (s, k))
    for h in hs:
        L.mp3b200_destroy(h)
    return fails
