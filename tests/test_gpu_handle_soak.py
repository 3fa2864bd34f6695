"""The streaming handle API under random call schedules (tests/handle_schedule.py) and at its per-handle error paths: every
call's bytes and byte count, and the tag of the tagged streams, equal what one lamejs encoder per stream would hand out for
the same calls (the oracle); after every operation, the state each named handle carries into its next call (its exported
blob's header and halo: ATH adjust, block-type state, OldValue / CurrentStep, frame count, FIFO fill, the masking handed to
the next granule) equals that stream's OracleEncoder.state(), through hand-overs and flush-then-reuse.  The directed tests
cover a handle listed twice in one batch call, a failed handle inside a batch,
NULL handles, a handle of another configuration, state blobs of different chunkings, and blobs whose bookkeeping was
tampered with."""
import ctypes
import struct

import numpy as np
import pytest

import handle_schedule as HS
import oracle_lib
from synth import make_signal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


@pytest.mark.parametrize("cfg,K,nops,seed", [(cfg, 32, 300, 100 + i) for i, cfg in enumerate(HS.CONFIGS)],
                         ids=["%d-%d-%d" % c for c in HS.CONFIGS])
def test_handle_soak(M, oracle, cfg, K, nops, seed):
    s = HS.make_schedule(cfg, K, nops, seed)           # the schedules tests/test_handle_schedule_cpu.py checks
    ex = HS.replay(s)
    fails = HS.run(M, s, ex)
    assert not fails, fails[:20]


def _raw_batch(M, hs, lefts, rights, caps):
    """mp3b200_encode_batch through ctypes: (per-entry bytes or error, return code)"""
    L = M.lib()
    m = len(hs)
    vp = ctypes.c_void_p
    outs = [np.zeros(max(c, 1) + 16, np.uint8) for c in caps]
    lefts = [np.ascontiguousarray(x, dtype=np.int16) for x in lefts]
    rights = [np.ascontiguousarray(x, dtype=np.int16) for x in rights] if rights is not None else None
    ns = np.array([len(x) for x in lefts], dtype=np.int32)
    got = np.zeros(m, np.int32)
    c = np.array(caps, dtype=np.int32)
    rc = L.mp3b200_encode_batch((vp * m)(*[h.value if h is not None else None for h in hs]), (vp * m)(*[x.ctypes.data for x in lefts]),
                                (vp * m)(*[x.ctypes.data for x in rights]) if rights is not None else None, ns.ctypes.data,
                                (vp * m)(*[o.ctypes.data for o in outs]), c.ctypes.data, m, got.ctypes.data)
    return [o[:g].tobytes() if g >= 0 else int(g) for o, g in zip(outs, got)], rc


def _raw_flush_batch(M, hs, cap=20000):
    L = M.lib()
    m = len(hs)
    vp = ctypes.c_void_p
    outs = [np.zeros(cap, np.uint8) for _ in hs]
    got = np.zeros(m, np.int32)
    caps = np.full(m, cap, np.int32)
    rc = L.mp3b200_flush_batch((vp * m)(*[h.value if h is not None else None for h in hs]), (vp * m)(*[o.ctypes.data for o in outs]),
                               caps.ctypes.data, m, got.ctypes.data)
    return [o[:g].tobytes() if g >= 0 else int(g) for o, g in zip(outs, got)], rc


def test_repeated_handle_in_batches(M, oracle):
    """encode_batch([a, b, a, a]) equals a's three calls and b's one in list order; flush_batch([a, b, a]) gives a's flush and
    then 0 bytes; the handles stay usable, and a's state equals that of a handle that made the same calls one by one."""
    l, r = make_signal("burst", 60000, 44100, 3)
    l2, r2 = make_signal("noise", 30000, 44100, 4)
    a, b, a1 = (M.Mp3Encoder(2, 44100, 128) for _ in range(3))
    ra, rb = oracle.OracleEncoder(2, 44100, 128), oracle.OracleEncoder(2, 44100, 128)
    cuts = [(0, 5000), (5000, 5001), (5001, 20000)]
    got = M.encode_batch([a, b, a, a], [l[0:5000], l2[:7000], l[5000:5001], l[5001:20000]],
                         [r[0:5000], r2[:7000], r[5000:5001], r[5001:20000]])
    want_a = [ra.encode_buffer(l[lo:hi], r[lo:hi]) for lo, hi in cuts]
    assert got == [want_a[0], rb.encode_buffer(l2[:7000], r2[:7000]), want_a[1], want_a[2]]
    for lo, hi in cuts:
        a1.encodeBuffer(l[lo:hi], r[lo:hi])
    assert a.export_state() == a1.export_state()
    got = M.flush_batch([a, b, a])
    assert got == [ra.flush(), rb.flush(), b""]
    assert got[0] and got[1]
    # reuse after the repeated flush, in a batch that repeats a NULL-free handle twice more
    got = M.encode_batch([a, a], [l[20000:41000], l[41000:]], [r[20000:41000], r[41000:]])
    assert got == [ra.encode_buffer(l[20000:41000], r[20000:41000]), ra.encode_buffer(l[41000:], r[41000:])]
    assert M.flush_batch([a, a, a]) == [ra.flush(), b"", b""]
    for e in (a, b, a1, ra, rb):
        e.close()


def test_failed_handle_inside_a_batch(M, oracle):
    """A too small buffer fails only its own handle (-1); the others are unaffected, and the failed handle's next call hands
    out the frames it held back in front of its own, so its stream equals the oracle's.  A NULL handle gets -3."""
    sigs = [make_signal(k, 40000, 44100, 10 + i) for i, k in enumerate(("burst", "noise", "sweep", "white"))]
    encs = [M.Mp3Encoder(2, 44100, 128) for _ in sigs]
    refs = [oracle.OracleEncoder(2, 44100, 128) for _ in sigs]
    streams = [bytearray() for _ in sigs]
    held = [b""] * len(sigs)                                # what a failed call held back
    hs = [e._h for e in encs]
    for rnd, (lo, hi) in enumerate([(0, 9000), (9000, 21000), (21000, 40000)]):
        want = [h + ref.encode_buffer(x[lo:hi], y[lo:hi]) for h, ref, (x, y) in zip(held, refs, sigs)]
        bad = rnd % 2 + 1                                   # handle 1, then 2, then 1 again gets a one-byte buffer
        assert len(want[bad]) > 1
        caps = [1 if i == bad else len(w) for i, w in enumerate(want)]
        got, rc = _raw_batch(M, hs + [None], [x[lo:hi] for x, _ in sigs] + [sigs[0][0][:10]],
                             [y[lo:hi] for _, y in sigs] + [sigs[0][1][:10]], caps + [100])
        assert rc == 0
        assert got[-1] == HS.ERR_HANDLE
        for i, g in enumerate(got[:-1]):
            if i == bad:
                assert g == HS.ERR_BUFFER, rnd
                held[i] = want[i]
            else:
                assert g == want[i], (rnd, i)
                held[i] = b""
                streams[i] += g
    got, rc = _raw_flush_batch(M, [None] + hs)
    assert rc == 0 and got[0] == HS.ERR_HANDLE
    for i, (g, ref) in enumerate(zip(got[1:], refs)):
        assert g == held[i] + ref.flush(), i
        streams[i] += g
    for i, (x, y) in enumerate(sigs):
        assert bytes(streams[i]) == oracle_lib.encode_stream(2, 44100, 128, x, y)[0], i
    for e in encs + refs:
        e.close()


def test_handle_of_another_configuration_in_a_batch(M, oracle):
    """A handle of another configuration than the batch's first one gets -1; it keeps its samples and frames, and a later
    call of its own hands them out."""
    l, r = make_signal("burst", 30000, 44100, 6)
    a, b = M.Mp3Encoder(2, 44100, 128), M.Mp3Encoder(2, 44100, 128)
    odd = M.Mp3Encoder(1, 44100, 128)
    ra, rb, ro = oracle.OracleEncoder(2, 44100, 128), oracle.OracleEncoder(2, 44100, 128), oracle.OracleEncoder(1, 44100, 128)
    got, rc = _raw_batch(M, [a._h, odd._h, b._h], [l[:9000], l[:9000], l[:5000]], [r[:9000], r[:9000], r[:5000]], [20000] * 3)
    assert rc == 0
    assert got[0] == ra.encode_buffer(l[:9000], r[:9000]) and got[2] == rb.encode_buffer(l[:5000], r[:5000])
    assert got[1] == HS.ERR_BUFFER
    held = ro.encode_buffer(l[:9000])
    assert held                                               # the failed call did complete frames
    assert odd.encodeBuffer(l[9000:12000]) == held + ro.encode_buffer(l[9000:12000])
    assert odd.flush() == ro.flush()
    for e in (a, b, odd, ra, rb, ro):
        e.close()


@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 22050, 32)])
def test_blobs_agree_across_chunkings(M, cfg):
    """Handles fed the same samples in different call sizes export equal blobs whenever they have been fed the same samples
    and handed out the same number of bytes."""
    ch, sr, kbps = cfg
    l, r = make_signal("burst", 80000, sr, 8)
    r = r if ch == 2 else None
    cuts = {}
    # three chunkings that meet every 4608 samples: tiny and odd calls, one MPEG-1 frame per call, four per call
    for name, sizes in (("a", [1, 1151, 577, 575, 2, 1150]), ("b", [1152, 1152, 2304]), ("c", [4608])):
        e = M.Mp3Encoder(ch, sr, kbps)
        pos, out, k = 0, 0, 0
        while pos < len(l):
            n = sizes[k % len(sizes)]
            out += len(e.encodeBuffer(l[pos:pos + n], None if r is None else r[pos:pos + n]))
            pos = min(pos + n, len(l))
            k += 1
            cuts.setdefault(name, {})[pos] = (out, e.export_state())
        e.close()
    for x, y in (("a", "b"), ("a", "c")):
        same = [p for p in cuts[x] if p in cuts[y] and cuts[x][p][0] == cuts[y][p][0]]
        assert len(same) >= 10, (x, y, same)
        for p in same:
            assert cuts[x][p][1] == cuts[y][p][1], (x, y, p)


def test_tampered_state_is_refused(M):
    """Blobs whose retained samples do not start at max(0, framesize * frames_done - 1104) are refused before anything is
    launched, and leave the importing handle as it was."""
    L = M.lib()
    l, r = make_signal("noise", 30000, 44100, 2)
    a = M.Mp3Encoder(2, 44100, 128)
    a.encodeBuffer(l, r)
    blob = bytearray(a.export_state())
    a.close()
    hist_base, fed, frames_done, pcm = struct.unpack_from("<4q", blob, 32)
    assert hist_base == 1152 * frames_done - 1104 and pcm == fed - hist_base
    tampered = []
    for hb, fd, fe in ((hist_base + 1152, frames_done, fed + 1152),      # retained samples start one frame late
                       (hist_base - 1, frames_done, fed - 1),
                       (hist_base, frames_done + 1, fed),                  # one more frame claimed done
                       (hist_base, frames_done - 1, fed),
                       (hist_base, -1, fed)):
        t = bytearray(blob)
        struct.pack_into("<3q", t, 32, hb, fe, fd)
        tampered.append(bytes(t))
    b = M.Mp3Encoder(2, 44100, 128)
    b.encodeBuffer(l[:3000], r[:3000])
    before = b.export_state()
    for t in tampered:
        n0 = L.mp3b200_launch_count()
        with pytest.raises(M.Mp3B200Error):
            b.import_state(t)
        assert L.mp3b200_launch_count() == n0
        assert b.export_state() == before
    b.import_state(bytes(blob))                               # the untampered blob is taken
    assert b.export_state() == bytes(blob)
    b.close()


def test_tag_placeholder_with_no_room_left(M, oracle):
    """A tagged handle's first call whose buffer holds the placeholder frame and nothing more: the frames fail (-1) without
    a byte written past the buffer, and the next call hands out the placeholder, the held-back frames and its own; the
    same inside a batch.  The stream and the finished tag equal the oracle's."""
    l, r = make_signal("burst", 40000, 44100, 5)
    tag = M.lametag_size(2, 44100, 128)
    L = M.lib()
    for batch in (False, True):
        e = M.Mp3Encoder(2, 44100, 128, write_vbr_tag=True)
        ref = oracle.OracleEncoder(2, 44100, 128, write_vbr_tag=True)
        want = ref.encode_buffer(l[:10000], r[:10000])
        assert len(want) > tag
        if batch:
            got, rc = _raw_batch(M, [e._h], [l[:10000]], [r[:10000]], [tag + 1])
            assert rc == 0 and got == [HS.ERR_BUFFER]
        else:
            buf = np.full(tag + 64, 0xA5, np.uint8)
            assert L.mp3b200_encode(e._h, l[:10000].ctypes.data, r[:10000].ctypes.data, 10000, buf.ctypes.data, tag) == HS.ERR_BUFFER
            assert (buf[tag:] == 0xA5).all()
        out = e.encodeBuffer(l[10000:], r[10000:])
        assert out == want + ref.encode_buffer(l[10000:], r[10000:])
        assert e.flush() == ref.flush()
        assert e.lametag_frame() == ref.lametag_frame()
        assert e.music_crc() == ref.music_crc() and e.bytes_written() == ref.bytes_written()
        e.close(); ref.close()
