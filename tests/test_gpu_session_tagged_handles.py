"""Tagged and ReplayGain streaming handles inside an encode session (DESIGN.md 17): the seeded handle schedules with their
tagged streams against the oracle, plain, tagged and ReplayGain handles mixed in one call against twins on the synchronous
calls (Int16, Float32, the switch, a flush in mid-stream, session rounds mixed with host calls across release and rebind),
refused rounds, calls that return while the stream is busy, the live shape of 64 handles fed from a side stream, the
ReplayGain schedules against the CPU restatement (tests/replaygain_ref.py), and lamejs's own ReplayGain, Float32 ReplayGain
and tagged fixtures."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import float_signals as FS  # noqa: E402
import handle_schedule as HS  # noqa: E402
import oracle_lib  # noqa: E402
from synth import make_signal  # noqa: E402
from test_gpu_session_handles import LOUD_GOLDEN, SLEEP_CYCLES, cuda, got_bytes, session_ops  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def tag_facts(M, e):
    """what a released handle's host getters say"""
    return {"tag": e.lametag_frame(), "crc": e.music_crc(), "bytes": e.bytes_written(), "rg": e.replay_gain}


def frames_of(M, sess, encs):
    o, off, lens, st = sess.lametag_frames(encs)
    M.check_status(st)
    return got_bytes(o, off, lens)


# ---- oracle parity on the handle schedules, tagged streams kept ----

@pytest.mark.parametrize("cfg", HS.CONFIGS + HS.RESAMPLED_CONFIGS, ids=lambda c: "%d_%d_%d" % c)
def test_tagged_schedule_parity_with_the_oracle(M, cfg):
    ch, sr, kb = cfg
    full = HS.make_schedule(cfg, 6, 40, seed=sr + kb + 1, big=0.02)
    s = session_ops(full)
    sched = HS.Schedule(s.cfg, s.signals, s.kinds, full.tagged, s.ops)
    assert sched.tagged
    ex = HS.replay(sched)
    encs = [M.Mp3Encoder(ch, sr, kb, resample=sched.resample, write_vbr_tag=k in sched.tagged) for k in range(sched.nstreams)]
    rows = [(cuda(l), None if r is None else cuda(r)) for l, r in sched.signals]
    fails, pending = [], []

    def settle():
        for j, (o, off, lens, st) in pending:
            M.check_status(st)
            for c, w, g in zip(sched.ops[j][1], ex.results[j], got_bytes(o, off, lens)):
                if g != w:
                    fails.append("op %d stream %d: %d bytes, want %d" % (j, c.s, len(g), len(w)))
        pending.clear()

    with M.EncodeSession() as sess:
        for i, (kind, entries) in enumerate(sched.ops):
            if kind == "handover":                       # never a tagged stream (the tag is not part of a state blob)
                k = entries[0].s
                sess.release(encs)
                settle()
                e = M.Mp3Encoder(ch, sr, kb, resample=sched.resample)
                e.import_state(encs[k].export_state())
                encs[k].close()
                encs[k] = e
                continue
            es = [encs[c.s] for c in entries]
            if kind == "encode_batch":
                ls = [rows[c.s][0][c.lo:c.hi] for c in entries]
                rs = None if ch == 1 else [rows[c.s][1][c.lo:c.hi] for c in entries]
                pending.append((i, sess.encode_batch_tagged(es, ls, rs)))
            else:
                pending.append((i, sess.flush_batch_tagged(es)))
        tagged = sorted(sched.tagged)
        frames = frames_of(M, sess, [encs[k] for k in tagged])
        sess.release(encs)
        settle()
    for k, f in zip(tagged, frames):
        t = ex.tags[k]
        assert f == t["tag"], k
        assert encs[k].lametag_frame() == t["tag"]
        if t["tag_on"]:                                  # where the tag does not fit, lamejs switches it off
            assert encs[k].music_crc() == t["music_crc"] and encs[k].bytes_written() == t["bytes_written"]
    for e in encs:
        e.close()
    assert not fails, fails[:10]


# ---- twins on the synchronous calls: plain, tagged and ReplayGain handles in one call ----

def make_mix(M, cfg, rs):
    ch, sr, kb = cfg
    kinds = [(False, False), (True, False), (True, True)] * 2
    return [M.Mp3Encoder(ch, sr, kb, resample=rs, write_vbr_tag=t, find_replay_gain=g) for t, g in kinds]


@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 24000, 64), (2, 48000, 64)], ids=lambda c: "%d_%d_%d" % c)
def test_mixed_handles_match_the_synchronous_calls(M, cfg):
    import torch
    ch, sr, kb = cfg
    rs = sr == 48000 and kb == 64
    rng = np.random.default_rng(17)
    A, B = make_mix(M, cfg, rs), make_mix(M, cfg, rs)
    K = len(A)
    assert A[2].replay_gain_on and A[1].tag_on
    sig = [make_signal(("noise", "sweep", "burst", "octave", "noise", "sweep")[k], 400000, sr, seed=k + 20) for k in range(K)]
    pos = [0] * K
    fails = []
    sess = M.EncodeSession()

    def compare(g, w, what):
        o, off, lens, st = g
        M.check_status(st)
        if got_bytes(o, off, lens) != w:
            fails.append(what)

    for rnd in range(30):
        if rnd in (12, 22):                               # flush, then the stream goes on: a new ReplayGain title
            compare(sess.flush_batch_tagged(A), M.flush_batch(B), "flush %d" % rnd)
            frames = frames_of(M, sess, A)
            sess.release(A)                               # the gains and CRCs come back; the next call binds again
            assert frames == [b.lametag_frame() for b in B]
            assert [tag_facts(M, a) for a in A] == [tag_facts(M, b) for b in B]
            continue
        f32 = rnd >= 6 and rnd % 4 != 1                   # Int16 first, then Float32 with Int16 rounds between
        ls, rs_ = [], []
        for k in range(K):
            n = int(rng.choice([0, 1, 577, 1152, 2400, 4000, 11025]))
            l, r = sig[k][0][pos[k]:pos[k] + n], sig[k][1][pos[k]:pos[k] + n]
            pos[k] += n
            if f32:
                l, r = l.astype(np.float32) / 32768, r.astype(np.float32) / 32768
            ls.append(cuda(l)); rs_.append(cuda(r))
        w = M.encode_batch(B, ls, None if ch == 1 else rs_)
        if 16 <= rnd < 19:                                # released: host calls on A, then the session binds it again
            if rnd == 16:
                sess.release(A)
            if M.encode_batch(A, ls, None if ch == 1 else rs_) != w:
                fails.append("host round %d" % rnd)
            continue
        compare(sess.encode_batch_tagged(A, ls, None if ch == 1 else rs_), w, "round %d" % rnd)
    compare(sess.flush_batch_tagged(A), M.flush_batch(B), "last flush")
    frames = frames_of(M, sess, A)
    album, st = sess.album_gain(A)
    M.check_status(st)
    sess.release(A)
    assert not fails, fails
    assert frames == [b.lametag_frame() for b in B]
    assert float(album.cpu()[0]) == M.album_gain(B) == M.album_gain(A)
    assert [tag_facts(M, a) for a in A] == [tag_facts(M, b) for b in B]
    assert A[2].replay_gain is not None
    assert [a.export_state() for a in A if not a.replay_gain_on] == [b.export_state() for b in B if not b.replay_gain_on]
    sess.close()
    torch.cuda.synchronize()
    for e in A + B:
        e.close()


# ---- refusals ----

def tagged_loud_case(M):
    """the first loud case of loud_case's kind whose configuration fits the tag and whose refused call has calls before it"""
    for name, c in sorted(LOUD_GOLDEN.items()):
        if c["rg"] or not c["thrown"] or FS.loud_peak(c) > 2.0 ** 40 or FS.loud_case_signal(c)[2][c["thrown"]] is None:
            continue
        ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
        if M.lametag_size(ch, sr, kb, M.out_samplerate(ch, sr, kb) != sr) > 0:
            return c
    raise AssertionError("no loud case with a tag")


@pytest.mark.parametrize("kind", ["loud", "nan"])
def test_refused_round_on_replaygain_handles(M, kind):
    c = tagged_loud_case(M)
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    _, _, calls = FS.loud_case_signal(c)
    k = c["thrown"]
    base = make_signal("noise", 400000, sr, seed=9)
    quiet = [(base[0][i * 20000:(i + 1) * 20000].astype(np.float32) / 65536, base[1][i * 20000:(i + 1) * 20000].astype(np.float32) / 65536)
             for i in range(k + 3)]
    rs = M.out_samplerate(ch, sr, kb) != sr

    def enc():
        return M.Mp3Encoder(ch, sr, kb, resample=rs, write_vbr_tag=True, find_replay_gain=True)

    A, T = [enc() for _ in range(3)], [enc() for _ in range(3)]     # T: twins that never see the refused rounds
    D = enc()
    assert A[0].replay_gain_on

    def rows(i):
        x = calls[i] if kind == "loud" and i <= k else (quiet[i][0][:4000], quiet[i][1][:4000])
        if kind == "nan" and i == k:
            x = (x[0].copy(), x[1].copy())
            x[0][1234] = np.nan
        xs = [x, (quiet[i][0][:len(x[0])], quiet[i][1][:len(x[0])]), (quiet[i][1][:len(x[0])], quiet[i][0][:len(x[0])])]
        return [cuda(a) for a, _ in xs], [cuda(b if b is not None else a) for a, b in xs]

    sess = M.EncodeSession()
    for i in range(k):
        if kind == "loud" and calls[i] is None:
            o, off, lens, st = sess.flush_batch_tagged(A)
            M.check_status(st)
            assert got_bytes(o, off, lens) == M.flush_batch(T)
            continue
        lp, rp = rows(i)
        o, off, lens, st = sess.encode_batch_tagged(A, lp, None if ch == 1 else rp)
        M.check_status(st)
        assert got_bytes(o, off, lens) == M.encode_batch(T, lp, None if ch == 1 else rp)
    lp, rp = rows(k)
    st_k = sess.encode_batch_tagged(A, lp, None if ch == 1 else rp)[3]
    lp, rp = rows(k + 1)
    st_k1 = sess.encode_batch_tagged([A[1], D], lp[1:], None if ch == 1 else rp[1:])[3]
    frames_st = sess.lametag_frames(A)[3]
    msg = "bit budget" if kind == "loud" else "non-finite"
    for st in (st_k, st_k1, frames_st):
        with pytest.raises(M.Mp3B200Error, match=msg):
            M.check_status(st)
    sess.release(A + [D])
    assert [tag_facts(M, a) for a in A] == [tag_facts(M, t) for t in T]

    def outcome(fn):          # the loud samples the FIFO still holds may refuse the next frames: then both refuse alike
        try:
            return fn()
        except M.Mp3B200Error as e:
            return str(e)

    lp = [cuda(quiet[k + 2][j % 2][:6000]) for j in range(3)]
    rp = [cuda(quiet[k + 2][(j + 1) % 2][:6000]) for j in range(3)]
    assert outcome(lambda: M.encode_batch(A, lp, None if ch == 1 else rp)) == outcome(lambda: M.encode_batch(T, lp, None if ch == 1 else rp))
    assert outcome(lambda: M.flush_batch(A)) == outcome(lambda: M.flush_batch(T))
    assert [tag_facts(M, a) for a in A] == [tag_facts(M, t) for t in T]
    assert M.album_gain(A) == M.album_gain(T)
    sess.close()


# ---- asynchrony ----

def test_tagged_calls_return_while_the_stream_is_busy(M):
    import torch
    side = torch.cuda.Stream()

    def encs():
        return [M.Mp3Encoder(2, 44100, 128, write_vbr_tag=True, find_replay_gain=k % 2 == 0) for k in range(8)]

    A, B = encs(), encs()
    l, r = make_signal("sweep", 30000, 44100, seed=2)
    x, y = cuda(l[:4000]), cuda(r[:4000])
    with M.EncodeSession(side) as sess:
        res = [sess.encode_batch_tagged(A, [x] * 8, [y] * 8) for _ in range(4)]   # binds, warms the shapes and the buffers
        side.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
        for k in range(3 * 4):                                   # more calls in flight than MP3B200_SESSION_SLOTS
            res.append(sess.encode_batch_tagged(A, [x] * 8, [y] * 8))
            if k == 0:
                assert not side.query()                          # returned with the stream still busy
        res.append(sess.flush_batch_tagged(A))
        frames = frames_of(M, sess, A)
        side.synchronize()
        sess.release(A)
    for o, off, lens, st in res[:-1]:
        M.check_status(st)
        assert got_bytes(o, off, lens) == M.encode_batch(B, [l[:4000]] * 8, [r[:4000]] * 8)
    o, off, lens, st = res[-1]
    assert got_bytes(o, off, lens) == M.flush_batch(B)
    assert frames == [b.lametag_frame() for b in B]
    assert [tag_facts(M, a) for a in A] == [tag_facts(M, b) for b in B]


# ---- the live shape ----

def test_live_shape_64_replaygain_handles_from_a_side_stream(M):
    import torch
    N, sr, n = 64, 24000, 2400
    kb = 64
    assert M.out_samplerate(1, sr, kb) == sr
    side = torch.cuda.Stream()
    A = [M.Mp3Encoder(1, sr, kb, write_vbr_tag=True, find_replay_gain=True) for _ in range(N)]
    B = [M.Mp3Encoder(1, sr, kb, write_vbr_tag=True, find_replay_gain=True) for _ in range(N)]
    g = torch.Generator(device="cuda").manual_seed(5)
    chunks, res, graphs = [], [], []
    with M.EncodeSession(side) as sess:
        for rnd in range(50):
            with torch.cuda.stream(side):
                t = torch.arange(n, device="cuda", dtype=torch.float32) + rnd * n
                f = torch.linspace(100, 3000, N, device="cuda")[:, None]
                x = 0.3 * torch.sin(t[None, :] * f * (2 * np.pi / sr)) + 0.01 * torch.randn(N, n, device="cuda", generator=g)
            chunks.append(x)
            res.append(sess.encode_batch_tagged(A, list(x)))
            graphs.append(sess.graph_instantiations())
        res.append(sess.flush_batch_tagged(A))
        frames = frames_of(M, sess, A)
        album, st = sess.album_gain(A)
        M.check_status(st)
        side.synchronize()
        for x, (o, off, lens, st) in zip(chunks, res):
            M.check_status(st)
            assert got_bytes(o, off, lens) == M.encode_batch(B, list(x))
        o, off, lens, st = res[-1]
        assert got_bytes(o, off, lens) == M.flush_batch(B)
        assert frames == [b.lametag_frame() for b in B]
        assert float(album.cpu()[0]) == M.album_gain(B)
        sess.release(A)
    assert graphs[-1] == graphs[20], graphs          # a steady workload instantiates nothing once warm
    assert [tag_facts(M, a) for a in A] == [tag_facts(M, b) for b in B]


# ---- ReplayGain schedules against the CPU restatement (tests/replaygain_ref.py) ----

def play_session(M, sched):
    """replaygain_worker.play through session calls: every stream on a tagged + ReplayGain handle driven by the session and a
    tagged plain twin on the synchronous calls.  After every flush (flush-then-continue starts a new title) the handle is
    released and its title and radio gain must be the restatement's; at the end its session-made tag frame must be the
    twin's with the Radio Replay Gain field set, and the album gain, in the session and after release, GetAlbumGain of all
    titles.  Returns what differed."""
    import replaygain_ref as RG
    import replaygain_worker as W
    ch, sr, kb = sched.cfg
    rs = sched.resample
    K = sched.nstreams
    rg = [M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs, find_replay_gain=True) for _ in range(K)]
    plain = [M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs) for _ in range(K)]
    assert all(e.replay_gain_on for e in rg)
    rows = [(cuda(l), None if r is None else cuda(r)) for l, r in sched.signals]
    steps = [[] for _ in range(K)]
    seen = [[] for _ in range(K)]
    fail = []
    sess = M.EncodeSession()
    for kind, cs in session_ops(sched).ops:
        if kind == "handover":
            continue
        if kind == "encode_batch":
            g = sess.encode_batch_tagged([rg[c.s] for c in cs], [rows[c.s][0][c.lo:c.hi] for c in cs],
                                         None if ch == 1 else [rows[c.s][1][c.lo:c.hi] for c in cs])
            w = M.encode_batch([plain[c.s] for c in cs], [sched.signals[c.s][0][c.lo:c.hi] for c in cs],
                               None if ch == 1 else [sched.signals[c.s][1][c.lo:c.hi] for c in cs])
            for c in cs:
                steps[c.s].append(("enc", c.hi - c.lo))
        else:
            g = sess.flush_batch_tagged([rg[c.s] for c in cs])
            w = M.flush_batch([plain[c.s] for c in cs])
        M.check_status(g[3])
        if got_bytes(*g[:3]) != w:
            fail.append("%s bytes differ from the plain handle's" % kind)
        if kind == "flush_batch":
            sess.release([rg[c.s] for c in cs])
            for c in cs:
                steps[c.s].append(("flush",))
                seen[c.s].append((len(steps[c.s]), rg[c.s].replay_gain))
    frames = got_bytes(*sess.lametag_frames(rg)[:3])
    album, st = sess.album_gain(rg)
    M.check_status(st)
    album = float(album.cpu()[0])
    sess.close()
    out_sr = M.out_samplerate(ch, sr, kb)
    hist = np.zeros(RG.HIST, dtype=np.int64)

    def fed(sig, st):
        m = sum(k[1] for k in st if k[0] == "enc")
        return None if sig is None else sig[:m]

    for s in range(K):
        x, y = sched.signals[s]
        for n, got in seen[s]:
            ref = RG.analyze_stream(ch, sr, kb, fed(x, steps[s][:n]), fed(y, steps[s][:n]), schedule=steps[s][:n])
            want = (ref.title_db[-1], ref.radio[-1]) if ref.title_db else None
            if got != want:
                fail.append("stream %d after step %d: %r != %r" % (s, n, got, want))
        ref = RG.analyze_stream(ch, sr, kb, fed(x, steps[s]), fed(y, steps[s]), schedule=steps[s])
        for a in ref.hist:
            hist += a
        want_tag = W.patched_tag(plain[s].lametag_frame(), ch, out_sr, RG.tag_field(ref.radio[-1]))
        if frames[s] != want_tag or rg[s].lametag_frame() != want_tag:
            fail.append("stream %d: tag frame" % s)
    want = RG.analyze_result(hist.astype(np.int32))
    if album != want or M.album_gain(rg) != want:
        fail.append("album gain %r / %r != %r" % (album, M.album_gain(rg), want))
    for e in rg + plain:
        e.close()
    return fail


@pytest.mark.parametrize("i", range(4))
def test_replaygain_schedules_against_the_restatement(M, i):
    import replaygain_worker as W
    cfg = W.CONFIGS[i]
    fail = play_session(M, HS.make_schedule(cfg, 5, 30, seed=700 + i))
    assert not fail, fail[:10]


# ---- lamejs itself: the golden fixtures through session calls with CUDA-tensor rows ----

RG_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_replaygain_golden.json")))
TAG_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_tag_golden.json")))["tagged"]
FLOAT_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))
FRACTIONAL = (44100, 22050, 11025)     # lamejs's fractional frame sizes: see tests/test_float_golden_cpu.py


def rg_field_at(ch, out_sr):
    return 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19


def run_calls(M, e, calls):
    """calls: (left, right) numpy rows, or None for a flush, each one session call on `e`; after every flush e is released
    and its radio gain read.  Returns (the bytes of every call, the radio gain after every flush, the session-made tag
    frame at the end)."""
    sess = M.EncodeSession()
    out, radio = [], []
    for x in calls:
        if x is None:
            g = sess.flush_batch_tagged([e])
        else:
            g = sess.encode_batch_tagged([e], [cuda(x[0])], None if x[1] is None else [cuda(x[1])])
        M.check_status(g[3])
        out += got_bytes(*g[:3])
        if x is None:
            sess.release([e])
            radio.append(e.replay_gain[1] if e.replay_gain else None)
    frame = got_bytes(*sess.lametag_frames([e])[:3])[0]
    sess.close()
    return out, radio, frame


def check_fixture(M, name, c, e, out, radio, frame):
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    out_sr = M.out_samplerate(ch, sr, kb)
    at = rg_field_at(ch, out_sr)
    assert radio == c["radio_gain"], name
    assert frame == e.lametag_frame() and frame[at:at + 2] == bytes.fromhex(c["tag"])[at:at + 2], name
    data = b"".join(out)
    audio = data[len(frame):]                                    # behind the placeholder
    assert e.music_crc() == oracle_lib.crc16(audio) and e.bytes_written() == len(audio), name
    if out_sr not in FRACTIONAL:
        assert [len(b) for b in out] == c["sizes"], name
        assert hashlib.sha256(data).hexdigest() == c["sha256"], name


@pytest.mark.parametrize("name", sorted(RG_GOLDEN))
def test_lamejs_replaygain_fixture(M, name):
    c = RG_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    l, r = make_signal(c["kind"], c["samples"], sr, seed=c["seed"])
    calls, at = [], 0
    for n in c["schedule"]:
        if n < 0:
            calls.append(None)
        else:
            calls.append((l[at:at + n], r[at:at + n] if ch == 2 else None))
            at += n
    if calls[-1] is not None:
        calls.append(None)
    e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, find_replay_gain=True, resample=M.out_samplerate(ch, sr, kb) != sr)
    assert e.replay_gain_on
    out, radio, frame = run_calls(M, e, calls)
    check_fixture(M, name, c, e, out, radio, frame)
    e.close()


@pytest.mark.parametrize("name", sorted(n for n, c in FLOAT_GOLDEN.items() if c["rg"]))
def test_lamejs_float_replaygain_fixture(M, name):
    c = FLOAT_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    _, _, calls = FS.case_signal(c)
    calls = list(calls)
    if calls[-1] is not None:
        calls.append(None)
    e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, find_replay_gain=True, resample=M.out_samplerate(ch, sr, kb) != sr)
    out, radio, frame = run_calls(M, e, calls)
    check_fixture(M, name, c, e, out, radio, frame)
    e.close()


@pytest.mark.parametrize("name", sorted(TAG_GOLDEN))
def test_lamejs_tag_fixture(M, name):
    """lamejs's tagged streams: per-call sizes and the stream's SHA-256 (placeholder in front, as lamejs hands it out), and
    after release the music CRC and byte count; where the tag does not fit, no placeholder and no frame"""
    c = TAG_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    l, r = make_signal(c["kind"], c["samples"], sr, seed=c["seed"])
    step = c["chunk"] or max(len(l), 1)
    calls = [(l[i:i + step], r[i:i + step] if ch == 2 else None) for i in range(0, len(l), step)] + [None]
    e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=M.out_samplerate(ch, sr, kb) != sr)
    assert e.tag_on == c["write_tag"]
    out, _, frame = run_calls(M, e, calls)
    data = b"".join(out)
    if c["write_tag"]:
        assert frame == e.lametag_frame() and len(frame) == int(c["total_frame_size"])
        assert e.music_crc() == c["music_crc"] and e.bytes_written() == c["bytes_written"] == len(data) - len(frame)
    else:
        assert frame == b"" and e.music_crc() == -1
    if c["total_frame_size"] == int(c["total_frame_size"]):       # integer frame size: the JavaScript stream is this stream
        assert [len(b) for b in out] == c["sizes"] and hashlib.sha256(data).hexdigest() == c["sha256"]
    e.close()
