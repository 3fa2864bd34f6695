"""Streaming handles inside an encode session (DESIGN.md 16): the seeded handle schedules played through session calls
against the oracle, Float32 and Int16 -> Float32 handles against twins fed by the synchronous device calls, session rounds
mixed with host calls, the live shape of 512 handles fed from a side stream, calls that return while the stream is busy,
refusals and binding errors."""
import ctypes
import json
import os
import sys
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import float_signals as FS  # noqa: E402
import handle_schedule as HS  # noqa: E402
from synth import make_signal  # noqa: E402

pytestmark = pytest.mark.gpu
vp = ctypes.c_void_p
ERR_CONFIG, ERR_HANDLE = -1, -3
SLEEP_CYCLES = 400_000_000           # torch.cuda._sleep: ~0.2 s on an H100
LOUD_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def got_bytes(out, off, lens):
    host = out.cpu().numpy()
    return [host[o:o + n].tobytes() for o, n in zip(off, lens)]


# ---- oracle parity on the handle schedules ----

def session_ops(sched):
    """the schedule with what sessions refuse left out: no tag, no one-byte buffers, no NULL entries; a batch that names a
    stream twice becomes consecutive calls (round k holds each stream's k-th entry)"""
    ops = []
    for kind, entries in sched.ops:
        if kind == "handover":
            ops.append((kind, entries))
            continue
        kind = "encode_batch" if kind.startswith("encode") else "flush_batch"
        rounds = []
        for c in entries:
            if c.s is None:
                continue
            k = next((j for j, r in enumerate(rounds) if c.s not in {x.s for x in r}), len(rounds))
            if k == len(rounds):
                rounds.append([])
            rounds[k].append(c._replace(fail=False))
        ops += [(kind, r) for r in rounds if r]
    return HS.Schedule(sched.cfg, sched.signals, sched.kinds, set(), ops)


@pytest.mark.parametrize("cfg", HS.CONFIGS + HS.RESAMPLED_CONFIGS, ids=lambda c: "%d_%d_%d" % c)
def test_schedule_parity_with_the_oracle(M, cfg):
    ch, sr, kb = cfg
    sched = session_ops(HS.make_schedule(cfg, 6, 40, seed=sr + kb, big=0.02))
    ex = HS.replay(sched)
    L = M.lib()
    encs = [M.Mp3Encoder(ch, sr, kb, resample=sched.resample) for _ in range(sched.nstreams)]
    rows = [(cuda(l), None if r is None else cuda(r)) for l, r in sched.signals]
    fails = []
    with M.EncodeSession() as sess:
        pending = []
        for i, ((kind, entries), want) in enumerate(zip(sched.ops, ex.results)):
            if kind == "handover":
                s = entries[0].s
                sess.release(encs)
                for j, (o, off, lens, st) in pending:
                    M.check_status(st)
                    for c, w, g in zip(sched.ops[j][1], ex.results[j], got_bytes(o, off, lens)):
                        if g != w:
                            fails.append("op %d stream %d: %d bytes, want %d" % (j, c.s, len(g), len(w)))
                pending = []
                for t, st in ex.states[i].items():
                    bad = HS.blob_state_diff(np.frombuffer(encs[t].export_state(), np.uint8), st, ch)
                    if bad:
                        fails.append("op %d: state of stream %d differs in %s" % (i, t, bad))
                blob = encs[s].export_state()
                e = M.Mp3Encoder(ch, sr, kb, resample=sched.resample)
                e.import_state(blob)
                encs[s].close()
                encs[s] = e
                continue
            es = [encs[c.s] for c in entries]
            if kind == "encode_batch":
                ls = [rows[c.s][0][c.lo:c.hi] for c in entries]
                rs = None if ch == 1 else [rows[c.s][1][c.lo:c.hi] for c in entries]
                pending.append((i, sess.encode_batch(es, ls, rs)))
            else:
                pending.append((i, sess.flush_batch(es)))
        sess.release(encs)
        for j, (o, off, lens, st) in pending:
            M.check_status(st)
            for c, w, g in zip(sched.ops[j][1], ex.results[j], got_bytes(o, off, lens)):
                if g != w:
                    fails.append("op %d stream %d: %d bytes, want %d" % (j, c.s, len(g), len(w)))
    for e in encs:
        e.close()
    assert not fails, fails[:10]


# ---- Float32 and the Int16 -> Float32 switch, against twins on the synchronous device calls ----

@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 16000, 32), (2, 48000, 64)], ids=lambda c: "%d_%d_%d" % c)
def test_float32_and_switch_match_the_synchronous_calls(M, cfg):
    import torch
    ch, sr, kb = cfg
    rs = sr == 48000 and kb == 64
    rng = np.random.default_rng(7)
    K = 4
    sig = [make_signal(("noise", "sweep", "burst", "octave")[k], 200000, sr, seed=k) for k in range(K)]
    A = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(K)]
    B = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(K)]
    pos = [0] * K
    want, got = [], []
    with M.EncodeSession() as sess:
        for rnd in range(24):
            f32 = rnd >= 8 and (rnd % 3 != 0 or rnd >= 16)       # Int16 first, then Float32 with Int16 rounds between
            ls, rs_ = [], []
            for k in range(K):
                n = int(rng.choice([0, 1, 577, 1152, 2400, 4000, 11025]))
                l, r = sig[k][0][pos[k]:pos[k] + n], sig[k][1][pos[k]:pos[k] + n]
                pos[k] += n
                if f32:
                    l, r = l.astype(np.float32) / 32768, r.astype(np.float32) / 32768
                ls.append(cuda(l)); rs_.append(cuda(r))
            want.append(M.encode_batch(B, ls, None if ch == 1 else rs_))
            got.append(sess.encode_batch(A, ls, None if ch == 1 else rs_))
        want.append(M.flush_batch(B))
        got.append(sess.flush_batch(A))
        sess.release(A)
    for w, (o, off, lens, st) in zip(want, got):
        M.check_status(st)
        assert got_bytes(o, off, lens) == w
    assert [a.export_state() for a in A] == [b.export_state() for b in B]
    torch.cuda.synchronize()
    for e in A + B:
        e.close()


def test_mixed_session_and_host_calls(M):
    ch, sr, kb = 2, 32000, 96
    l, r = make_signal("noise", 120000, sr, seed=11)
    A = [M.Mp3Encoder(ch, sr, kb) for _ in range(3)]
    B = [M.Mp3Encoder(ch, sr, kb) for _ in range(3)]
    sess = M.EncodeSession()
    at = 0

    def chunk(n):
        nonlocal at
        x, y = l[at:at + n], r[at:at + n]
        at += n
        return x, y

    for phase in range(3):
        for rnd in range(5):
            x, y = chunk(1500 + 701 * rnd)
            w = M.encode_batch(B, [x] * 3, [y] * 3)
            if phase == 1:                       # host and device calls on the released handles
                g = M.encode_batch(A, [x] * 3, [y] * 3) if rnd % 2 else M.encode_batch(A, [cuda(x)] * 3, [cuda(y)] * 3)
            else:
                o, off, lens, st = sess.encode_batch(A, [cuda(x)] * 3, [cuda(y)] * 3)
                M.check_status(st)
                g = got_bytes(o, off, lens)
            assert g == w
        if phase != 1:
            sess.release(A)
        assert [a.export_state() for a in A] == [b.export_state() for b in B]
    o, off, lens, st = sess.flush_batch(A)
    M.check_status(st)
    assert got_bytes(o, off, lens) == M.flush_batch(B)
    sess.close()
    assert [a.export_state() for a in A] == [b.export_state() for b in B]


# ---- the live shape ----

def test_live_shape_512_handles_from_a_side_stream(M):
    import torch
    N, sr, n = 512, 24000, 2400
    kb = next(k for k in (64, 48, 56, 40, 32) if M.out_samplerate(1, sr, k) == sr)
    side = torch.cuda.Stream()
    A = [M.Mp3Encoder(1, sr, kb) for _ in range(N)]
    B = [M.Mp3Encoder(1, sr, kb) for _ in range(N)]
    g = torch.Generator(device="cuda").manual_seed(5)
    chunks, res = [], []
    with M.EncodeSession(side) as sess:
        for rnd in range(50):
            with torch.cuda.stream(side):
                t = torch.arange(n, device="cuda", dtype=torch.float32) + rnd * n
                f = torch.linspace(100, 3000, N, device="cuda")[:, None]
                x = 0.3 * torch.sin(t[None, :] * f * (2 * np.pi / sr)) + 0.01 * torch.randn(N, n, device="cuda", generator=g)
            chunks.append(x)
            res.append(sess.encode_batch(A, list(x)))
        res.append(sess.flush_batch(A))
        side.synchronize()
        for x, (o, off, lens, st) in zip(chunks, res):
            M.check_status(st)
            assert got_bytes(o, off, lens) == M.encode_batch(B, list(x))
        o, off, lens, st = res[-1]
        assert got_bytes(o, off, lens) == M.flush_batch(B)


# ---- asynchrony ----

def test_call_returns_while_the_stream_is_busy(M):
    import torch
    side = torch.cuda.Stream()
    A = [M.Mp3Encoder(2, 44100, 128) for _ in range(8)]
    B = [M.Mp3Encoder(2, 44100, 128) for _ in range(8)]
    l, r = make_signal("sweep", 30000, 44100, seed=2)
    with M.EncodeSession(side) as sess:
        x, y = cuda(l[:4000]), cuda(r[:4000])
        res = [sess.encode_batch(A, [x] * 8, [y] * 8) for _ in range(4)]   # binds, warms the shapes and grows the buffers
        side.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
        t0 = time.perf_counter()
        for k in range(3 * 4):                                 # more calls in flight than MP3B200_SESSION_SLOTS
            res.append(sess.encode_batch(A, [x] * 8, [y] * 8))
            if k == 0:
                first = time.perf_counter() - t0
                assert not side.query()
        assert first < 0.1
        side.synchronize()
    for o, off, lens, st in res:
        M.check_status(st)
        assert got_bytes(o, off, lens) == M.encode_batch(B, [l[:4000]] * 8, [r[:4000]] * 8)


def test_two_sessions_from_two_threads(M):
    import torch
    l, r = make_signal("noise", 60000, 44100, seed=4)
    out, errs = {}, []

    def worker(k):
        try:
            st = torch.cuda.Stream()
            A = [M.Mp3Encoder(2, 44100, 128) for _ in range(4)]
            got = []
            with M.EncodeSession(st) as sess:
                for i in range(10):
                    x, y = cuda(l[i * 3000:(i + 1) * 3000]), cuda(r[i * 3000:(i + 1) * 3000])
                    got.append(sess.encode_batch(A, [x] * 4, [y] * 4))
                got.append(sess.flush_batch(A))
                st.synchronize()
                out[k] = [got_bytes(o, off, lens) for o, off, lens, _ in got]
        except Exception as e:   # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    B = [M.Mp3Encoder(2, 44100, 128) for _ in range(4)]
    want = [M.encode_batch(B, [l[i * 3000:(i + 1) * 3000]] * 4, [r[i * 3000:(i + 1) * 3000]] * 4) for i in range(10)]
    want.append(M.flush_batch(B))
    assert out[0] == want and out[1] == want


# ---- refusals ----

def loud_case():
    name = sorted(n for n, c in LOUD_GOLDEN.items() if not c["rg"] and c["thrown"] is not None
                  and FS.loud_peak(c) <= 2.0 ** 40 and FS.loud_case_signal(c)[2][c["thrown"]] is not None)[0]
    return LOUD_GOLDEN[name]


@pytest.mark.parametrize("kind", ["loud", "nan"])
def test_refused_round_and_release(M, kind):
    c = loud_case()
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    _, _, calls = FS.loud_case_signal(c)
    k = c["thrown"]
    base = make_signal("noise", 400000, sr, seed=9)
    quiet = [(base[0][i * 20000:(i + 1) * 20000].astype(np.float32) / 65536, base[1][i * 20000:(i + 1) * 20000].astype(np.float32) / 65536)
             for i in range(k + 3)]
    rs = M.out_samplerate(ch, sr, kb) != sr
    A = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(3)]
    D = M.Mp3Encoder(ch, sr, kb, resample=rs)                     # named only with the others after the refusal

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
            M.check_status(sess.flush_batch(A)[3])
            continue
        lp, rp = rows(i)
        M.check_status(sess.encode_batch(A, lp, None if ch == 1 else rp)[3])
    sess.release(A)
    before = [a.export_state() for a in A]
    lp, rp = rows(k)
    st_k = sess.encode_batch(A, lp, None if ch == 1 else rp)[3]
    lp, rp = rows(k + 1)
    st_k1 = sess.encode_batch([A[1], D], lp[1:], None if ch == 1 else rp[1:])[3]
    st_d = sess.encode_batch([D], lp[2:], None if ch == 1 else rp[2:])[3]
    msg = "bit budget" if kind == "loud" else "non-finite"
    for st in (st_k, st_k1):
        with pytest.raises(M.Mp3B200Error, match=msg):
            M.check_status(st)
    with pytest.raises(M.Mp3B200Error, match=msg):   # D was named by round k + 1: refused with it
        M.check_status(st_d)
    E = M.Mp3Encoder(ch, sr, kb, resample=rs)
    st_e = sess.encode_batch([E], lp[2:], None if ch == 1 else rp[2:])[3]
    M.check_status(st_e)                              # a round naming only other handles stands
    sess.release(A + [D, E])
    assert [a.export_state() for a in A] == before
    # synchronous calls continue them as twins that never saw the refused rounds
    T = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(3)]
    for a, t in zip(A, T):
        t.import_state(a.export_state())
    lp = [cuda(quiet[k + 2][j % 2][:6000]) for j in range(3)]
    rp = [cuda(quiet[k + 2][(j + 1) % 2][:6000]) for j in range(3)]
    assert M.encode_batch(A, lp, None if ch == 1 else rp) == M.encode_batch(T, lp, None if ch == 1 else rp)
    assert M.flush_batch(A) == M.flush_batch(T)
    sess.close()


# ---- binding errors ----

def test_binding_errors(M):
    import torch
    L = M.lib()
    e = M.Mp3Encoder(2, 44100, 128)
    f = M.Mp3Encoder(1, 44100, 128)
    t = M.Mp3Encoder(2, 44100, 128, write_vbr_tag=True)
    x = cuda(np.zeros(3000, np.int16))
    s1, s2 = M.EncodeSession(), M.EncodeSession(torch.cuda.Stream())
    M.check_status(s1.encode_batch([e], [x], [x])[3])
    for call in (lambda: e.encodeBuffer(np.zeros(10, np.int16)), e.flush, e.export_state,
                 lambda: e.import_state(b"\0" * 64), lambda: e.seek(1, np.zeros(272, np.int16)),
                 lambda: M.encode_batch([e], [np.zeros(5, np.int16)]), lambda: M.flush_batch([e]),
                 lambda: e.encodeBuffer(x, x), lambda: e.replay_gain, e.lametag_frame):
        with pytest.raises(M.Mp3B200Error, match="bound to an encode session"):
            call()
    with pytest.raises(M.Mp3B200Error, match="another encode session"):
        s2.encode_batch([e], [x], [x])
    n = np.array([3000, 3000], np.int32)
    got = np.zeros(2, np.int32)
    off = np.zeros(2, np.int64)
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")

    def raw(hs, rows, fn=L.mp3b200_session_encode_batch, sess=s1):
        k = len(hs)
        hp = (vp * k)(*[h._h.value if h else None for h in hs])
        lp = (vp * k)(*rows)
        return fn(sess._h, hp, lp, lp, n.ctypes.data, k, out.data_ptr(), off.ctypes.data, got.ctypes.data, status.data_ptr())

    assert raw([e, None], [x.data_ptr()] * 2) == ERR_HANDLE
    assert raw([e, e], [x.data_ptr()] * 2) == ERR_HANDLE
    assert raw([e, f], [x.data_ptr()] * 2) == ERR_CONFIG
    assert raw([t], [x.data_ptr()]) == ERR_HANDLE
    host = np.zeros(3000, np.int16)
    assert raw([f], [host.ctypes.data]) == ERR_HANDLE
    pinned = torch.zeros(3000, dtype=torch.int16).pin_memory()
    assert raw([f], [pinned.data_ptr()]) == ERR_HANDLE
    cap_st = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    cs = M.EncodeSession(cap_st)
    with torch.cuda.graph(g, stream=cap_st, capture_error_mode="relaxed"):
        y = x + 1
        rc = raw([f], [x.data_ptr()], sess=cs)
    assert rc == ERR_HANDLE
    assert L.mp3b200_encode_bytes(e._h, 1152) >= 0           # host arithmetic, bound or not
    s1.release([e])
    assert len(e.export_state()) > 0
    for s in (s1, s2, cs):
        s.close()
