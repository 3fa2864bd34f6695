"""Streaming handles fed from device memory (mp3b200_encode_device / _f32 / _batch_device / _batch_device_f32, and CUDA
tensors through Mp3Encoder.encodeBuffer / encode_batch): call by call the bytes, errors and exported state of the same
handles fed from host memory, and the oracle's bytes; the lamejs fixtures; random call schedules mixing host and device
calls; batch semantics; tags and ReplayGain; refusals before anything changes; pointer checks; ordering behind torch work."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import float_signals as FS
import handle_schedule as HS
import oracle_lib as O
from synth import make_signal

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FIX = json.load(open(os.path.join(HERE, "golden", "lamejs_golden.json")))["cases"]
FLOAT_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))
LOUD_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
FRACTIONAL = (44100, 22050, 11025)     # see tests/test_float_golden_cpu.py
ERR_CONFIG, ERR_HANDLE = -1, -3
vp = ctypes.c_void_p


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def sha(b):
    return hashlib.sha256(b).hexdigest()


def cuda(a):
    """a device copy of the numpy row `a`, 3 samples into a larger allocation, so that rows do not start aligned"""
    import torch
    t = torch.zeros(len(a) + 8, dtype=torch.from_numpy(np.asarray(a)[:0]).dtype, device="cuda")
    t[3:3 + len(a)] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t[3:3 + len(a)]


def rs_of(M, ch, sr, kb):
    return M.out_samplerate(ch, sr, kb) != sr


def handle(M, ch, sr, kb, **kw):
    return M.Mp3Encoder(ch, sr, kb, resample=rs_of(M, ch, sr, kb), **kw)


# ---- 1. parity matrix ----

def sizes_for(chunk, n):
    if chunk == "whole":
        return [n]
    out, pos, k = [], 0, 0
    while pos < n:
        s = (1903 if k % 2 else 0) if chunk == 0 else chunk
        s = min(s, n - pos)
        out.append(s)
        pos += s
        k += 1
    return out


@pytest.mark.parametrize("chunk", [0, 1, 575, 1152, 1903, 1904, 5000, "whole"])
@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
@pytest.mark.parametrize("cfg", HS.CONFIGS + HS.RESAMPLED_CONFIGS, ids=lambda c: "%d_%d_%d" % c)
def test_parity_call_by_call(M, cfg, f32, chunk):
    """after every call: the device-fed handle's bytes equal the host-fed handle's (and, for Int16 rows, the oracle's),
    and both export byte-identical state blobs"""
    ch, sr, kb = cfg
    n = 3000 if chunk == 1 else 14000
    l, r = make_signal("noise" if f32 else "burst", n, sr, seed=11)
    if f32:
        l, r = (l * 0.71 + 0.3).astype(np.float32), (r * -0.53).astype(np.float32)
    r = r if ch == 2 else None
    dl, dr = cuda(l), None if r is None else cuda(r)
    H, D = handle(M, ch, sr, kb), handle(M, ch, sr, kb)
    oracle = None
    if not f32:
        try:
            oracle = O.OracleEncoder(ch, sr, kb)
        except ValueError:
            oracle = None
    pos = 0
    for k, s in enumerate(sizes_for(chunk, n)):
        sl = slice(pos, pos + s)
        a = H.encodeBuffer(l[sl], None if r is None else r[sl])
        b = D.encodeBuffer(dl[sl], None if dr is None else dr[sl])
        assert a == b, (k, s)
        if oracle is not None:
            assert oracle.encode_buffer(l[sl], None if r is None else r[sl]) == a, (k, s)
        assert H.export_state() == D.export_state(), (k, s)
        pos += s
    a, b = H.flush(), D.flush()
    assert a == b
    if oracle is not None:
        assert oracle.flush() == a
        oracle.close()
    H.close()
    D.close()


# ---- 2. lamejs fixtures through device calls ----

ODD_FIX = sorted(k for k, v in FIX.items() if "error" not in v and v["chunk"] and v["chunk"] % 576)


@pytest.mark.parametrize("name", ODD_FIX)
def test_lamejs_fixture_with_odd_chunks(M, name):
    c = FIX[name]
    ch = c["channels"]
    try:
        e = M.Mp3Encoder(ch, c["samplerate"], c["kbps"])
    except M.Mp3B200Error:
        pytest.skip("configuration lamejs resamples")
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], c["seed"])
    dl, dr = cuda(l), cuda(r) if ch == 2 else None
    step = c["chunk"]
    out = [e.encodeBuffer(dl[i:i + step], None if dr is None else dr[i:i + step]) for i in range(0, len(l), step)]
    out.append(e.flush())
    e.close()
    data = b"".join(out)
    assert len(data) == c["bytes"] and sha(data) == c["sha256"]
    assert len(out) == c["calls"]
    assert sha(json.dumps([len(b) for b in out]).encode()) == c["sizes_sha256"]


@pytest.mark.parametrize("name", sorted(FLOAT_GOLDEN))
def test_float_fixture(M, name):
    """lamejs's Float32 fixtures (Int16, Float32 and float64 calls), ReplayGain ones included"""
    c = FLOAT_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    _, _, calls = FS.case_signal(c)
    kw = dict(write_vbr_tag=True, find_replay_gain=True) if c["rg"] else {}
    e = handle(M, ch, sr, kb, **kw)
    out = [e.flush() if x is None else e.encodeBuffer(cuda(x[0]), None if x[1] is None else cuda(x[1])) for x in calls[:-1]]
    out.append(e.flush())
    if c["rg"]:
        out_sr = M.out_samplerate(ch, sr, kb)
        at = 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19
        assert e.replay_gain[1] == c["radio_gain"][-1] and e.lametag_frame()[at:at + 2] == bytes.fromhex(c["tag"])[at:at + 2]
        if out_sr in FRACTIONAL:
            e.close()
            return
    e.close()
    assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"]


# ---- 3. random schedules, every call host-fed or device-fed at random ----

class _DeviceFed:
    """the library, with mp3b200_encode / mp3b200_encode_batch made device calls at random (the rows copied to the GPU)"""

    def __init__(self, L, seed):
        self._L, self._rng, self.device_calls = L, np.random.default_rng(seed), 0

    def __getattr__(self, k):
        return getattr(self._L, k)

    def _dev(self, p, n, f32):
        if not p or n <= 0:
            return None
        t = ctypes.c_float if f32 else ctypes.c_int16
        return cuda(np.ctypeslib.as_array((t * n).from_address(p)).copy())

    def mp3b200_encode(self, h, l, r, n, out, cap):
        if self._rng.random() < 0.5 or n <= 0:
            return self._L.mp3b200_encode(h, l, r, n, out, cap)
        self.device_calls += 1
        dl, dr = self._dev(l, n, False), self._dev(r, n, False)
        return self._L.mp3b200_encode_device(h, dl.data_ptr(), None if dr is None else dr.data_ptr(), n, out, cap)

    def mp3b200_encode_batch(self, hp, lp, rp, ns, op, caps, m, got):
        if self._rng.random() < 0.5:
            return self._L.mp3b200_encode_batch(hp, lp, rp, ns, op, caps, m, got)
        self.device_calls += 1
        n = (ctypes.c_int32 * m).from_address(ns)
        keep = [self._dev(lp[j], n[j], False) for j in range(m)] + [self._dev(rp[j], n[j], False) if rp else None for j in range(m)]
        dp = lambda t: None if t is None else t.data_ptr()     # noqa: E731
        dl = (vp * m)(*[dp(t) for t in keep[:m]])
        dr = (vp * m)(*[dp(t) for t in keep[m:]]) if rp else None
        return self._L.mp3b200_encode_batch_device(hp, dl, dr, ns, op, caps, m, got)


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("cfg", [HS.CONFIGS[0], HS.CONFIGS[2], HS.RESAMPLED_CONFIGS[0]], ids=lambda c: "%d_%d_%d" % c)
def test_schedule_mixing_host_and_device_calls(M, cfg, seed):
    sched = HS.make_schedule(cfg, 6, 60, seed)
    ex = HS.replay(sched)
    L = _DeviceFed(M.lib(), seed)

    class Lib:
        @staticmethod
        def lib():
            return L

    assert HS.run(Lib, sched, ex) == []
    assert L.device_calls > 5
    assert any(k == "handover" for k, _ in sched.ops)


# ---- 4. batch semantics through the C ABI: device-fed handles against host-fed ones ----

class Pair:
    """handles fed from the host and their twins fed from the device, driven with the same batches"""

    def __init__(self, M, cfgs):
        self.M, self.L = M, M.lib()
        self.cfgs = cfgs
        self.h = [[M.Mp3Encoder(*c, resample=rs_of(M, *c)) for c in cfgs] for _ in range(2)]

    def batch(self, entries, f32=False, caps=None):
        """entries: (handle index or None, left, right) with numpy rows; returns (rc, out_bytes, bytes) of both sides"""
        m = len(entries)
        res = []
        for side in range(2):
            keep = []

            def ptr(a):
                if a is None:
                    return None
                a = np.ascontiguousarray(a, dtype=np.float32 if f32 else np.int16)
                t = cuda(a) if side else a
                keep.append(t)
                return t.data_ptr() if side else t.ctypes.data

            hp = (vp * m)(*[None if i is None else self.h[side][i]._h.value for i, _, _ in entries])
            lp = (vp * m)(*[ptr(l) for _, l, _ in entries])
            rp = (vp * m)(*[ptr(r) for _, _, r in entries])
            ns = np.array([0 if l is None else len(l) for _, l, _ in entries], dtype=np.int32)
            cap = np.array(caps if caps else [int(1.25 * n + 7200) for n in ns], dtype=np.int32)
            bufs = [np.zeros(int(1.25 * n + 7200), dtype=np.uint8) for n in ns]
            op = (vp * m)(*[b.ctypes.data for b in bufs])
            got = np.zeros(m, dtype=np.int32)
            name = "mp3b200_encode_batch" + ("_device" if side else "") + ("_f32" if f32 else "")
            rc = getattr(self.L, name)(hp, lp, rp, ns.ctypes.data, op, cap.ctypes.data, m, got.ctypes.data)
            res.append((rc, got.tolist(), [b[:max(int(g), 0)].tobytes() for b, g in zip(bufs, got)]))
        return res

    def same(self, entries, **kw):
        a, b = self.batch(entries, **kw)
        assert a == b
        for x, y in zip(*self.h):
            assert x.export_state() == y.export_state()
        return a

    def close(self):
        for side in self.h:
            for e in side:
                e.close()


def test_batch_semantics(M):
    ch, sr, kb = 2, 44100, 128
    P = Pair(M, [(ch, sr, kb)] * 3 + [(1, 22050, 64)])
    sig = [make_signal(k, 40000, sr, seed=i) for i, k in enumerate(["noise", "sweep", "burst", "white"])]
    pos = [0] * 4

    def take(i, n):
        l, r = sig[i]
        s = slice(pos[i], pos[i] + n)
        pos[i] += n
        return i, l[s], r[s] if P.cfgs[i][0] == 2 else None

    # a repeated handle runs as rounds; a NULL handle is -3; another configuration with frames to encode is -1
    rc, got, _ = P.same([take(0, 3000), take(1, 700), take(0, 2500), (None, None, None), take(0, 1152), take(3, 4000)])
    assert rc == 0 and got[3] == ERR_HANDLE and got[5] == ERR_CONFIG and got[0] > 0
    # a cap too small: -1, the frames come with the handle's next call
    rc, got, _ = P.same([take(0, 5000), take(1, 5000)], caps=[1, 0])
    assert rc == 0 and got[0] == -1 and got[1] > 0
    rc, got, out = P.same([take(0, 10), take(2, 6000)])
    assert rc == 0 and got[0] > 1000
    # Float32 calls on the same handles, then Int16 again: the handles switch to Float32 and stay there
    f = lambda t: (t[0], None if t[1] is None else (t[1] * 0.5 + 0.25).astype(np.float32),       # noqa: E731
                   None if t[2] is None else (t[2] * 0.5).astype(np.float32))
    rc, got, _ = P.same([f(take(0, 3001)), f(take(1, 2999)), f(take(0, 100)), f(take(2, 0))], f32=True)
    assert rc == 0
    rc, got, _ = P.same([take(1, 4000), take(0, 1), take(2, 5555), take(1, 33)])
    assert rc == 0
    # a stereo call without right rows encodes left on both channels
    rc, got, _ = P.same([(0, sig[0][0][:4000], None), (2, sig[2][0][:3000], None)])
    assert rc == 0
    P.close()


# ---- 5. tagged and ReplayGain handles ----

@pytest.mark.parametrize("cfg", [(2, 44100, 128), (1, 16000, 32), (2, 48000, 64)], ids=lambda c: "%d_%d_%d" % c)
def test_tagged_and_replaygain_handles(M, cfg):
    ch, sr, kb = cfg
    encs = [[handle(M, ch, sr, kb, write_vbr_tag=True, find_replay_gain=True) for _ in range(2)] for _ in range(2)]
    for t in range(2):
        l, r = make_signal("sweep" if t else "noise", 3 * sr + 77, sr, seed=5 + t)
        r = r if ch == 2 else None
        dl, dr = cuda(l), None if r is None else cuda(r)
        for a, b in ((0, 1733), (1733, 5000), (6733, len(l))):
            h = encs[0][t].encodeBuffer(l[a:b], None if r is None else r[a:b])
            d = encs[1][t].encodeBuffer(dl[a:b], None if dr is None else dr[a:b])
            assert h == d
        assert encs[0][t].flush() == encs[1][t].flush()
        H, D = encs[0][t], encs[1][t]
        assert H.lametag_frame() == D.lametag_frame() and H.music_crc() == D.music_crc()
        assert H.replay_gain == D.replay_gain and H.bytes_written() == D.bytes_written()
    assert M.album_gain(encs[0]) == M.album_gain(encs[1])
    for side in encs:
        for e in side:
            e.close()


# ---- 6. refusals ----

@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 3e12], ids=["nan", "inf", "-inf", "beyond_2^40"])
@pytest.mark.parametrize("frames", [True, False], ids=["completes_frames", "completes_none"])
def test_refused_float32_call_changes_nothing(M, bad, frames):
    ch, sr, kb = 2, 32000, 96
    L = M.lib()
    l, r = make_signal("noise", 20000, sr, seed=3)
    lf, rf = (l * 0.5).astype(np.float32), (r * 0.5).astype(np.float32)
    H = [M.Mp3Encoder(ch, sr, kb) for _ in range(2)]
    D = [M.Mp3Encoder(ch, sr, kb) for _ in range(2)]
    for e in H + D:
        e.encodeBuffer(lf[:3000], rf[:3000])
    n = 6000 if frames else 40
    before = [e.export_state() for e in D]
    x = rf[3000:3000 + n].copy()
    x[n // 2] = bad
    rows = [cuda(lf[3000:3000 + n]), cuda(rf[3000:3000 + n]), cuda(lf[3000:3000 + n]), cuda(x)]
    hp = (vp * 2)(D[0]._h.value, D[1]._h.value)
    lp, rp = (vp * 2)(rows[0].data_ptr(), rows[2].data_ptr()), (vp * 2)(rows[1].data_ptr(), rows[3].data_ptr())
    ns, cap, got = np.array([n, n], np.int32), np.array([0, 0], np.int32), np.zeros(2, np.int32)
    outs = [np.zeros(20000, np.uint8) for _ in range(2)]
    op = (vp * 2)(*[o.ctypes.data for o in outs])
    assert L.mp3b200_encode_batch_device_f32(hp, lp, rp, ns.ctypes.data, op, cap.ctypes.data, 2, got.ctypes.data) == ERR_CONFIG
    assert b"non-finite" in L.mp3b200_last_error()
    assert L.mp3b200_encode_device_f32(D[1]._h, rows[2].data_ptr(), rows[3].data_ptr(), n, outs[0].ctypes.data, 0) == ERR_CONFIG
    assert [e.export_state() for e in D] == before
    for h, d in zip(H, D):
        assert h.encodeBuffer(lf[3000:], rf[3000:]) == d.encodeBuffer(cuda(lf[3000:]), cuda(rf[3000:]))
        assert h.flush() == d.flush()
    for e in H + D:
        e.close()


def test_loud_call_lamejs_throws_on_is_undone(M):
    name = sorted(n for n, c in LOUD_GOLDEN.items() if not c["rg"] and c["thrown"] is not None
                  and FS.loud_peak(c) <= 2.0 ** 40)[0]
    c = LOUD_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    _, _, calls = FS.loud_case_signal(c)
    e = handle(M, ch, sr, kb)
    out = []
    for i, x in enumerate(calls):
        if i == c["thrown"]:
            before = e.export_state()
            with pytest.raises(M.Mp3B200Error, match="bit budget"):
                e.flush() if x is None else e.encodeBuffer(cuda(x[0]), None if x[1] is None else cuda(x[1]))
            assert e.export_state() == before
            break
        out.append(e.flush() if x is None else e.encodeBuffer(cuda(x[0]), None if x[1] is None else cuda(x[1])))
    e.close()
    assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"]


# ---- 7. pointer validation ----

def test_rows_not_on_the_handles_device_are_refused(M):
    import torch
    L = M.lib()
    e = M.Mp3Encoder(2, 44100, 128)
    e.encodeBuffer(*make_signal("noise", 3000, 44100, seed=1))
    before = e.export_state()
    out = np.zeros(20000, np.uint8)
    host = np.zeros(5000, np.int16)
    pinned = torch.zeros(5000, dtype=torch.int16, pin_memory=True)
    good = torch.zeros(5000, dtype=torch.int16, device="cuda")
    for p in (host.ctypes.data, pinned.data_ptr()):
        assert L.mp3b200_encode_device(e._h, p, p, 5000, out.ctypes.data, 0) == ERR_HANDLE
        assert L.mp3b200_encode_device(e._h, good.data_ptr(), p, 5000, out.ctypes.data, 0) == ERR_HANDLE
        assert b"device" in L.mp3b200_last_error()
    # a batch is refused as a whole: the good entry is not taken either
    hp, lp = (vp * 2)(e._h.value, e._h.value), (vp * 2)(good.data_ptr(), host.ctypes.data)
    ns, cap, got = np.array([5000, 5000], np.int32), np.zeros(2, np.int32), np.zeros(2, np.int32)
    op = (vp * 2)(out.ctypes.data, out.ctypes.data)
    assert L.mp3b200_encode_batch_device(hp, lp, None, ns.ctypes.data, op, cap.ctypes.data, 2, got.ctypes.data) == ERR_HANDLE
    assert e.export_state() == before
    if torch.cuda.device_count() > 1:
        other = torch.zeros(5000, dtype=torch.int16, device="cuda:1")
        assert L.mp3b200_encode_device(e._h, other.data_ptr(), other.data_ptr(), 5000, out.ctypes.data, 0) == ERR_HANDLE
        assert e.export_state() == before
        with pytest.raises(ValueError):
            e.encodeBuffer(other, other)
    e.close()


# ---- 8. ordering ----

@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_waits_for_torch_work_on_the_default_stream(M, f32):
    import torch
    n = 44100
    t = torch.arange(2 * n, device="cuda", dtype=torch.float64)
    d = torch.zeros(2 * n, dtype=torch.float32 if f32 else torch.int16, device="cuda")
    out = np.zeros(int(1.25 * n + 7200), np.uint8)
    fn = M.lib().mp3b200_encode_device_f32 if f32 else M.lib().mp3b200_encode_device

    def write():
        x = torch.sin(t * 0.031) * 12000 + torch.sin(t * 0.0007) * 9000
        d.copy_(x if f32 else x.round())

    # everything once with the same shapes, so that nothing below allocates (which would synchronise the device)
    warm = M.Mp3Encoder(2, 44100, 128)
    write()
    torch.cuda._sleep(1000)
    fn(warm._h, d[:n].data_ptr(), d[n:].data_ptr(), n, out.ctypes.data, 0)
    warm.close()
    e = M.Mp3Encoder(2, 44100, 128)
    d.zero_()
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    write()
    k = fn(e._h, d[:n].data_ptr(), d[n:].data_ptr(), n, out.ctypes.data, 0)
    got = out[:k].tobytes() + e.flush()
    e.close()
    pcm = d.cpu().numpy()
    h = M.Mp3Encoder(2, 44100, 128)
    want = h.encodeBuffer(pcm[:n], pcm[n:]) + h.flush()
    h.close()
    assert got == want and len(got) > 1000


def test_rows_made_on_a_side_stream(M):
    import torch
    n = 30000
    l, r = make_signal("noise", n, 44100, seed=9)
    src = torch.from_numpy(np.stack([l, r]).astype(np.float32)).cuda()
    torch.cuda.synchronize()
    e = M.Mp3Encoder(2, 44100, 128)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(100_000_000)
        x = src * 0.5
        got = e.encodeBuffer(x[0], x[1]) + e.flush()
    e.close()
    h = M.Mp3Encoder(2, 44100, 128)
    xf = (np.stack([l, r]).astype(np.float32) * np.float32(0.5))
    want = h.encodeBuffer(xf[0], xf[1]) + h.flush()
    h.close()
    assert got == want


# ---- 9. Python dispatch ----

def test_python_dispatch(M):
    import torch
    l, r = make_signal("sweep", 20000, 44100, seed=4)
    for dt in (torch.int16, torch.float32, torch.float64):
        a = l if dt == torch.int16 else (l * 0.37).astype(np.float64)
        b = r if dt == torch.int16 else (r * 0.41).astype(np.float64)
        H, D = M.Mp3Encoder(2, 44100, 128), M.Mp3Encoder(2, 44100, 128)
        ta, tb = torch.from_numpy(np.asarray(a)).to(dt).cuda(), torch.from_numpy(np.asarray(b)).to(dt).cuda()
        assert H.encodeBuffer(a, b) == D.encodeBuffer(ta, tb)
        assert M.encode_batch([H], [a[:7000]], [b[:7000]]) == M.encode_batch([D], [ta[:7000]], [tb[:7000]])
        assert H.export_state() == D.export_state()
        assert H.flush() == D.flush()
        with pytest.raises(ValueError):
            M.encode_batch([H, D], [a[:100], ta[:100]], [b[:100], tb[:100]])
        with pytest.raises(ValueError):
            D.encodeBuffer(ta[:100], b[:100])
        assert H.export_state() == D.export_state()
        H.close()
        D.close()
    mono = M.Mp3Encoder(1, 22050, 32)
    ref = M.Mp3Encoder(1, 22050, 32)
    assert mono.encodeBuffer(torch.from_numpy(l[:9000]).cuda()) == ref.encodeBuffer(l[:9000])
    mono.close()
    ref.close()


def test_two_dimensional_rows(M):
    """encode_batch with lefts and rights as 2-D arrays [S, n]: numpy takes the host path as before, CUDA tensors (rows of
    one tensor, as a model's output is laid out) the device path, with the same bytes"""
    import torch
    S, n = 3, 6000
    x = np.stack([np.stack(make_signal("noise", n, 44100, seed=20 + s)) for s in range(S)])     # [S, 2, n] Int16
    H = [M.Mp3Encoder(2, 44100, 128) for _ in range(S)]
    R = [M.Mp3Encoder(2, 44100, 128) for _ in range(S)]
    D = [M.Mp3Encoder(2, 44100, 128) for _ in range(S)]
    want = [R[s].encodeBuffer(x[s, 0], x[s, 1]) for s in range(S)]
    assert M.encode_batch(H, x[:, 0], x[:, 1]) == want
    t = torch.from_numpy(x).cuda()
    assert M.encode_batch(D, t[:, 0], t[:, 1]) == want
    tf = (t.double() * 0.5).float()
    assert M.encode_batch(D, tf[:, 0], tf[:, 1]) == M.encode_batch(H, (x[:, 0] * 0.5).astype(np.float32),
                                                                    (x[:, 1] * 0.5).astype(np.float32))
    assert [e.export_state() for e in H] == [e.export_state() for e in D]
    for e in H + R + D:
        e.close()


def test_one_long_row_among_many_short_ones(M):
    """a batch of one whole-file row and many live chunks: each descriptor of the gather gets only the blocks its rows need,
    and every handle's bytes equal the host-fed handle's"""
    S = 300
    long_l = make_signal("sweep", 400 * 576 + 77, 24000, seed=1)[0]
    rows = [long_l] + [make_signal("noise", 2400, 24000, seed=s)[0] for s in range(1, S)]
    H = [M.Mp3Encoder(1, 24000, 64) for _ in range(S)]
    D = [M.Mp3Encoder(1, 24000, 64) for _ in range(S)]
    for rnd in range(2):
        a = [r[rnd * 1000:] for r in rows]
        assert M.encode_batch(H, a) == M.encode_batch(D, [cuda(r) for r in a])
    assert M.flush_batch(H) == M.flush_batch(D)
    for e in H + D:
        e.close()
