"""Encode sessions (DESIGN.md 14): whole device-resident streams queued on the caller's CUDA stream.  The same bytes and
pass counts as encode_streams_device on the same device buffers, the fixed-point loop iterating on the device (a library
built with bad speculation guesses, tests/async_worker.py), no wait for the device on a warm shape, ordering by the
session's stream alone, isolated sessions, more calls in flight than the descriptor ring holds, and the refusals."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import float_signals as FS  # noqa: E402
from synth import make_signal, sweep, white  # noqa: E402

pytestmark = pytest.mark.gpu
LOUD = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
SLEEP_CYCLES = 400_000_000           # torch.cuda._sleep: ~0.2 s on an H100


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def signals(ch, sr, lens, seed, f32=False):
    sigs = []
    for i, n in enumerate(lens):
        l, r = white(n, seed + i) if i % 3 == 0 else make_signal(("burst", "noise", "sweep")[i % 3], n, sr, seed + i)
        if f32:
            l, r = l.astype(np.float32) / 32768, r.astype(np.float32) / 32768
        sigs.append((l, r if ch == 2 else None))
    return sigs


class Batch:
    """one packed batch in device memory, laid out as encode_streams_device reads it"""

    def __init__(self, M, ch, sr, kbps, sigs, resample=False):
        import torch
        self.cfg, self.resample = (ch, sr, kbps), resample
        self.ns = np.array([len(l) for l, _ in sigs], dtype=np.int64)
        dt = sigs[0][0].dtype if sigs else np.int16
        rows = [np.concatenate([l, r]) if ch == 2 else l for l, r in sigs]
        host = np.concatenate(rows + [np.zeros(8, dt)])
        self.f32 = host.dtype == np.float32
        self.pcm_off = np.cumsum([0] + [n * ch for n in self.ns])[:-1].astype(np.int64)
        nbs = {int(n): M.stream_bytes(ch, sr, kbps, int(n), resample) for n in np.unique(self.ns)}
        self.nb = np.array([nbs[int(n)] for n in self.ns], dtype=np.int64)
        self.out_off = np.cumsum([0] + list(self.nb))[:-1].astype(np.int64)
        self.out_len = int(self.nb.sum()) + 8
        self.pcm = torch.from_numpy(host).cuda()

    def out(self):
        import torch
        return torch.full((self.out_len,), 0xA5, dtype=torch.uint8, device="cuda")

    def sync(self, M, pcm=None):
        """encode_streams_device into a fresh buffer: (bytes, timings_ms[7])"""
        o = self.out()
        tm = M.encode_streams_device(*self.cfg, (self.pcm if pcm is None else pcm).data_ptr(), self.pcm_off, self.ns,
                                     o.data_ptr(), self.out_off, resample=self.resample, float32=self.f32)
        return o.cpu().numpy().tobytes(), int(tm[7])

    def run(self, sess, out, pcm=None):
        return sess.encode_streams(*self.cfg, self.pcm if pcm is None else pcm, self.pcm_off, self.ns, out, self.out_off,
                                   resample=self.resample)


def async_once(M, b, sess=None):
    own = sess is None
    sess = sess or M.EncodeSession()
    o = b.out()
    st = b.run(sess, o)
    passes = M.check_status(st)
    got = o.cpu().numpy().tobytes()
    status = st.cpu().tolist()
    if own:
        sess.close()
    return got, passes, status


CASES = {
    "mpeg1_stereo": (2, 44100, 128, False, False),
    "mpeg1_mono": (1, 32000, 48, False, False),
    "mpeg2_stereo": (2, 22050, 64, False, False),
    "mpeg2_mono": (1, 16000, 24, False, False),
    "mpeg25_stereo": (2, 11025, 32, False, False),
    "mpeg25_mono": (1, 8000, 16, False, False),
    "resample_48_24": (2, 48000, 64, True, False),
    "float32_mpeg1": (2, 44100, 128, False, True),
    "float32_resample": (2, 48000, 64, True, True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_same_bytes_and_passes_as_the_synchronous_call(M, name):
    ch, sr, kbps, rs, f32 = CASES[name]
    frame = 1152 if (M.granules_per_frame(ch, sr, kbps, rs) == 2) else 576
    lens = [0, 1, 700, 1377, 5000, frame * 31 + 5, 0, frame * 64, frame * 150 + 3]
    b = Batch(M, ch, sr, kbps, signals(ch, sr, lens, 0xA5E0 + sr, f32), resample=rs)
    ref, ref_passes = b.sync(M)
    got, passes, status = async_once(M, b)
    assert got == ref, name
    assert passes == ref_passes and status == [0, 0, ref_passes, 0], (status, ref_passes)


def test_c2_length_stream(M):
    l, r = sweep(10000 * 1152, 44100)
    b = Batch(M, 2, 44100, 128, [(l, r)])
    ref, ref_passes = b.sync(M)
    got, passes, _ = async_once(M, b)
    assert got == ref and passes == ref_passes


def test_more_than_65535_streams(M):
    lens = [(i * 37) % 1500 for i in range(65600)]
    sigs = [(np.full(n, (i % 200) - 100, dtype=np.int16) + (np.arange(n) % 13).astype(np.int16), None) for i, n in enumerate(lens)]
    sigs[65599] = (white(30000, 11)[0], None)           # the second launch group speculates
    b = Batch(M, 1, 8000, 16, sigs)
    ref, ref_passes = b.sync(M)
    got, passes, _ = async_once(M, b)
    assert got == ref and passes == ref_passes


def test_the_device_loop_iterates(M, tmp_path):
    """with every speculated frame landing on gain 255 and no folded repair, the graph's WHILE loop does all the repair, in
    the session and in the synchronous call alike: the same passes and the same launch count"""
    from lamejs_b200 import build
    lib = build.build(variant="async_nofold", defines=["Q_SPEC_START=255", "Q_SPEC_STEP=1", "Q_SPEC_FOLD=0"], out_dir=str(tmp_path))
    env = dict(os.environ, MP3B200_LIB=lib)
    p = subprocess.run([sys.executable, os.path.join(HERE, "async_worker.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    print("async passes", res["passes"])
    assert not res["fail"], res["fail"][:20]
    assert min(res["passes"].values()) >= 3, res["passes"]


def test_the_call_does_not_wait(M):
    import torch
    s = torch.cuda.Stream()
    b = Batch(M, 2, 44100, 128, signals(2, 44100, [5000, 1152 * 40 + 3, 1152 * 90], 0xD00D))
    ref, _ = b.sync(M)
    with M.EncodeSession(s) as sess:
        o = b.out()
        s.wait_stream(torch.cuda.current_stream())
        M.check_status(b.run(sess, o))                   # the shape is warm: workspace, staging and loop graph exist
        o2 = b.out()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
        st = b.run(sess, o2)
        assert not s.query(), "the call waited for the device"
        s.synchronize()
        assert o2.cpu().numpy().tobytes() == ref
        assert M.check_status(st) >= 2


def test_ordered_by_the_sessions_stream_alone(M):
    import torch
    s = torch.cuda.Stream()
    b = Batch(M, 2, 22050, 64, signals(2, 22050, [4000, 576 * 70 + 9, 576 * 33], 0x0DE7))
    ref, _ = b.sync(M)
    src = b.pcm.clone()
    with M.EncodeSession(s) as sess:
        warm = b.out()
        s.wait_stream(torch.cuda.current_stream())
        M.check_status(b.run(sess, warm))
        with torch.cuda.stream(s):
            pcm = torch.zeros_like(src)
            o = b.out()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            pcm.copy_(src)                               # a torch kernel writes the PCM ...
        st = b.run(sess, o, pcm=pcm)                     # ... the encode reads it ...
        with torch.cuda.stream(s):
            seen = o.clone()                             # ... and a torch kernel reads the bytes, no synchronise between
            words = st.clone()
        s.synchronize()
        assert seen.cpu().numpy().tobytes() == ref
        assert words.cpu().tolist()[:2] == [0, 0] and words.cpu().tolist()[3] == 0


def test_sessions_are_isolated(M):
    import torch
    b1 = Batch(M, 2, 44100, 128, signals(2, 44100, [1152 * 50 + 7, 3000], 0x1501))
    b2 = Batch(M, 1, 16000, 24, signals(1, 16000, [576 * 120, 9000, 576 * 7 + 1], 0x1502))
    refs = [b1.sync(M)[0], b2.sync(M)[0]]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    # one thread, interleaved calls
    with M.EncodeSession(s1) as a, M.EncodeSession(s2) as c:
        outs = []
        for _ in range(3):
            for sess, b in ((a, b1), (c, b2)):
                with torch.cuda.stream(sess.stream):
                    o = b.out()
                outs.append((o, b.run(sess, o), 0 if b is b1 else 1))
        torch.cuda.synchronize()
        for o, st, k in outs:
            M.check_status(st)
            assert o.cpu().numpy().tobytes() == refs[k]
    # two threads, one session each
    errors = []

    def work(b, k, s):
        try:
            with M.EncodeSession(s) as sess:
                for _ in range(4):
                    with torch.cuda.stream(s):
                        o = b.out()
                    st = b.run(sess, o)
                    s.synchronize()
                    M.check_status(st)
                    if o.cpu().numpy().tobytes() != refs[k]:
                        errors.append("thread %d" % k)
        except Exception as e:                           # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(b1, 0, s1)), threading.Thread(target=work, args=(b2, 1, s2))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_calls_in_flight(M):
    import torch
    s = torch.cuda.Stream()
    small = Batch(M, 2, 44100, 128, signals(2, 44100, [3000, 1152 * 6], 0xF117))
    large = Batch(M, 2, 44100, 128, signals(2, 44100, [1152 * 400 + 5, 1152 * 300, 5000, 1152 * 50], 0xF118))
    refs = {id(small): small.sync(M)[0], id(large): large.sync(M)[0]}
    torch.cuda.synchronize()
    with M.EncodeSession(s) as sess:
        pending = []
        order = [small, large] + [small] * (3 * 4) + [large] * 3   # the first large call grows the workspace, unsynchronised
        for b in order:
            with torch.cuda.stream(s):
                o = b.out()
            pending.append((b, o, b.run(sess, o)))
        s.synchronize()
        for b, o, st in pending:
            M.check_status(st)
            assert o.cpu().numpy().tobytes() == refs[id(b)]


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")     # the refused call leaves torch's capture empty
def test_refusals(M):
    import torch
    with M.EncodeSession() as sess:
        good = Batch(M, 2, 44100, 128, signals(2, 44100, [5000, 1152 * 20], 0xBAD0, f32=True))
        ref, _ = good.sync(M)
        # a non-finite Float32 sample
        sigs = signals(2, 44100, [5000, 1152 * 20], 0xBAD0, f32=True)
        sigs[1][0][777] = np.nan
        bad = Batch(M, 2, 44100, 128, sigs)
        with pytest.raises(M.Mp3B200Error) as sync_err:
            bad.sync(M)
        st = bad.run(sess, bad.out())
        with pytest.raises(M.Mp3B200Error) as async_err:
            M.check_status(st)
        assert st.cpu().tolist()[0] != 0
        assert str(async_err.value) == str(sync_err.value)
        assert async_once(M, good, sess)[0] == ref        # the session's next call is right
        # loud Float32 input with a frame over its bit budget (lamejs throws)
        c = next(c for _, c in sorted(LOUD.items()) if c["thrown"] is not None and not c["rg"] and
                 FS.loud_peak(c) <= 2.0 ** 40 and c["channels"] == 1 and M.out_samplerate(1, c["samplerate"], c["kbps"]) == c["samplerate"])
        lf, _, _ = FS.loud_case_signal(c)
        loud = Batch(M, 1, c["samplerate"], c["kbps"], [(lf.astype(np.float32), None)])
        with pytest.raises(M.Mp3B200Error, match="bit budget") as sync_err:
            loud.sync(M)
        st = loud.run(sess, loud.out())
        with pytest.raises(M.Mp3B200Error, match="bit budget") as async_err:
            M.check_status(st)
        assert st.cpu().tolist()[1] != 0
        assert str(async_err.value) == str(sync_err.value)
        assert async_once(M, good, sess)[0] == ref
        # refused before anything is queued, with the synchronous call's errors
        i16 = Batch(M, 2, 44100, 128, signals(2, 44100, [3000], 0xBAD1))
        neg = np.array([-5], dtype=np.int64)
        ok, c2 = (i16.pcm_off.ctypes.data, i16.ns.ctypes.data), (2, 44100, 128)
        for cfg, flags, rows in ((c2, M.REPLAYGAIN, ok), (c2, 8, ok), ((3, 44100, 128), 0, ok), ((2, 44100, 7), 0, ok),
                                 (c2, 0, (None, ok[1])), (c2, 0, (ok[0], None)), (c2, 0, (ok[0], neg.ctypes.data))):
            for fn in (M.lib().mp3b200_encode_streams_async, M.lib().mp3b200_encode_streams_device_ex):
                o = i16.out()
                st = torch.zeros(4, dtype=torch.int32, device="cuda")
                args = (*cfg, flags, 1, i16.pcm.data_ptr(), *rows, o.data_ptr(), i16.out_off.ctypes.data)
                rc = fn(sess._h, *args, st.data_ptr()) if fn is M.lib().mp3b200_encode_streams_async else fn(*args, None)
                msg = M.lib().mp3b200_last_error()
                if fn is M.lib().mp3b200_encode_streams_async:
                    rc_async, msg_async = rc, msg
                    torch.cuda.synchronize()
                    assert (o == 0xA5).all() and (st == 0).all()
            assert rc_async == rc < 0 and msg_async == msg, (cfg, flags)
        rc = M.lib().mp3b200_encode_streams_async(sess._h, 2, 44100, 128, 0, -1, None, None, None, None, None, None)
        assert rc == -3 and M.lib().mp3b200_last_error() == b"negative stream count"
    # a stream capturing a graph
    s = torch.cuda.Stream()
    with M.EncodeSession(s) as sess:
        g = torch.cuda.CUDAGraph()
        o = i16.out()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            with pytest.raises(M.Mp3B200Error, match="capturing"):
                i16.run(sess, o)
        torch.cuda.synchronize()
        assert async_once(M, i16, sess)[0] == i16.sync(M)[0]


def test_python_wrapper_checks(M):
    import torch
    b = Batch(M, 1, 16000, 24, signals(1, 16000, [4000], 0xC0DE))
    with M.EncodeSession() as sess:
        with pytest.raises(TypeError):
            sess.encode_streams(1, 16000, 24, b.pcm.to(torch.int32), b.pcm_off, b.ns, b.out(), b.out_off)
        with pytest.raises(TypeError):
            sess.encode_streams(1, 16000, 24, b.pcm, b.pcm_off, b.ns, b.out().to(torch.int16), b.out_off)
        with pytest.raises(ValueError):
            sess.encode_streams(1, 16000, 24, b.pcm.cpu(), b.pcm_off, b.ns, b.out(), b.out_off)
        with pytest.raises(ValueError):
            sess.encode_streams(1, 16000, 24, b.pcm, b.pcm_off, b.ns, b.out()[:10], b.out_off)
