"""Finished files from an encode session (DESIGN.md 15): EncodeSession.encode_streams_tagged against
encode_streams_device_tagged on the same device buffers -- the same files, lengths, gains and pass counts, with the tag
frame finished and the ReplayGain repair loop resolved on the device; the lamejs fixtures; a configuration whose tag does
not fit; a library whose analysis needs many repair passes (tests/async_tagged_worker.py); ordering by the session's stream
alone; no wait on a warm shape; more calls in flight than the ring holds, mixed with untagged calls; the refusals."""
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
from synth import make_signal, white  # noqa: E402
from test_gpu_async import CASES, SLEEP_CYCLES, signals  # noqa: E402

pytestmark = pytest.mark.gpu
LOUD = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
RG_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_replaygain_golden.json")))
FLOAT_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))
FRACTIONAL = (44100, 22050, 11025)     # lamejs's own tagged stream differs from the oracle's there (tests/test_tag_oracle.py)
FILL = 0xA5


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


class Tagged:
    """one packed batch in device memory and the room of its files, a few bytes apart"""

    def __init__(self, M, ch, sr, kbps, sigs, resample=False):
        import torch
        self.cfg, self.resample = (ch, sr, kbps), resample
        self.sigs = sigs
        self.ns = np.array([len(l) for l, _ in sigs], dtype=np.int64)
        dt = sigs[0][0].dtype if sigs else np.int16
        host = np.concatenate([np.concatenate([l, r]) if ch == 2 else l for l, r in sigs] + [np.zeros(8, dt)])
        self.f32 = host.dtype == np.float32
        self.pcm_off = np.cumsum([0] + [n * ch for n in self.ns])[:-1].astype(np.int64)
        self.tfs = M.lametag_size(ch, sr, kbps, resample=resample)
        self.audio = [M.stream_bytes(ch, sr, kbps, int(n), resample) for n in self.ns]
        self.room = [a + self.tfs for a in self.audio]
        self.out_off = (np.cumsum([0] + [r + 3 for r in self.room])[:-1] + 5).astype(np.int64)
        self.out_len = int(sum(self.room)) + 3 * len(self.room) + 16
        self.pcm = torch.from_numpy(host).cuda()

    def out(self):
        import torch
        return torch.full((self.out_len,), FILL, dtype=torch.uint8, device="cuda")

    def sync(self, M, rg, pcm=None):
        """encode_streams_device_tagged into a fresh buffer: (buffer bytes, out_bytes, gains)"""
        o = self.out()
        ob, title, album = M.encode_streams_device_tagged(*self.cfg, (self.pcm if pcm is None else pcm).data_ptr(), self.pcm_off, self.ns,
                                                          o.data_ptr(), self.out_off, resample=self.resample, float32=self.f32,
                                                          find_replay_gain=rg)
        return o.cpu().numpy().tobytes(), ob, title + [album]

    def quant_passes(self, M):
        """the quantizer's pass count of the synchronous untagged call on the same PCM"""
        import torch
        o = torch.zeros(sum(self.audio) + 8, dtype=torch.uint8, device="cuda")
        tm = M.encode_streams_device(*self.cfg, self.pcm.data_ptr(), self.pcm_off, self.ns, o.data_ptr(),
                                     np.cumsum([0] + self.audio)[:-1], resample=self.resample, float32=self.f32)
        return int(tm[7])

    def rg_passes(self, M):
        """the analysis's pass count on the synchronous path: a batch needs what its slowest stream needs"""
        ch = self.cfg[0]
        return max(M.debug_replaygain(*self.cfg, l, r if ch == 2 else None, resample=self.resample)["passes"] for l, r in self.sigs)

    def run(self, sess, out, rg, pcm=None):
        return sess.encode_streams_tagged(*self.cfg, self.pcm if pcm is None else pcm, self.pcm_off, self.ns, out, self.out_off,
                                          resample=self.resample, find_replay_gain=rg)

    def files(self, buf, out_bytes):
        return [buf[o:o + n] for o, n in zip(self.out_off, out_bytes)]


def async_once(M, b, rg, sess=None):
    own = sess is None
    sess = sess or M.EncodeSession()
    o = b.out()
    ob, gains, st = b.run(sess, o, rg)
    M.check_status(st)
    got = o.cpu().numpy().tobytes()
    if own:
        sess.close()
    return got, ob, (gains.cpu().tolist() if gains is not None else None), st.cpu().tolist()


@pytest.mark.parametrize("rg", [False, True], ids=["tag", "replaygain"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_same_files_lengths_and_gains_as_the_synchronous_call(M, name, rg):
    ch, sr, kbps, rs, f32 = CASES[name]
    frame = 1152 if (M.granules_per_frame(ch, sr, kbps, rs) == 2) else 576
    out_sr = M.out_samplerate(ch, sr, kbps)
    lens = [0, 1, out_sr // 40, 1377, 5000, frame * 31, 0, frame * 64, frame * 150 + 3]
    b = Tagged(M, ch, sr, kbps, signals(ch, sr, lens, 0x7A60 + sr, f32), resample=rs)
    ref, ref_ob, ref_gains = b.sync(M, rg)
    with M.EncodeSession() as sess:
        o = b.out()
        ob, gains, st = b.run(sess, o, rg)
        assert ob == ref_ob == b.room                     # known before anything is synchronised
        assert (gains is None) == (not rg)
        M.check_status(st)
        got = o.cpu().numpy().tobytes()
    assert got == ref, name                               # the files, and the fill everywhere else
    assert all(f[:4] != bytes([FILL] * 4) for f in b.files(got, ob))
    status = st.cpu().tolist()
    assert status[:4] == [0, 0, b.quant_passes(M), 0], status
    if rg:
        assert gains.cpu().tolist() == ref_gains
    if rg and b.tfs > 0:
        assert ref_gains[-2] != M.GAIN_NOT_ENOUGH_SAMPLES
        assert status[4:] == [b.rg_passes(M), status[5], 0, 0] and status[5] >= 0, status
    else:                                                 # no analysis asked for, or the tag does not fit: none ran
        assert status[4:] == [0, 0, 0, 0]
        assert not rg or ref_gains == [M.GAIN_NOT_ENOUGH_SAMPLES] * (len(lens) + 1)


def _at(ch, out_sr):
    """offset of the tag's Radio Replay Gain field"""
    return 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19


def _check_fixture(M, name, c, l, r):
    import hashlib
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    out_sr = M.out_samplerate(ch, sr, kb)
    rs = out_sr != sr
    b = Tagged(M, ch, sr, kb, [(l, r)], resample=rs)
    got, ob, gains, _ = async_once(M, b, True)
    f = b.files(got, ob)[0]
    at = _at(ch, out_sr)
    assert M.radio_gain(gains[0]) == c["radio_gain"][-1], name
    assert f[at:at + 2] == bytes.fromhex(c["tag"])[at:at + 2], name
    if out_sr not in FRACTIONAL:
        e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs)
        ph = e.flush()[:b.tfs]
        e.close()
        assert hashlib.sha256(ph + f[len(ph):]).hexdigest() == c["sha256"], name


@pytest.mark.parametrize("name", sorted(n for n, c in RG_GOLDEN.items() if len(c["schedule"]) == 2 and c["schedule"][1] == -1))
def test_replaygain_fixture(M, name):
    """lamejs's ReplayGain fixtures of one encodeBuffer call and a flush, Int16 rows"""
    c = RG_GOLDEN[name]
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], seed=c["seed"])
    _check_fixture(M, name, c, l, r if c["channels"] == 2 else None)


@pytest.mark.parametrize("name", sorted(n for n, c in FLOAT_GOLDEN.items()
                                        if c["rg"] and len(c["schedule"]) == 2 and c["schedule"][0][1] == "f"))
def test_float_replaygain_fixture(M, name):
    """lamejs's Float32 ReplayGain fixtures of one encodeBuffer call and a flush"""
    c = FLOAT_GOLDEN[name]
    l, r, _ = FS.case_signal(c)
    _check_fixture(M, name, c, l.astype(np.float32), None if r is None else r.astype(np.float32))


def test_a_tag_that_does_not_fit(M):
    """(1, 8000, 8): no tag frame, nothing analysed -- audio only, every gain -24601, as the synchronous call"""
    b = Tagged(M, 1, 8000, 8, signals(1, 8000, [0, 700, 9000, 576 * 40 + 1], 0x0F17))
    assert b.tfs == 0
    ref, ref_ob, ref_gains = b.sync(M, True)
    got, ob, gains, status = async_once(M, b, True)
    assert got == ref and ob == ref_ob == b.audio
    assert gains == ref_gains == [M.GAIN_NOT_ENOUGH_SAMPLES] * 5
    assert status[4:] == [0, 0, 0, 0]


def test_the_repair_loop_iterates_on_the_device(M, tmp_path):
    """A C2-length stream needs more repair passes than are queued ahead, so the graph's WHILE loop runs the rest, pass
    after pass, and reports the synchronous loop's count.  Libraries built with one-window chunks from a wrong guess and no
    pass queued ahead (every repair is the graph's), and with 64-window chunks, give the default build's files and gains."""
    from concurrent.futures import ThreadPoolExecutor

    from lamejs_b200 import build
    from test_gpu_replaygain_variants import VARIANTS
    l, r = make_signal("sweep", 10000 * 1152, 44100, seed=1)
    b = Tagged(M, 2, 44100, 128, [(l, r)])
    ref, ref_ob, ref_gains = b.sync(M, True)
    _, _, _, status = async_once(M, b, True)
    assert status[4] == b.rg_passes(M) > 4, status         # 4: the default RG_QUEUED_PASSES
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        libs = {n: f.result() for n, f in {n: ex.submit(build.build, variant="tagged_" + n, defines=d, out_dir=str(tmp_path))
                                           for n, d in VARIANTS.items()}.items()}
    import hashlib
    want = {"sha256": hashlib.sha256(ref).hexdigest(), "gains": ref_gains}
    for n, lib in sorted(libs.items()):
        env = dict(os.environ, MP3B200_LIB=lib)
        p = subprocess.run([sys.executable, os.path.join(HERE, "async_tagged_worker.py")], env=env, capture_output=True, text=True, timeout=1800)
        assert p.returncode == 0, p.stderr[-4000:]
        res = json.loads(p.stdout.strip().splitlines()[-1])
        print(n, "status", res["status"], "default", status)
        assert res["sha256"] == want["sha256"] and res["gains"] == want["gains"], n
        assert res["status"][:2] == [0, 0] and res["status"][3] == 0
        assert res["status"][4] == res["sync_passes"] >= 1, (n, res)
        if "RG_QUEUED_PASSES=0" in VARIANTS[n]:           # no pass queued ahead: the graph's body ran every chunk again
            assert res["status"][5] > 1000, (n, res)


def test_ordered_by_the_sessions_stream_alone(M):
    import torch
    s = torch.cuda.Stream()
    b = Tagged(M, 2, 22050, 64, signals(2, 22050, [4000, 576 * 70 + 9, 576 * 33], 0x0DE8))
    ref, _, ref_gains = b.sync(M, True)
    src = b.pcm.clone()
    with M.EncodeSession(s) as sess:
        warm = b.out()
        s.wait_stream(torch.cuda.current_stream())
        M.check_status(b.run(sess, warm, True)[2])       # the shape is warm: no buffer grows below
        with torch.cuda.stream(s):
            pcm = torch.zeros_like(src)
            o = b.out()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            pcm.copy_(src)                               # a torch kernel writes the PCM ...
        _, gains, st = b.run(sess, o, True, pcm=pcm)     # ... the encode and the analysis read it ...
        with torch.cuda.stream(s):
            seen = o.clone()                             # ... and torch kernels read the results, no synchronise between
            g, words = gains.clone(), st.clone()
        s.synchronize()
        assert seen.cpu().numpy().tobytes() == ref
        assert g.cpu().tolist() == ref_gains
        assert words.cpu().tolist()[:2] == [0, 0] and words.cpu().tolist()[3] == 0


@pytest.mark.parametrize("rg", [False, True], ids=["tag", "replaygain"])
def test_the_call_does_not_wait(M, rg):
    import torch
    s = torch.cuda.Stream()
    b = Tagged(M, 2, 44100, 128, signals(2, 44100, [5000, 1152 * 40 + 3, 1152 * 90], 0xD00E))
    ref, _, ref_gains = b.sync(M, rg)
    with M.EncodeSession(s) as sess:
        o = b.out()
        s.wait_stream(torch.cuda.current_stream())
        M.check_status(b.run(sess, o, rg)[2])            # warm: workspace, staging and both loop graphs exist
        o2 = b.out()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
        _, gains, st = b.run(sess, o2, rg)
        assert not s.query(), "the call waited for the device"
        s.synchronize()
        assert o2.cpu().numpy().tobytes() == ref
        assert M.check_status(st) >= 2
        assert not rg or gains.cpu().tolist() == ref_gains


def test_calls_in_flight_mixed_with_untagged_calls(M):
    import torch
    from test_gpu_async import Batch
    s = torch.cuda.Stream()
    sigs = signals(2, 44100, [3000, 1152 * 6, 1152 * 60 + 5], 0xF119)
    t = Tagged(M, 2, 44100, 128, sigs)
    u = Batch(M, 2, 44100, 128, sigs)
    refs = {"tag": t.sync(M, False), "rg": t.sync(M, True), "plain": u.sync(M)[0]}
    torch.cuda.synchronize()
    with M.EncodeSession(s) as sess:
        pending = []
        for i in range(3 * 4 + 2):                       # more than MP3B200_SESSION_SLOTS calls queued before any is looked at
            kind = ("tag", "rg", "plain")[i % 3]
            with torch.cuda.stream(s):
                o = u.out() if kind == "plain" else t.out()
            pending.append((kind, o) + ((None, None, u.run(sess, o)) if kind == "plain" else t.run(sess, o, kind == "rg")))
        s.synchronize()
        for kind, o, ob, gains, st in pending:
            M.check_status(st)
            if kind == "plain":
                assert o.cpu().numpy().tobytes() == refs[kind]
                continue
            assert o.cpu().numpy().tobytes() == refs[kind][0] and ob == refs[kind][1]
            assert gains is None or gains.cpu().tolist() == refs[kind][2]


def test_two_sessions_from_two_threads(M):
    import torch
    b1 = Tagged(M, 2, 44100, 128, signals(2, 44100, [1152 * 50 + 7, 3000], 0x1503))
    b2 = Tagged(M, 1, 16000, 24, signals(1, 16000, [576 * 120, 9000, 576 * 7 + 1], 0x1504))
    refs = [b1.sync(M, True), b2.sync(M, True)]
    torch.cuda.synchronize()
    errors = []

    def work(b, k):
        try:
            s = torch.cuda.Stream()
            with M.EncodeSession(s) as sess:
                for i in range(4):
                    with torch.cuda.stream(s):
                        o = b.out()
                    ob, gains, st = b.run(sess, o, True)
                    s.synchronize()
                    M.check_status(st)
                    if (o.cpu().numpy().tobytes(), ob, gains.cpu().tolist()) != refs[k]:
                        errors.append("thread %d call %d" % (k, i))
        except Exception as e:                           # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(b1, 0)), threading.Thread(target=work, args=(b2, 1))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_more_than_65535_streams(M):
    """two launch groups and two k_music_crc groups, the same files; with the analysis the batch is refused as the
    synchronous call refuses it"""
    rng = np.random.default_rng(3)
    sigs = [(rng.integers(-3000, 3000, size=int(n), dtype=np.int16), None) for n in rng.integers(0, 700, size=65535 + 100)]
    b = Tagged(M, 1, 8000, 24, sigs)
    ref, ref_ob, _ = b.sync(M, False)
    with M.EncodeSession() as sess:
        got, ob, _, _ = async_once(M, b, False, sess)
        assert got == ref and ob == ref_ob
        with pytest.raises(M.Mp3B200Error, match="error -3: ReplayGain batches hold at most 65535 streams"):
            b.run(sess, b.out(), True)
        with pytest.raises(M.Mp3B200Error, match="error -3: ReplayGain batches hold at most 65535 streams"):
            b.sync(M, True)


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")     # the refused call leaves torch's capture empty
def test_refusals(M):
    import torch
    L = M.lib()
    with M.EncodeSession() as sess:
        good = Tagged(M, 2, 44100, 128, signals(2, 44100, [5000, 1152 * 20], 0xBAD2, f32=True))
        ref = good.sync(M, True)
        # a non-finite Float32 sample
        sigs = signals(2, 44100, [5000, 1152 * 20], 0xBAD2, f32=True)
        sigs[1][0][777] = np.nan
        bad = Tagged(M, 2, 44100, 128, sigs)
        with pytest.raises(M.Mp3B200Error) as sync_err:
            bad.sync(M, True)
        _, _, st = bad.run(sess, bad.out(), True)
        with pytest.raises(M.Mp3B200Error) as async_err:
            M.check_status(st)
        assert st.cpu().tolist()[0] != 0
        assert str(async_err.value) == str(sync_err.value)
        assert async_once(M, good, True, sess)[:3] == ref            # the session's next call is right
        # loud Float32 input with a frame over its bit budget (lamejs throws)
        c = next(c for _, c in sorted(LOUD.items()) if c["thrown"] is not None and not c["rg"] and
                 FS.loud_peak(c) <= 2.0 ** 40 and c["channels"] == 1 and M.out_samplerate(1, c["samplerate"], c["kbps"]) == c["samplerate"])
        lf, _, _ = FS.loud_case_signal(c)
        loud = Tagged(M, 1, c["samplerate"], c["kbps"], [(lf.astype(np.float32), None)])
        with pytest.raises(M.Mp3B200Error, match="bit budget") as sync_err:
            loud.sync(M, False)
        _, _, st = loud.run(sess, loud.out(), False)
        with pytest.raises(M.Mp3B200Error, match="bit budget") as async_err:
            M.check_status(st)
        assert st.cpu().tolist()[1] != 0
        assert str(async_err.value) == str(sync_err.value)
        assert async_once(M, good, True, sess)[:3] == ref
        # refused before anything is queued, with the synchronous call's codes and texts
        i16 = Tagged(M, 2, 44100, 128, signals(2, 44100, [3000], 0xBAD3))
        ob = np.zeros(1, dtype=np.int64)
        neg = np.array([-5], dtype=np.int64)
        ok, c2 = (i16.pcm_off.ctypes.data, i16.ns.ctypes.data), (2, 44100, 128)
        for cfg, flags, rows in ((c2, 4, ok), (c2, 8 | M.REPLAYGAIN, ok), ((3, 44100, 128), 0, ok), ((2, 44100, 7), M.REPLAYGAIN, ok),
                                 (c2, M.REPLAYGAIN, (None, ok[1])), (c2, 0, (ok[0], None)), (c2, M.REPLAYGAIN, (ok[0], neg.ctypes.data))):
            o = i16.out()
            st = torch.zeros(8, dtype=torch.int32, device="cuda")
            gains = torch.zeros(2, dtype=torch.float64, device="cuda")
            args = (*cfg, flags, 1, i16.pcm.data_ptr(), *rows, o.data_ptr(), i16.out_off.ctypes.data, ob.ctypes.data)
            rc_async = L.mp3b200_encode_streams_tagged_async(sess._h, *args, gains.data_ptr(), st.data_ptr())
            msg_async = L.mp3b200_last_error()
            torch.cuda.synchronize()
            assert (o == FILL).all() and (st == 0).all() and (gains == 0).all()
            rc = L.mp3b200_encode_streams_tagged_device(*args, None, None)
            assert rc_async == rc < 0 and msg_async == L.mp3b200_last_error(), (cfg, flags)
        args = (2, 44100, 128, 0, -1, None, None, None, None, None, None, None, None)
        assert L.mp3b200_encode_streams_tagged_async(sess._h, *args) == -3 and L.mp3b200_last_error() == b"negative stream count"
        o, st = i16.out(), torch.zeros(8, dtype=torch.int32, device="cuda")
        head = (i16.pcm.data_ptr(), i16.pcm_off.ctypes.data, i16.ns.ctypes.data, o.data_ptr(), i16.out_off.ctypes.data)
        for flags, tail, text in ((M.REPLAYGAIN, (ob.ctypes.data, None, st.data_ptr()), b"d_gain is NULL"),
                                  (0, (ob.ctypes.data, None, None), b"d_status is NULL"),
                                  (0, (None, None, st.data_ptr()), b"out_bytes is NULL")):
            assert L.mp3b200_encode_streams_tagged_async(sess._h, 2, 44100, 128, flags, 1, *head, *tail) == -3
            assert L.mp3b200_last_error() == text
        torch.cuda.synchronize()
        assert (o == FILL).all() and (st == 0).all()
    # a stream capturing a graph
    s = torch.cuda.Stream()
    with M.EncodeSession(s) as sess:
        g = torch.cuda.CUDAGraph()
        o = i16.out()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            with pytest.raises(M.Mp3B200Error, match="capturing"):
                i16.run(sess, o, True)
        torch.cuda.synchronize()
        assert async_once(M, i16, True, sess)[:3] == i16.sync(M, True)


def test_python_wrapper_checks(M):
    import torch
    b = Tagged(M, 1, 16000, 24, signals(1, 16000, [4000], 0xC0DF))
    with M.EncodeSession() as sess:
        with pytest.raises(TypeError):
            sess.encode_streams_tagged(1, 16000, 24, b.pcm.to(torch.int32), b.pcm_off, b.ns, b.out(), b.out_off)
        with pytest.raises(ValueError):
            sess.encode_streams_tagged(1, 16000, 24, b.pcm.cpu(), b.pcm_off, b.ns, b.out(), b.out_off)
        room = int(b.out_off[0]) + b.room[0]
        with pytest.raises(ValueError):                  # room for the audio, not for the tag frame
            sess.encode_streams_tagged(1, 16000, 24, b.pcm, b.pcm_off, b.ns, b.out()[:room - 1], b.out_off)
        o = b.out()[:room]
        ob, _, st = sess.encode_streams_tagged(1, 16000, 24, b.pcm, b.pcm_off, b.ns, o, b.out_off)
        M.check_status(st)
        assert ob == b.room
