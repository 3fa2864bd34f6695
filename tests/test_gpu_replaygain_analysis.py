"""ReplayGain of whole streams without the encoder (mp3b200_replaygain_streams / _f32 / _device / _device_f32,
replay_gain_streams / replay_gain_streams_device): bit for bit the title and album gains of the tagged whole-stream encode
(encode_streams_replaygain) wherever the tag fits, the CPU restatement of lamejs's analysis (tests/replaygain_ref.py) also
where it does not, lamejs's own fixtures, device rows laid out with gaps, refusals and the ordering behind torch work."""
import json
import os

import numpy as np
import pytest

import replaygain_ref as RG
from synth import make_signal

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = [(2, 48000, 128), (1, 48000, 128), (2, 44100, 128), (1, 44100, 128), (2, 32000, 128), (1, 32000, 64), (2, 24000, 64),
          (1, 24000, 64), (2, 22050, 64), (1, 22050, 64), (2, 16000, 40), (1, 16000, 40), (2, 12000, 32), (1, 12000, 32),
          (2, 11025, 32), (1, 11025, 32), (2, 8000, 24), (1, 8000, 24)]
RESAMPLED = [(2, 48000, 64), (2, 48000, 40), (2, 32000, 24), (2, 16000, 24), (2, 48000, 24), (2, 24000, 24)]
NO_TAG = [(1, 22050, 32), (1, 8000, 16), (2, 8000, 16), (1, 16000, 24), (2, 24000, 56)]     # lametag_size == 0
KINDS = ("noise", "sweep", "silence", "burst")


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def _rs(M, ch, sr, kb):
    return M.out_samplerate(ch, sr, kb) != sr


def _lengths(M, ch, sr, kb):
    """0, below one RMS window, exactly one, one + 1 (at the input rate) and about 400 frames"""
    w = (sr + 19) // 20
    return [0, w - 1, w, w + 1, 400 * 576 * M.granules_per_frame(ch, sr, kb, resample=_rs(M, ch, sr, kb)) + 77]


def _batch(M, ch, sr, kb, f32, seed=0):
    lefts, rights = [], []
    for i, n in enumerate(_lengths(M, ch, sr, kb)):
        for j, kind in enumerate(KINDS):
            l, r = make_signal(kind, n, sr, seed=seed + 10 * i + j)
            if f32:
                l, r = (l * 0.7).astype(np.float32), (r * 1.3).astype(np.float32)
            lefts.append(l)
            rights.append(r)
    return lefts, rights if ch == 2 else None


def _same(M, ch, sr, kb, lefts, rights, resample=False):
    title, album = M.replay_gain_streams(ch, sr, kb, lefts, rights, resample=resample)
    _, t_enc, a_enc = M.encode_streams_replaygain(ch, sr, kb, lefts, rights, resample=resample)
    assert title == t_enc
    assert album == a_enc
    return title, album


@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
@pytest.mark.parametrize("ch,sr,kb", NATIVE)
def test_host_entry_equals_the_tagged_encode(M, ch, sr, kb, f32):
    lefts, rights = _batch(M, ch, sr, kb, f32, seed=sr + ch)
    title, _ = _same(M, ch, sr, kb, lefts, rights)
    assert any(t != M.GAIN_NOT_ENOUGH_SAMPLES for t in title)


@pytest.mark.parametrize("ch,sr,kb", RESAMPLED)
def test_resampled_configurations(M, ch, sr, kb):
    for f32 in (False, True):
        lefts, rights = _batch(M, ch, sr, kb, f32, seed=kb)
        _same(M, ch, sr, kb, lefts, rights, resample=True)


def test_batches_of_1_to_17_streams(M):
    rng = np.random.default_rng(5)
    for S in range(1, 18):
        lens = rng.integers(0, 30000, size=S)
        sig = [make_signal(KINDS[i % 4], int(n), 44100, seed=S * 100 + i) for i, n in enumerate(lens)]
        _same(M, 2, 44100, 128, [s[0] for s in sig], [s[1] for s in sig])


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 8000, 24), (2, 22050, 64)] + NO_TAG)
def test_against_the_cpu_restatement(M, ch, sr, kb):
    """also where the tag does not fit: the encode analyses nothing there, this entry analyses the same pieces"""
    assert (M.lametag_size(ch, sr, kb) == 0) == ((ch, sr, kb) in NO_TAG)
    lens = [0, 1000, sr // 2 + 3, 3 * sr + 17]
    sig = [make_signal(k, n, sr, seed=i + 3) for i, (k, n) in enumerate(zip(KINDS, lens))]
    lefts, rights = [s[0] for s in sig], [s[1] for s in sig] if ch == 2 else None
    title, album = M.replay_gain_streams(ch, sr, kb, lefts, rights)
    hist = np.zeros(RG.HIST, dtype=np.int64)
    for i in range(len(lens)):
        ref = RG.analyze_stream(ch, sr, kb, lefts[i], rights[i] if ch == 2 else None)
        assert title[i] == ref.title_db[0], i
        hist += ref.hist[0]
    assert album == RG.analyze_result(hist.astype(np.int32))
    if (ch, sr, kb) in NO_TAG:
        _, t_enc, a_enc = M.encode_streams_replaygain(ch, sr, kb, lefts, rights)
        assert t_enc == [M.GAIN_NOT_ENOUGH_SAMPLES] * len(lens) and a_enc == M.GAIN_NOT_ENOUGH_SAMPLES


RG_GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_replaygain_golden.json")))


@pytest.mark.parametrize("name", sorted(n for n, c in RG_GOLDEN.items() if len(c["schedule"]) == 2 and c["schedule"][1] == -1))
def test_lamejs_whole_call_fixtures(M, name):
    """lamejs's fixtures of one encodeBuffer call and a flush: its gfc.RadioGain"""
    c = RG_GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    l, r = make_signal(c["kind"], c["samples"], sr, seed=c["seed"])
    title, _ = M.replay_gain_streams(ch, sr, kb, [l], [r] if ch == 2 else None, resample=_rs(M, ch, sr, kb))
    assert M.radio_gain(title[0]) == c["radio_gain"][0]


def _device_pcm(ch, lefts, rights, f32):
    """one device tensor of every stream's rows (left, then right), each stream behind a gap: (tensor, offsets)"""
    import torch
    dt = np.float32 if f32 else np.int16
    parts, offs, at = [], [], 0
    for i, l in enumerate(lefts):
        gap = np.full(3 + i % 5, 7, dtype=dt)
        parts.append(gap)
        at += len(gap)
        offs.append(at)
        rows = [np.asarray(l, dtype=dt)] + ([np.asarray(rights[i], dtype=dt)] if ch == 2 else [])
        parts += rows
        at += sum(len(x) for x in rows)
    return torch.from_numpy(np.concatenate(parts + [np.zeros(8, dtype=dt)])).cuda(), offs


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 22050, 64), (2, 8000, 24), (2, 48000, 64), (1, 8000, 16)])
@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_device_entry_equals_the_host_entry(M, ch, sr, kb, f32):
    rs = _rs(M, ch, sr, kb)
    lefts, rights = _batch(M, ch, sr, kb, f32, seed=7)
    d_pcm, offs = _device_pcm(ch, lefts, rights, f32)
    title, album = M.replay_gain_streams_device(ch, sr, kb, d_pcm.data_ptr(), offs, [len(l) for l in lefts], resample=rs,
                                                float32=f32)
    assert (title, album) == M.replay_gain_streams(ch, sr, kb, lefts, rights, resample=rs)
    assert M.replay_gain_streams_device(ch, sr, kb, 0, [], [], resample=rs) == ([], M.GAIN_NOT_ENOUGH_SAMPLES)


def test_non_finite_float_is_refused(M):
    import torch
    l, r = make_signal("noise", 20000, 44100, seed=8)
    lf, rf = (l * 0.5).astype(np.float32), (r * 0.25).astype(np.float32)
    for bad in (np.nan, np.inf, 3e38):
        x = rf.copy()
        x[12345] = bad
        d_pcm = torch.from_numpy(np.concatenate([lf, x])).cuda()
        with pytest.raises(M.Mp3B200Error, match="error -1: non-finite"):
            M.replay_gain_streams_device(2, 44100, 128, d_pcm.data_ptr(), [0], [len(lf)], float32=True)
        with pytest.raises(M.Mp3B200Error, match="error -1: non-finite"):
            M.replay_gain_streams(2, 44100, 128, [lf], [x])
    d_pcm = torch.from_numpy(np.concatenate([lf, rf])).cuda()
    assert M.replay_gain_streams_device(2, 44100, 128, d_pcm.data_ptr(), [0], [len(lf)], float32=True) == \
        M.replay_gain_streams(2, 44100, 128, [lf], [rf])


def test_more_than_65535_streams_are_refused(M):
    lefts = [np.zeros(10, np.int16)] * 65536
    with pytest.raises(M.Mp3B200Error, match="error -3: ReplayGain batches hold at most 65535 streams"):
        M.replay_gain_streams(1, 8000, 24, lefts)


@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_waits_for_torch_work_on_the_default_stream(M, f32):
    """PCM written by a torch kernel just before the call, without a synchronise, behind a long kernel: the analysis reads
    that PCM (Int16 rows are analysed where the caller left them)"""
    import torch
    n = 3 * 44100
    t = torch.arange(2 * n, device="cuda", dtype=torch.float64)

    def write_pcm(dst):
        x = torch.sin(t * 0.031) * 12000 + torch.sin(t * 0.0007) * 9000
        dst.copy_(x if f32 else x.round())

    def call():
        return M.replay_gain_streams_device(2, 44100, 128, d_pcm.data_ptr(), [0], [n], float32=f32)

    # everything once with the same shapes, so that nothing below loads a module or grows a buffer (which synchronises)
    d_pcm = torch.zeros(2 * n, dtype=torch.float32 if f32 else torch.int16, device="cuda")
    write_pcm(d_pcm)
    torch.cuda._sleep(1000)
    call()
    torch.cuda.synchronize()
    d_pcm.zero_()
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    write_pcm(d_pcm)
    title, album = call()
    pcm = d_pcm.cpu().numpy()
    assert (title, album) == M.replay_gain_streams(2, 44100, 128, [pcm[:n]], [pcm[n:]])
    assert title[0] != M.GAIN_NOT_ENOUGH_SAMPLES
