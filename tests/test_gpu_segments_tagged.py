"""Finished files of streams encoded in segments: the tag step on audio already in device memory (finish_tags_device,
mp3b200_finish_tags_device) against encode_streams_device_tagged, and lamejs_b200/sharding.py's segmented files against the
whole-stream encode_streams_replaygain file and title gain, locally and over two gloo ranks on one GPU."""
import os
import sys

import numpy as np
import pytest

from synth import make_signal

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CANARY = 0x5A


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def _rs(M, ch, sr, kb):
    return M.out_samplerate(ch, sr, kb) != sr


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 48000, 64), (2, 22050, 64), (1, 16000, 40), (2, 8000, 24),
                                      (1, 11025, 32), (2, 48000, 64), (2, 32000, 24), (1, 8000, 16)])
@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_finish_tags_reproduces_the_tagged_device_files(M, ch, sr, kb, f32):
    """the audio of encode_streams_device, placed behind the room of its tag, finished with the gains of
    replay_gain_streams_device and without: encode_streams_device_tagged's files, canaries around every file untouched"""
    import torch
    rs = _rs(M, ch, sr, kb)
    lens = [0, 900, 5 * 1152 + 1, sr // 2, 2 * sr + 333]
    sig = [make_signal(k, n, sr, seed=i + 11) for i, (k, n) in enumerate(zip(("noise", "sweep", "burst", "silence", "noise"), lens))]
    dt = np.float32 if f32 else np.int16
    rows = [np.concatenate([np.asarray(l * (0.6 if f32 else 1), dt)] + ([np.asarray(r, dt)] if ch == 2 else [])) for l, r in sig]
    d_pcm = torch.from_numpy(np.concatenate(rows + [np.zeros(8, dt)])).cuda()
    pcm_off = np.cumsum([0] + [len(x) for x in rows[:-1]])
    tfs = M.lametag_size(ch, sr, kb, resample=rs)
    audio = [M.stream_bytes(ch, sr, kb, n, resample=rs) for n in lens]
    files = [a + tfs for a in audio]
    gap = 13
    file_off = np.cumsum([gap] + [f + gap for f in files[:-1]])
    size = int(file_off[-1] + files[-1] + gap)
    for rg in (False, True):
        want = torch.full((size,), CANARY, dtype=torch.uint8, device="cuda")
        got_b, _, _ = M.encode_streams_device_tagged(ch, sr, kb, d_pcm.data_ptr(), pcm_off, lens, want.data_ptr(), file_off,
                                                     resample=rs, float32=f32, find_replay_gain=rg)
        assert got_b == files
        buf = torch.full((size,), CANARY, dtype=torch.uint8, device="cuda")
        M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, lens, buf.data_ptr(), file_off + tfs, resample=rs,
                                float32=f32)
        title = None
        if rg:
            title, _ = M.replay_gain_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, lens, resample=rs, float32=f32)
        before = buf.cpu().numpy().copy()
        got = M.finish_tags_device(ch, sr, kb, buf.data_ptr(), file_off, lens, title, resample=rs)
        assert got == files
        after = buf.cpu().numpy()
        outside = np.ones(size, dtype=bool)
        for o, f in zip(file_off, files):
            outside[o:o + f] = False
        assert (after[outside] == CANARY).all()
        assert (after[outside] == before[outside]).all()
        assert after.tobytes() == want.cpu().numpy().tobytes(), rg
        if tfs == 0:
            assert (after == before).all()                     # no room: the call writes nothing
        for n, o, a in zip(lens, file_off, audio):
            if tfs:
                t = M.get_vbr_tag(after[o:o + tfs].tobytes())
                assert t["frames"] == M.stream_frames(n, ch, sr, kb, resample=rs)
                assert t["bytes"] == a + tfs


def test_config_whose_tag_does_not_fit(M):
    assert M.lametag_size(1, 8000, 16) == 0
    import torch
    l, _ = make_signal("noise", 20000, 8000, seed=1)
    d_pcm = torch.from_numpy(l).cuda()
    n = M.stream_bytes(1, 8000, 16, len(l))
    buf = torch.full((n + 10,), CANARY, dtype=torch.uint8, device="cuda")
    assert M.finish_tags_device(1, 8000, 16, buf.data_ptr(), [5], [len(l)], [3.5]) == [n]
    assert (buf.cpu().numpy() == CANARY).all()
    del d_pcm


SEG_CONFIGS = [(2, 44100, 128), (1, 44100, 128), (2, 48000, 320), (2, 24000, 64), (1, 22050, 32), (1, 8000, 16)]


def _whole(M, ch, sr, kb, l, r, rg):
    files, title, _ = M.encode_streams_replaygain(ch, sr, kb, [l], None if r is None else [r], find_replay_gain=rg)
    return files[0], title[0]


@pytest.mark.parametrize("ch,sr,kb", SEG_CONFIGS)
@pytest.mark.parametrize("f32", [False, True], ids=["int16", "float32"])
def test_local_segments_equal_the_whole_stream_file(M, ch, sr, kb, f32):
    from lamejs_b200 import sharding
    fs = 576 * M.granules_per_frame(ch, sr, kb)
    l, r = make_signal("sweep", 37 * fs + 517, sr, seed=9)
    if f32:
        l, r = (l * 0.8).astype(np.float32), (r * 0.5).astype(np.float32)
    r = r if ch == 2 else None
    for rg in (False, True):
        want, w_title = _whole(M, ch, sr, kb, l, r, rg)
        for nseg in (1, 2, 3, 8):
            for warmup in (1, 8):
                got, _, title = sharding.encode_stream_segments_tagged_local(ch, sr, kb, l, r, nseg, warmup, find_replay_gain=rg)
                assert got == want, (rg, nseg, warmup)
                assert title == w_title
        if rg and M.lametag_size(ch, sr, kb):
            assert w_title != M.GAIN_NOT_ENOUGH_SAMPLES
            tag = M.get_vbr_tag(want)
            assert tag["frames"] == M.stream_frames(len(l), ch, sr, kb)
            assert tag["bytes"] == len(want)
            assert tag["enc_padding"] > 0


def test_cuda_rows(M):
    """CUDA tensors as rows: the same file and gain as host rows"""
    import torch
    from lamejs_b200 import sharding
    l, r = make_signal("noise", 50 * 1152 + 3, 44100, seed=2)
    want, w_title = _whole(M, 2, 44100, 128, l, r, True)
    for f32 in (False, True):
        dl, dr = (torch.from_numpy(x.astype(np.float32) if f32 else x).cuda() for x in (l, r))
        got, _, title = sharding.encode_stream_segments_tagged_local(2, 44100, 128, dl, dr, 3, 8, find_replay_gain=True)
        assert got == want and title == w_title


def test_quiet_passage_re_encodes_and_is_still_equal(M):
    from lamejs_b200 import sharding
    rng = np.random.default_rng(4)
    loud = (rng.standard_normal(60 * 1152) * 6000).astype(np.int16)
    quiet = (rng.standard_normal(120 * 1152) * 12).astype(np.int16)
    l = np.concatenate([loud, quiet, loud])
    want, w_title = _whole(M, 1, 44100, 128, l, None, True)
    got, redone, title = sharding.encode_stream_segments_tagged_local(1, 44100, 128, l, None, 6, 4, find_replay_gain=True)
    assert redone >= 1
    assert got == want and title == w_title


def test_short_streams_and_more_segments_than_frames(M):
    from lamejs_b200 import sharding
    for n in (0, 700, 3 * 1152):                              # shorter than one frame, and fewer frames than segments
        l, r = make_signal("noise", n, 44100, seed=n + 1)
        for rg in (False, True):
            want, w_title = _whole(M, 2, 44100, 128, l, r, rg)
            got, _, title = sharding.encode_stream_segments_tagged_local(2, 44100, 128, l, r, 8, 8, find_replay_gain=rg)
            assert got == want and title == w_title, (n, rg)


def test_resampled_configuration_is_refused(M):
    from lamejs_b200 import sharding
    with pytest.raises(ValueError, match="resampled"):
        sharding.encode_stream_segments_tagged_local(2, 48000, 64, np.zeros(5000, np.int16), np.zeros(5000, np.int16), 2)


def _rank(rank, world, port, q):
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
    from synth import make_signal as sig
    from lamejs_b200 import sharding
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        l, r = sig("burst", 40 * 1152 + 11, 44100, seed=6)
        out = []
        for rg in (False, True):
            got, redone, title = sharding.encode_stream_segments_tagged(2, 44100, 128, l, r, warmup=4, find_replay_gain=rg)
            local = sharding.encode_stream_segments_tagged_local(2, 44100, 128, l, r, world, 4, find_replay_gain=rg) if rank == 0 else None
            out.append((got, title, local))
        q.put((rank, out, None))
    except Exception as e:                                    # reported to the test, which fails on it
        q.put((rank, None, repr(e)))
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_equal_the_local_form(M):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29750 + os.getpid() % 200
    procs = [ctx.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict((rank, (out, err)) for rank, out, err in (q.get(timeout=600) for _ in procs))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert res[0][1] is None and res[1][1] is None, res
    for got, title, local in res[0][0]:
        assert got == local[0] and title == local[2]
    for got, title, _ in res[1][0]:
        assert got is None and title is None
