"""Host logic of segmented finished files (lamejs_b200/sharding.py encode_segments_tagged / _local): the ranges' audio joined
in order behind the tag frame's room, the analysis run once and on rank 0 only, and the re-encode path, with the toy encoder
of test_segments_cpu.py and stand-ins for the analysis and the tag step; world-size-2 and -3 gloo runs on CPU.  Also the
argument checks of the C entry points behind them, which refuse bad calls before touching the device."""
import ctypes
import hashlib
import os
import struct
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from lamejs_b200 import sharding  # noqa: E402
from test_segments_cpu import FS, ToyEncoder, signal, whole  # noqa: E402

ROOM = 29


def toy_finish(buf, title_db):
    """a stand-in for the tag step: the room must still be zero and the audio behind it; writes a digest of both"""
    assert not buf[:ROOM].any()
    audio = buf[ROOM:].numpy().tobytes()
    tag = b"T" + struct.pack("<d", -1.0 if title_db is None else title_db) + hashlib.sha1(audio).digest()
    buf[:ROOM] = torch.frombuffer(bytearray(tag), dtype=torch.uint8)
    return len(buf)


def expected(pcm, shift, title_db):
    audio = whole(pcm, shift)
    return b"T" + struct.pack("<d", -1.0 if title_db is None else title_db) + hashlib.sha1(audio).digest() + audio


@pytest.mark.parametrize("nseg,warmup,shift", [(1, 8, 4), (3, 8, 4), (4, 2, 1), (6, 3, 4)])
@pytest.mark.parametrize("gain", [None, -3.75])
def test_local_file_is_the_whole_stream_behind_its_tag(nseg, warmup, shift, gain):
    pcm = signal(40 * FS + 321)
    calls = []

    def analyse():
        calls.append(1)
        return gain

    got, redone, title = sharding.encode_segments_tagged_local(lambda: ToyEncoder(shift), pcm, None, FS, nseg, warmup, ROOM,
                                                               None if gain is None else analyse, toy_finish)
    assert got == expected(pcm, shift, gain)
    assert title == gain and len(calls) == (0 if gain is None else 1)
    if shift == 1 and nseg > 1:
        assert redone >= 1


def test_no_room_and_short_streams():
    for n in (0, 300, 2 * FS):
        pcm = signal(n, seed=n + 2)
        got, _, _ = sharding.encode_segments_tagged_local(lambda: ToyEncoder(4), pcm, None, FS, 5, 3, 0, None,
                                                          lambda buf, t: len(buf))
        assert got == whole(pcm, 4)


def test_analysis_error_is_raised():
    def bad():
        raise RuntimeError("analysis failed")
    with pytest.raises(RuntimeError, match="analysis failed"):
        sharding.encode_segments_tagged_local(lambda: ToyEncoder(4), signal(5 * FS), None, FS, 2, 2, ROOM, bad, toy_finish)


def _worker(rank, world, port, shift, warmup, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pcm = signal(50 * FS + 99)
    ran = []

    def analyse():
        ran.append(rank)
        return 0.5 + rank

    got, redone, title = sharding.encode_segments_tagged(lambda: ToyEncoder(shift), pcm, None, FS, ROOM, analyse, toy_finish,
                                                         warmup=warmup)
    q.put((rank, got == expected(pcm, shift, 0.5) if rank == 0 else got is None, redone, title, ran))
    dist.destroy_process_group()


@pytest.mark.parametrize("world,shift,warmup", [(2, 4, 8), (3, 4, 8), (3, 1, 2)])
def test_tagged_segments_over_gloo(world, shift, warmup):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29950 + (os.getpid() % 300) + 7 * world + shift
    procs = [ctx.Process(target=_worker, args=(r, world, port, shift, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    for rank, ok, redone, title, ran in got:
        assert ok, rank
        assert ran == ([0] if rank == 0 else [])                 # the stream is analysed once, on rank 0
        assert title == (0.5 if rank == 0 else None)
        assert (redone == 0) if shift == 4 else (redone >= 1)


@pytest.fixture(scope="module")
def L():
    from lamejs_b200 import encoder
    return encoder.lib()


def test_c_entries_refuse_bad_arguments_before_the_device(L):
    vp = ctypes.c_void_p
    one = np.array([1000], dtype=np.int64)
    row = np.zeros(1000, dtype=np.int16)
    rows = (vp * 1)(row.ctypes.data)
    title = np.zeros(1, dtype=np.float64)
    got = np.zeros(1, dtype=np.int64)
    for host in ("mp3b200_replaygain_streams", "mp3b200_replaygain_streams_f32"):
        fn = getattr(L, host)
        assert fn(2, 44100, 128, 0, -1, rows, None, one.ctypes.data, title.ctypes.data, None) == -3
        assert fn(2, 44100, 128, 0, 1, None, None, one.ctypes.data, title.ctypes.data, None) == -3
        assert fn(2, 44100, 128, 0, 1, rows, None, None, title.ctypes.data, None) == -3
        assert fn(2, 44100, 128, 0, 1, (vp * 1)(None), None, one.ctypes.data, title.ctypes.data, None) == -3
        assert fn(2, 44100, 128, 4, 1, rows, None, one.ctypes.data, title.ctypes.data, None) == -1
        assert fn(2, 44100, 128, 2, 1, rows, None, one.ctypes.data, title.ctypes.data, None) == -1      # REPLAYGAIN is implied
        assert fn(2, 44100, 128, 0, 1, rows, None, np.array([-5], np.int64).ctypes.data, title.ctypes.data, None) == -3
    off = np.zeros(1, dtype=np.int64)
    for dev in ("mp3b200_replaygain_streams_device", "mp3b200_replaygain_streams_device_f32"):
        fn = getattr(L, dev)
        assert fn(2, 44100, 128, 0, -1, row.ctypes.data, off.ctypes.data, one.ctypes.data, None, None) == -3
        assert fn(2, 44100, 128, 0, 1, None, off.ctypes.data, one.ctypes.data, None, None) == -3
        assert fn(2, 44100, 128, 0, 1, row.ctypes.data, None, one.ctypes.data, None, None) == -3
        assert fn(2, 44100, 128, 0, 1, row.ctypes.data, off.ctypes.data, None, None, None) == -3
        assert fn(2, 44100, 128, 8, 1, row.ctypes.data, off.ctypes.data, one.ctypes.data, None, None) == -1
    fn = L.mp3b200_finish_tags_device
    assert fn(2, 44100, 128, 0, -1, row.ctypes.data, off.ctypes.data, one.ctypes.data, None, got.ctypes.data) == -3
    assert fn(2, 44100, 128, 0, 1, None, off.ctypes.data, one.ctypes.data, None, got.ctypes.data) == -3
    assert fn(2, 44100, 128, 0, 1, row.ctypes.data, None, one.ctypes.data, None, got.ctypes.data) == -3
    assert fn(2, 44100, 128, 0, 1, row.ctypes.data, off.ctypes.data, None, None, got.ctypes.data) == -3
    assert fn(2, 44100, 128, 0, 1, row.ctypes.data, off.ctypes.data, one.ctypes.data, None, None) == -3
    assert fn(2, 44100, 128, 2, 1, row.ctypes.data, off.ctypes.data, one.ctypes.data, None, got.ctypes.data) == -1


def test_resampled_configuration_is_refused_for_segments():
    with pytest.raises(ValueError, match="resampled"):
        sharding.encode_stream_segments_tagged_local(2, 48000, 64, np.zeros(5000, np.int16), None, 2)
