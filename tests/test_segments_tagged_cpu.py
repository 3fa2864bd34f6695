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


# Every synchronous whole-stream entry point: its arguments in order (F: flags, N: nstreams, or a buffer role), and which
# flag bits it takes.  MP3B200_REPLAYGAIN (2) belongs to the tagged encodes alone.
HOST = ("left", "right", "nsamples")
DEVICE = ("d_pcm", "pcm_off", "nsamples")
ENTRIES = {
    "mp3b200_encode_streams": (("N",) + HOST + ("out", "cap", "out_bytes"), None),
    "mp3b200_encode_streams_ex": (("F", "N") + HOST + ("out", "cap", "out_bytes"), 1),
    "mp3b200_encode_streams_f32": (("F", "N") + HOST + ("out", "cap", "out_bytes"), 1),
    "mp3b200_encode_streams_tagged": (("N",) + HOST + ("out", "cap", "out_bytes"), None),
    "mp3b200_encode_streams_tagged_ex": (("F", "N") + HOST + ("out", "cap", "out_bytes", "title", "album"), 3),
    "mp3b200_encode_streams_tagged_f32": (("F", "N") + HOST + ("out", "cap", "out_bytes", "title", "album"), 3),
    "mp3b200_replaygain_streams": (("F", "N") + HOST + ("title", "album"), 1),
    "mp3b200_replaygain_streams_f32": (("F", "N") + HOST + ("title", "album"), 1),
    "mp3b200_encode_streams_device": (("N",) + DEVICE + ("d_out", "out_off", "timings"), None),
    "mp3b200_encode_streams_device_ex": (("F", "N") + DEVICE + ("d_out", "out_off", "timings"), 1),
    "mp3b200_encode_streams_device_f32": (("F", "N") + DEVICE + ("d_out", "out_off", "timings"), 1),
    "mp3b200_encode_streams_tagged_device": (("F", "N") + DEVICE + ("d_out", "out_off", "out_bytes", "title", "album"), 3),
    "mp3b200_encode_streams_tagged_device_f32": (("F", "N") + DEVICE + ("d_out", "out_off", "out_bytes", "title", "album"), 3),
    "mp3b200_replaygain_streams_device": (("F", "N") + DEVICE + ("title", "album"), 1),
    "mp3b200_replaygain_streams_device_f32": (("F", "N") + DEVICE + ("title", "album"), 1),
    "mp3b200_finish_tags_device": (("F", "N", "d_pcm", "pcm_off", "nsamples", "title", "out_bytes"), 1),
}
# what each entry cannot do without: the rows, the offsets of device rows, and the arrays it writes
OPTIONAL = {"right", "d_out", "title", "album", "timings"}


def test_c_entries_refuse_bad_arguments_before_the_device(L):
    """every bad argument of a whole-stream call is refused by one gate before the configuration and before any CUDA call,
    so a machine without a device answers with the gate's code, never MP3B200_ERR_CUDA"""
    import torch

    vp = ctypes.c_void_p
    C = ctypes.CDLL(L._name)                      # a handle of our own: argtypes set here leave the binding's alone
    i16, f32 = np.zeros(2000, np.int16), np.zeros(2000, np.float32)
    bufs = {"nsamples": np.array([1000], np.int64), "pcm_off": np.zeros(1, np.int64), "out_off": np.zeros(1, np.int64),
            "cap": np.array([1 << 16], np.int64), "out_bytes": np.zeros(1, np.int64), "title": np.zeros(1, np.float64),
            "album": np.zeros(1, np.float64), "timings": np.zeros(16, np.float32), "d_out": np.zeros(1 << 16, np.uint8)}
    out = np.zeros(1 << 16, np.uint8)
    for name, (roles, takes) in ENTRIES.items():
        rows = f32 if name.endswith("_f32") else i16
        fn = getattr(C, name)
        fn.argtypes = [ctypes.c_int] * 3 + [ctypes.c_int if r in ("F", "N") else vp for r in roles]

        def call(n=1, flags=0, **over):
            host = {"left": (vp * 1)(rows.ctypes.data), "right": None, "d_pcm": rows.ctypes.data, "out": (vp * 1)(out.ctypes.data)}
            args = []
            for r in roles:
                v = {"F": flags, "N": n}.get(r, host.get(r, bufs[r].ctypes.data if r in bufs else None))
                args.append(over.get(r, v))
            return fn(2, 44100, 128, *args)

        if not torch.cuda.is_available():             # the base call is valid: only the missing device refuses it
            assert call() == -100, name
        assert call(n=-1) == -3 and L.mp3b200_last_error() == b"negative stream count", name
        for r in roles:
            if r in ("F", "N") or r in OPTIONAL:
                continue
            want = {"out_bytes": b"file_bytes is NULL" if "finish_tags" in name else b"out_bytes is NULL"}.get(r, b"null array")
            assert call(**{r: None}) == -3 and L.mp3b200_last_error() == want, (name, r)
        if "left" in roles:
            assert call(left=(vp * 1)(None)) == -3 and L.mp3b200_last_error() == b"null row", name
        assert call(nsamples=np.array([-5], np.int64).ctypes.data) == -3, name
        assert L.mp3b200_last_error() == b"negative sample count", name
        if takes is not None:
            for flags in (4, 8, 1 << 30, 2 | 4, 2):
                if flags & ~takes:
                    assert call(flags=flags) == -1 and L.mp3b200_last_error() == b"unknown flags", (name, flags)
    for name in ("mp3b200_debug_replaygain", "mp3b200_debug_replaygain_f32"):       # one stream of its own
        fn = getattr(C, name)
        fn.argtypes = [ctypes.c_int] * 4 + [vp, vp, ctypes.c_int64, vp, vp, ctypes.c_int64, vp, vp, vp]
        rows = f32 if name.endswith("_f32") else i16
        assert fn(2, 44100, 128, 0, None, None, 1000, None, None, 0, None, None, None) == -3, name
        assert L.mp3b200_last_error() == b"null row", name
        assert fn(2, 44100, 128, 0, rows.ctypes.data, None, -5, None, None, 0, None, None, None) == -3, name


def test_resampled_configuration_is_refused_for_segments():
    with pytest.raises(ValueError, match="resampled"):
        sharding.encode_stream_segments_tagged_local(2, 48000, 64, np.zeros(5000, np.int16), None, 2)
