"""Tagged and ReplayGain handles in encode sessions without a GPU: the entry points are exported with the arity
include/mp3b200.h declares (and the Python binding passes), each returns MP3B200_ERR_CUDA without a device, the Python
argument checks, and the bytes each call hands out (the arithmetic behind out_bytes, placeholder included) against the
oracle on the handle schedules with their tagged streams."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import handle_schedule as HS  # noqa: E402
from test_gpu_session_handles import session_ops  # noqa: E402
ARITY = {"mp3b200_session_encode_batch_tagged": 10, "mp3b200_session_encode_batch_tagged_f32": 10,
         "mp3b200_session_flush_batch_tagged": 7, "mp3b200_session_lametag_frames": 7, "mp3b200_session_album_gain": 5,
         "mp3b200_session_graph_instantiations": 1, "mp3b200_encode_bytes_schedule": 8}
ERR_CUDA = -100


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    lamejs_b200.lib()
    return lamejs_b200


def _declared_arity(name):
    hdr = open(os.path.join(ROOT, "include", "mp3b200.h")).read()
    m = re.search(r"\b(?:int|int64_t)\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
    assert m, name
    return len(m.group(1).split(","))


@pytest.mark.parametrize("name", sorted(ARITY))
def test_exported_with_declared_arity(M, name):
    assert _declared_arity(name) == ARITY[name]
    L = ctypes.CDLL(os.path.join(ROOT, "lamejs_b200", "libmp3b200.so"))
    assert hasattr(L, name)
    assert len(getattr(M.lib(), name).argtypes) == ARITY[name]


def test_no_device_is_a_cuda_error(M):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    L = M.lib()
    n = np.zeros(1, np.int32)
    off = np.zeros(1, np.int64)
    got = np.zeros(1, np.int32)
    hp = (ctypes.c_void_p * 1)(None)
    for fn in (L.mp3b200_session_encode_batch_tagged, L.mp3b200_session_encode_batch_tagged_f32):
        assert fn(None, hp, hp, hp, n.ctypes.data, 1, None, off.ctypes.data, got.ctypes.data, None) == ERR_CUDA
    assert L.mp3b200_session_flush_batch_tagged(None, hp, 1, None, off.ctypes.data, got.ctypes.data, None) == ERR_CUDA
    assert L.mp3b200_session_lametag_frames(None, hp, 1, None, off.ctypes.data, got.ctypes.data, None) == ERR_CUDA
    assert L.mp3b200_session_album_gain(None, hp, 1, None, None) == ERR_CUDA


def test_python_argument_checks(M):
    sess = object.__new__(M.EncodeSession)
    sess._h = None
    for call in (lambda: sess.encode_batch_tagged([], []), lambda: sess.flush_batch_tagged([]),
                 lambda: sess.lametag_frames([]), lambda: sess.album_gain([]), sess.graph_instantiations):
        with pytest.raises(ValueError, match="closed"):
            call()
    sess._h = ctypes.c_void_p(1)
    sess.device = "cuda:0"
    with pytest.raises(ValueError, match="one row"):
        sess.encode_batch_tagged([object()], [])
    with pytest.raises(ValueError, match="CUDA tensors"):
        sess.encode_batch_tagged([object()], [np.zeros(4, np.int16)])
    for call in (sess.flush_batch_tagged, sess.lametag_frames, sess.album_gain):
        with pytest.raises(ValueError, match="Mp3Encoder"):
            call([object()])
    sess._h = None


@pytest.mark.parametrize("cfg", HS.CONFIGS + HS.RESAMPLED_CONFIGS, ids=lambda c: "%d_%d_%d" % c)
def test_call_bytes_match_the_oracle_call_by_call(M, cfg):
    """mp3b200_encode_bytes_schedule (the arithmetic of mp3b200_encode_bytes and of a session call's out_bytes) walks each
    stream of the schedule, tagged streams included, and gives the length of every oracle call, the placeholder of a tagged
    stream's first feeding call included"""
    ch, sr, kb = cfg
    L = M.lib()
    checked_tagged = 0
    for seed in range(3):
        full = HS.make_schedule(cfg, 6, 60, seed=seed + 40)
        s = session_ops(full)
        sched = HS.Schedule(s.cfg, s.signals, s.kinds, full.tagged, s.ops)
        ex = HS.replay(sched)
        calls = [[] for _ in range(sched.nstreams)]
        want = [[] for _ in range(sched.nstreams)]
        for (kind, entries), res in zip(sched.ops, ex.results):
            if kind == "handover":                 # the handle's accounting carries over in the state blob
                continue
            for c, w in zip(entries, res):
                calls[c.s].append(c.hi - c.lo if kind == "encode_batch" else -1)
                want[c.s].append(len(w))
        flags = 1 if sched.resample else 0
        for k in range(sched.nstreams):
            n = np.array(calls[k], np.int32)
            got = np.zeros(max(len(n), 1), np.int32)
            assert L.mp3b200_encode_bytes_schedule(ch, sr, kb, flags, int(k in sched.tagged), n.ctypes.data, len(n),
                                                   got.ctypes.data) == 0
            assert list(got[:len(n)]) == want[k], (seed, k)
            checked_tagged += int(k in sched.tagged and ex.tags[k]["tag_on"])
    if M.lametag_size(ch, sr, kb, HS.ratio_of(cfg) > 1) > 0:
        assert checked_tagged > 0


def test_call_bytes_arguments(M):
    L = M.lib()
    n = np.array([1152], np.int32)
    got = np.zeros(1, np.int32)
    assert L.mp3b200_encode_bytes_schedule(2, 44100, 128, 2, 1, n.ctypes.data, 1, got.ctypes.data) == -1      # unknown flag
    assert L.mp3b200_encode_bytes_schedule(2, 44101, 128, 0, 1, n.ctypes.data, 1, got.ctypes.data) == -1
    assert L.mp3b200_encode_bytes_schedule(2, 44100, 128, 0, 1, None, 1, got.ctypes.data) == -3
    assert L.mp3b200_encode_bytes_schedule(2, 44100, 128, 0, 1, None, 0, None) == 0
