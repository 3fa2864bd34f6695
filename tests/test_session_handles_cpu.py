"""Streaming handles in encode sessions without a GPU: the entry points are exported with the arity include/mp3b200.h
declares (and the Python binding passes), each returns MP3B200_ERR_CUDA without a device, the Python argument checks, and
the tail capacity against every state the handle schedules reach."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import handle_schedule as HS  # noqa: E402

ARITY = {"mp3b200_session_encode_batch": 10, "mp3b200_session_encode_batch_f32": 10, "mp3b200_session_flush_batch": 7,
         "mp3b200_encode_bytes": 2, "mp3b200_session_release": 3, "mp3b200_session_tail_capacity": 4}
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
    for fn in (L.mp3b200_session_encode_batch, L.mp3b200_session_encode_batch_f32):
        assert fn(None, hp, hp, hp, n.ctypes.data, 1, None, off.ctypes.data, got.ctypes.data, None) == ERR_CUDA
    assert L.mp3b200_session_flush_batch(None, hp, 1, None, off.ctypes.data, got.ctypes.data, None) == ERR_CUDA
    assert L.mp3b200_session_release(None, hp, 1) == ERR_CUDA


def test_python_argument_checks(M):
    sess = object.__new__(M.EncodeSession)
    sess._h = None
    with pytest.raises(ValueError, match="closed"):
        sess.encode_batch([], [])
    with pytest.raises(ValueError, match="closed"):
        sess.flush_batch([])
    with pytest.raises(ValueError, match="closed"):
        sess.release([])
    sess._h = ctypes.c_void_p(1)
    sess.device = "cuda:0"
    with pytest.raises(ValueError, match="one row"):
        sess.encode_batch([object()], [])
    with pytest.raises(ValueError, match="CUDA tensors"):
        sess.encode_batch([object()], [np.zeros(4, np.int16)])
    with pytest.raises(ValueError, match="Mp3Encoder"):
        sess.flush_batch([object()])
    sess._h = None


def _capacity(M, cfg):
    ch, sr, kb = cfg
    return int(M.lib().mp3b200_session_tail_capacity(ch, sr, kb, 1 if HS.ratio_of(cfg) > 1 else 0))


@pytest.mark.parametrize("cfg", HS.CONFIGS + HS.RESAMPLED_CONFIGS, ids=lambda c: "%d_%d_%d" % c)
def test_tail_capacity_holds_every_state_the_schedules_reach(M, cfg):
    """fed - hist_base after each call, from the oracle's FIFO state: every call of the schedules, resampled ones included"""
    cap = _capacity(M, cfg)
    assert cap > 0
    r = HS.ratio_of(cfg)
    G = 2 if cfg[1] // r >= 32000 else 1
    worst = 0
    for seed in range(3):
        sched = HS.make_schedule(cfg, 6, 60, seed=seed)
        ex = HS.replay(sched)
        for states in ex.states:
            for st in states.values():
                # the outputs fed: the FIFO holds 528 delay zeros + outputs - 576 G frames; flush zeros count as fed
                out_fed = int(st["mf_size"]) - 528 + 576 * G * int(st["frames_done"])
                hist_out = max(0, 576 * G * int(st["frames_done"]) - 1104)
                hist_in = max(0, r * hist_out - HS.RS_HALF) if r > 1 else hist_out
                fed_in = r * out_fed + (HS.RS_HALF if r > 1 else 0)
                worst = max(worst, fed_in - hist_in)
    assert worst <= cap, (worst, cap)
    assert worst > cap // 2                     # the bound is not loose by a wide margin
