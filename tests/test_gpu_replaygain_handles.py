"""ReplayGain on streaming handles (mp3b200_set_find_replay_gain, _get_replay_gain, _album_gain) under the random call
schedules of tests/handle_schedule.py, flush-then-continue included (tests/replaygain_worker.py), and the refusals of the
state calls."""
import ctypes

import numpy as np
import pytest

import handle_schedule as HS
import replaygain_worker as W
from synth import make_signal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("i,cfg", list(enumerate(W.CONFIGS)), ids=[str(c) for c in W.CONFIGS])
def test_random_schedules(i, cfg):
    import lamejs_b200 as M
    fail = W.play(M, HS.make_schedule(cfg, 8, 60, seed=300 + i))
    assert not fail, fail[:10]


def test_switches_and_refusals():
    import lamejs_b200 as M
    L = M.lib()
    e = M.Mp3Encoder(2, 44100, 128, write_vbr_tag=True, find_replay_gain=True)
    assert e.replay_gain_on and e.replay_gain is None
    assert L.mp3b200_export_state(e._h, None, 0) == -2
    blob = np.zeros(64, dtype=np.uint8)
    assert L.mp3b200_import_state(e._h, blob.ctypes.data, 64) == -2
    assert L.mp3b200_seek(e._h, 1, None, None, 0) == -2
    assert not M.Mp3Encoder(2, 44100, 128, find_replay_gain=True).replay_gain_on      # needs the tag
    assert not M.Mp3Encoder(1, 8000, 8, write_vbr_tag=True, find_replay_gain=True).replay_gain_on   # the tag does not fit
    l, r = make_signal("noise", 5000, 44100, seed=1)
    e.encodeBuffer(l, r)
    assert L.mp3b200_set_find_replay_gain(e._h, 0) == -3                              # only before the first sample
    e.flush()
    db, radio = e.replay_gain
    assert radio == M.radio_gain(db)
    out = ctypes.c_double(0)
    assert L.mp3b200_album_gain(None, 1, ctypes.byref(out)) == -3
