"""The graphs of the device loops belong to a thread's context (DESIGN.md 14): a bounded cache of at most MP3_LOOP_GRAPHS
(32) of them, the least recently used going first.  More speculated launch shapes than the bound go through the
synchronous call on one thread and the first shape runs again, evicted and captured anew; a larger call between two calls
of one shape reallocates the workspace, which drops its graphs.  Every result must be the oracle's bytes and the pass count
a fresh context gives for that shape."""
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle_lib as O  # noqa: E402
from synth import white  # noqa: E402

pytestmark = pytest.mark.gpu
CFG = (1, 16000, 24)                 # MPEG-2 mono: 576-sample frames, cheap for the oracle
LOOP_GRAPHS = 32


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def on_fresh_thread(fn):
    """fn() on a new thread, whose context (and graph cache) starts empty"""
    out = {}

    def run():
        try:
            out["r"] = fn()
        except BaseException as e:  # noqa: BLE001
            out["e"] = e
    t = threading.Thread(target=run)
    t.start()
    t.join()
    if "e" in out:
        raise out["e"]
    return out["r"]


def encode(M, sigs):
    """one encode_streams_device call of the streams `sigs`: (bytes per stream, quantizer passes)"""
    import torch
    ns = np.array([len(x) for x in sigs], dtype=np.int64)
    nb = [M.stream_bytes(*CFG, int(n)) for n in ns]
    pcm = torch.from_numpy(np.concatenate(sigs + [np.zeros(8, np.int16)])).cuda()
    out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
    pcm_off = np.cumsum([0] + list(ns))[:-1]
    out_off = np.cumsum([0] + nb)[:-1]
    tm = M.encode_streams_device(*CFG, pcm.data_ptr(), pcm_off, ns, out.data_ptr(), out_off)
    o = out.cpu().numpy()
    return [o[a:a + b].tobytes() for a, b in zip(out_off, nb)], int(tm[7])


def shape(k):
    """one stream of 10 + k frames: a launch shape of its own, which speculates"""
    return [white(576 * (10 + k) + 37, 0x100B + k)[0]]


def test_evicted_graphs_are_captured_again(M):
    shapes = [shape(k) for k in range(LOOP_GRAPHS + 2)]
    fresh = [on_fresh_thread(lambda s=s: encode(M, s)) for s in shapes]
    order = list(range(len(shapes))) + [0, 1]            # 0 and 1 are evicted by the time they run again
    got = on_fresh_thread(lambda: [encode(M, shapes[k]) for k in order])
    for k, (g, (ref_bytes, ref_passes)) in zip(order, zip(got, [fresh[k] for k in order])):
        assert g[0][0] == O.encode_stream(*CFG, shapes[k][0])[0], k
        assert g == (ref_bytes, ref_passes), k
    assert min(p for _, p in fresh) >= 2


def test_graphs_survive_a_workspace_reallocation(M):
    small = shape(3)
    large = [white(576 * 900 + 11, 0x2B00 + i)[0] for i in range(6)]
    ref = on_fresh_thread(lambda: encode(M, small))

    def run():
        first = encode(M, small)
        encode(M, large)                                 # grows the workspace: the graphs of `small` hold stale addresses
        return first, encode(M, small)
    first, again = on_fresh_thread(run)
    assert first == ref and again == ref
    assert again[0][0] == O.encode_stream(*CFG, small[0])[0]
