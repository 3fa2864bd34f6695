"""The edge corpus (tests/edge_signals.py: full scale, -32768, DC, Nyquist, +-1 LSB, click trains over every attack sub-block
and across the 16-frame chunks of the block-type scan, a silent channel, L = -R, level jumps, tones near 20 kHz) through
the CUDA path: every stage tap and all side-info columns bit-equal to the oracle, MPEG-1 and LSF, mono and stereo; and
the whole corpus once more as one ragged batch per configuration.  The resampled corpus (edge_signals.RESAMPLED_CASES)
takes the same two tests through k_resample and the Float32 input path (MP3B200_RESAMPLE)."""
import pytest

import edge_signals
import stage_taps

pytestmark = pytest.mark.gpu

ALL_CASES = [(c, False) for c in edge_signals.CASES] + [(c, True) for c in edge_signals.RESAMPLED_CASES]


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


@pytest.mark.parametrize("case,resample", ALL_CASES, ids=[edge_signals.case_id(c) + ("-rs" if rs else "") for c, rs in ALL_CASES])
def test_edge_stage_parity(M, oracle, case, resample):
    kind, ch, sr, kbps, frames = case
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(ch, sr, kbps, resample)
    F = M.stream_frames(len(l), ch, sr, kbps, resample)
    ref, _, tr = oracle.encode_stream(ch, sr, kbps, l, r, trace_frames=F + 2)
    assert len(tr) == F
    g = M.debug_stages(ch, sr, kbps, l, r, want=stage_taps.ALL_TAPS, resample=resample)
    stage_taps.compare(g, tr, ref, G, ch, edge_signals.case_id(case))


def _batches(M, oracle, cases, resample):
    by_cfg = {}
    for c in cases:
        by_cfg.setdefault(c[1:4], []).append(c)
    for (ch, sr, kbps), cases in by_cfg.items():
        sigs = [edge_signals.signal(c) for c in cases]
        sigs += [(l[:len(l) * 2 // 3 + 17], None if r is None else r[:len(r) * 2 // 3 + 17]) for l, r in sigs]
        outs = M.encode_streams(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None, resample=resample)
        for (l, r), o in zip(sigs, outs):
            assert o == oracle.encode_stream(ch, sr, kbps, l, r)[0], (ch, sr, kbps, len(l))


def test_edge_corpus_as_batches(M, oracle):
    """Each configuration's cases in one encode_streams call, together with prefixes of themselves (other chunk phases)."""
    _batches(M, oracle, edge_signals.CASES, False)


def test_resampled_edge_corpus_as_batches(M, oracle):
    """The same for the resampled corpus, through encode_streams(..., resample=True)."""
    _batches(M, oracle, edge_signals.RESAMPLED_CASES, True)


@pytest.mark.parametrize("tagged", [False, True])
def test_stereo_host_streams_without_right(M, tagged):
    """Stereo whole streams from host buffers: right == NULL, or right[s] == NULL, encodes left[s] on both channels."""
    import ctypes

    import numpy as np
    from synth import make_signal

    L = M.lib()
    fn = L.mp3b200_encode_streams_tagged if tagged else L.mp3b200_encode_streams
    lefts = [np.ascontiguousarray(make_signal("noise", n, 44100, seed=n)[0], dtype=np.int16) for n in (5000, 12345)]
    want = (M.encode_streams_tagged if tagged else M.encode_streams)(2, 44100, 128, lefts, lefts)
    room = M.lametag_size(2, 44100, 128) if tagged else 0
    ns = np.array([len(x) for x in lefts], dtype=np.int64)
    caps = np.array([M.stream_bytes(2, 44100, 128, int(n)) + room for n in ns], dtype=np.int64)
    lp = (ctypes.c_void_p * 2)(*[x.ctypes.data for x in lefts])
    for rp in (None, (ctypes.c_void_p * 2)(lefts[0].ctypes.data, None)):
        outs = [np.zeros(int(c), dtype=np.uint8) for c in caps]
        op = (ctypes.c_void_p * 2)(*[o.ctypes.data for o in outs])
        got = np.zeros(2, dtype=np.int64)
        assert fn(2, 44100, 128, 2, lp, rp, ns.ctypes.data, op, caps.ctypes.data, got.ctypes.data) == 0
        assert [o[: int(g)].tobytes() for o, g in zip(outs, got)] == want
