"""Keeps the handle soak (tests/handle_schedule.py, tests/test_gpu_handle_soak.py) honest, on the oracle alone: the schedules
split every stream into calls without losing or repeating a sample, the expected results hand out every byte exactly once,
and the schedules reach the call patterns they exist for -- calls that complete 0, 1 and 16 or more frames, call boundaries
right after a START and after a SHORT granule, flush then reuse, hand-overs, repeated handles, NULL handles and failed calls.
The resampled schedules (48 -> 24 and 48 -> 8 kHz) must reach the same minimum counts.  A schedule that silently stopped
reaching them would leave the GPU soak green for the wrong reason."""
import pytest

import handle_schedule as HS
import oracle_lib

# seeds and sizes of the GPU soak; the totals below are asserted over all of its configurations, native and resampled
SOAK = [(cfg, 32, 300, 100 + i) for i, cfg in enumerate(HS.CONFIGS)] + [(cfg, 32, 300, 200 + i) for i, cfg in enumerate(HS.RESAMPLED_CONFIGS)]

MIN_PER_CONFIG = {"calls_0_frames": 50, "calls_1_frame": 50, "calls_16plus_frames": 20, "after_start": 10, "after_short": 20,
                  "handovers": 10, "repeated_batches": 20, "null_entries": 5, "injected_failures": 10, "flush_then_reuse": 20}


@pytest.fixture(scope="module")
def soaks(oracle):
    out = []
    for cfg, K, nops, seed in SOAK:
        s = HS.make_schedule(cfg, K, nops, seed)
        out.append((s, HS.replay(s, trace=True)))
    return out


@pytest.mark.parametrize("i", range(len(SOAK)), ids=["%d-%d-%d" % c[0] for c in SOAK])
def test_calls_concatenate_to_the_whole_stream(soaks, i):
    """Per stream: the oracle's bytes call by call equal one encodeBuffer per flush-delimited range plus its flush (for a
    stream never flushed before the end: oracle.encode_stream of the whole signal); the expected results hand out those
    bytes, each exactly once, in order."""
    s, ex = soaks[i]
    ch, sr, kbps = s.cfg
    whole = 0
    for k in range(s.nstreams):
        l, r = s.signals[k]
        e = oracle_lib.OracleEncoder(ch, sr, kbps, write_vbr_tag=k in s.tagged)
        want = bytearray()
        for lo, hi in ex.epochs[k]:
            if hi > lo:
                want += e.encode_buffer(l[lo:hi], None if r is None else r[lo:hi])
            want += e.flush()
        e.close()
        assert ex.raw[k] == bytes(want), k
        assert ex.epochs[k][-1][1] == len(l) or (len(l) == 1 and ex.epochs[k][-1][1] == 0)
        if k not in s.tagged and all(lo == hi for lo, hi in ex.epochs[k][1:]):      # flushed only at the end
            assert ex.raw[k] == oracle_lib.encode_stream(ch, sr, kbps, l, r)[0], k
            whole += 1
        delivered = b"".join(res[j] for (_, entries), res in zip(s.ops, ex.results)
                             for j, c in enumerate(entries) if c.s == k and isinstance(res[j], bytes))
        assert delivered == ex.raw[k], k
    assert whole >= s.nstreams // 4, whole


def test_schedules_reach_what_they_exist_for(soaks):
    total = {}
    for s, ex in soaks:
        r = HS.reached(s, ex)
        print(s.cfg, r)
        for k, v in MIN_PER_CONFIG.items():
            assert r[k] >= v, (s.cfg, k, r[k])
        # 16 kbps at 8 kHz, and 8 kbps resampled to 8 kHz: the tag does not fit
        assert any(t["tag_on"] for t in ex.tags) or s.cfg in ((1, 8000, 16), (1, 48000, 8)), s.cfg
        for k, v in r.items():
            total[k] = total.get(k, 0) + v
    print("all configurations:", total)
    assert total["frames"] >= 20000
    assert total["after_start"] >= 20 and total["after_short"] >= 20
