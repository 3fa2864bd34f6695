"""ReplayGain on streaming handles under the random call schedules of tests/handle_schedule.py, against the CPU restatement
(tests/replaygain_ref.py).  Imported by tests/test_gpu_replaygain_handles.py; run as a script (one process per library,
MP3B200_LIB naming it) by tests/test_gpu_replaygain_variants.py, where it prints one JSON line {"fail": [...]}.

Every logical stream of a schedule runs on two tagged handles, one with find_replay_gain: their bytes must be equal call for
call (the analysis changes no audio byte); after every flush the analysing handle's title gain must be the restatement's for
that stream's calls so far (flush-then-continue starts a new title); at the end its tag frame must be the plain one with the
Radio Replay Gain field set, and the album gain over all handles must be GetAlbumGain of all their titles."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import handle_schedule as HS  # noqa: E402
import oracle_lib  # noqa: E402
import replaygain_ref as RG  # noqa: E402
from synth import make_signal  # noqa: E402

# handle_schedule's configurations whose tag fits the frame (lamejs analyses only with the tag on), and a resampled one
CONFIGS = [(2, 44100, 128), (1, 48000, 320), (2, 22050, 64), (2, 48000, 64)]


def patched_tag(frame, ch, out_sr, field):
    """a tag frame with its Radio Replay Gain field set and the tag CRC recomputed"""
    q = 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116
    b = bytearray(frame)
    b[q + 19:q + 21] = field.to_bytes(2, "big")
    b[q + 38:q + 40] = oracle_lib.crc16(bytes(b[:q + 38])).to_bytes(2, "big")
    return bytes(b)


def play(M, sched):
    """plays `sched`; returns a list of what differed"""
    ch, sr, kb = sched.cfg
    rs = sched.resample
    K = sched.nstreams
    rg = [M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs, find_replay_gain=True) for _ in range(K)]
    plain = [M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs) for _ in range(K)]
    assert all(e.replay_gain_on for e in rg)
    steps = [[] for _ in range(K)]
    seen = [[] for _ in range(K)]          # (steps so far, replay_gain) after every flush
    fail = []
    for op, calls in sched.ops:
        cs = [c for c in calls if c.s is not None]
        if not cs or op == "handover":
            continue
        if op in ("encode", "encode_batch"):
            L = [sched.signals[c.s][0][c.lo:c.hi] for c in cs]
            R = [sched.signals[c.s][1][c.lo:c.hi] for c in cs] if ch == 2 else None
            a = M.encode_batch([rg[c.s] for c in cs], L, R)
            b = M.encode_batch([plain[c.s] for c in cs], L, R)
            for c in cs:
                steps[c.s].append(("enc", c.hi - c.lo))
        else:
            a = M.flush_batch([rg[c.s] for c in cs])
            b = M.flush_batch([plain[c.s] for c in cs])
            for c in cs:
                steps[c.s].append(("flush",))
                seen[c.s].append((len(steps[c.s]), rg[c.s].replay_gain))
        if a != b:
            fail.append("%s bytes differ from the plain handle's" % op)
    out_sr = oracle_lib.out_samplerate(ch, sr, kb)
    hist = np.zeros(RG.HIST, dtype=np.int64)
    def fed(sig, st):                       # the samples the calls `st` took from a signal
        m = sum(k[1] for k in st if k[0] == "enc")
        return None if sig is None else sig[:m]

    for s in range(K):
        x, y = sched.signals[s]
        for n, got in seen[s]:
            ref = RG.analyze_stream(ch, sr, kb, fed(x, steps[s][:n]), fed(y, steps[s][:n]), schedule=steps[s][:n])
            want = (ref.title_db[-1], ref.radio[-1]) if ref.title_db else None
            if got != want:
                fail.append("stream %d after step %d: %r != %r" % (s, n, got, want))
        ref = RG.analyze_stream(ch, sr, kb, fed(x, steps[s]), fed(y, steps[s]), schedule=steps[s])
        for a in ref.hist:
            hist += a
        want_tag = patched_tag(plain[s].lametag_frame(), ch, out_sr, RG.tag_field(ref.radio[-1]))
        if rg[s].lametag_frame() != want_tag:
            fail.append("stream %d: tag frame" % s)
    album = M.album_gain(rg)
    if album != RG.analyze_result(hist.astype(np.int32)):
        fail.append("album gain %r != %r" % (album, RG.analyze_result(hist.astype(np.int32))))
    return fail


def window_fails(M):
    """whole streams through the debug tap: every window's sum bits and index, native and resampled"""
    fail = []
    for ch, sr, kb in [(2, 44100, 128), (1, 8000, 24), (2, 48000, 64), (1, 22050, 64)]:
        l, r = make_signal("sweep" if ch == 2 else "noise", 3 * sr + 1234, sr, seed=sr)
        rs = oracle_lib.out_samplerate(ch, sr, kb) != sr
        got = M.debug_replaygain(ch, sr, kb, l, r if ch == 2 else None, resample=rs)
        ref = RG.analyze_stream(ch, sr, kb, l, r if ch == 2 else None)
        w = ref.windows[0]
        if not (np.array_equal(got["sums"].view(np.uint64), w[:, :2]) and np.array_equal(got["idx"], w[:, 2].astype(np.int32))
                and got["title_db"] == ref.title_db[0]):
            fail.append("windows %r" % ((ch, sr, kb),))
    return fail


def main():
    import lamejs_b200 as M
    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    fail = window_fails(M)
    for i, cfg in enumerate(CONFIGS):
        fail += ["%r: %s" % (cfg, f) for f in play(M, HS.make_schedule(cfg, 5, 30, seed=700 + i))]
    print(json.dumps({"fail": fail}))


if __name__ == "__main__":
    main()
