"""Runs in a subprocess of tests/test_gpu_loud_beyond_gate.py with MP3B200_LIB naming a library built with another input
limit (lamejs_b200.lib() is a process singleton, so one process per library).  Prints one JSON line.

`compare NAME...`: the loud fixtures NAME (tests/golden/lamejs_loud_golden.json) against lamejs and the oracle -- the handle
with the fixture's calls, whole streams host / device / tagged, every stage tap, and for the ReplayGain fixtures the window
sums and gains of tests/replaygain_ref_f32.py.  {"fail": [what differed, ...], "taps": {name: [[tap, first index], ...]}}.

`domain NAME...`: the domain-check build (-DMP3_DOMAIN_CHECK): encodes the fixtures NAME (one group per rung), the edge
corpus and the Int16 lamejs fixtures, and reads the device's out-of-domain counters after each group.
{"hits": {group: [count per site]}}.  `domain-loud NAME...`: the fixtures alone."""
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import float_signals as FS  # noqa: E402
import oracle_f32  # noqa: E402
import oracle_lib  # noqa: E402
import replaygain_ref_f32 as RGF  # noqa: E402
import stage_taps  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))


def sha(b):
    return hashlib.sha256(b).hexdigest()


def cfg_of(c):
    return c["channels"], c["samplerate"], c["kbps"]


def rows(c):
    l, r, calls = FS.loud_case_signal(c)
    return l.astype(np.float32), None if r is None else r.astype(np.float32), calls


def oracle_whole(ch, sr, kb, l, r, trace_frames=0):
    """the oracle on one whole stream: (bytes, traces), or None where it throws"""
    try:
        b, _, tr = oracle_f32.encode_stream(ch, sr, kb, l, r, trace_frames=trace_frames)
    except oracle_lib.LamejsThrows:
        return None
    return b, tr


def whole_frame_prefix(M, c, l, r, rs):
    """the longest prefix of whole frames (in input samples) that the oracle encodes as a whole stream without throwing"""
    ch, sr, kb = cfg_of(c)
    fsz = 576 * M.granules_per_frame(ch, sr, kb, resample=rs) * (sr // M.out_samplerate(ch, sr, kb))
    for k in range(len(l) // fsz, 0, -1):
        n = k * fsz
        if oracle_whole(ch, sr, kb, l[:n], None if r is None else r[:n]) is not None:
            return n
    return 0


def compare(M, names):
    import torch

    fail, taps = [], {}
    for name in names:
        c = GOLDEN[name]
        ch, sr, kb = cfg_of(c)
        rs = M.out_samplerate(ch, sr, kb) != sr
        lf, rf, calls = rows(c)
        kw = dict(write_vbr_tag=True, find_replay_gain=True) if c["rg"] else {}
        # the handle with the fixture's calls: lamejs's per-call sizes and bytes, then its throw as a refusal that changes
        # nothing
        e = M.Mp3Encoder(ch, sr, kb, resample=rs, **kw)
        out = []
        try:
            for i, x in enumerate(calls):
                if i == c["thrown"]:
                    # (state blobs do not carry the ReplayGain analysis: test_gpu_loud_float.py's batch test covers it)
                    state = (lambda: None) if c["rg"] else e.export_state
                    before = state()
                    try:
                        e.flush() if x is None else e.encodeBuffer(*x)
                        fail.append("%s: handle call %d encoded where lamejs threw" % (name, i))
                    except M.Mp3B200Error as err:
                        if "bit budget" not in str(err):
                            fail.append("%s: handle call %d refused for another reason: %s" % (name, i, err))
                    if state() != before:
                        fail.append("%s: the refused call %d changed the handle's state" % (name, i))
                    break
                out.append(e.flush() if x is None else e.encodeBuffer(*x))
        except M.Mp3B200Error as err:
            fail.append("%s: handle call %d refused: %s" % (name, len(out), err))
        if [len(b) for b in out] != c["sizes"][:len(out)] or len(out) != len(c["sizes"]) or sha(b"".join(out)) != c["sha256"]:
            fail.append("%s: handle bytes or per-call sizes differ from lamejs" % name)
        if c["rg"] and c["thrown"] is None:
            if e.replay_gain[1] != c["radio_gain"][-1]:
                fail.append("%s: handle RadioGain %s, lamejs %s" % (name, e.replay_gain[1], c["radio_gain"][-1]))
        e.close()
        # whole streams where lamejs encoded the stream whole
        rr = None if rf is None else [rf]
        if c["thrown"] is None:
            try:
                if sha(M.encode_streams(ch, sr, kb, [lf], rr, resample=rs)[0]) != c["sha256"]:
                    fail.append("%s: host whole stream" % name)
                pcm = np.concatenate([lf, rf]) if ch == 2 else lf
                nb = M.stream_bytes(ch, sr, kb, len(lf), resample=rs)
                d_pcm = torch.from_numpy(pcm).cuda()
                d_out = torch.zeros(nb, dtype=torch.uint8, device="cuda")
                M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [len(lf)], d_out.data_ptr(), [0], resample=rs,
                                        float32=True)
                if sha(d_out.cpu().numpy().tobytes()) != c["sha256"]:
                    fail.append("%s: device whole stream" % name)
                tagged = M.encode_streams_tagged(ch, sr, kb, [lf], rr, resample=rs)[0]
                if sha(tagged[len(tagged) - c["bytes"]:]) != c["sha256"]:
                    fail.append("%s: tagged whole stream" % name)
                if c["rg"]:
                    streams, title, _ = M.encode_streams_replaygain(ch, sr, kb, [lf], rr, resample=rs)
                    if M.radio_gain(title[0]) != c["radio_gain"][-1]:
                        fail.append("%s: whole-stream RadioGain %d, lamejs %d" % (name, M.radio_gain(title[0]), c["radio_gain"][-1]))
            except M.Mp3B200Error as err:
                fail.append("%s: whole stream refused: %s" % (name, err))
        # stage taps: the whole stream, or the longest whole-frame prefix the oracle encodes without throwing
        n = len(lf) if c["thrown"] is None else whole_frame_prefix(M, c, lf, rf, rs)
        if n:
            l, r = lf[:n], None if rf is None else rf[:n]
            F = M.stream_frames(n, ch, sr, kb, resample=rs)
            G = M.granules_per_frame(ch, sr, kb, resample=rs)
            ref, tr = oracle_whole(ch, sr, kb, l, r, trace_frames=F + 2)
            try:
                g = M.debug_stages(ch, sr, kb, l, r, want=stage_taps.ALL_TAPS, resample=rs)
            except M.Mp3B200Error as err:
                fail.append("%s: stage taps of %d samples refused: %s" % (name, n, err))
            else:
                d = stage_taps.differences(g, tr, ref, G, ch)
                if d:
                    taps[name] = d
                    fail.append("%s: %d samples: first differing tap %s at (frame, granule, channel, index) %s" % (name, n, d[0][0], d[0][1]))
            if c["rg"]:
                got = M.debug_replaygain(ch, sr, kb, l, r, resample=rs)
                ref_rg = RGF.analyze_calls(ch, sr, kb, l, r, [("enc", n), ("flush",)])
                w = ref_rg.windows[0] if ref_rg.windows else np.zeros((0, 3), np.uint64)
                if not (len(got["sums"]) == len(w) and np.array_equal(got["sums"].view(np.uint64), w[:, :2])
                        and np.array_equal(got["idx"], w[:, 2].astype(np.int32))):
                    fail.append("%s: ReplayGain window sums" % name)
                if got["title_db"] != ref_rg.title_db[0]:
                    fail.append("%s: ReplayGain title gain %r, reference %r" % (name, got["title_db"], ref_rg.title_db[0]))
    return {"fail": fail, "taps": taps}


def domain(M, names, corpora):
    import edge_signals

    def group(fn):
        M.debug_domain_hits()                   # clear what earlier work left
        fn()
        return M.debug_domain_hits().tolist()

    hits = {}

    def fixtures(ns):
        def run():
            for n in ns:
                c = GOLDEN[n]
                ch, sr, kb = cfg_of(c)
                rs = M.out_samplerate(ch, sr, kb) != sr
                lf, rf, calls = rows(c)
                e = M.Mp3Encoder(ch, sr, kb, resample=rs)
                try:
                    for x in calls:
                        e.flush() if x is None else e.encodeBuffer(*x)
                except M.Mp3B200Error:
                    pass
                e.close()
        return run

    by_rung = {}
    for n in names:
        by_rung.setdefault(GOLDEN[n]["magnitude"], []).append(n)
    for m, ns in by_rung.items():
        hits["loud %s" % m] = group(fixtures(ns))
    if not corpora:
        return {"hits": hits}

    def edges():
        for case in edge_signals.CASES:
            kind, ch, sr, kb, _ = case
            l, r = edge_signals.signal(case)
            M.encode_streams(ch, sr, kb, [l], [r] if ch == 2 else None)
        for case in edge_signals.RESAMPLED_CASES:
            kind, ch, sr, kb, _ = case
            l, r = edge_signals.signal(case)
            M.encode_streams(ch, sr, kb, [l], [r] if ch == 2 else None, resample=True)
    hits["edge corpus"] = group(edges)

    def int16_fixtures():
        from synth import make_signal
        cases = json.load(open(os.path.join(HERE, "golden", "lamejs_golden.json")))["cases"]
        for c in cases.values():
            ch, sr, kb = cfg_of(c)
            out_sr = M.out_samplerate(ch, sr, kb)
            if out_sr <= 0 or sr % out_sr:
                continue                        # the non-integer resampling ratios are not encoded (DESIGN.md 9)
            l, r = make_signal(c["kind"], c["samples"], sr, c["seed"])
            M.encode_streams(ch, sr, kb, [l], [r] if ch == 2 else None, resample=out_sr != sr)
    hits["int16 lamejs fixtures"] = group(int16_fixtures)
    return {"hits": hits}


def main():
    import lamejs_b200 as M

    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    mode, names = sys.argv[1], sys.argv[2:]
    print(json.dumps(compare(M, names) if mode == "compare" else domain(M, names, corpora=mode == "domain")))


if __name__ == "__main__":
    main()
