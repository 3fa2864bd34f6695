"""Runs in a subprocess of tests/test_gpu_speculation.py with MP3B200_LIB naming a library built with other speculation
guesses (lamejs_b200.lib() is a process singleton, so one process per library).  Encodes, compares with the oracle, and
prints one JSON line: {"fail": [what differed, ...], "passes": {workload: quantizer passes}}."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import edge_signals  # noqa: E402
import handle_schedule as HS  # noqa: E402
import oracle_lib as O  # noqa: E402
import stage_taps  # noqa: E402
from synth import make_signal, white  # noqa: E402


def device_encode(M, torch, ch, sr, kbps, sigs, resample=False):
    """encode_streams_device on a packed device copy of `sigs`: (list of bytes, quantizer passes)."""
    ns = [len(l) for l, _ in sigs]
    pcm = np.concatenate([np.concatenate([l, r]) if ch == 2 else l for l, r in sigs] + [np.zeros(8, np.int16)])
    pcm_off = np.cumsum([0] + [n * ch for n in ns])[:-1]
    nb = [M.stream_bytes(ch, sr, kbps, n, resample) for n in ns]
    out_off = np.cumsum([0] + nb)[:-1]
    d_pcm = torch.from_numpy(pcm).cuda()
    d_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
    tm = M.encode_streams_device(ch, sr, kbps, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off, resample=resample)
    out = d_out.cpu().numpy()
    return [out[o:o + b].tobytes() for o, b in zip(out_off, nb)], int(tm[7])


def main():
    import torch

    import lamejs_b200 as M

    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    fail, passes = [], {}

    def check(tag, got, ch, sr, kbps, sigs):
        for i, ((l, r), o) in enumerate(zip(sigs, got)):
            if o != O.encode_stream(ch, sr, kbps, l, r if ch == 2 else None)[0]:
                fail.append("%s stream %d (%d samples)" % (tag, i, len(l)))

    def check_taps(tag, ch, sr, kbps, sigs, resample=False):
        """every stage tap of each stream, the quantizer's carried state included: where a stale speculated state would
        show although the bytes agree"""
        G = M.granules_per_frame(ch, sr, kbps, resample)
        for i, (l, r) in enumerate(sigs):
            r = r if ch == 2 else None
            F = M.stream_frames(len(l), ch, sr, kbps, resample)
            ref, _, tr = O.encode_stream(ch, sr, kbps, l, r, trace_frames=F + 2)
            try:
                stage_taps.compare(M.debug_stages(ch, sr, kbps, l, r, want=stage_taps.ALL_TAPS, resample=resample), tr, ref, G, ch)
            except AssertionError as e:
                fail.append("%s stream %d taps: %s" % (tag, i, str(e)[:300]))

    # ragged batches through the device entry point (the pass count is reported there): MPEG-1 (verify, repair stream)
    # and LSF (verify(1) with predict_step)
    for tag, ch, sr, kbps, frame in (("mpeg1", 2, 44100, 128, 1152), ("lsf", 2, 22050, 64, 576), ("lsf_mono", 1, 16000, 24, 576)):
        lens = [1, 700, 1377, 5000, frame * 31 + 5, frame * 64, frame * 150 + 3]
        sigs = []
        for i, n in enumerate(lens):
            l, r = white(n, 0x5EED0030 + i) if i % 3 == 0 else make_signal(("burst", "noise", "sweep")[i % 3], n, sr, 90 + i)
            sigs.append((l, r if ch == 2 else l))
        got, passes[tag] = device_encode(M, torch, ch, sr, kbps, sigs)
        check(tag, got, ch, sr, kbps, sigs)
        check(tag + " host", M.encode_streams(ch, sr, kbps, [s[0] for s in sigs], [s[1] for s in sigs] if ch == 2 else None),
              ch, sr, kbps, sigs)
        check_taps(tag, ch, sr, kbps, sigs)

    # a resampled ragged batch (48 -> 24 kHz, MP3B200_RESAMPLE): lengths around the first output sample and the output frame
    # edges, in input samples
    ch, sr, kbps, r = 2, 48000, 64, 2
    lens = [1, 17, r * 800 + 16, 5000, r * 576 * 31 + 5, r * 576 * 64, r * 576 * 150 + 3]
    sigs = []
    for i, n in enumerate(lens):
        l, rt = white(n, 0x5EED0040 + i) if i % 3 == 0 else make_signal(("burst", "noise", "sweep")[i % 3], n, sr, 70 + i)
        sigs.append((l, np.roll(rt, 7)))
    got, passes["resampled"] = device_encode(M, torch, ch, sr, kbps, sigs, resample=True)
    check("resampled", got, ch, sr, kbps, sigs)
    check_taps("resampled", ch, sr, kbps, sigs, resample=True)

    # live handles fed 5000-sample calls: several frames per call, so the handle path speculates too
    for ch, sr, kbps in ((2, 44100, 128), (1, 24000, 48)):
        sigs = [make_signal(k, n, sr, 60 + i) for i, (k, n) in enumerate([("burst", 41000), ("noise", 33000), ("sweep", 26000)])]
        encs = [M.Mp3Encoder(ch, sr, kbps) for _ in sigs]
        refs = [O.OracleEncoder(ch, sr, kbps) for _ in sigs]
        for pos in range(0, 41000, 5000):
            ls = [l[pos:pos + 5000] for l, _ in sigs]
            rs = [r[pos:pos + 5000] for _, r in sigs] if ch == 2 else None
            got = M.encode_batch(encs, ls, rs)
            for i in range(len(sigs)):
                if len(ls[i]) and got[i] != refs[i].encode_buffer(ls[i], rs[i] if rs else None):
                    fail.append("handles %d/%d/%d stream %d call at %d" % (ch, sr, kbps, i, pos))
        for i, (a, b) in enumerate(zip(M.flush_batch(encs), [r.flush() for r in refs])):
            if a != b:
                fail.append("handles %d/%d/%d stream %d flush" % (ch, sr, kbps, i))
        for e, r in zip(encs, refs):
            e.close(); r.close()

    # one reduced call schedule per configuration family (tests/handle_schedule.py), with many calls of up to 200 frames
    for cfg, seed in (((2, 44100, 128), 7), ((2, 22050, 64), 8)):
        s = HS.make_schedule(cfg, 8, 40, seed, big=0.3)
        fail += ["schedule %d/%d/%d: %s" % (cfg + (f,)) for f in HS.run(M, s, HS.replay(s))]

    # the edge corpus, one batch per configuration
    by_cfg = {}
    for c in edge_signals.CASES:
        by_cfg.setdefault(c[1:4], []).append(edge_signals.signal(c))
    edge_passes = 0
    for (ch, sr, kbps), sigs in by_cfg.items():
        sigs = [(l, r if ch == 2 else l) for l, r in sigs]
        got, p = device_encode(M, torch, ch, sr, kbps, sigs)
        edge_passes = max(edge_passes, p)
        check("edge %d/%d/%d" % (ch, sr, kbps), got, ch, sr, kbps, sigs)
        check_taps("edge %d/%d/%d" % (ch, sr, kbps), ch, sr, kbps, sigs)
    passes["edge"] = edge_passes

    # the resampled edge corpus, one batch per configuration
    by_cfg = {}
    for c in edge_signals.RESAMPLED_CASES:
        by_cfg.setdefault(c[1:4], []).append(edge_signals.signal(c))
    edge_passes = 0
    for (ch, sr, kbps), sigs in by_cfg.items():
        sigs = [(l, r if ch == 2 else l) for l, r in sigs]
        got, p = device_encode(M, torch, ch, sr, kbps, sigs, resample=True)
        edge_passes = max(edge_passes, p)
        check("resampled edge %d/%d/%d" % (ch, sr, kbps), got, ch, sr, kbps, sigs)
        check_taps("resampled edge %d/%d/%d" % (ch, sr, kbps), ch, sr, kbps, sigs, resample=True)
    passes["resampled_edge"] = edge_passes
    print(json.dumps({"fail": fail, "passes": passes}))


if __name__ == "__main__":
    main()
