"""The front end's rows against the oracle, row for row and bit for bit (tests/psy_rows.py, tests/front_rows.py): the psy rows
of k_psy_analysis and k_attack_prepass, the short list and short rows of k_psy_short, the block types and ATH adjustments of
k_stream_scan, the masking rows of k_psy_masking and the xr rows of k_mdct, all from one capture of each launch.  In every
launch shape the rows depend on: whole streams of every native configuration, ragged batches, upload slices, the edge
corpus, the bench's bursts, streaming handles (odd chunks, calls that start on a short granule, batches of handles at
different frames, state blobs, seek), device-resident and session calls, Float32 and resampled input; and the library built
with other PSY_UNITS, FB_G and SCAN_FRAMES.  Each call runs on a poisoned workspace and its bytes must equal the oracle's,
which shows that no kernel read a row the launch left poisoned, and no quantizer a short half the encoder skipped."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import edge_signals
import float_signals
import front_rows as F
import psy_rows as P
from synth import bursts

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


def _ok(fail):
    assert not fail, "%d rows differ; first: %s" % (len(fail), fail[:10])


def _has_short(launches):
    return any((s["bt"] == P.BT_SHORT).any() for rec in launches for s in rec["streams"])


def test_whole_streams_every_native_configuration(M):
    fail = []
    P.shape_whole(M, fail, F.check_rows)
    _ok(fail)


def test_ragged_batches(M):
    fail = []
    P.shape_batches(M, fail, F.check_rows)
    _ok(fail)


def test_upload_slices(M):
    fail = []
    P.shape_slices(M, fail, F.check_rows)
    _ok(fail)


# kinds whose every case has short granules: first in the stream, on both sides of frame boundaries, in long runs and near
# the end
SHORT_KINDS = ("square", "click_pairs", "loud_silent", "clicks1", "clicks3", "clicks5")
EDGE = [c for c in edge_signals.CASES if c[0] in SHORT_KINDS + ("dc_max", "dc_min", "nyquist", "lsb_dither", "lsb_clicks",
                                                                "clicks4", "silent_right")]


@pytest.mark.parametrize("case", EDGE, ids=edge_signals.case_id)
def test_edge_corpus(M, case):
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    fail = []
    launches = P.whole_streams(M, ch, sr, kb, [(l, r)], edge_signals.case_id(case), fail, F.check_rows)
    _ok(fail)
    assert case[0] not in SHORT_KINDS or _has_short(launches)


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 44100, 128), (2, 22050, 64), (1, 16000, 32)])
def test_bursts(M, ch, sr, kb):
    """the bench's C5 signal: a quarter of the units do the short half"""
    l, r = bursts(120 * 576 * M.granules_per_frame(ch, sr, kb) + 333, 0xC5)
    fail = []
    launches = P.whole_streams(M, ch, sr, kb, [(l, r)], "bursts %d/%d/%d" % (ch, sr, kb), fail, F.check_rows)
    _ok(fail)
    assert _has_short(launches)


def test_short_granules_in_float32_and_resampled_input(M):
    """Float32 bursts (k_stage_f32, fractional samples) and a configuration lamejs resamples (k_resample), both with short
    granules"""
    l, r = bursts(120 * 1152 + 333, 0xC5)
    l, r = l.astype(np.float32) * np.float32(0.75), r.astype(np.float32) + np.float32(0.25)
    fail = []
    assert _has_short(P.whole_streams(M, 2, 44100, 128, [(l, r)], "float32 bursts", fail, F.check_rows, f32=True))
    case = ("clicks1", 2, 48000, 64, 56)
    assert case in edge_signals.RESAMPLED_CASES
    l, r = edge_signals.signal(case)
    assert _has_short(P.whole_streams(M, 2, 48000, 64, [(l, r)], "resampled clicks1", fail, F.check_rows, resample=True))
    _ok(fail)


def test_unread_rows_stay_poisoned_and_capture_off_changes_nothing(M):
    """a capture call is recorded as one launch; for a silent stream (no short blocks) it leaves the short half of nearly
    every masking row poisoned (only the last unit needs it); a stream of the same length with short blocks, encoded next
    with capture off, still encodes the bytes it encoded before: it writes every row its kernels read"""
    n = 40 * 1152 + 77
    l, r = P.k2_signal("mixed", n, 3)
    before = M.encode_streams(2, 44100, 128, [l], [r])[0]
    z = np.zeros(n, np.int16)
    with M.debug_psy_capture() as cap:
        M.encode_streams(2, 44100, 128, [z], [z])
    assert len(cap.launches) == 1
    (s,) = cap.launches[0]["streams"]
    assert not (s["bt"] == P.BT_SHORT).any()
    assert np.isnan(s["ratio"]["en_s"][1:-1]).all() and not np.isnan(s["ratio"]["en_s"][-1]).any()
    assert M.encode_streams(2, 44100, 128, [l], [r])[0] == before


@pytest.mark.parametrize("case", [c for c in EDGE if c[0] in SHORT_KINDS], ids=edge_signals.case_id)
def test_stage_taps_compute_every_short_unit(M, case):
    """the stage taps run the short-block half for every (unit, channel), the halo included, so that they can compare
    en_s / thm_s everywhere"""
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    with M.debug_psy_capture() as cap:
        M.debug_stages(ch, sr, kb, l, r, want=("en_s",))
    (rec,) = cap.launches
    (s,) = rec["streams"]
    want = [(0, u, c) for u in range(-1, s["G"] * s["nframes"]) for c in range(ch)]
    assert sorted(tuple(int(v) for v in e) for e in rec["short"]) == want


def _handle(M, ch, sr, kb, l, r, bounds, label, fail, blob_after=(), f32=False):
    """one handle fed l[bounds[i]:bounds[i + 1]] for each i, then flushed, each call under capture; after the calls whose index
    is in blob_after the handle is exported and replaced by a fresh one that imports the blob.  Returns (launches, Ref)."""
    ref = P.make_ref(ch, sr, kb, f32)
    enc = M.Mp3Encoder(ch, sr, kb)
    recs = []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        ra = r[a:b] if ch == 2 else None
        got, launches = P.capture_call(M, lambda: enc.encodeBuffer(l[a:b], ra))
        if got != ref.call(l[a:b], ra):
            fail.append("%s: bytes of call %d" % (label, k))
        recs += launches
        if k in blob_after:
            blob = enc.export_state()
            enc.close()
            enc = M.Mp3Encoder(ch, sr, kb)
            enc.import_state(blob)
            assert enc.export_state() == blob, label
    got, launches = P.capture_call(M, enc.flush)
    if got != ref.flush():
        fail.append("%s: bytes of flush" % label)
    recs += launches
    enc.close()
    ref.done()
    for rec in recs:
        F.check_rows(rec, [ref], label, fail)
    return recs, ref


CHUNKS = [1, 575, 576, 577, 1151, 1152, 1153, 4097]


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 22050, 64)])
def test_handle_chunks(M, ch, sr, kb):
    """encodeBuffer with chunks of 1, 575, 576, 577, 1151, 1152, 1153 and 4097 samples, then flush, a state blob halfway:
    frame0 > 0, the halo unit recomputed from the carried tail, the halo row carried from the previous call, the scan
    starting from the carried state"""
    l, r = P.k2_signal("mixed", 60 * 1152 + 333, 11)
    bounds, i, k = [0], 0, 0
    while i < len(l):
        i = min(len(l), i + CHUNKS[k % len(CHUNKS)])
        k += 1
        bounds.append(i)
    fail = []
    recs, _ = _handle(M, ch, sr, kb, l, r, bounds, "handle %d/%d/%d" % (ch, sr, kb), fail, blob_after=(len(bounds) // 2,))
    assert sum(1 for rec in recs for s in rec["streams"] if s["frame0"] % 2) > 0
    _ok(fail)


@pytest.mark.parametrize("case", [("clicks1", 2, 44100, 128, 56), ("click_pairs", 1, 16000, 32, 120)], ids=edge_signals.case_id)
def test_handle_calls_that_start_on_a_short_granule(M, case):
    """handles cut so that a call starts on a short granule or ends just before one (found from the oracle's block types):
    its masking reads the short half of the carried halo row.  A state blob between the calls.  The stream cut into
    segments, and encoded whole, gives the oracle's bytes too."""
    from lamejs_b200 import sharding

    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(ch, sr, kb)
    fs = 576 * G
    whole = P.make_ref(ch, sr, kb)
    want = whole.stream(l, r)
    is_short = [bool((b == P.BT_SHORT).any()) for b in whole.done().bt]
    runs = [u for u in range(1, len(is_short)) if is_short[u] and not is_short[u - 1]]
    short = [u for u in range(G, len(is_short), G) if is_short[u]]
    assert len(short) >= 3 and len(runs) >= 3
    # lamejs holds 576 + 48 samples back (MDCT lookahead, encoder delay) before frame f completes: the first and the last
    # cut after which f frames are done, for the first of a short run where one starts a frame and granules inside runs;
    # and cuts around the completion of the frame before the one that starts a run
    cuts = set()
    for u in set([u for u in short if u in runs][:2] + short[:2] + short[-2:]):
        f = u // G
        cuts |= {f * fs + fs // 2 + 48, (f + 1) * fs + fs // 2 + 47}
    for u in runs[:3] + runs[-2:]:
        f = u // G
        cuts |= {f * fs + 576 + fs // 2, f * fs + 576 + fs // 2 + 48, (f + 1) * fs}
    fail, starts = [], 0
    for cut in sorted({min(max(c, 1), len(l) - 1) for c in cuts}):
        mid = cut + (len(l) - cut) // 3
        recs, ref = _handle(M, ch, sr, kb, l, r, [0, cut, mid, len(l)], "%s cut %d" % (edge_signals.case_id(case), cut), fail,
                            blob_after=(0,))
        starts += sum(1 for rec in recs for s in rec["streams"]
                      if s["nframes"] and s["frame0"] and (ref.bt[G * s["frame0"]] == P.BT_SHORT).any())
    assert starts > 0, "no call started on a short granule"
    _ok(fail)
    for nseg, warmup in ((3, 8), (5, 1)):
        got, _ = sharding.encode_stream_segments_local(lambda: M.Mp3Encoder(ch, sr, kb), l, r, fs, nseg, warmup)
        assert got == want, (nseg, warmup)
    assert M.encode_streams(ch, sr, kb, [l], None if r is None else [r])[0] == want


def test_handle_batch_state_blobs_and_seek(M):
    """encode_batch over handles whose frame0 differ in parity; a handle exported and imported mid-stream; a handle seeked into
    the middle of a stream: its psy rows depend on the PCM only and equal the stream's oracle, and the rows after them start
    from the stream-start state and hold no poison"""
    ch, sr, kb = 2, 44100, 128
    fs = 1152
    sigs = [P.k2_signal(k, 50 * fs + 100 * i, 20 + i) for i, k in enumerate(("mixed", "impulses", "quiet8"))]
    refs = [P.make_ref(ch, sr, kb) for _ in sigs]
    encs = [M.Mp3Encoder(ch, sr, kb) for _ in sigs]
    fail, recs = [], []
    # stagger the handles: 0, 1 and 2 frames ahead before the batch calls
    pos = [0, 0, 0]
    for j, (e, rf, (l, r)) in enumerate(zip(encs, refs, sigs)):
        n = 2000 + j * fs
        got, launches = P.capture_call(M, lambda: e.encodeBuffer(l[:n], r[:n]))
        if got != rf.call(l[:n], r[:n]):
            fail.append("warm-up %d" % j)
        recs += [(rec, [j]) for rec in launches]
        pos[j] = n
    for step in (4097, 3 * fs + 1, 577, 7 * fs):
        ls = [l[p:p + step] for (l, _), p in zip(sigs, pos)]
        rs = [r[p:p + step] for (_, r), p in zip(sigs, pos)]
        got, launches = P.capture_call(M, lambda: M.encode_batch(encs, ls, rs))
        for j, rf in enumerate(refs):
            if got[j] != rf.call(ls[j], rs[j]):
                fail.append("batch step %d handle %d" % (step, j))
        recs += [(rec, list(range(len(encs)))) for rec in launches]
        pos = [p + step for p in pos]
    assert len({s["frame0"] % 2 for rec, zs in recs if len(zs) > 1 for s in rec["streams"]}) == 2
    blob = encs[1].export_state()
    encs[1].close()
    encs[1] = M.Mp3Encoder(ch, sr, kb)
    encs[1].import_state(blob)
    for j, (e, rf, (l, r)) in enumerate(zip(encs, refs, sigs)):
        got, launches = P.capture_call(M, lambda: e.encodeBuffer(l[pos[j]:], r[pos[j]:]))
        got2, launches2 = P.capture_call(M, e.flush)
        if got != rf.call(l[pos[j]:], r[pos[j]:]) or got2 != rf.flush():
            fail.append("tail %d" % j)
        recs += [(rec, [j]) for rec in launches + launches2]
        e.close()
    for rf in refs:
        rf.done()
    for rec, zs in recs:
        F.check_rows(rec, [refs[z] for z in zs], "handles", fail)
    # seek: a fresh handle at frame 17 of stream 0, fed the rest of it
    l, r = sigs[0]
    frame = 17
    lo, hi = max(0, frame * fs - 1104), frame * fs + 224
    e = M.Mp3Encoder(ch, sr, kb)
    e.seek(frame, l[lo:hi], r[lo:hi])
    _, launches = P.capture_call(M, lambda: e.encodeBuffer(l[hi:], r[hi:]))
    _, launches2 = P.capture_call(M, e.flush)
    e.close()
    assert launches and launches[0]["streams"][0]["frame0"] == frame and launches[0]["streams"][0]["nframes"] > 0
    F.check_unpoisoned(launches[0], "seek", fail, halo_start=True)
    for rec in launches[1:] + launches2:
        F.check_unpoisoned(rec, "seek, later calls", fail)
    for rec in launches + launches2:
        P.check_launch(rec, [refs[0]], "seek", fail)
    _ok(fail)


def _packed(torch, ch, sigs):
    ns = [len(l) for l, _ in sigs]
    pcm = np.concatenate([np.concatenate([l, r]) if ch == 2 else l for l, r in sigs] + [np.zeros(8, np.int16)]).astype(np.int16)
    pcm_off = np.cumsum([0] + [n * ch for n in ns])[:-1]
    return torch.from_numpy(pcm).cuda(), pcm_off, ns


def test_device_and_session_entries(M):
    """encode_streams_device, EncodeSession.encode_streams and EncodeSession.encode_batch"""
    import torch

    ch, sr, kb = 2, 44100, 128
    sigs = [P.k2_signal(k, n, 40 + i) for i, (k, n) in enumerate((("mixed", 30 * 1152 + 5), ("impulses", 1377), ("silence", 0),
                                                                    ("nyquist", 9 * 1152)))]
    fail = []
    d_pcm, pcm_off, ns = _packed(torch, ch, sigs)
    nb = [M.stream_bytes(ch, sr, kb, n) for n in ns]
    out_off = np.cumsum([0] + nb)[:-1]
    for entry in ("device", "session"):
        rf = [P.make_ref(ch, sr, kb) for _ in sigs]
        want = [x.stream(l, r) for x, (l, r) in zip(rf, sigs)]
        for x in rf:
            x.done()
        d_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
        if entry == "device":
            _, launches = P.capture_call(M, lambda: M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off))
        else:
            with M.EncodeSession() as sess:
                _, launches = P.capture_call(M, lambda: M.check_status(sess.encode_streams(ch, sr, kb, d_pcm, pcm_off, ns, d_out, out_off)))
        out = d_out.cpu().numpy()
        for i, (o, b, w) in enumerate(zip(out_off, nb, want)):
            if out[o:o + b].tobytes() != w:
                fail.append("%s: bytes of stream %d" % (entry, i))
        base = 0
        for rec in launches:
            F.check_rows(rec, rf[base:base + len(rec["streams"])], entry, fail)
            base += len(rec["streams"])
        assert base == len(sigs)
    # session handles: three live encoders fed device rows in two rounds
    rf = [P.make_ref(ch, sr, kb) for _ in range(3)]
    hs = [M.Mp3Encoder(ch, sr, kb) for _ in range(3)]
    src = [P.k2_signal(k, 20 * 1152, 60 + i) for i, k in enumerate(("mixed", "impulses", "quiet1"))]
    recs = []
    with M.EncodeSession() as sess:
        for a, b in ((0, 5000), (5000, 20 * 1152)):
            ls = [torch.from_numpy(l[a:b].copy()).cuda() for l, _ in src]
            rs = [torch.from_numpy(r[a:b].copy()).cuda() for _, r in src]

            def run():
                out, offs, lens, st = sess.encode_batch(hs, ls, rs)
                M.check_status(st)
                return out.cpu().numpy(), offs, lens
            (out, offs, lens), launches = P.capture_call(M, run)
            for j, x in enumerate(rf):
                if out[offs[j]:offs[j] + lens[j]].tobytes() != x.call(src[j][0][a:b], src[j][1][a:b]):
                    fail.append("session batch %d handle %d" % (a, j))
            recs += launches
        sess.release(hs)
    for x in rf:
        x.done()
    for rec in recs:
        F.check_rows(rec, rf, "session handles", fail)
    for h in hs:
        h.close()
    _ok(fail)


def test_float32_and_resampled_input(M):
    """Float32 rows (k_stage_f32), loud values (10^4 x full scale, below the gate), and configurations lamejs resamples (rows
    at the output rate; the oracle resamples on the CPU)"""
    fail = []
    for kind in ("webaudio", "unit", "x4"):
        for (ch, sr, kb) in ((2, 44100, 128), (1, 22050, 64)):
            sigs = [float_signals.make(kind, n, sr, 70 + n % 7) for n in (1377, 30 * 1152 + 11)]
            P.whole_streams(M, ch, sr, kb, sigs, "float32 %s %d/%d/%d" % (kind, ch, sr, kb), fail, F.check_rows, f32=True)
    for kind in ("burst", "impulse", "nyquist"):
        sigs = [float_signals.loud(kind, 1e4, n, 44100, 80 + n % 5, 1.0) for n in (5000, 20 * 1152 + 3)]
        P.whole_streams(M, 2, 44100, 128, sigs, "loud float32 %s" % kind, fail, F.check_rows, f32=True)
    for case in [c for c in edge_signals.RESAMPLED_CASES if c[0] in ("clicks1", "square", "dc_min", "lsb_dither")]:
        _, ch, sr, kb, _ = case
        l, r = edge_signals.signal(case)
        P.whole_streams(M, ch, sr, kb, [(l, r if r is not None else l)], "resampled " + edge_signals.case_id(case), fail,
                        F.check_rows, resample=True)
    _ok(fail)


# ---- the PSY_UNITS, FB_G and SCAN_FRAMES knobs ----------------------------------------------------------------------------

# PSY_UNITS units per k_psy_analysis block; FB_G granules per k_mdct block (FB_G + 1 slabs per k_subband_analysis block): 1,
# 3 and 5 put block starts inside MPEG-1 frames; SCAN_FRAMES frames per speculative scan chunk
VARIANTS = {
    "psy1_fb1_scan3": ["PSY_UNITS=1", "FB_G=1", "SCAN_FRAMES=3"],
    "psy3_fb3_scan1": ["PSY_UNITS=3", "PSY_MIN_BLOCKS=5", "FB_G=3", "SCAN_FRAMES=1"],
    "psy4_fb5": ["PSY_UNITS=4", "PSY_MIN_BLOCKS=4", "FB_G=5"],
}


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("front_end_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_launch_shape_variants(variant_libs, name):
    """whole streams, ragged batches and upload slices with other k_psy_analysis, k_mdct / k_subband_analysis blocks and scan
    chunks"""
    env = dict(os.environ, MP3B200_LIB=variant_libs[name])
    p = subprocess.run([sys.executable, os.path.join(HERE, "front_rows.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert not res["fail"], (res["nfail"], res["fail"][:10])
