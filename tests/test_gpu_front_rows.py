"""k_stream_scan's block types and ATH adjustments, k_psy_masking's masking rows and k_mdct's xr row for row against the
oracle's traces (tests/front_rows.py), in every launch shape: whole streams of every native configuration, ragged batches,
upload slices, the edge corpus, streaming handles (odd chunks, calls that start on a short granule, batches of handles at
different frames, state blobs, seek), device-resident and session calls, Float32 and resampled input; and the library built
with other k_mdct / k_subband_analysis block sizes (FB_G) and scan chunk lengths (SCAN_FRAMES).  Each call runs on a
poisoned workspace and its bytes must equal the oracle's, which shows that no quantizer read a masking row left poisoned."""
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

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHECK = F.check_front


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


def _ok(fail):
    assert not fail, "%d rows differ; first: %s" % (len(fail), fail[:10])


def test_whole_streams_every_native_configuration(M):
    fail = []
    P.shape_whole(M, fail, check=CHECK)
    _ok(fail)


def test_ragged_batches(M):
    fail = []
    P.shape_batches(M, fail, check=CHECK)
    _ok(fail)


def test_upload_slices(M):
    fail = []
    P.shape_slices(M, fail, check=CHECK)
    _ok(fail)


@pytest.mark.parametrize("case", [c for c in edge_signals.CASES if c[0] in ("square", "dc_max", "dc_min", "nyquist", "lsb_dither",
                                                                           "lsb_clicks", "clicks1", "clicks4", "click_pairs",
                                                                           "loud_silent", "silent_right")],
                         ids=edge_signals.case_id)
def test_edge_corpus(M, case):
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    fail = []
    P.whole_streams(M, ch, sr, kb, [(l, r)], edge_signals.case_id(case), fail, check=CHECK)
    _ok(fail)


def test_unread_short_halves_stay_poisoned_and_capture_off_changes_nothing(M):
    """a capture call of a silent stream (no short blocks) leaves the short half of nearly every masking row poisoned (only the
    last unit needs it); a stream of the same length with short blocks, encoded next with capture off, still encodes the
    bytes it encoded before: it writes every masking row its quantizer reads"""
    n = 40 * 1152 + 77
    l, r = P.k2_signal("mixed", n, 3)
    before = M.encode_streams(2, 44100, 128, [l], [r])[0]
    z = np.zeros(n, np.int16)
    with M.debug_psy_capture() as cap:
        M.encode_streams(2, 44100, 128, [z], [z])
    (s,) = cap.launches[0]["streams"]
    assert not (s["bt"] == F.BT_SHORT).any()
    assert np.isnan(s["ratio"]["en_s"][1:-1]).all() and not np.isnan(s["ratio"]["en_s"][-1]).any()
    assert M.encode_streams(2, 44100, 128, [l], [r])[0] == before


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
    got, launches = P.capture_call(M, enc.flush)
    if got != ref.flush():
        fail.append("%s: bytes of flush" % label)
    recs += launches
    enc.close()
    ref.done()
    for rec in recs:
        CHECK(rec, [ref], label, fail)
    return recs, ref


CHUNKS = [1, 575, 576, 577, 1151, 1152, 1153, 4097]


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 22050, 64)])
def test_handle_chunks(M, ch, sr, kb):
    """encodeBuffer with chunks of 1, 575, 576, 577, 1151, 1152, 1153 and 4097 samples, then flush: frame0 > 0, the halo row
    carried from the previous call, the scan starting from the carried state"""
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
    """handles cut so that the next call starts on a short granule (found from the oracle's block types; the first of a short
    run where one starts a frame, and granules inside runs): its masking reads the short half of the carried halo row.  A
    state blob between the calls."""
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    G = M.granules_per_frame(ch, sr, kb)
    fs = 576 * G
    whole = P.make_ref(ch, sr, kb)
    whole.stream(l, r if ch == 2 else None)
    bt = whole.done().bt
    short = [u for u in range(G, len(bt), G) if (bt[u] == P.BT_SHORT).any()]
    first = [u for u in short if not (bt[u - 1] == P.BT_SHORT).any()]
    assert len(short) >= 3
    fail, starts = [], 0
    for u in sorted(set(first[:2] + short[:2] + short[-2:])):
        f = u // G
        # lamejs holds 576 + 48 samples back (MDCT lookahead, encoder delay) before frame f completes: the first and the last
        # cut after which f frames are done
        for cut in (f * fs + fs // 2 + 48, (f + 1) * fs + fs // 2 + 47):
            cut = min(cut, len(l) - 1)
            mid = cut + (len(l) - cut) // 3
            recs, ref = _handle(M, ch, sr, kb, l, r, [0, cut, mid, len(l)], "%s cut %d" % (edge_signals.case_id(case), cut), fail,
                                blob_after=(0,))
            starts += sum(1 for rec in recs for s in rec["streams"]
                          if s["nframes"] and s["frame0"] and (ref.bt[G * s["frame0"]] == P.BT_SHORT).any())
    assert starts > 0, "no call started on a short granule"
    _ok(fail)


def test_handle_batch_state_blobs_and_seek(M):
    """encode_batch over handles whose frame0 differ in parity; a handle exported and imported mid-stream; a handle seeked into
    the middle of a stream (no oracle: its rows start from the stream-start state and hold no poison)"""
    ch, sr, kb = 2, 44100, 128
    fs = 1152
    sigs = [P.k2_signal(k, 50 * fs + 100 * i, 20 + i) for i, k in enumerate(("mixed", "impulses", "quiet8"))]
    refs = [P.make_ref(ch, sr, kb) for _ in sigs]
    encs = [M.Mp3Encoder(ch, sr, kb) for _ in sigs]
    fail, recs = [], []
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
        CHECK(rec, [refs[z] for z in zs], "handles", fail)
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
            CHECK(rec, rf[base:base + len(rec["streams"])], entry, fail)
            base += len(rec["streams"])
        assert base == len(sigs)
    # session handles: three live encoders fed device rows in two rounds, then flushed
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
        CHECK(rec, rf, "session handles", fail)
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
            P.whole_streams(M, ch, sr, kb, sigs, "float32 %s %d/%d/%d" % (kind, ch, sr, kb), fail, f32=True, check=CHECK)
    for kind in ("burst", "impulse", "nyquist"):
        sigs = [float_signals.loud(kind, 1e4, n, 44100, 80 + n % 5, 1.0) for n in (5000, 20 * 1152 + 3)]
        P.whole_streams(M, 2, 44100, 128, sigs, "loud float32 %s" % kind, fail, f32=True, check=CHECK)
    for case in [c for c in edge_signals.RESAMPLED_CASES if c[0] in ("clicks1", "square", "dc_min", "lsb_dither")]:
        _, ch, sr, kb, _ = case
        l, r = edge_signals.signal(case)
        P.whole_streams(M, ch, sr, kb, [(l, r if r is not None else l)], "resampled " + edge_signals.case_id(case), fail,
                        resample=True, check=CHECK)
    _ok(fail)


# ---- the FB_G and SCAN_FRAMES knobs ---------------------------------------------------------------------------------------

# FB_G granules per k_mdct block (FB_G + 1 slabs per k_subband_analysis block): 1, 3 and 5 put block starts inside MPEG-1
# frames; SCAN_FRAMES frames per speculative scan chunk
VARIANTS = {
    "fb1_scan3": ["FB_G=1", "SCAN_FRAMES=3"],
    "fb3_scan1": ["FB_G=3", "SCAN_FRAMES=1"],
    "fb5": ["FB_G=5"],
}


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("front_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_launch_shape_variants(variant_libs, name):
    """whole streams, ragged batches and upload slices with other k_mdct / k_subband_analysis blocks and scan chunks"""
    env = dict(os.environ, MP3B200_LIB=variant_libs[name])
    p = subprocess.run([sys.executable, os.path.join(HERE, "front_rows.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert not res["fail"], (res["nfail"], res["fail"][:10])
