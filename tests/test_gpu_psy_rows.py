"""k_psy_analysis, k_attack_prepass and k_psy_short row for row against the oracle's psy trace (tests/psy_rows.py), in every
launch shape the rows depend on: whole streams of every native configuration, ragged batches, upload slices, streaming
handles (odd chunks, batches of handles at different frames, state blobs, seek), device-resident and session calls, Float32
and resampled input; and the library built with PSY_UNITS = 1, 3 and 4.  Each call runs on a poisoned workspace and its
bytes must equal the oracle's."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import edge_signals
import float_signals
import psy_rows as P

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


def _ok(fail):
    assert not fail, "%d rows differ; first: %s" % (len(fail), fail[:10])


def test_whole_streams_every_native_configuration(M):
    fail = []
    P.shape_whole(M, fail)
    _ok(fail)


def test_ragged_batches(M):
    fail = []
    P.shape_batches(M, fail)
    _ok(fail)


def test_upload_slices(M):
    fail = []
    P.shape_slices(M, fail)
    _ok(fail)


@pytest.mark.parametrize("case", [c for c in edge_signals.CASES if c[0] in ("square", "dc_max", "dc_min", "nyquist", "lsb_dither",
                                                                           "lsb_clicks", "clicks1", "clicks4", "click_pairs",
                                                                           "loud_silent", "silent_right")],
                         ids=edge_signals.case_id)
def test_edge_corpus(M, case):
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    fail = []
    P.whole_streams(M, ch, sr, kb, [(l, r)], edge_signals.case_id(case), fail)
    _ok(fail)


def test_the_poison_reaches_no_kernel_and_capture_off_changes_nothing(M):
    """a capture launch leaves rows the launch does not use poisoned for the next one; the next call with capture off
    encodes the same bytes as before (it overwrites every row it reads)"""
    l, r = P.k2_signal("mixed", 40 * 1152 + 77, 3)
    before = M.encode_streams(2, 44100, 128, [l], [r])[0]
    with M.debug_psy_capture() as cap:
        M.encode_streams(2, 44100, 128, [l[:5000]], [r[:5000]])
    assert len(cap.launches) == 1
    assert M.encode_streams(2, 44100, 128, [l], [r])[0] == before


CHUNKS = [1, 575, 576, 577, 1151, 1152, 1153, 4097]


def _handle_calls(M, ch, sr, kb, l, r, chunks, label, fail):
    """one handle fed `chunks` (cycled) and flushed, each call under capture; returns the rows' oracle"""
    ref = P.make_ref(ch, sr, kb)
    enc = M.Mp3Encoder(ch, sr, kb)
    recs = []
    i = k = 0
    while i < len(l):
        n = chunks[k % len(chunks)]
        k += 1
        got, launches = P.capture_call(M, lambda: enc.encodeBuffer(l[i:i + n], r[i:i + n] if ch == 2 else None))
        if got != ref.call(l[i:i + n], r[i:i + n] if ch == 2 else None):
            fail.append("%s: bytes of call %d" % (label, k))
        recs += launches
        i += n
    got, launches = P.capture_call(M, enc.flush)
    if got != ref.flush():
        fail.append("%s: bytes of flush" % label)
    recs += launches
    enc.close()
    ref.done()
    for rec in recs:
        P.check_launch(rec, [ref], label, fail)
    return recs


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 22050, 64)])
def test_handle_chunks(M, ch, sr, kb):
    """encodeBuffer with chunks of 1, 575, 576, 577, 1151, 1152, 1153 and 4097 samples, then flush: frame0 > 0, the halo unit
    recomputed from the carried tail"""
    l, r = P.k2_signal("mixed", 60 * 1152 + 333, 11)
    fail = []
    recs = _handle_calls(M, ch, sr, kb, l, r, CHUNKS, "handle %d/%d/%d" % (ch, sr, kb), fail)
    assert sum(1 for rec in recs for s in rec["streams"] if s["frame0"] % 2) > 0
    _ok(fail)


def test_handle_batch_state_blobs_and_seek(M):
    """encode_batch over handles whose frame0 differ in parity; a handle exported and imported mid-stream; a handle seeked into
    the middle of a stream, its halo rebuilt from the history"""
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
        if e.encodeBuffer(l[:n], r[:n]) != rf.call(l[:n], r[:n]):
            fail.append("warm-up %d" % j)
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
    assert len({s["frame0"] % 2 for rec, _ in recs for s in rec["streams"]}) == 2
    # export / import the second handle, go on with the imported one
    blob = encs[1].export_state()
    encs[1].close()
    encs[1] = M.Mp3Encoder(ch, sr, kb)
    encs[1].import_state(blob)
    for j, (e, rf, (l, r)) in enumerate(zip(encs, refs, sigs)):
        got, launches = P.capture_call(M, lambda: e.encodeBuffer(l[pos[j]:], r[pos[j]:]) + e.flush())
        if got != rf.call(l[pos[j]:], r[pos[j]:]) + rf.flush():
            fail.append("tail %d" % j)
        recs += [(rec, [j]) for rec in launches]
        e.close()
    for rf in refs:
        rf.done()
    for rec, zs in recs:
        P.check_launch(rec, [refs[z] for z in zs], "handles", fail)
    # seek: a fresh handle at frame 17 of stream 0, fed the rest of it
    l, r = sigs[0]
    frame = 17
    lo, hi = max(0, frame * fs - 1104), frame * fs + 224
    e = M.Mp3Encoder(ch, sr, kb)
    e.seek(frame, l[lo:hi], r[lo:hi])
    got, launches = P.capture_call(M, lambda: e.encodeBuffer(l[hi:], r[hi:]) + e.flush())
    e.close()
    assert launches and launches[0]["streams"][0]["frame0"] == frame
    for rec in launches:
        P.check_launch(rec, [refs[0]], "seek", fail)
    _ok(fail)


def _packed(M, torch, ch, sigs, f32=False):
    ns = [len(l) for l, _ in sigs]
    dt = np.float32 if f32 else np.int16
    pcm = np.concatenate([np.concatenate([l, r]).astype(dt) if ch == 2 else l.astype(dt) for l, r in sigs] + [np.zeros(8, dt)])
    pcm_off = np.cumsum([0] + [n * ch for n in ns])[:-1]
    return torch.from_numpy(pcm).cuda(), pcm_off, ns


def test_device_and_session_entries(M):
    """encode_streams_device, EncodeSession.encode_streams and EncodeSession.encode_batch"""
    import torch

    ch, sr, kb = 2, 44100, 128
    sigs = [P.k2_signal(k, n, 40 + i) for i, (k, n) in enumerate((("mixed", 30 * 1152 + 5), ("impulses", 1377), ("silence", 0),
                                                                    ("nyquist", 9 * 1152)))]
    fail = []
    d_pcm, pcm_off, ns = _packed(M, torch, ch, sigs)
    nb = [M.stream_bytes(ch, sr, kb, n) for n in ns]
    out_off = np.cumsum([0] + nb)[:-1]

    def refs():
        rf = [P.make_ref(ch, sr, kb) for _ in sigs]
        want = [x.stream(l, r) for x, (l, r) in zip(rf, sigs)]
        return [x.done() for x in rf], want

    for entry in ("device", "session"):
        rf, want = refs()
        d_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
        if entry == "device":
            _, launches = P.capture_call(M, lambda: M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off))
        else:
            with M.EncodeSession() as sess:
                def run():
                    st = sess.encode_streams(ch, sr, kb, d_pcm, pcm_off, ns, d_out, out_off)
                    M.check_status(st)
                _, launches = P.capture_call(M, run)
        out = d_out.cpu().numpy()
        for i, (o, b, w) in enumerate(zip(out_off, nb, want)):
            if out[o:o + b].tobytes() != w:
                fail.append("%s: bytes of stream %d" % (entry, i))
        base = 0
        for rec in launches:
            P.check_launch(rec, rf[base:base + len(rec["streams"])], entry, fail)
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
        P.check_launch(rec, rf, "session handles", fail)
    for h in hs:
        h.close()
    _ok(fail)


def test_float32_and_resampled_input(M):
    """Float32 rows (k_stage_f32), loud values below the gate, and configurations lamejs resamples (rows at the output
    rate; the oracle resamples on the CPU)"""
    fail = []
    for kind in ("webaudio", "unit", "x4"):
        for (ch, sr, kb) in ((2, 44100, 128), (1, 22050, 64)):
            sigs = [float_signals.make(kind, n, sr, 70 + n % 7) for n in (1377, 30 * 1152 + 11)]
            P.whole_streams(M, ch, sr, kb, sigs, "float32 %s %d/%d/%d" % (kind, ch, sr, kb), fail, f32=True)
    for kind in ("burst", "impulse", "nyquist"):        # 10^4 x full scale: far above it, below the 2^40 gate
        sigs = [float_signals.loud(kind, 1e4, n, 44100, 80 + n % 5, 1.0) for n in (5000, 20 * 1152 + 3)]
        P.whole_streams(M, 2, 44100, 128, sigs, "loud float32 %s" % kind, fail, f32=True)
    for case in [c for c in edge_signals.RESAMPLED_CASES if c[0] in ("clicks1", "square", "dc_min", "lsb_dither")]:
        _, ch, sr, kb, _ = case
        l, r = edge_signals.signal(case)
        P.whole_streams(M, ch, sr, kb, [(l, r if r is not None else l)], "resampled " + edge_signals.case_id(case), fail, resample=True)
    _ok(fail)


# ---- the PSY_UNITS knob ---------------------------------------------------------------------------------------------------

VARIANTS = {
    "psy_units1": ["PSY_UNITS=1"],
    "psy_units3": ["PSY_UNITS=3", "PSY_MIN_BLOCKS=5"],
    "psy_units4": ["PSY_UNITS=4", "PSY_MIN_BLOCKS=4"],
}


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("psy_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_psy_units_variants(variant_libs, name):
    """whole streams, ragged batches and upload slices with PSY_UNITS units per k_psy_analysis block"""
    env = dict(os.environ, MP3B200_LIB=variant_libs[name])
    p = subprocess.run([sys.executable, os.path.join(HERE, "psy_rows.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert not res["fail"], (res["nfail"], res["fail"][:10])
