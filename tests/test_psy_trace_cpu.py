"""The oracle's psy trace means what it says: its peaks, attack candidates and loudness are recomputed in plain numpy from the
same PCM and tied to the values the encoder consumes (the ath_adjust of the frame trace).  tests/test_gpu_psy_rows.py
compares the GPU's psy rows with this trace, so a trace that recorded the wrong thing would let a wrong kernel pass."""
import ctypes

import numpy as np
import pytest

import edge_signals

# PsyModel.js:994-998: the fs/4 high-pass FIR, fircoef[i] = 2 x the listed half-coefficients
FIRCOEF = np.array([-8.65163e-18, -0.00851586, -6.74764e-18, 0.0209036, -3.36639e-17, -0.0438162, -1.54175e-17, 0.0931738,
                    -5.52212e-17, -0.313819]) * 2

EDGE = [c for c in edge_signals.CASES if c[0] in ("square", "dc_max", "dc_min", "nyquist", "lsb_dither", "lsb_clicks", "clicks1",
                                                 "click_pairs", "loud_silent", "silent_right", "fs_white")]


def quiet_case(lsb, ch, sr, kb, n, seed):
    rng = np.random.default_rng(seed)
    l = rng.integers(-lsb, lsb + 1, n).astype(np.int16)
    r = rng.integers(-lsb, lsb + 1, n).astype(np.int16) if ch == 2 else None
    return l, r


QUIET = [(lsb, ch, sr, kb) for lsb in (1, 4, 16, 64) for ch, sr, kb in ((2, 44100, 128), (1, 22050, 64))]


def encode(oracle, ch, sr, kb, l, r):
    enc = oracle.OracleEncoder(ch, sr, kb, trace_frames=len(l) // 576 + 8, psy_trace=True)
    enc.encode_buffer(l, r)
    enc.flush()
    L = enc.L
    L.lj_get_scale.argtypes = [ctypes.c_void_p]
    L.lj_get_scale.restype = ctypes.c_double
    out = dict(psy=enc.psy_traces(), bt_old=enc.psy_block_traces(), tr=enc.traces(), thr=enc.attack_threshold(), sens=enc.ath_aa_sensitivity(),
               scale=L.lj_get_scale(enc.h))
    enc.close()
    assert len(out["psy"]) == len(out["tr"])
    return out


def f32_ulps(a, b):
    """distance in float32 units in the last place (both finite, same sign)"""
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


def check_peaks(o, x, G, ch):
    """peaks[s] of unit c = max(1, |hp|) over hp outputs 64 s .. 64 s + 63, hp output q centred on stream sample 576 c + 183 + q
    (sum x[m] + fir[j] (x[m - 10 + j] + x[m + 11 - j])), each output stored as float32 (ns_hpfsmpl)"""
    psy = o["psy"]
    U = G * len(psy)
    pad = 1024
    xp = np.concatenate([np.zeros(pad), x, np.zeros(576 * U + 2048)])
    q = np.arange(576)
    for c in range(U):
        m = pad + 576 * c + 183 + q
        hp = xp[m].copy()
        for j in range(10):
            hp += FIRCOEF[j] * (xp[m - 10 + j] + xp[m + 11 - j])
        want = np.maximum(1.0, np.abs(hp.astype(np.float32)).reshape(9, 64).max(axis=1).astype(np.float64)).astype(np.float32)
        got = psy["peaks"][c // G, c % G, ch]
        assert (f32_ulps(got, want) <= 1).all(), (c, ch, got, want)


def attack_from_peaks(prev, cur, thr):
    """k_attack_prepass / PsyModel.js:1108-1183 up to the lastAttacks rule, from the float32 peaks of units c - 1 and c"""
    f32 = np.float32
    en_subshort = [f32(0)] * 12
    ai = [f32(0)] * 12
    en_short = [0.0] * 4
    for i in range(3):
        en_subshort[i] = f32(prev[i + 6])
        ai[i] = f32(float(en_subshort[i]) / float(prev[i + 4]))
        en_short[0] += float(en_subshort[i])
    for i in range(9):
        p = float(cur[i])
        en_subshort[i + 3] = f32(p)
        if i % 3 == 0:
            en_short[1 + i // 3] += p
        e2 = float(en_subshort[i + 1])
        if p > e2:
            p = p / e2
        elif e2 > p * 10.0:
            p = e2 / (p * 10.0)
        else:
            p = 0.0
        ai[i + 3] = f32(p)
    a = [0, 0, 0, 0]
    for i in range(0, 12, 3):
        if float(ai[i]) > thr:
            a[i // 3] = 1
    for i in range(1, 4):
        ratio = en_short[i - 1] / en_short[i] if en_short[i - 1] > en_short[i] else en_short[i] / en_short[i - 1]
        if ratio < 1.7:
            a[i] = 0
            if i == 1:
                a[0] = 0
    return a


def check_attacks(o, G, ch):
    psy = o["psy"]
    init = np.full(9, 10.0, np.float32)
    for c in range(G * len(psy)):
        prev = init if c == 0 else psy["peaks"][(c - 1) // G, (c - 1) % G, ch]
        cur = psy["peaks"][c // G, c % G, ch]
        assert list(psy["attack"][c // G, c % G, ch]) == attack_from_peaks(prev, cur, o["thr"]), (c, ch)


def check_ath_adjust(o, G, nch):
    """Encoder.js adjust_ATH in Python doubles from the traced loudness: loudness_sq[gr] of frame k is the loudness of unit
    G k + gr - 1 (one call late; unit -1 has 0), summed over the channels (doubled for mono)"""
    psy, tr = o["psy"], o["tr"]

    def pw(c):
        if c < 0:
            return 0.0
        loud = psy["loudness"][c // G, c % G]
        v = float(loud[0])
        return v + (float(loud[1]) if nch == 2 else v)
    adjust, limit = 0.01, 1.0
    for k in range(len(tr)):
        max_pow = pw(G * k - 1)
        if G == 2:
            gr2 = pw(G * k)
            max_pow = max(max_pow, gr2)
        max_pow *= 0.5
        max_pow *= o["sens"]
        if max_pow > 0.03125:
            if adjust >= 1.0:
                adjust = 1.0
            elif adjust < limit:
                adjust = limit
            limit = 1.0
        else:
            new = 31.98 * max_pow + 0.000625
            if adjust >= new:
                adjust *= new * 0.075 + 0.925
                if adjust < new:
                    adjust = new
            else:
                if limit >= new:
                    adjust = new
                elif adjust < limit:
                    adjust = limit
            limit = new
        assert np.float64(adjust).tobytes() == np.float64(tr["ath_adjust"][k]).tobytes(), (k, adjust, tr["ath_adjust"][k])


NORM, START, SHORT, STOP = 0, 1, 2, 3


def check_block_types(o, G, nch):
    """blocktype_old as each psy call found it, tied to the traced block types (block_type_set, PsyModel.js:784-826): the
    stream starts from NORM; a unit is short exactly when the next call finds SHORT, and then its block type is blocktype_old
    promoted (NORM -> START, STOP -> SHORT), else blocktype_old itself; a long unit hands on STOP after SHORT, NORM otherwise"""
    psy, tr = o["psy"], o["tr"]
    U = G * len(psy)
    assert len(o["bt_old"]) == len(psy)
    prev = o["bt_old"][:, :G, :nch].reshape(U, nch)
    bt = tr["blocktype"][:, :G, :nch].reshape(U, nch)
    assert (prev[0] == NORM).all()
    assert np.isin(prev, (NORM, SHORT, STOP)).all(), np.unique(prev)
    for c in range(U - 1):
        short = prev[c + 1] == SHORT
        promoted = np.where(prev[c] == NORM, START, np.where(prev[c] == STOP, SHORT, prev[c]))
        assert (bt[c] == np.where(short, promoted, prev[c])).all(), (c, bt[c], prev[c], prev[c + 1])
        assert (short | (prev[c + 1] == np.where(prev[c] == SHORT, STOP, NORM))).all(), (c, prev[c], prev[c + 1])


def run_case(oracle, ch, sr, kb, l, r):
    assert oracle.out_samplerate(ch, sr, kb) == sr
    G = 2 if sr >= 32000 else 1
    o = encode(oracle, ch, sr, kb, l, r)
    for c in range(ch):
        x = (l if c == 0 else r).astype(np.float64)
        if o["scale"] not in (0.0, 1.0):       # lame_encode_buffer_sample scales the stored Float32 samples
            x = (x * o["scale"]).astype(np.float32).astype(np.float64)
        check_peaks(o, x, G, c)
        check_attacks(o, G, c)
    check_ath_adjust(o, G, ch)
    return o


@pytest.mark.parametrize("case", EDGE, ids=edge_signals.case_id)
def test_trace_of_the_edge_corpus(oracle, case):
    _, ch, sr, kb, _ = case
    l, r = edge_signals.signal(case)
    o = run_case(oracle, ch, sr, kb, l, r if ch == 2 else None)
    check_block_types(o, 2 if sr >= 32000 else 1, ch)


@pytest.mark.parametrize("lsb,ch,sr,kb", QUIET)
def test_trace_of_quiet_signals(oracle, lsb, ch, sr, kb):
    """1 to 64 LSB: the loudness decides ath_adjust frame by frame"""
    l, r = quiet_case(lsb, ch, sr, kb, 40 * 1152 + 99, lsb)
    o = run_case(oracle, ch, sr, kb, l, r)
    assert (o["tr"]["ath_adjust"] < 1.0).any()


def test_trace_of_silence(oracle):
    """digital silence: every peak at the 1.0 clamp, loudness 0, no attack"""
    z = np.zeros(20 * 1152, np.int16)
    o = run_case(oracle, 2, 44100, 128, z, z)
    assert (o["psy"]["peaks"][:, :, :2] == 1.0).all() and (o["psy"]["loudness"] == 0).all() and not o["psy"]["attack"].any()
