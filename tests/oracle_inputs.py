"""Every input the GPU tests compare with the oracle stage by stage or byte for byte, in one place.

The GPU copy of a branch of the encoder is only checked where some input the GPU tests feed drives the oracle through that
branch, so the branch ledger (tests/branch_ledger.py, tests/test_branch_ledger_cpu.py) runs the oracle, built with coverage,
over exactly these inputs.  The GPU tests import their case lists from here (or from edge_signals / float_signals, which
this module gathers), so what the ledger accounts for is what they run.

runs() lists them all as (id, channels, samplerate, kbps, calls) with calls() -> [(left, right or None), ...]: the
encodeBuffer calls of the stream (Int16 arrays, or floating arrays for lamejs's Float32 store), flush() after the last."""
import json
import os

import numpy as np

import edge_signals
import float_signals
import oracle_lib
from synth import make_signal

HERE = os.path.dirname(os.path.abspath(__file__))

# tests/test_gpu_parity.py: test_stage_parity, MPEG-1 (kind, channels, samplerate, kbps, frames), seed 21
STAGE_PARITY_CASES = [
    ("noise", 2, 44100, 128, 60), ("burst", 2, 44100, 128, 80), ("white", 2, 48000, 320, 50), ("sine", 1, 44100, 128, 40),
    ("octave", 1, 44100, 128, 60), ("sweep", 2, 44100, 128, 120), ("noise", 2, 32000, 160, 40), ("white", 1, 48000, 320, 30),
    ("silence", 2, 44100, 128, 12), ("burst", 1, 44100, 192, 60)]

# test_stage_parity_lsf: MPEG-2 / MPEG-2.5, seed 23
LSF_STAGE_PARITY_CASES = [
    ("noise", 2, 22050, 64, 80), ("burst", 2, 24000, 96, 100), ("octave", 1, 16000, 32, 80), ("white", 2, 16000, 160, 60),
    ("burst", 1, 22050, 32, 90), ("noise", 1, 8000, 8, 60), ("burst", 2, 12000, 32, 70), ("sine", 2, 11025, 40, 50), ("sine", 1, 11025, 24, 50),
    ("silence", 2, 24000, 64, 14)]


def stage_parity_signal(case):
    kind, ch, sr, kbps, frames = case
    l, r = make_signal(kind, frames * 1152 + 211, sr, 21)
    return l, (r if ch == 2 else None)


def lsf_stage_parity_signal(case):
    kind, ch, sr, kbps, frames = case
    l, r = make_signal(kind, frames * 576 + 211, sr, 23)
    return l, (r if ch == 2 else None)


# test_config_matrix: every bitrate of each rate's MPEG version and an off-ladder one lamejs snaps, mono and stereo; the
# configurations lamejs encodes at the input rate (the others the C ABI refuses without MP3B200_RESAMPLE)
CONFIG_MATRIX_RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)
CONFIG_MATRIX_KBPS = (8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 123, 128, 144, 160, 192, 224, 256, 320)


def config_matrix_signals(sr):
    """the two streams every configuration of rate `sr` encodes: a short burst and a short noise stream"""
    return make_signal("burst", 9 * 1152 + 100, sr, 77), make_signal("noise", 7 * 1152, sr, 78)


# tests/test_gpu_float.py: MPEG-1, MPEG-2, MPEG-2.5 and resampled (48 -> 24, 44.1 -> 22.05, 48 -> 8 kHz) configurations
FLOAT_CFGS = [(2, 44100, 128), (1, 48000, 160), (2, 32000, 96), (2, 22050, 64), (1, 24000, 48), (2, 16000, 40), (1, 11025, 24),
              (2, 12000, 32), (1, 8000, 16), (2, 48000, 64), (2, 44100, 48), (1, 48000, 8)]
# the float inputs lamejs callers pass: Web Audio x * 32767 with fractions, unscaled [-1, 1], 1.5 and 4 x full scale,
# +-0.5 dither, Float32 denormals and -0.0
FLOAT_KINDS = ["webaudio", "unit", "x1.5", "x4", "dither", "denormal"]
FLOAT_TAP_KINDS = ("webaudio", "unit")


def float_signal(kind, n, sr, seed):
    """(left, right) float32 arrays of a FLOAT_KINDS kind"""
    l, r = float_signals.make(kind, n, sr, seed)
    return l.astype(np.float32), r.astype(np.float32)


def frame_input_samples(ch, sr, kbps):
    """input samples per frame (more than the output's where lamejs resamples)"""
    out = oracle_lib.out_samplerate(ch, sr, kbps)
    return (1152 if out >= 32000 else 576) * (sr // out)


def float_entry_signals(cfg):
    """test_entry_points_match_the_oracle: one stream of each FLOAT_KINDS kind, six frames and a ragged tail"""
    ch, sr, kb = cfg
    n = 6 * frame_input_samples(ch, sr, kb) + 123
    return [float_signal(k, n, sr, 30 + i) for i, k in enumerate(FLOAT_KINDS)]


def float_tap_samples(cfg):
    """test_stage_taps_match_the_oracle: twelve granules and a ragged tail (seed 7)"""
    ch, sr, kb = cfg
    out = oracle_lib.out_samplerate(ch, sr, kb)
    return (sr // out) * (12 * 576 * (2 if out >= 32000 else 1) + 211) + 5


# test_edge_corpus_as_floats: these edge cases, /32768 as Float32 (Web Audio's range), against the oracle's Float32 store
EDGE_AS_FLOAT_CASES = edge_signals.CASES[::2] + edge_signals.RESAMPLED_CASES[::3]


def edge_as_float(case):
    l, r = edge_signals.signal(case)
    return (l.astype(np.float64) / 32768.0).astype(np.float32), None if r is None else (r.astype(np.float64) / 32768.0).astype(np.float32)


def loud_golden():
    """tests/golden/lamejs_loud_golden.json: loud Float32 input, pinned to lamejs (tests/test_gpu_loud_float.py)"""
    return json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))


def _lazy(fn, *args):
    def calls():
        l, r = fn(*args)
        return [(l, r)]
    return calls


def runs():
    """[(id, channels, samplerate, kbps, calls)]: every stream above as the oracle is given it"""
    out = []
    for c in edge_signals.CASES + edge_signals.RESAMPLED_CASES:
        out.append(("edge/" + edge_signals.case_id(c), c[1], c[2], c[3], _lazy(edge_signals.signal, c)))
    for c in EDGE_AS_FLOAT_CASES:
        out.append(("edge_as_float/" + edge_signals.case_id(c), c[1], c[2], c[3], _lazy(edge_as_float, c)))
    for c in STAGE_PARITY_CASES:
        out.append(("parity/%s-%d-%d-%d" % c[:4], c[1], c[2], c[3], _lazy(stage_parity_signal, c)))
    for c in LSF_STAGE_PARITY_CASES:
        out.append(("parity_lsf/%s-%d-%d-%d" % c[:4], c[1], c[2], c[3], _lazy(lsf_stage_parity_signal, c)))
    for sr in CONFIG_MATRIX_RATES:
        for kbps in CONFIG_MATRIX_KBPS:
            for ch in (1, 2):
                if oracle_lib.out_samplerate(ch, sr, kbps) != sr:
                    continue
                for j in range(2):
                    def calls(sr=sr, ch=ch, j=j):
                        l, r = config_matrix_signals(sr)[j]
                        return [(l, r if ch == 2 else None)]
                    out.append(("config_matrix/%d-%d-%d-%d" % (ch, sr, kbps, j), ch, sr, kbps, calls))
    for cfg in FLOAT_CFGS:
        ch, sr, kb = cfg
        for k in range(len(FLOAT_KINDS)):
            def calls(cfg=cfg, k=k):
                l, r = float_entry_signals(cfg)[k]
                return [(l, r if cfg[0] == 2 else None)]
            out.append(("float/%s-%d-%d-%d" % ((FLOAT_KINDS[k],) + cfg), ch, sr, kb, calls))
        for kind in FLOAT_TAP_KINDS:
            def calls(cfg=cfg, kind=kind):
                l, r = float_signal(kind, float_tap_samples(cfg), cfg[1], 7)
                return [(l, r if cfg[0] == 2 else None)]
            out.append(("float_taps/%s-%d-%d-%d" % ((kind,) + cfg), ch, sr, kb, calls))
    for name, c in sorted(loud_golden().items()):
        if float_signals.loud_peak(c) > float_signals.LOUD_GATE:
            continue                                  # the library refuses these before anything is encoded

        def calls(c=c):
            l, r, cl = float_signals.loud_case_signal(c)
            return [x for x in cl if x is not None]
        out.append(("loud/" + name, c["channels"], c["samplerate"], c["kbps"], calls))
    return out
