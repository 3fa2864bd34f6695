"""Edge-of-range PCM corpus: deterministic Int16 generators for the inputs where the encoder's data-dependent branches turn
(full scale and -32768, DC, Nyquist, +-1 LSB, clicks at every attack sub-block, a silent channel, L = -R, level jumps,
tones near 20 kHz), and the configurations each one is encoded with.

CASES drives tests/test_gpu_edges.py (every stage tap and the bytes against the oracle) and tests/test_edge_corpus_cpu.py
(the oracle, built with coverage, reaches the branches the corpus is meant to reach).  RESAMPLED_CASES are the same
generators fed to configurations lamejs resamples by an integer ratio r (MP3B200_RESAMPLE): the signals are made at the
input rate and sized and laid out in output samples times r, so the clicks still walk through every sub-block of the
output granules.  tests/test_gpu_edges.py runs them through every stage tap too, and tests/test_resample_cpu.py checks what
the resampler turns them into."""
import numpy as np

import oracle_lib
from synth import white

FULL = 32767
GRANULE = 576
SUBBLOCK = 192          # a short block: 3 per granule


def _noise(n, seed):
    a, b = white(n, 0x5EED0E00 + seed)
    return a, b


def square(n, period=100):
    """+-full-scale square wave (+32767 / -32768), the right channel in anti-phase."""
    x = np.where((np.arange(n) // (period // 2)) % 2 == 0, FULL, -FULL - 1).astype(np.int16)
    return x, (-x.astype(np.int32) - 1).astype(np.int16)


def dc(n, value):
    x = np.full(n, value, dtype=np.int16)
    return x, x.copy()


def nyquist(n):
    """Alternating +32767 / -32768: all energy at fs/2."""
    x = np.where(np.arange(n) % 2 == 0, FULL, -FULL - 1).astype(np.int16)
    return x, x[::-1].copy()


def clipped_sine(n, sr, f=997.0, gain=3.0):
    t = np.arange(n, dtype=np.float64)
    x = np.clip(np.rint(gain * FULL * np.sin(2 * np.pi * f * t / sr)), -FULL - 1, FULL).astype(np.int16)
    y = np.clip(np.rint(gain * FULL * np.sin(2 * np.pi * 1.5 * f * t / sr)), -FULL - 1, FULL).astype(np.int16)
    return x, y


def lsb_dither(n, seed=1):
    """Independent -1 / 0 / +1 samples."""
    a, b = _noise(n, seed)
    return (a.astype(np.int32) % 3 - 1).astype(np.int16), (b.astype(np.int32) % 3 - 1).astype(np.int16)


def lsb_clicks(n, seed=2):
    """Silence with a single +-1 sample every 300-ish samples."""
    a, b = _noise(n, seed)
    i = np.arange(n)
    l = np.where(i % 311 == 0, np.where(a > 0, 1, -1), 0).astype(np.int16)
    r = np.where(i % 257 == 5, np.where(b > 0, 1, -1), 0).astype(np.int16)
    return l, r


def fs_white(n, seed=3):
    """Full-scale white noise."""
    return _noise(n, seed)


def click_train(n, spacing, seed=4, ratio=1):
    """Full-scale clicks (a short noise burst of 16 samples) on a +-1 LSB floor, `spacing` granules apart; the offset of
    each click inside its granule walks through every sub-block quarter (48 samples), so that over the train the
    attacks land in every sub-block of the attack detector, and across the 16-frame boundaries of the block-type scan.
    With `ratio` r (input samples per output sample of a resampled configuration) granules and offsets are r times longer:
    they are those of the output."""
    a, b = _noise(n, seed)
    l = (a.astype(np.int32) % 3 - 1).astype(np.int16)
    r = (b.astype(np.int32) % 3 - 1).astype(np.int16)
    k = 0
    pos = GRANULE * ratio // 2
    while True:
        at = pos + (k * 48 * ratio) % (GRANULE * ratio)
        if at + 16 > n:
            break
        burst_l, burst_r = _noise(16, 100 + k)
        l[at:at + 16] = np.where(burst_l >= 0, FULL, -FULL - 1)
        if k % 3:                                  # every third click is left only
            r[at:at + 16] = np.where(burst_r >= 0, FULL, -FULL - 1)
        k += 1
        pos += spacing * GRANULE * ratio
    return l, r


def click_pairs(n, seed=9, ratio=1):
    """Pairs of full-scale clicks one short block (192 samples) apart, every other granule, the pair's offset walking
    through the granule in 32-sample steps: the second click of a pair is an attack in the last sub-block of one granule
    while the first one left lastAttacks set -- the case in which an attack in sub-block 0 is suppressed.  `ratio`: as in
    click_train."""
    a, b = _noise(n, seed)
    l = (a.astype(np.int32) % 3 - 1).astype(np.int16)
    r = (b.astype(np.int32) % 3 - 1).astype(np.int16)
    k = 0
    while True:
        at = ratio * (2 * GRANULE * k + (32 * k) % GRANULE)
        if at + SUBBLOCK * ratio + 8 > n:
            break
        for x in (at, at + SUBBLOCK * ratio):
            l[x:x + 8] = FULL
            r[x:x + 8] = -FULL - 1
        k += 1
    return l, r


def silent_right(n, seed=5):
    a, _ = _noise(n, seed)
    return (a >> 2).astype(np.int16), np.zeros(n, dtype=np.int16)


def l_minus_r(n, seed=6):
    a, _ = _noise(n, seed)
    l = (a >> 1).astype(np.int16)
    return l, (-l.astype(np.int32)).astype(np.int16)


def loud_silent(n, framesize, seed=7):
    """Full-scale noise and digital silence alternating frame by frame, then every 3 frames."""
    a, b = _noise(n, seed)
    f = np.arange(n) // framesize
    on = np.where(f < 40, f % 2 == 0, f % 3 == 0)
    return np.where(on, a, 0).astype(np.int16), np.where(on, b, 0).astype(np.int16)


def hf_tone(n, sr, seed=8):
    """19.5 kHz (left) and a 19-20 kHz sweep (right) at -6 dBFS, over a -60 dB noise floor."""
    t = np.arange(n, dtype=np.float64)
    a, b = _noise(n, seed)
    l = np.rint(16384 * np.sin(2 * np.pi * 19500.0 * t / sr)) + (a >> 10)
    f = 19000.0 + 1000.0 * t / max(n, 1)
    r = np.rint(16384 * np.sin(2 * np.pi * np.cumsum(f) / sr)) + (b >> 10)
    return l.astype(np.int16), r.astype(np.int16)


def tone_comb(n, sr, level):
    """40 tones spaced evenly in log frequency from 60 Hz to 0.45 fs, each at (f / 1 kHz) x level / 10 (rising 6 dB per
    octave), the right channel 1 radian later: quantizes to values of at most 15 with table 14 best in region 2, the
    region whose table 14 -> 16 remap the side-info writer has."""
    t = np.arange(n, dtype=np.float64)
    out = []
    for ph in (0.0, 1.0):
        x = sum((f / 1000.0) * np.sin(2 * np.pi * f * t / sr + f + ph) for f in np.geomspace(60.0, sr * 0.45, 40))
        out.append(np.clip(np.rint(x * level / 10.0), -FULL - 1, FULL).astype(np.int16))
    return out[0], out[1]


def make(kind, n, sr, framesize, ratio=1):
    """`n` samples of `kind` at `sr`; `framesize` and `ratio` are in input samples (a resampled configuration's output frame
    and granule are `ratio` times longer at the input)."""
    if kind == "square":
        return square(n)
    if kind == "dc_max":
        return dc(n, FULL)
    if kind == "dc_min":
        return dc(n, -FULL - 1)
    if kind == "nyquist":
        return nyquist(n)
    if kind == "clipped_sine":
        return clipped_sine(n, sr)
    if kind == "lsb_dither":
        return lsb_dither(n)
    if kind == "lsb_clicks":
        return lsb_clicks(n)
    if kind == "fs_white":
        return fs_white(n)
    if kind.startswith("clicks"):
        return click_train(n, int(kind[6:]), ratio=ratio)
    if kind == "click_pairs":
        return click_pairs(n, ratio=ratio)
    if kind == "silent_right":
        return silent_right(n)
    if kind == "l_minus_r":
        return l_minus_r(n)
    if kind == "loud_silent":
        return loud_silent(n, framesize)
    if kind == "hf_tone":
        return hf_tone(n, sr)
    if kind.startswith("tone_comb"):
        return tone_comb(n, sr, int(kind[9:]))
    raise ValueError(kind)


# (kind, channels, samplerate, kbps, frames).  MPEG-1 and LSF (MPEG-2 / 2.5), mono and stereo.  fs_white runs at the lowest
# bitrate the configuration encodes natively (no resampling) and the +-1 LSB inputs at the highest, to drive the global
# gain to 255 and to 0.
CASES = [
    ("square", 2, 44100, 128, 40), ("square", 1, 22050, 64, 60),
    ("dc_max", 1, 44100, 128, 20), ("dc_min", 2, 24000, 64, 30), ("dc_min", 2, 48000, 192, 20),
    ("nyquist", 2, 48000, 192, 30), ("nyquist", 1, 16000, 32, 40),
    ("clipped_sine", 2, 32000, 128, 40), ("clipped_sine", 2, 22050, 96, 50),
    ("lsb_dither", 2, 48000, 320, 30), ("lsb_dither", 1, 44100, 320, 30), ("lsb_dither", 2, 24000, 160, 40),
    ("lsb_clicks", 1, 44100, 320, 30), ("lsb_clicks", 2, 24000, 160, 40),
    ("fs_white", 1, 32000, 48, 40), ("fs_white", 2, 44100, 112, 40), ("fs_white", 1, 8000, 8, 60), ("fs_white", 2, 16000, 32, 60),
] + [("clicks%d" % s, 2, 44100, 128, 56) for s in range(1, 7)] + [("clicks%d" % s, 1, 22050, 64, 100) for s in (1, 2, 3, 5)] + [
    ("click_pairs", 2, 44100, 128, 60), ("click_pairs", 1, 16000, 32, 120),
    ("silent_right", 2, 44100, 128, 40), ("silent_right", 2, 22050, 64, 60),
    ("l_minus_r", 2, 48000, 256, 30), ("l_minus_r", 2, 16000, 48, 60),
    ("loud_silent", 2, 44100, 128, 60), ("loud_silent", 1, 24000, 56, 80),
    ("hf_tone", 2, 44100, 320, 30), ("hf_tone", 1, 48000, 128, 30),
    ("tone_comb5000", 2, 44100, 128, 12),
]


# (kind, channels, input samplerate, kbps, output frames): configurations lamejs resamples by an integer ratio, all of them
# MPEG-2 or MPEG-2.5 at the output and all with gfp.scale = 0.95 (scale_applied), spread over the ratios 2, 3, 4 and 6 and
# mono / stereo.  After the filter these inputs are what Int16 input never is: full-scale squares, DC and click trains
# overshoot +-32768, and +-1 LSB input becomes fractional samples.  nyquist puts all its energy where the filter removes
# it, hf_tone above the output's Nyquist frequency.
RESAMPLED_CASES = [
    ("square", 2, 48000, 64, 40), ("square", 1, 48000, 8, 40),
    ("dc_max", 1, 32000, 16, 30), ("dc_max", 2, 24000, 24, 30), ("dc_min", 1, 48000, 24, 30), ("dc_min", 2, 32000, 8, 30),
    ("nyquist", 2, 24000, 16, 40), ("nyquist", 1, 48000, 40, 40),
    ("hf_tone", 2, 48000, 64, 30), ("hf_tone", 1, 44100, 32, 40),
    ("lsb_dither", 2, 48000, 56, 30), ("lsb_dither", 1, 16000, 8, 40), ("lsb_dither", 2, 32000, 16, 40),
    ("lsb_clicks", 1, 48000, 40, 30), ("lsb_clicks", 2, 48000, 16, 40),
    ("fs_white", 1, 48000, 8, 40), ("fs_white", 2, 24000, 8, 40),
] + [("clicks%d" % s, 2, 48000, 64, 56) for s in range(1, 7)] + [("clicks%d" % s, 1, 48000, 16, 60) for s in (1, 2, 3, 5)] + [
    ("click_pairs", 2, 44100, 48, 60), ("click_pairs", 1, 32000, 8, 80),
    ("loud_silent", 2, 48000, 64, 60), ("loud_silent", 1, 24000, 8, 60),
    ("silent_right", 2, 32000, 40, 40), ("silent_right", 2, 48000, 8, 40),
    ("l_minus_r", 2, 16000, 24, 40), ("l_minus_r", 2, 48000, 32, 40),
    ("clipped_sine", 2, 48000, 40, 40), ("clipped_sine", 1, 32000, 24, 40),
]


def case_id(c):
    kind, ch, sr, kbps, frames = c
    return "%s-%dch-%d-%dk" % (kind, ch, sr, kbps)


def ratio(case):
    """input samples per output sample of a case's configuration (1: lamejs encodes at the input rate)"""
    _, ch, sr, kbps, _ = case
    return sr // oracle_lib.out_samplerate(ch, sr, kbps)


def signal(case):
    """(left, right or None) of a case: `frames` frames of its configuration plus a ragged tail.  For a resampled case the
    frames are output frames and the signal is r times as long (r = ratio(case)), its tail too."""
    kind, ch, sr, kbps, frames = case
    r = ratio(case)
    out_rate = sr // r
    framesize = (1152 if out_rate >= 32000 else 576) * r
    n = frames * framesize + 211 * r
    l, rt = make(kind, n, sr, framesize, r)
    return l, (rt if ch == 2 else None)
