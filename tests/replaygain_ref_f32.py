"""The ReplayGain restatement (tests/replaygain_ref.py / .cpp) fed with Float32 input: what AnalyzeSamples sees when
encodeBuffer is given Float32Arrays (or Int16Arrays and Float32Arrays in turn).  Test infrastructure only.

lamejs stores the caller's values into Float32Arrays and scales them in place, so the analysed rows are
Float32((double)Float32(v) * scale) at native rates, and the resampler's outputs of those rows at resampled rates (the
integer-ratio FIR model, equal to the oracle's resampler: tests/test_resample_cpu.py)."""
import numpy as np

import replaygain_ref as RG
import resample_tap


def analysed(channels, samplerate, kbps, left, right, schedule):
    """replaygain_ref.analysed for Float32 samples (left / right: any values, rounded to Float32 once)"""
    import oracle_lib
    out_sr = oracle_lib.out_samplerate(channels, samplerate, kbps)
    ratio = samplerate // out_sr
    mode_gr = 2 if out_sr >= 32000 else 1
    left = np.asarray(left, dtype=np.float32)
    right = left if (right is None or channels == 1) else np.asarray(right, dtype=np.float32)
    fifo = RG.Fifo(mode_gr, ratio)
    titles, cur, rows, pos = [], [], [[] for _ in range(channels)], 0
    for step in schedule:
        if step[0] == "enc":
            n = step[1]
            cur += fifo.feed(n)
            for c, x in enumerate((left, right)[:channels]):
                rows[c].append(x[pos:pos + n])
            pos += n
        else:
            if fifo.to_encode < 1:
                continue
            p, z = fifo.flush()
            cur += p
            for c in range(channels):
                rows[c].append(np.zeros(z, dtype=np.float32))
            titles.append(cur)
            cur = []
    if cur:
        titles.append(cur)
    assert pos == len(left)
    if ratio > 1:
        total = sum(sum(t) for t in titles)
        _, h, scale, _ = resample_tap.record(channels, samplerate, kbps, np.zeros(4096, np.int16))
        y = np.stack([resample_tap.fir(np.concatenate(rows[c]).astype(np.float64), h, scale, ratio, total) for c in range(channels)])
        return np.ascontiguousarray(y[:, :total]), out_sr, titles
    scale = RG._scale(channels, samplerate, kbps)
    out = []
    for c in range(channels):
        x = np.concatenate(rows[c]).astype(np.float64) if rows[c] else np.zeros(0)
        xs = x if scale in (0.0, 1.0) else x * scale
        out.append(xs.astype(np.float32))
    return np.ascontiguousarray(np.stack(out)), out_sr, titles


def analyze_calls(channels, samplerate, kbps, left, right, schedule):
    """ReplayGain of the schedule's calls (replaygain_ref.schedule_of format): a replaygain_ref.Result"""
    rows, out_sr, titles = analysed(channels, samplerate, kbps, left, right, schedule)
    return RG.run(rows, out_sr, titles)
