"""Float input signals and call schedules shared by tests/golden/make_lamejs_float_golden.py and the tests that replay its
fixtures: deterministic from (kind, samples, rate, seed), so the fixtures store only those and hashes."""
import numpy as np

from synth import make_signal

KINDS = ("webaudio", "unit", "x1.5", "x4", "dither", "denormal", "array", "mixed")


def make(kind, n, sr, seed):
    """(left, right) float64 arrays.  Every kind but "array" holds Float32 values; "array" holds doubles that are not (a
    plain JS Array of numbers, which lamejs rounds to Float32 at its store); "mixed" is Web Audio scale, and the samples of
    its Int16 calls (see schedule) are integers."""
    base = "noise" if kind in ("dither", "denormal") else "burst"
    l, r = make_signal(base, n, sr, seed=seed)
    u = np.stack([l, r]).astype(np.float64) / 32768.0
    rng = np.random.default_rng(seed)
    if kind in ("webaudio", "mixed"):
        x = u * 32767.0
    elif kind == "unit":
        x = u
    elif kind == "x1.5":
        x = u * 32768.0 * 1.5
    elif kind == "x4":
        x = u * 32768.0 * 4.0
    elif kind == "dither":
        x = rng.uniform(-0.5, 0.5, size=u.shape)
    elif kind == "denormal":
        x = rng.integers(-3, 4, size=u.shape) * np.float64(np.float32(1e-45))
        x[:, ::7] = -0.0
        x[:, 5::11] = np.float64(np.float32(1.1754942e-38))
    elif kind == "array":
        return (u * 32767.0 + rng.uniform(-1e-3, 1e-3, size=u.shape))[0].copy(), (u * 32767.0)[1].copy()
    else:
        raise ValueError(kind)
    x = x.astype(np.float32).astype(np.float64)
    return x[0].copy(), x[1].copy()


def schedule(kind, n, ragged, seed):
    """encodeBuffer calls [size, type] (type "f": Float32Array, "i": Int16Array, "a": plain Array) and [-1] for flush()"""
    typ = "a" if kind == "array" else "f"
    if not ragged:
        sizes = [n]
    else:
        rng = np.random.default_rng(seed)
        sizes, i = [], 0
        while i < n:
            k = int(min(n - i, rng.choice([1, 7, 333, 576, 1151, 1152, 1153, 2000, 4099])))
            sizes.append(k)
            i += k
    out = []
    for j, k in enumerate(sizes):
        out.append([k, ("i" if j % 2 else "f") if kind == "mixed" else typ])
    return out + [[-1]]


def integer_calls(l, r, sched):
    """rounds the samples of the Int16 calls to integers in place (Int16Array values); returns l, r"""
    pos = 0
    for step in sched:
        if step[0] < 0:
            continue
        k, t = step
        if t == "i":
            for x in (l, r):
                x[pos:pos + k] = np.clip(np.round(x[pos:pos + k]), -32768, 32767)
        pos += k
    return l, r


def case_signal(c):
    """(left, right or None, calls): the fixture case's input and its encodeBuffer calls as arrays (int16 for "i", float32
    for "f", float64 for "a"), None for flush()"""
    l, r = make(c["kind"], c["samples"], c["samplerate"], c["seed"])
    l, r = integer_calls(l, r, c["schedule"])
    calls, pos = [], 0
    for step in c["schedule"]:
        if step[0] < 0:
            calls.append(None)
            continue
        k, t = step
        dt = {"i": np.int16, "f": np.float32, "a": np.float64}[t]
        a, b = l[pos:pos + k].astype(dt), r[pos:pos + k].astype(dt)
        calls.append((a, b if c["channels"] == 2 else None))
        pos += k
    return l, (r if c["channels"] == 2 else None), calls
