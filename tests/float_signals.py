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


# Loud input (tests/golden/make_lamejs_loud_golden.py): a unit-peak signal times magnitude x 32768, where the magnitude
# is a number or "max", the largest Float32 that stays finite once scaled by the configuration's `scale`.
LOUD_KINDS = ("burst", "noise", "nyquist", "impulse", "dcstep")
LOUD_MAGNITUDES = (16, 256, 4096, 65536, 2 ** 18, 2 ** 20, 2 ** 22, 2 ** 24, 3.3e7, 1e9, 1e15, 1e20, 1e30, "max")
# across the magnitude at which lamejs's frames stop fitting their slots (between 2e5 and 1e6 x full scale)
LOUD_FINE = (3e5, 4e5, 5e5, 6e5, 7e5, 8e5)
# the library's input limit (MP3_F32_MAX_SAMPLE, k_resample.cuh): it refuses samples beyond it once scaled
LOUD_GATE = 2.0 ** 40


def _unit(kind, n, sr, seed):
    """(left, right) float64 in [-1, 1]"""
    if kind in ("burst", "noise"):
        l, r = make_signal(kind, n, sr, seed=seed)
        return l / 32768.0, r / 32768.0
    t = np.arange(n)
    if kind == "nyquist":
        w = 2 * np.pi * 0.49 * t
        return np.sin(w), np.cos(w * 0.995)
    l, r = np.zeros(n), np.zeros(n)
    if kind == "impulse":
        l[n // 3] = 1.0
        r[n // 2] = -1.0
    elif kind == "dcstep":
        l[n // 3:] = 1.0
        r[n // 2:] = -1.0
    else:
        raise ValueError(kind)
    return l, r


def max_finite(scale):
    """the largest Float32 v with Float32(v * scale) finite (lamejs's scale of a Float32Array, k_stage_f32)"""
    top = np.float32(np.finfo(np.float32).max)
    v = np.float32(min(float(top), float(top) / scale))

    def ok(x):
        with np.errstate(over="ignore"):
            return np.isfinite(np.float32(float(x) * scale))
    while not ok(v):
        v = np.nextafter(v, np.float32(0))
    while v < top and ok(np.nextafter(v, top)):
        v = np.nextafter(v, top)
    return float(v)


def loud(kind, magnitude, n, sr, seed, scale):
    """(left, right): float64 holding Float32 values"""
    l, r = _unit(kind, n, sr, seed)
    if magnitude == "max":
        vmax = max_finite(scale)
        a = vmax / max(np.abs(l).max(), np.abs(r).max())
        x = np.clip(np.stack([l, r]) * a, -vmax, vmax)
    else:
        x = np.stack([l, r]) * (float(magnitude) * 32768.0)
    with np.errstate(over="ignore"):
        x = x.astype(np.float32).astype(np.float64)
    assert np.isfinite(x).all()
    return x[0].copy(), x[1].copy()


def loud_case_signal(c):
    """case_signal for a loud fixture case (its "scale" is the configuration's)"""
    l, r = loud(c["kind"], c["magnitude"], c["samples"], c["samplerate"], c["seed"], c["scale"])
    calls, pos = [], 0
    for step in c["schedule"]:
        if step[0] < 0:
            calls.append(None)
            continue
        k = step[0]
        calls.append((l[pos:pos + k].astype(np.float32), r[pos:pos + k].astype(np.float32) if c["channels"] == 2 else None))
        pos += k
    return l, (r if c["channels"] == 2 else None), calls


def loud_peak(c):
    """the largest sample of a loud fixture case once lamejs has scaled it (what the library's input limit compares)"""
    l, r = loud(c["kind"], c["magnitude"], c["samples"], c["samplerate"], c["seed"], c["scale"])
    return max(np.abs(l).max(), np.abs(r).max() if c["channels"] == 2 else 0.0) * c["scale"]


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
