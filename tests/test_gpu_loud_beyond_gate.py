"""Loud Float32 input beyond the library's input limit (MP3_F32_MAX_SAMPLE, k_resample.cuh) against lamejs and the oracle.

The library is rebuilt with the limit lifted to the largest finite Float32 (non-finite samples stay refused), and every
loud fixture (tests/golden/lamejs_loud_golden.json) that the default build refuses, at the rungs where the oracle's
intermediates are still finite (below 1e15 x full scale), goes through tests/loud_beyond_gate_worker.py in a subprocess:
the handle with the fixture's call schedule (lamejs's per-call sizes and bytes, its throw as a "bit budget" refusal that
leaves the state blob unchanged), host, device and tagged whole streams where lamejs encoded the stream whole, every stage
tap against the oracle's traces (of the whole stream, or of the longest whole-frame prefix the oracle encodes without
throwing), and for the ReplayGain fixtures the window sums and title gain of tests/replaygain_ref_f32.py.  A failure names
the first differing tap and its (frame, granule, channel, index).

The domain-check build (-DMP3_DOMAIN_CHECK) counts every argument of a device helper or a narrowing store that falls
outside the domain it is exact on (mp3b200_debug_domain_hits); the Int16 lamejs fixtures, the edge corpus and every loud
fixture up to the default limit must leave every counter at zero."""
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import float_signals as FS  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
from test_gpu_loud_float import GATE  # noqa: E402
from lamejs_b200 import DOMAIN_SITES  # noqa: E402

LIFTED = ["MP3_F32_MAX_SAMPLE=3.40282347e38f"]      # FLT_MAX: only non-finite samples are refused
FINITE = 1e15                                       # from here lamejs's masking energies overflow (test_loud_float_cpu.py)


def finite_rung(c):
    return c["magnitude"] != "max" and c["magnitude"] < FINITE


# the rungs where the rate loop works at global_gain 255 and granules reach their bit budget, up to the last rung whose
# intermediates are finite: the input limit lies among them
LOUDEST = sorted(n for n, c in GOLDEN.items() if finite_rung(c) and c["magnitude"] >= 2 ** 20)
WITHIN = sorted(n for n, c in GOLDEN.items() if FS.loud_peak(c) <= GATE)
BEYOND = sorted(n for n, c in GOLDEN.items() if FS.loud_peak(c) > GATE)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("loud_variants"))
    return {"lifted": build.build(variant="lifted", defines=LIFTED, out_dir=d),
            "domain": build.build(variant="domain", defines=LIFTED + ["MP3_DOMAIN_CHECK"], out_dir=d)}


def _run(lib, mode, names):
    env = dict(os.environ, MP3B200_LIB=lib)
    p = subprocess.run([sys.executable, os.path.join(HERE, "loud_beyond_gate_worker.py"), mode] + names, env=env,
                       capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0, p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_the_fixtures_reach_the_gate_and_beyond():
    rungs = {GOLDEN[n]["magnitude"] for n in LOUDEST}
    assert len(LOUDEST) >= 100 and len(rungs) >= 5, rungs
    assert any(GOLDEN[n]["thrown"] is None for n in LOUDEST) and any(GOLDEN[n]["thrown"] is not None for n in LOUDEST)
    assert any(GOLDEN[n]["rg"] for n in LOUDEST)
    # the gate lies among them: compared on both sides of it
    assert any(FS.loud_peak(GOLDEN[n]) <= GATE for n in LOUDEST) and any(FS.loud_peak(GOLDEN[n]) > GATE for n in LOUDEST)
    assert BEYOND


def test_loudest_rungs_match_lamejs_tap_by_tap(libs):
    res = _run(libs["lifted"], "compare", LOUDEST)
    assert not res["fail"], res["fail"][:20]


def test_domain_counters_stay_zero_within_the_gate(libs):
    """every site in its domain for the Int16 fixtures, the edge corpus and the loud fixtures the default build encodes;
    the louder rungs' counts are printed (DESIGN.md 12 names the sites that leave their domain there)"""
    within = _run(libs["domain"], "domain", WITHIN)["hits"]
    beyond = _run(libs["domain"], "domain-loud", BEYOND)["hits"]
    for group, hits in beyond.items():
        print("beyond the gate:", group, dict(zip(DOMAIN_SITES, hits)))
    for group, hits in within.items():
        print(group, dict(zip(DOMAIN_SITES, hits)))
        assert not any(hits), (group, dict(zip(DOMAIN_SITES, hits)))
