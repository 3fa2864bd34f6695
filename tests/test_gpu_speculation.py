"""The speculation machinery under adversarial guesses (DESIGN.md 5): what the speculated in-states are must change only the
speed, never the bytes.  The library is rebuilt with deliberately bad guesses -- the quantizer's speculative start gain and
step (Q_SPEC_START, Q_SPEC_STEP), the start step handed to gr1 (Q_SPEC_GR1_STEP), the in-state of the block-type / ATH scan
chunks (SCAN_GUESS_LA, SCAN_GUESS_BT, SCAN_GUESS_ATH) -- and with the re-validation folded into the first pass switched off
(Q_SPEC_FOLD=0), so that every wrong guess is repaired by the fixed-point loop.  Each variant encodes ragged MPEG-1 and LSF
batches, live handles fed 5000-sample calls, one MPEG-1 and one LSF handle call schedule (tests/handle_schedule.py) with many
calls of up to 200 frames, and the edge corpus, all byte-equal to the oracle (tests/speculation_worker.py,
one subprocess per library because the library is loaded once per process).  The streams of the ragged batches and the
edge corpus also go through every stage tap, and the schedules compare each handle's state blob after every call: a
repaired frame that kept a state from its speculated start would show there even where the bytes agree."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))

VARIANTS = {
    # the worst guesses: a linear gain search from 0, a gr1 step far off, every scan chunk starting inside a short block
    # with lastAttacks = 3 and the ATH adjustment at its floor
    "worst": ["Q_SPEC_START=0", "Q_SPEC_STEP=1", "Q_SPEC_GR1_STEP=64", "SCAN_GUESS_LA=3", "SCAN_GUESS_BT=BT_SHORT", "SCAN_GUESS_ATH=0.01"],
    # no repair inside the first pass: every speculated frame lands on gain 255 and the fixed-point loop fixes them all
    "nofold": ["Q_SPEC_START=255", "Q_SPEC_STEP=1", "Q_SPEC_FOLD=0"],
    # speculative searches that overshoot both ends of the gain range (the clamps at 0 and 255), chunks starting in a STOP
    # block (an attack in their first granule rewrites it to SHORT)
    "clamp": ["Q_SPEC_START=128", "Q_SPEC_STEP=128", "SCAN_GUESS_LA=1", "SCAN_GUESS_BT=BT_STOP", "SCAN_GUESS_ATH=1e-3"],
}


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("spec_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


def _run(lib):
    env = dict(os.environ, MP3B200_LIB=lib)
    p = subprocess.run([sys.executable, os.path.join(HERE, "speculation_worker.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_bytes_do_not_depend_on_the_guess(variant_libs, name):
    res = _run(variant_libs[name])
    print("%s: quantizer passes %s" % (name, res["passes"]))
    assert not res["fail"], res["fail"][:20]
    if name == "nofold":
        # no folded repair: the first pass cannot be final, so the fixed-point loop ran (pass 3 onwards is the loop)
        assert min(res["passes"].values()) >= 3, res["passes"]
