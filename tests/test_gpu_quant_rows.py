"""The quantizer's rows against the oracle in other launch shapes of its kernels (tests/quant_rows.py through
front_rows.check_rows): whole streams of every native configuration, ragged MPEG-1 and LSF batches and the edge corpus, each
launch on a poisoned workspace, in library builds with other warps per block, blocks per SM, rate-loop task order and
repair-stream width.  The default build's shapes are checked by tests/test_gpu_front_end_rows.py, whose every launch runs
the same check.  And the poison itself: capture off, the bytes are the oracle's; capture on, the rows of granules without
energy hold what quant_rows documents for them."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import front_rows as F
import psy_rows as P
import quant_rows as Q

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))

# k_quant.cuh's knobs: Q_WARPS warps (tasks in flight) per block of the persistent task-pull kernels, Q_BLOCKS_PER_SM /
# Q_SLIM_BLOCKS blocks per SM of the rate-loop / search and finish kernels, Q_REVERSE: k_q_outer pulls the frames of its
# first passes last to first; Q_SPEC_START / Q_SPEC_STEP: the in-state guessed for every frame but a stream's first;
# Q_REPAIR_BLOCKS: blocks of the repair stream's kernels, which redo gr0 of the frames whose guess did not stand while the
# main stream runs gr1's rate loop.  A guessed start of 255 with step 1 is a search that stops at once at gain 255, which no
# granule with energy keeps: every such frame's gr0 goes on the repair list.  Later passes of the fixed point clear `redo`
# of the frames they list again, so the record shows the flag on those only the first pass redid.
VARIANTS = {
    "q_warps1_reverse": ["Q_WARPS=1", "Q_BLOCKS_PER_SM=16", "Q_SLIM_BLOCKS=16", "Q_REVERSE"],
    "q_warps8": ["Q_WARPS=8", "Q_BLOCKS_PER_SM=2", "Q_SLIM_BLOCKS=2"],
    "q_repair_heavy": ["Q_SPEC_START=255", "Q_SPEC_STEP=1", "Q_REPAIR_BLOCKS=1"],
}
SHAPES = ("whole", "batches", "edges")


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    return lamejs_b200


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("quant_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_quantizer_launch_shape_variants(variant_libs, name):
    """every row of every launch of whole streams, ragged batches and the edge corpus; in the repair-heavy build, over a tenth
    of the MPEG-1 frames after each stream's first must end with gr0 redone (redo & Q_R0_ANY), so that rows the two-stream
    repair left are among those checked (12 % on these inputs, against 6 % with a guessed start of 0)"""
    env = dict(os.environ, MP3B200_LIB=variant_libs[name])
    p = subprocess.run([sys.executable, os.path.join(HERE, "front_rows.py")] + list(SHAPES), env=env, capture_output=True,
                       text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert not res["fail"], (res["nfail"], res["fail"][:10])
    assert res["frames"] > 500, res["frames"]
    if name == "q_repair_heavy":
        assert 10 * res["repaired"] > res["frames"], (res["repaired"], res["frames"])


def test_silent_granules_hold_the_documented_rows_and_capture_off_changes_nothing(M):
    """a stream whose left channel falls silent for a stretch and whose right channel is digital silence throughout: under
    capture, every row equals the oracle's (check_rows), and each granule without energy has have 0, mnz 575, xrq and
    xrpow all 0, no line quantised, global_gain 210 and part2_3_length 0; the same stream with capture off gives the same
    bytes"""
    ch, sr, kb = 2, 44100, 128
    n = 30 * 1152 + 77
    l, _ = P.k2_signal("mixed", n, 5)
    r = np.zeros(n, np.int16)
    fail = []
    (rec,) = P.whole_streams(M, ch, sr, kb, [(l, r)], "silent granules", fail, F.check_rows)
    assert not fail, fail[:10]
    (s,) = rec["streams"]
    silent = s["prep"]["have"] == 0
    assert silent[:, 1].all() and silent[:, 0].sum() >= 4, silent.sum(axis=0)
    g = s["ginfo"][silent]
    assert (s["prep"]["mnz"][silent] == 575).all()
    assert not s["xrq"][silent].any() and not s["xrpow"][silent].any() and not s["l3enc"][silent].any()
    assert not s["neg"][silent].any()
    assert (g["global_gain"] == 210).all() and (g["part2_3_length"] == 0).all()
    assert not any(m.any() for m in Q.poisoned_rows(s).values())
    ref = P.make_ref(ch, sr, kb)
    assert M.encode_streams(ch, sr, kb, [l], [r])[0] == ref.stream(l, r)
