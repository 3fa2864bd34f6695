"""The ReplayGain speculation under hostile knobs (k_replaygain.cuh): one-window chunks, a deliberately wrong guess for every
chunk's start state and no repair pass queued ahead, so that every chunk is repaired by the repair loop's graph.  The knobs
change the speed only: each variant must give the restatement's window bits, gains, tags and album gain on whole streams and
on live handles under a random call schedule (tests/replaygain_worker.py, one subprocess per library)."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))

VARIANTS = {
    "one_window_garbage": ["RG_CHUNK_WINDOWS=1", "RG_GUESS=1", "RG_QUEUED_PASSES=0"],
    "long_chunks_garbage": ["RG_CHUNK_WINDOWS=64", "RG_GUESS=1", "RG_QUEUED_PASSES=1"],
}


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    from lamejs_b200 import build

    d = str(tmp_path_factory.mktemp("rg_variants"))
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(build.build, variant=name, defines=defs, out_dir=d) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_results_do_not_depend_on_the_knobs(variant_libs, name):
    env = dict(os.environ, MP3B200_LIB=variant_libs[name])
    p = subprocess.run([sys.executable, os.path.join(HERE, "replaygain_worker.py")], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert not res["fail"], res["fail"][:20]
