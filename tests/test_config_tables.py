"""The product's per-configuration constant block (lamejs_b200/csrc/mp3_config.cpp -> Mp3Tables, what every kernel reads)
against the oracle's lame_init_params / psymodel_init / iteration_init restatement, for every sample rate x bitrate x
channel count: scalefactor bands, psy partitions, spreading rows, ATH, filter gains, windows, masking adjustment -- bit for bit,
on CPU.  The product's tables are built with MP3B200_RESAMPLE, so the 29 configurations lamejs resamples by an integer ratio
are compared with the oracle's output-rate tables too (their filter taps are pinned by tests/test_resample_cpu.py).
(The oracle's tables are pinned to real lamejs through the byte fixtures of test_lamejs_pin.py.)"""
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_product_tables_equal_oracle_tables():
    exe = os.path.join(tempfile.mkdtemp(), "config_check")
    src = [os.path.join(ROOT, "tools", "cfgcheck", "config_check.cpp"), os.path.join(ROOT, "lamejs_b200", "csrc", "mp3_config.cpp")]
    src += [os.path.join(ROOT, "oracle", f) for f in ("lj_init.cpp", "lj_mdct.cpp", "lj_psy.cpp", "lj_quant.cpp", "lj_bitstream.cpp", "lj_vbrtag.cpp")]
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-o", exe] + src + ["-lm"])
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    assert "342 configurations, 0 with mismatches" in p.stdout
    assert "29 resampled configurations compared" in p.stdout, p.stdout[-3000:]
