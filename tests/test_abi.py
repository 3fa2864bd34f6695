"""C-ABI library: builds for sm_90a without a GPU, loads, exports every symbol include/mp3b200.h declares; the
closed-form stream geometry (no compute) matches the oracle; host-side logic fails loudly without a GPU."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    lamejs_b200.lib()
    return lamejs_b200


def test_exports_every_declared_symbol(M):
    hdr = open(os.path.join(ROOT, "include", "mp3b200.h")).read()
    names = set(re.findall(r"\b(mp3b200_[a-z_0-9]+)\s*\(", hdr))
    assert len(names) >= 12
    L = ctypes.CDLL(os.path.join(ROOT, "lamejs_b200", "libmp3b200.so"))
    for n in sorted(names):
        assert hasattr(L, n), n


@pytest.mark.parametrize("n", [0, 1, 1151, 1152, 1375, 1376, 1377, 2304, 44100, 11520000])
def test_stream_geometry_matches_oracle(M, oracle, n):
    F = M.stream_frames(n)
    if n <= 50000:
        x = np.zeros(n, dtype=np.int16)
        data, _, tr = oracle.encode_stream(2, 44100, 128, x, x, trace_frames=F + 4)
        assert len(tr) == F
        assert len(data) == M.stream_bytes(2, 44100, 128, n)
    else:
        assert F == (n - 1376) // 1152 + 1 + 2 or F == (n - 1376) // 1152 + 1 + 1


DEBUG_TAPS_FIELDS = ["size", "channels", "samplerate", "kbps", "left", "right", "nsamples", "force_blocktype", "xr", "blocktype",
                     "en_l", "thm_l", "en_s", "thm_s", "ath_adjust", "l3_enc", "ginfo", "bytes_out", "bytes_cap", "scalefac",
                     "subblock_gain", "xmin", "max_nonzero_coeff", "xrpow_max", "scfsi", "old_value", "cur_step"]


def test_debug_taps_layout(M, tmp_path):
    """mp3b200_debug_taps: the Python binding's ctypes struct has the C header's field order, offsets and size, and both are
    pinned (16 bytes of int32 header, then 8-byte pointers / int64; 200 bytes on LP64)."""
    from lamejs_b200.encoder import DebugTaps

    assert [f[0] for f in DebugTaps._fields_] == DEBUG_TAPS_FIELDS
    want = {n: 4 * i for i, n in enumerate(DEBUG_TAPS_FIELDS[:4])}
    want.update({n: 16 + 8 * i for i, n in enumerate(DEBUG_TAPS_FIELDS[4:])})
    assert {n: getattr(DebugTaps, n).offset for n in DEBUG_TAPS_FIELDS} == want
    assert ctypes.sizeof(DebugTaps) == 200
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mp3b200.h"\nint main(void) {\n' +
                   "".join('  printf("%%s %%zu\\n", "%s", offsetof(mp3b200_debug_taps, %s));\n' % (n, n) for n in DEBUG_TAPS_FIELDS) +
                   '  printf("sizeof %zu\\n", sizeof(mp3b200_debug_taps));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert {n: int(got[n]) for n in DEBUG_TAPS_FIELDS} == want and int(got["sizeof"]) == 200


def test_debug_taps_size_is_checked(M):
    """A struct of another size is refused before any device work (no GPU needed)."""
    from lamejs_b200.encoder import DebugTaps

    t = DebugTaps(size=ctypes.sizeof(DebugTaps) - 8)
    assert M.lib().mp3b200_debug_stages_ex(ctypes.byref(t)) == -3


def test_config_errors(M):
    assert M.stream_bytes(2, 44100, 64, 1000) == -1       # lamejs would resample to 32 kHz: not built
    assert M.stream_bytes(2, 22050, 64, 1000) == 835      # MPEG-2: 4 frames of 208/209 bytes
    assert M.stream_bytes(2, 48000, 64, 1000) == -1       # lamejs would resample to 24 kHz
    assert M.stream_bytes(3, 44100, 128, 1000) == -1
    assert M.stream_bytes(2, 44100, 123, 44100) == M.stream_bytes(2, 44100, 128, 44100)   # FindNearestBitrate


def test_no_cpu_fallback(M):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(M.Mp3B200Error):
        M.Mp3Encoder(2, 44100, 128)
    with pytest.raises(M.Mp3B200Error):
        M.encode_streams(1, 44100, 128, [np.zeros(5000, dtype=np.int16)])


def test_product_does_not_reference_oracle():
    """The shipped path must not import, link or execute anything under oracle/."""
    for d, _, files in os.walk(os.path.join(ROOT, "lamejs_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".inc")):
                s = open(os.path.join(d, f)).read()
                assert "oracle_lib" not in s and "liblamejs_oracle" not in s and "oracle/" not in s.replace("the oracle/", ""), f


def test_config_matrix_acceptance_and_sizes_match_oracle(M, oracle):
    """Host logic only: for every sample rate x bitrate x mono/stereo the library accepts exactly the configurations
    lamejs encodes at the input rate (MPEG-1, MPEG-2 and MPEG-2.5), and predicts the oracle's byte count -- including
    the flush quirk that a 1152-sample zero bunch can complete two 576-sample frames (Lame.js:1416-1443)."""
    from synth import make_signal
    for sr in (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000):
        l, r = make_signal("noise", 2000, sr, 1)
        for kbps in (8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 123, 128, 144, 160, 192, 224, 256, 320):
            for ch in (1, 2):
                # the product takes the configurations lamejs encodes at the input rate; where lamejs would resample
                # (oracle.out_samplerate != sr) it answers -1 (documented deviation, include/mp3b200.h)
                want = len(oracle.encode_stream(ch, sr, kbps, l, r if ch == 2 else None)[0]) if oracle.out_samplerate(ch, sr, kbps) == sr else -1
                assert M.stream_bytes(ch, sr, kbps, len(l)) == want, (ch, sr, kbps)
