"""Build libmp3b200.so in-tree for sm_90a (H100; nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmp3b200.so")
STAMP = LIB + ".flags"          # the flags LIB was built with: a library built with other flags is rebuilt
SOURCES = ["mp3_encoder.cu", "mp3_config.cpp", "mp3_tag.cpp", "mp3_id3.cpp"]
DEPS = SOURCES + ["mp3_config.h", "mp3_device.cuh", "mp3_math.cuh", "mp3_tables.h", "k_filterbank.cuh", "k_psy.cuh",
                  "k_quant.cuh", "k_tag.cuh", "k_resample.cuh", "k_replaygain.cuh", "k_stage.cuh", "mp3_tag.h", "mp3_handle.inc", "mp3_session.inc", "../../include/mp3b200.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # bit-exactness contract: no FMA contraction, IEEE div/sqrt, no flush-to-zero (DESIGN.md "numerics")
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math", "-diag-suppress", "222", "-shared",
]


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(STAMP) or open(STAMP).read() != " ".join(NVCC_FLAGS):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force=False, verbose=False, variant=None, defines=(), out_dir=None):
    """variant/defines: tuning or test builds (libmp3b200_<variant>.so with -D flags, in out_dir or next to the default
    library), selected at run time by MP3B200_LIB."""
    out = LIB if variant is None else os.path.join(out_dir or HERE, "libmp3b200_%s.so" % variant)
    if variant is None and not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    if variant is None:
        with open(STAMP, "w") as f:
            f.write(" ".join(NVCC_FLAGS))
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
