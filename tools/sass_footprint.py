#!/usr/bin/env python3
"""Instruction footprint of the encoder's kernels on sm_90a, read from the SASS (no GPU needed).

  python tools/sass_footprint.py                      build a cubin of mp3_encoder.cu with the production flags, report it
  python tools/sass_footprint.py --lib LIB.so         report the sm_90a cubin inside a built library (e.g. a tuning variant)
  python tools/sass_footprint.py -D Q_CN_UNROLL=1     build with extra -D knobs (tools/build_variants.py spells them the same)
  python tools/sass_footprint.py --lines 20           also the 20 source lines with the most code in k_q_outer's own body

Prints the .text bytes of every kernel, then for k_q_outer each subroutine (every __noinline__ helper is its own CALL
target, laid out as one address range inside the kernel's section) with its offset and size, and the rate loop's hot set:
the subroutines that run on every iteration of outer_loop_w, their total and the address span they are spread over.  A
helper that is inlined has no range of its own: its bytes count in the kernel body (--lines attributes them to source)."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lamejs_b200 import build as B  # noqa: E402

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
KERNEL = "k_q_outer"
# the noise-shaping loop of outer_loop_w (k_quant.cuh): what a warp of k_q_outer runs on every iteration.  LSF streams run
# scale_bitcount_lsf_w in place of scale_bitcount_w.
HOT = ["outer_loop_w", "balance_noise_w", "scale_xrpow_w", "scale_bitcount_w", "count_bits_w<true>", "noquant_count_bits_w",
       "region_table_w", "calc_noise_w", "q_log10", "copy_gi_w", "copy_ix_w"]


def build_cubin(defines, out_dir):
    out = os.path.join(out_dir, "mp3_encoder.cubin")
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    cmd = [os.path.join(CUDA, "bin", "nvcc"), "-cubin"] + flags + ["-D" + d for d in defines] + ["-o", out, "mp3_encoder.cu"]
    subprocess.check_call(cmd, cwd=B.CSRC)
    return out


def cubin_of_lib(lib, out_dir):
    subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(lib)], cwd=out_dir, check=True,
                   stdout=subprocess.DEVNULL)
    cubin = os.path.join(out_dir, "mp3_encoder.sm_90a.cubin")
    assert os.path.exists(cubin), "no sm_90a cubin of mp3_encoder.cu in %s" % lib
    return cubin


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return {n: (d.split("(")[0] if d else n) for n, d in zip(names, out)}


INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+\S")
SECTION = re.compile(r"^\s*\.section\s+\.text\.(\S+?),")
SUB = re.compile(r"^\$([^$]+)\$(\S+):\s*$")
LINE = re.compile(r'//## File "([^"]+)", line (\d+)')


def parse(cubin):
    """{kernel: {"size": bytes, "funcs": [(name, offset, bytes)], "lines": Counter((file, line) -> bytes of the kernel body)}}"""
    text = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "--print-line-info", cubin], capture_output=True, text=True,
                          check=True).stdout
    kernels, cur, fn, src = {}, None, None, None
    for line in text.splitlines():
        m = SECTION.match(line)
        if m:
            cur = {"size": 0, "funcs": [], "lines": collections.Counter()}
            kernels[m.group(1)] = cur
            fn, src = None, None
            continue
        if cur is None:
            continue
        m = SUB.match(line)
        if m:
            fn = [m.group(2), None, 0]
            cur["funcs"].append(fn)
            continue
        m = LINE.search(line)
        if m:
            src = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = INSN.match(line)
        if m:
            cur["size"] += 16
            if fn is None:
                cur["lines"][src] += 16
            else:
                if fn[1] is None:
                    fn[1] = int(m.group(1), 16)
                fn[2] += 16
    return kernels


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", help="built libmp3b200*.so to read instead of building a cubin")
    ap.add_argument("-D", dest="defines", action="append", default=[], help="extra -D knob for the cubin build")
    ap.add_argument("--lines", type=int, default=0, help="show the N source lines with the most code in k_q_outer's own body")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        cubin = cubin_of_lib(args.lib, d) if args.lib else build_cubin(args.defines, d)
        kernels = parse(cubin)
    names = demangle(list(kernels) + [f[0] for k in kernels.values() for f in k["funcs"]])

    print("kernel .text bytes (sm_90a)")
    for k, v in sorted(kernels.items(), key=lambda kv: -kv[1]["size"]):
        if v["size"] >= 1024:
            print("  %7d  %s" % (v["size"], names[k]))
    outer = [k for k in kernels if names[k] == KERNEL]
    assert len(outer) == 1, "no single %s kernel in the cubin" % KERNEL
    K = kernels[outer[0]]
    body = K["size"] - sum(f[2] for f in K["funcs"])
    print("\n%s: %d bytes" % (KERNEL, K["size"]))
    print("  %7s  %7s  %s" % ("offset", "bytes", "function"))
    print("  %7x  %7d  %s" % (0, body, "(kernel body, with the helpers inlined into it)"))
    hot, span = 0, []
    for name, off, size in K["funcs"]:
        dn = names[name]
        is_hot = dn.replace("int ", "") in HOT
        if is_hot:
            hot += size
            span += [off, off + size]
        print("  %7x  %7d  %s%s" % (off, size, dn, "  [hot]" if is_hot else ""))
    missing = [h for h in HOT if h not in [names[f[0]].replace("int ", "") for f in K["funcs"]]]
    print("hot set: %d bytes in %d subroutines over a span of %d bytes%s" % (
        hot, len(HOT) - len(missing), (max(span) - min(span)) if span else 0,
        ("; inlined (not separate): " + ", ".join(missing)) if missing else ""))
    if args.lines:
        print("\n%s body: bytes per source line" % KERNEL)
        srcs = {}
        for (f, ln), v in K["lines"].most_common(args.lines):
            if f and f not in srcs and os.path.exists(os.path.join(B.CSRC, f)):
                srcs[f] = open(os.path.join(B.CSRC, f)).read().split("\n")
            txt = srcs[f][ln - 1].strip()[:90] if f in srcs else ""
            print("  %6d  %s:%d  %s" % (v, f, ln, txt))


if __name__ == "__main__":
    main()
