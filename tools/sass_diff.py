#!/usr/bin/env python
"""tools/sass_diff.py — compare the machine code of vdl2_kernels.cu in two source trees, kernel by kernel (CPU only).

Each tree's csrc/vdl2_kernels.cu is compiled to an sm_90a cubin with build.NVCC_FLAGS (include paths of that tree) and
-Xptxas -v, disassembled with cuobjdump -sass, and one line per kernel is printed:
  SAME      identical instruction text
  SAME~PAR  identical apart from kernel-parameter offsets, all shifted by one amount: the parameter block changed, the code
            did not
  DIFF      anything else
  ONLY A/B  the kernel exists in one tree only
followed by the instruction counts (NOPs excluded) and the -Xptxas -v registers and stack, spill and shared-memory bytes of
A -> B.  Kernels are matched by demangled name; --sub renames tree A's kernels first.

    python tools/sass_diff.py <tree A> <tree B>      # e.g. a checkout of the parent commit and .
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dumpvdl2_b200 import build  # noqa: E402

CUDA_BIN = os.path.dirname(build._nvcc())


def compile_tree(tree, out):
    """{mangled kernel: (instruction list, resource summary)} of tree's vdl2_kernels.cu"""
    flags, skip = [], False
    for f in build.NVCC_FLAGS:                      # the flags of this build, the include paths of the tree compiled
        if skip or f == "-I":
            skip = f == "-I"
            continue
        flags.append(f)
    csrc = os.path.join(tree, "dumpvdl2_b200", "csrc")
    cubin = os.path.join(out, "k.cubin")
    cmd = [build._nvcc()] + flags + ["-I", csrc, "-I", os.path.join(tree, "include"), "-Xptxas", "-v", "-cubin", "-o", cubin,
                                     os.path.join(csrc, "vdl2_kernels.cu")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    res, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name, res[m.group(1)] = m.group(1), [0, 0, 0, 0]
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            res[name][1], res[name][2] = int(m.group(1)), int(m.group(2)) + int(m.group(3))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            res[name][0] = int(m.group(1))
        m = re.search(r"(\d+) bytes smem", line)
        if m and name:
            res[name][3] = int(m.group(1))
    sass = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    code, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\w+)", line)
        if m:
            cur = code.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur is not None and not m.group(1).startswith("NOP"):
            cur.append(m.group(1))
    return {k: (code[k], "%d regs, %d stack, %d spill, %d smem" % tuple(res.get(k, (0, 0, 0, 0)))) for k in code}


def number(tok):
    """the integer a SASS operand stands for: hex, or an fp16 subnormal (HFMA2 materialising a small integer), else None"""
    if re.fullmatch(r"-?0x[0-9a-f]+", tok):
        return int(tok, 16)
    if re.fullmatch(r"\d+\.\d+e-\d+", tok) and float(tok) * 2 ** 24 == round(float(tok) * 2 ** 24):
        return round(float(tok) * 2 ** 24)
    return None


def shifted(ia, ib):
    """the same code apart from kernel-parameter offsets: every token that differs is a number - a c[0x0][...] offset, or
    an offset the code forms itself for an indexed parameter load (hex, or an HFMA2 fp16 immediate) - and all differ
    by one common amount, the shift of the fields behind a removed or added one"""
    if len(ia) != len(ib):
        return False
    deltas = set()
    for x, y in zip(ia, ib):
        tx, ty = re.split(r"([\s,\[\]]+)", x), re.split(r"([\s,\[\]]+)", y)
        if len(tx) != len(ty):
            return False
        for u, v in zip(tx, ty):
            if u != v:
                nu, nv = number(u), number(v)
                if nu is None or nv is None:
                    return False
                deltas.add(nu - nv)
    return len(deltas) == 1


def demangled(kernels):
    """{demangled name: (instructions, resources)}"""
    names = sorted(kernels)
    out = subprocess.run([os.path.join(CUDA_BIN, "cu++filt")], input="\n".join(names), capture_output=True, text=True).stdout
    return dict(zip(out.split("\n"), (kernels[k] for k in names)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a", help="tree A (e.g. the parent commit)")
    ap.add_argument("b", help="tree B")
    ap.add_argument("--sub", nargs=2, action="append", default=[], metavar=("PATTERN", "REPL"),
                    help="re.sub applied to tree A's demangled kernel names before matching, e.g. for a removed template "
                         "parameter: --sub 'packed<(.*), \\(bool\\)0>' 'packed<\\1>'")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as ta, tempfile.TemporaryDirectory() as tb:
        A, B = demangled(compile_tree(args.a, ta)), demangled(compile_tree(args.b, tb))
    for pat, repl in args.sub:
        A = {re.sub(pat, repl, k): v for k, v in A.items()}

    tally = {}
    for k in sorted(set(A) | set(B)):
        if k not in A or k not in B:
            st, info = ("ONLY A" if k in A else "ONLY B"), "%d ins, %s" % (len((A.get(k) or B[k])[0]), (A.get(k) or B[k])[1])
        else:
            (ia, ra), (ib, rb) = A[k], B[k]
            st = "SAME" if ia == ib else "SAME~PAR" if shifted(ia, ib) else "DIFF"
            info = "%d -> %d ins, %s -> %s" % (len(ia), len(ib), ra, rb)
        tally[st] = tally.get(st, 0) + 1
        print("%-8s %s   %s" % (st, k, info))
    print("kernels: " + ", ".join("%d %s" % (n, s) for s, n in sorted(tally.items())))


if __name__ == "__main__":
    main()
