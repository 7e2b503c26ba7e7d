#!/usr/bin/env python
"""sass_census.py -- static instruction counts per issue pipe of named kernels in a built library.  Needs no GPU.

    python tools/sass_census.py [--lib stitching_b200/libstitch_b200.so] [--ptxas-log stitching_b200/csrc/build/X.ptxas.log]
                                [--pixels-per-thread N] 'k_collapse_tile<0,false>' 'k_collapse_tile<1,false>'

Runs `cuobjdump -sass` and `cuobjdump -res-usage` on the library and prints, per kernel, the number of SASS
instructions grouped by the pipe that issues them on sm_90 (ALU: integer / logic / lane arithmetic, issued at half the
FP32 rate; FMA: IMAD, FFMA, FMUL, FADD, IDP; conversion / MUFU; shared memory; global memory; barriers; control), plus
registers, stack and static shared memory, and the spill lines of a ptxas log when one is given.  The counts are
STATIC: instructions in the binary, not instructions executed (a loop body counts once, both sides of a branch count).
With --pixels-per-thread the counts are also printed divided by the pixels one thread produces, which is what makes
two tile shapes comparable.  A kernel is named as in the source; `true` / `false` may be written for bool arguments.
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PIPES = [  # first match wins; an opcode is matched without its .suffixes
    ("alu", r"LOP3|LOP|PRMT|SHF|SHL|SHR|IADD3|IADD|VIADD\w*|VIADDMNMX|VIMNMX\w*|VABSDIFF\w*|IMNMX|ISETP|FSETP|PLOP3|SEL|FSEL|"
            r"LEA|MOV|FMNMX|IABS|POPC|FLO|BREV|SGXT|BMSK|CS2R|R2P|P2R|FCHK|LEA_HI"),
    ("fma", r"IMAD|FFMA|FMUL|FADD|IDP\w*|HFMA2\w*|HADD2\w*|HMUL2\w*"),
    ("cvt_mufu", r"I2F\w*|F2I\w*|F2F\w*|I2I\w*|I2FP|F2FP|FRND|MUFU"),
    ("shared", r"LDS\w*|STS\w*|LDSM"),
    ("global", r"LDG|LDGSTS|STG|LD|ST|LDL|STL|ATOMG|RED|LDGDEPBAR|DEPBAR"),
    ("const_uniform", r"LDC|ULDC|S2R|S2UR|R2UR|UMOV|ULOP3|UIADD3|UIMAD|USHF|ULEA|UISETP|USEL|UPRMT|UFLO|UPOPC|VOTEU|VOTE|SHFL|"
                      r"UP2UR|UR2UP|UPLOP3|UVIADD|UVIMNMX|USGXT|UBMSK|REDUX"),
    ("barrier", r"BAR|ACQBULK|PREEXIT|ERRBAR|MEMBAR|CCTL|WARPSYNC"),
    ("control", r"BRA|BRX|JMP|EXIT|RET|CALL|BSSY|BSYNC|BREAK|ENDCOLLECTIVE|NOP|YIELD|NANOSLEEP|KILL|BPT"),
]
PIPES = [(name, re.compile(r"^(?:%s)$" % pat)) for name, pat in PIPES]
INSN = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)")


def tool(name):
    p = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    if not os.path.exists(p):
        sys.exit(f"sass_census: {name} not found (CUDA toolkit on PATH or CUDA_HOME)")
    return p


def normal(name):
    """`k<0, false>` and the demangler's `void sb::<unnamed>::k<(int)0, (bool)0>(sb::CollapseArgs)` in one spelling."""
    name = re.sub(r"\((?:int|bool|unsigned int)\)", "", name.replace(" ", ""))
    name = name.replace("false", "0").replace("true", "1")
    name = re.sub(r"\(.*\)$", "", name)  # the parameter list
    return name.split("::")[-1].removeprefix("void")


def demangle(names):
    out = subprocess.run([tool("cu++filt")] + names, capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, out))


def pipe_of(op):
    for name, rx in PIPES:
        if rx.match(op):
            return name
    return "other"


def census(lib):
    """{mangled name: (Counter per pipe, Counter per opcode)} of every kernel in the library"""
    sass = subprocess.run([tool("cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    kernels, cur = {}, None
    for line in sass.split("\n"):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = kernels[m.group(1)] = (Counter(), Counter())
            continue
        m = INSN.match(line)
        if m and cur is not None:
            cur[0][pipe_of(m.group(1))] += 1
            cur[1][m.group(1)] += 1
    return kernels


def resources(lib):
    text = subprocess.run([tool("cuobjdump"), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in text.split("\n"):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            res[cur] = dict(kv.split(":") for kv in line.split() if ":" in kv)
            cur = None
    return res


def spills(log):
    """{mangled name: 'N bytes stack frame, ... spill stores, ... spill loads'} from a `-Xptxas -v` log"""
    out, cur = {}, None
    for line in open(log):
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
        elif cur and "spill" in line:
            out[cur] = line.strip()
            cur = None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("kernels", nargs="+", help="kernel names as in the source, e.g. 'k_collapse_tile<0,false>'")
    ap.add_argument("--lib", default=os.path.join(ROOT, "stitching_b200", "libstitch_b200.so"))
    ap.add_argument("--ptxas-log", help="a `nvcc -Xptxas -v` log of the file that defines the kernels (spill lines)")
    ap.add_argument("--pixels-per-thread", type=float, help="also print the counts divided by this")
    ap.add_argument("--opcodes", action="store_true", help="also print the count of every opcode")
    args = ap.parse_args()

    kernels, res = census(args.lib), resources(args.lib)
    spill = spills(args.ptxas_log) if args.ptxas_log else {}
    by_name = {normal(d): m for m, d in demangle(list(kernels)).items()}
    cols = [name for name, _ in PIPES] + ["other"]
    print(f"{args.lib}: STATIC instruction counts (instructions in the binary, not instructions executed)")
    failed = False
    for want in args.kernels:
        m = by_name.get(normal(want))
        if m is None:
            print(f"{want}: not in the library", file=sys.stderr)
            failed = True
            continue
        pipes, ops = kernels[m]
        total = sum(pipes.values())
        r = res.get(m, {})
        print(f"\n{want}: {total} instructions; registers {r.get('REG', '?')}, stack {r.get('STACK', '?')} B, static shared "
              f"{r.get('SHARED', '?')} B, local {r.get('LOCAL', '?')} B" + (f"; ptxas: {spill[m]}" if m in spill else ""))
        print("  " + "  ".join(f"{c:>13}" for c in cols))
        print("  " + "  ".join(f"{pipes.get(c, 0):>13}" for c in cols))
        if args.pixels_per_thread:
            print("  " + "  ".join(f"{pipes.get(c, 0) / args.pixels_per_thread:>13.2f}" for c in cols) +
                  f"   per pixel ({args.pixels_per_thread:g} pixels per thread)")
            print(f"  BAR {ops.get('BAR', 0)} ({ops.get('BAR', 0) / args.pixels_per_thread:.2f} per pixel), total "
                  f"{total / args.pixels_per_thread:.1f} per pixel")
        if args.opcodes:
            print("  " + ", ".join(f"{op} {n}" for op, n in sorted(ops.items(), key=lambda kv: -kv[1])))
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
