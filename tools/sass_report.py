#!/usr/bin/env python3
"""What the compiler made of each kernel in ht2_gpu.cu, on the CPU (no GPU needed).

  python tools/sass_report.py [--filter SUBSTR] [--lines KERNEL] [--top 25]

Compiles hisat2_b200/csrc/ht2_gpu.cu for sm_90a with the library's flags plus `-Xptxas -v -lineinfo` into a
temporary directory, then prints per kernel: SASS code bytes, instruction count, local (LDL / STL) and generic
(LD / ST) memory instructions, registers, stack frame and spill bytes (from ptxas).  A kernel's SASS includes the
non-inlined device functions it calls.  With --lines KERNEL (a substring of the demangled name, e.g.
"ht2_sam_kernel<true>") it also lists the source lines with the most SASS instructions and with the most
local-memory instructions, attributed by `nvdisasm --print-line-info` to the innermost source line (the line
an inlined helper's instruction comes from, not its call site).
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def cuda_tool(name):
    home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    p = os.path.join(home, "bin", name)
    return p if os.path.exists(p) else name


def compile_cubin(tmp):
    from hisat2_b200 import build as b
    cubin = os.path.join(tmp, "ht2_gpu.cubin")
    flags = [f for f in b.NVCC_FLAGS if f not in ("-shared", "-cudart", "static")]
    flags = [f for i, f in enumerate(flags) if not (f == "-Xcompiler" or (i > 0 and flags[i - 1] == "-Xcompiler"))]
    cmd = [cuda_tool("nvcc")] + flags + ["-Xptxas", "-v", "-cubin", "-o", cubin, "ht2_gpu.cu"]
    r = subprocess.run(cmd, cwd=b.CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise SystemExit("nvcc failed")
    return cubin, r.stdout


def demangle(names):
    """mangled -> short name without the parameter list, e.g. ht2_sam_kernel<true>"""
    if not names:
        return {}
    r = subprocess.run([cuda_tool("cu++filt")], input="\n".join(names), stdout=subprocess.PIPE, universal_newlines=True, check=True)
    out = {}
    for m, d in zip(names, r.stdout.splitlines()):
        d = d.replace("(bool)1", "true").replace("(bool)0", "false").replace("(int)", "")
        d = re.sub(r"^void ", "", d)
        out[m] = d.split("(")[0] if "(" in d else d
    return out


def ptxas_info(log):
    """mangled entry -> {regs, stack, spill_st, spill_ld}"""
    info = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = info.setdefault(m.group(1), {})
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            cur.update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
            continue
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = info.setdefault(m.group(1), {})
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur is not None:
            cur["regs"] = int(m.group(1))
    return info


INSN = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[0-7T]\s+)?([A-Z][A-Z0-9_]*)(\.[A-Z0-9_.]+)?")


def sass_functions(cubin):
    """mangled kernel -> list of (opcode, file, line) in order, from nvdisasm with line info"""
    out = subprocess.run([cuda_tool("nvdisasm"), "--print-line-info", cubin], stdout=subprocess.PIPE,
                         universal_newlines=True, check=True).stdout
    funcs = collections.OrderedDict()
    cur = None
    loc = (None, 0)
    for line in out.splitlines():
        m = re.match(r"\s*\.text\.(\S+):\s*$", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            loc = (None, 0)
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', line)
        if m:
            loc = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        if cur is None:
            continue
        m = INSN.search(line)
        if m:
            cur.append((m.group(1), loc[0], loc[1]))
    return funcs


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--filter", default="", help="only kernels whose demangled name contains this")
    ap.add_argument("--lines", metavar="KERNEL", help="per-source-line SASS of the kernel whose demangled name contains this")
    ap.add_argument("--top", type=int, default=25)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="ht2_sass_") as tmp:
        cubin, log = compile_cubin(tmp)
        funcs = sass_functions(cubin)
    pinfo = ptxas_info(log)
    names = demangle(list(funcs) + [m for m in pinfo if m not in funcs])
    print("%-48s %9s %7s %6s %6s %6s %6s %5s %6s %9s" % ("kernel", "code B", "insns", "LDL", "STL", "LD", "ST", "regs", "stack", "spill B"))
    for mangled, insns in funcs.items():
        name = names.get(mangled, mangled)
        if args.filter not in name:
            continue
        cnt = collections.Counter(op for op, _, _ in insns)
        p = pinfo.get(mangled, {})
        print("%-48s %9d %7d %6d %6d %6d %6d %5s %6s %9s" % (
            name[:48], 16 * len(insns), len(insns), cnt["LDL"], cnt["STL"], cnt["LD"], cnt["ST"], p.get("regs", "-"),
            p.get("stack", "-"), "%d/%d" % (p.get("spill_st", 0), p.get("spill_ld", 0)) if p else "-"))
    # non-inlined device functions have frames of their own; ptxas reports them apart from the kernels that call them
    callees = [(m, p) for m, p in pinfo.items() if m not in funcs and p.get("stack", 0) > 0 and args.filter in names.get(m, m)]
    if callees:
        print("\nnon-inlined device functions with a stack frame (ptxas; their code is counted in the calling kernels):")
        for m, p in sorted(callees, key=lambda x: -x[1]["stack"]):
            print("  %6d B stack, spill %d/%d  %s" % (p["stack"], p.get("spill_st", 0), p.get("spill_ld", 0), names.get(m, m)[:100]))
    if args.lines:
        hits = [m for m in funcs if args.lines in names.get(m, m)]
        if not hits:
            raise SystemExit("no kernel matches %r" % args.lines)
        for mangled in hits:
            insns = funcs[mangled]
            allc = collections.Counter((f, l) for _, f, l in insns)
            locc = collections.Counter((f, l) for op, f, l in insns if op in ("LDL", "STL"))
            print("\n%s: %d instructions, %d LDL/STL" % (names.get(mangled, mangled), len(insns), sum(locc.values())))
            print("  most SASS instructions:")
            for (f, l), c in allc.most_common(args.top):
                print("    %7d  %s:%d" % (c, f, l))
            print("  most local-memory instructions (LDL / STL):")
            for (f, l), c in locc.most_common(args.top):
                print("    %7d  %s:%d" % (c, f, l))


if __name__ == "__main__":
    main()
