#!/usr/bin/env python3
"""Static report of the built librtb200.so (no GPU needed): ptxas resource lines of every kernel from the build log and the
SASS mnemonic mix of one kernel (default: the shipped rt_wavefront_kernel<MODE_TREE,no lights>).

    python tools/sass_report.py [substring-of-mangled-name] > sass_static.txt
"""
import collections, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rust-raytracer_b200")
want = sys.argv[1] if len(sys.argv) > 1 else "rt_wavefront_kernelILj0ELb0"

print("== ptxas resource usage (rust-raytracer_b200/build.log, -Xptxas -v) ==")
log = open(os.path.join(PKG, "build.log")).read().splitlines()
name = None
for i, ln in enumerate(log):
    m = re.search(r"Compiling entry function '(\S+)'", ln)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        name = re.sub(r"\(rtk::TraceParams\)|\(.*\)$", "", name)
        continue
    if name and "bytes stack frame" in ln:
        stack = ln.strip()
    if name and "Used " in ln:
        used = re.sub(r"ptxas info\s*:\s*", "", ln).strip()
        print(f"{name}\n    {used}\n    {stack}")
        name = None

sass = subprocess.run(["cuobjdump", "-sass", os.path.join(PKG, "librtb200.so")], capture_output=True, text=True).stdout
blocks = re.split(r"\n\s*Function : ", sass)
for b in blocks[1:]:
    fn = b.split("\n", 1)[0].strip()
    if want not in fn:
        continue
    ops = collections.Counter()
    n = 0
    for ln in b.splitlines():
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Z0-9_]+)*)", ln)
        if m:
            ops[m.group(1).split(".")[0]] += 1
            n += 1
    print(f"\n== SASS mnemonic mix of {fn} ==")
    print(f"instructions: {n}  ({n * 16 / 1024:.1f} KiB of code)")
    groups = [
        ("packed f32 (FFMA2/FMUL2/FADD2)", ("FFMA2", "FMUL2", "FADD2")),
        ("scalar f32 (FFMA/FMUL/FADD)", ("FFMA", "FMUL", "FADD")),
        ("3-input min/max (FMNMX3)", ("FMNMX3",)),
        ("f32 min/max, compare, select", ("FMNMX", "FSETP", "FSEL", "FSET")),
        ("f64 (DFMA/DMUL/DADD/DSETP)", ("DFMA", "DMUL", "DADD", "DSETP")),
        ("MUFU (rcp/rsq/sqrt seeds)", ("MUFU",)),
        ("integer / logic", ("IMAD", "IADD3", "IADD", "LOP3", "SHF", "LEA", "ISETP", "SEL", "PRMT", "POPC", "FLO", "BREV", "IABS", "IMNMX", "VIMNMX", "VIMNMX3", "I2F", "F2I", "F2F", "I2FP", "F2FP", "MOV", "CS2R", "S2R", "R2P", "P2R", "PLOP3")),
        ("shared loads/stores (LDS/STS)", ("LDS", "STS")),
        ("shared atomics (ATOMS)", ("ATOMS",)),
        ("global/constant loads (LDG/LD/LDC/LDCU)", ("LDG", "LD", "LDC", "LDCU", "ULDC")),
        ("global stores/atomics (STG/ST/ATOMG/RED/ATOM)", ("STG", "ST", "ATOMG", "RED", "ATOM")),
        ("local (spill) LDL/STL", ("LDL", "STL")),
        ("warp shuffle/vote/match (SHFL/VOTE/VOTEU/MATCH/REDUX)", ("SHFL", "VOTE", "VOTEU", "MATCH", "REDUX")),
        ("CTA barriers (BAR)", ("BAR",)),
        ("warp sync / reconvergence (WARPSYNC/BSSY/BSYNC/BRA/...)", ("WARPSYNC", "BSSY", "BSYNC", "BRA", "BRX", "EXIT", "CALL", "RET", "NANOSLEEP", "YIELD", "BREAK")),
        ("TMA bulk copy + mbarrier (UBLKCP/SYNCS/...)", ("UBLKCP", "SYNCS", "UTMALDG", "FENCE", "MEMBAR", "ERRBAR", "CCTL")),
    ]
    seen = set()
    for title, keys in groups:
        c = sum(ops[k] for k in keys)
        seen.update(keys)
        detail = ", ".join(f"{k} {ops[k]}" for k in keys if ops[k])
        print(f"  {title:58s} {c:6d}   {detail}")
    rest = {k: v for k, v in ops.items() if k not in seen}
    print(f"  {'other':58s} {sum(rest.values()):6d}   " + ", ".join(f"{k} {v}" for k, v in sorted(rest.items(), key=lambda kv: -kv[1])))
