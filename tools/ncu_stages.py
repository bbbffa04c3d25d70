#!/usr/bin/env python3
"""Stage breakdown of an ncu capture of rt_wavefront_kernel (instructions, samples, active lanes, top stalls per stage).
Every SASS instruction is attributed through its INLINE CHAIN (nvdisasm --print-line-info-inline): the kernel-level line in
rtb200_wavefront.cu picks the stage, and inside closest_hit() the outermost frame in rtb200_trace.cuh picks the step.
Stage boundaries are found from the marker comments in the sources, so the tool follows the code.
usage: ncu_stages.py <rep> [kernel-substr] [lib.so]"""
import collections, csv, os, re, subprocess, sys, tempfile
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rep = sys.argv[1]
kname = sys.argv[2] if len(sys.argv) > 2 else "rt_wavefront_kernelILj0ELb0"
lib = sys.argv[3] if len(sys.argv) > 3 else os.path.join(REPO, "rust-raytracer_b200", "librtb200.so")
WF = os.path.join(REPO, "rust-raytracer_b200", "csrc", "rtb200_wavefront.cu")
TR = os.path.join(REPO, "rust-raytracer_b200", "csrc", "rtb200_trace.cuh")

def line_of(path, needle, after=0):
    for i, l in enumerate(open(path).read().splitlines(), 1):
        if i > after and needle in l:
            return i
    raise KeyError(needle)

# kernel-level stages (rtb200_wavefront.cu)
k_fill = line_of(WF, "initial fill of the pool")
k_ch = line_of(WF, "closest_hit<MODE>(")
k_sort = line_of(WF, "=== sort: compact")
k_A = line_of(WF, "// A: class counts and perm complete")
k_shade = line_of(WF, "shade_slot<LIGHTS>(p, sc")
k_regen = line_of(WF, "regenerate_slot<LIGHTS>(p, P, active && done")
k_C = line_of(WF, "// C: pool written back")
k_stats = line_of(WF, "flush_stats(p, st, lane)")
def kernel_stage(l):
    if l < k_fill: return "setup"
    if l == k_fill: return "regen"
    if l < k_ch: return "loop_ctl"
    if l == k_ch: return "closest_hit"
    if l < k_A: return "sort"
    if l == k_A: return "barrier_A"
    if l <= k_shade: return "shade"
    if l == k_regen: return "regen"
    if l <= k_C: return "barrier_C"
    if l >= k_stats: return "exit"
    return "loop_ctl"
# steps inside closest_hit (rtb200_trace.cuh)
t_ch0 = line_of(TR, "RT_DEV uint32_t closest_hit(")
t_const = line_of(TR, "per-ray constants in the recentred f32 frame")
t_trav = line_of(TR, "warp-cooperative traversal ----")
t_node = line_of(TR, "node step: lane")
t_leaf = line_of(TR, "leaf step: lane")
t_exact = line_of(TR, "exact step: lane")
t_brute = line_of(TR, "MODE_BRUTE: hit_world")
t_merge = line_of(TR, "if (alive) {", t_brute)
t_end = line_of(TR, "// Regenerate pool slot")
def ch_step(l):
    if l < t_const: return "ch_setup"
    if l < t_trav: return "ch_setup"
    if l < t_node: return "ch_control"
    if l < t_leaf: return "node_step"
    if l < t_exact: return "leaf_step"
    if l < t_brute: return "exact_step"
    if l < t_merge: return "ch_control"
    return "ch_merge"

tmp = tempfile.mkdtemp()
subprocess.run(f"cd {tmp} && cuobjdump -xelf all {os.path.abspath(lib)}", shell=True, capture_output=True)
seq = None
for f in sorted(os.listdir(tmp)):
    if not f.endswith(".cubin"): continue
    out = subprocess.run(["nvdisasm", "--print-line-info-inline", "-c", os.path.join(tmp, f)], capture_output=True, text=True).stdout
    infn = False; cur = []; chain = []; fresh = True; s = []
    for ln in out.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+),", ln)
        if m:
            if infn and s: break
            infn = kname in m.group(1); s = []; chain = []; fresh = True; continue
        if not infn: continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            if fresh: chain = []; fresh = False
            chain.append((os.path.basename(m.group(1)), int(m.group(2)))); continue
        if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", ln):
            s.append(list(chain)); fresh = True
    if infn and s: seq = s; break
assert seq, "kernel not found in " + lib

def stage_of(chain):
    if not chain: return "other"
    outer = chain[-1]
    if outer[0] != "rtb200_wavefront.cu": return "other"
    st = kernel_stage(outer[1])
    if st == "closest_hit":
        for fr in reversed(chain[:-1]):          # outermost frame inside rtb200_trace.cuh
            if fr[0] == "rtb200_trace.cuh" and t_ch0 <= fr[1] < t_end:
                return ch_step(fr[1])
        return "ch_control"
    return st

csvout = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(csvout.splitlines())); hdr = rows[1]; data = rows[2:]
assert len(seq) == len(data), (len(seq), len(data))
iex = hdr.index("Instructions Executed"); ismp = hdr.index("# Samples"); ithr = hdr.index("Thread Instructions Executed")
stall = {h: i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h}
order = ["setup", "regen", "ch_setup", "ch_control", "node_step", "leaf_step", "exact_step", "ch_merge", "sort", "barrier_A", "shade", "barrier_C", "loop_ctl", "exit", "other"]
agg = collections.OrderedDict((k, [0, 0, 0, 0, collections.Counter()]) for k in order)
tot = [0, 0]; bar = 0
for ch, r in zip(seq, data):
    a = agg[stage_of(ch)]
    a[0] += int(r[iex]); a[1] += int(r[ismp]); a[2] += int(r[ithr]); a[3] += 1
    for h, c in stall.items():
        if r[c] not in ("", "0"):
            a[4][h] += int(r[c])
            if h == "stall_barrier": bar += int(r[c])
    tot[0] += int(r[iex]); tot[1] += int(r[ismp])
print(f"{'stage':12s} {'sass':>5s} {'instr%':>7s} {'smp%':>6s} {'lanes':>6s}  top stalls (share of the stage's samples)")
for nm, a in agg.items():
    if a[3] == 0: continue
    top = ", ".join(f"{k[6:]}={100*v/max(a[1],1):.0f}%" for k, v in a[4].most_common(4))
    print(f"{nm:12s} {a[3]:5d} {100*a[0]/tot[0]:7.2f} {100*a[1]/tot[1]:6.2f} {a[2]/max(a[0],1):6.1f}  {top}")
print(f"total warp instructions {tot[0]}, samples {tot[1]}, of which waiting at a CTA barrier {100*bar/max(tot[1],1):.1f} %")
