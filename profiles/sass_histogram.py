"""Static SASS opcode histogram of the hot kernels in libpinn_b200.so (cuobjdump -sass; needs no GPU).
    python profiles/sass_histogram.py > sass_opcodes.md"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pinns-tf2.0_b200", "lib", "libpinn_b200.so")
WANT = ["burgers215fused_loss_grad", "7burgers15fused_loss_grad", "3nls15fused_loss_grad", "7generic15fused_loss_grad",
        "4nsid15fused_loss_grad", "reduce_tail", "adam_update", "lbfgs_iterateILi12ELi256", "lbfgs_dots", "lbfgs_solve", "lbfgs_apply"]
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
usage = {m.group(1): m.group(2) for m in re.finditer(r"Function (\S+?):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+)", res)}
funcs, cur = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1); funcs[cur] = collections.Counter(); continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*(?:\.[A-Za-z0-9_.]+)?)", line)
    if m and cur:
        op = m.group(2)
        base = op.split(".")[0]
        key = op if base in ("DMMA", "UBLKCP", "SYNCS", "LDGSTS", "MUFU", "HMMA", "UTCHMMA", "UTMALDG") else base
        funcs[cur][key] += 1
print("# Static SASS opcode histogram of the hot kernels (`cuobjdump -sass pinns-tf2.0_b200/lib/libpinn_b200.so`, sm_90a)\n")
print("FP64 tensor work is `DMMA.8x8x4` (tcgen05 has no FP64 kind: no UTC*MMA / LDTM is expected); `UBLKCP` = TMA bulk copy,\n"
      "`SYNCS.*` = mbarrier, `LDGSTS` = cp.async.  LDL+STL counts local-memory (spill) instructions: none in the two specialised fused\n"
      "kernels; the generic kernel (128-register cap for 2 CTAs per SM) spills a few values.\n")
for name, c in funcs.items():
    if not any(w in name for w in WANT):
        continue
    tot = sum(c.values())
    u = usage.get(name, "")
    top = ", ".join("%s %d" % kv for kv in c.most_common(14))
    spill = c.get("LDL", 0) + c.get("STL", 0)
    print("* `%s`  \n  %s; %d instructions; LDL+STL = %d  \n  %s\n" % (name, u, tot, spill, top))
