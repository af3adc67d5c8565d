"""SASS evidence that the kernels use the Hopper instructions they are written for: per kernel of libcgd_b200.so, the counts of the
mnemonics that identify wgmma (HGMMA), TMA (UTMALDG / UTMASTG / UBLKCP), legacy warp MMA (HMMA), cp.async
(LDGSTS), plus registers / shared memory from `cuobjdump -res-usage`.
    python scripts/sass_summary.py > profiles/sass_summary.txt     (no GPU needed)"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "clip_guided_diffusion_b200", "libcgd_b200.so")
KEYS = ["HGMMA", "UTMALDG", "UTMASTG", "UTMAPF", "UBLKCP", "HMMA", "LDGSTS", "LDSM", "MUFU", "ATOM", "RED", "SYNCS", "UCGABAR", "BAR"]
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout
usage = {}
cur = None
for line in res.splitlines():
    m = re.search(r"Function (\S+):", line)
    if m:
        cur = m.group(1)
        continue
    m = re.search(r"REG:(\d+).*?SHARED:(\d+)", line)
    if m and cur:
        usage[cur] = (int(m.group(1)), int(m.group(2)))
counts, name = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        name = m.group(1)
        counts[name] = collections.Counter()
        continue
    if name is None:
        continue
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m:
        op = m.group(1)
        counts[name]["_total"] += 1
        for k in KEYS:
            if op.split(".")[0] == k or (k in ("UTMALDG", "UTMASTG") and op.startswith(k)):
                counts[name][k] += 1
def demangle(n):
    try:
        return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    except Exception:
        return n
print(f"# SASS summary of {os.path.relpath(so, ROOT)} (cuobjdump -sass / -res-usage, sm_90a); columns: instructions | registers | static smem | mnemonic counts")
tot = collections.Counter()
for n, c in counts.items():
    d = re.sub(r"\(.*", "", demangle(n))
    d = d.replace("void cgd::", "").replace("cgd::", "")
    reg, sh = usage.get(n, (0, 0))
    flags = " ".join(f"{k}={c[k]}" for k in KEYS if c[k])
    print(f"{d[:72]:72s} {c['_total']:6d} instr  {reg:3d} regs {sh:6d} B smem  {flags}")
    tot.update({k: v for k, v in c.items() if k != "_total"})
print("# totals:", " ".join(f"{k}={tot[k]}" for k in KEYS if tot[k]))
