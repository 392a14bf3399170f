"""What the kernels are made of: per kernel of build/llama.cu.o, build/vision.cu.o and build/tp.cpp.o the counts of the SASS mnemonics that prove
the Hopper paths: HGMMA / IGMMA (wgmma f16 / s8), WARPGROUP (wgmma fences and waits), UTMALDG (TMA tensor load), UBLKCP
(cp.async.bulk), SYNCS (mbarrier), IDP.4A (dp4a).   python tools/sass_census.py   (after a build; prints to stdout)"""
import re, subprocess, sys, collections
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
PAT = ["HGMMA", "IGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "UBLKPF", "SYNCS", "IDP.4A", "HMMA", "IMMA", "LDG", "LDS", "SHFL", "BAR.SYNC", "ATOMG", "REDG"]
for obj in ("llama.cu.o", "vision.cu.o", "tp.cpp.o"):
    out = subprocess.run(["cuobjdump", "-sass", str(ROOT / "build" / obj)], capture_output=True, text=True).stdout
    cur, counts = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); counts[cur] = collections.Counter(); continue
        if cur:
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
            if m:
                op = m.group(1)
                for p in PAT:
                    if op == p or op.startswith(p + "."):
                        counts[cur][p] += 1
                counts[cur]["(all)"] += 1
    print(f"== {obj}")
    for fn, c in counts.items():
        name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()[:110]
        keys = " ".join(f"{p}={c[p]}" for p in PAT if c[p])
        print(f"{c['(all)']:6d} instr  {name}\n        {keys}")
