"""Guard against unintended code-generation changes in kernels that have been measured: md5 of each kernel's SASS (addresses and encodings
stripped) in build/llama.cu.o and build/vision.cu.o against build/sass_hashes.json (a local record, not committed).

    python tools/sass_guard.py            # compare; lists changed / new / vanished / renamed kernels
    python tools/sass_guard.py --write    # record the current build as the baseline (do this right after a measured GPU run)

Use: record after a measured run, then add experimental variants while proving that every measured kernel stayed byte-identical
(ptxas output is sensitive even to a kernel-parameter struct growing)."""
import hashlib
import json
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
BASE = ROOT / "build" / "sass_hashes.json"


def hashes() -> dict[str, str]:
    out = {}
    for obj in ("llama.cu.o", "vision.cu.o"):
        txt = subprocess.run(["cuobjdump", "-sass", str(ROOT / "build" / obj)], capture_output=True, text=True, check=True).stdout
        cur, buf = None, []
        for line in txt.split("\n"):
            m = re.search(r"Function : (\S+)", line)
            if m:
                if cur:
                    out[cur] = hashlib.md5("".join(buf).encode()).hexdigest()
                cur, buf = m.group(1), []
            elif cur and re.match(r"\s+/\*[0-9a-f]{4,5}\*/", line):
                buf.append(re.sub(r"/\* 0x[0-9a-f]+ \*/", "", re.sub(r"/\*[0-9a-f]{4,5}\*/", "", line)).strip() + "\n")
        if cur:
            out[cur] = hashlib.md5("".join(buf).encode()).hexdigest()
    return out


if __name__ == "__main__":
    cur = hashes()
    if "--write" in sys.argv:
        BASE.write_text(json.dumps(cur, indent=0, sort_keys=True))
        print(f"recorded {len(cur)} kernels in {BASE}")
        sys.exit(0)
    if not BASE.exists():
        sys.exit(f"no baseline recorded: run with --write after a measured run ({BASE})")
    base = json.loads(BASE.read_text())
    changed = sorted(k for k in base if k in cur and base[k] != cur[k])
    gone = sorted(k for k in base if k not in cur)
    new = sorted(k for k in cur if k not in base)
    # a vanished kernel whose code a new kernel has, hash for hash, was renamed (a wrapper turned into a template instantiation, say)
    renamed = []
    for k in list(gone):
        match = next((m for m in new if cur[m] == base[k]), None)
        if match:
            renamed.append((k, match))
            gone.remove(k)
            new.remove(match)
    for title, lst in (("CHANGED", changed), ("VANISHED", gone), ("new", new)):
        for k in lst:
            print(f"{title:9s} {k[:120]}")
    for old, now in renamed:
        print(f"RENAMED   {old[:120]} -> {now[:120]}")
    print(f"{len(base) - len(changed) - len(gone)} of {len(base)} recorded kernels unchanged ({len(renamed)} renamed), {len(changed)} changed, "
          f"{len(gone)} vanished, {len(new)} new")
    sys.exit(1 if changed or gone else 0)
