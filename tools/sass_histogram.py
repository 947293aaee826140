"""Per-kernel SASS mnemonic histogram of the built library (evidence that wgmma / TMA are on the hot path).
Usage: python tools/sass_histogram.py [library.so] > profiles/<name>.md"""
import collections
import re
import subprocess
import sys

lib = sys.argv[1] if len(sys.argv) > 1 else "defensegan_b200/libdefensegan_b200.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], stdout=subprocess.PIPE, text=True).stdout
fn, hist = None, collections.defaultdict(collections.Counter)
for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        fn = m.group(1)
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
    if m and fn:
        hist[fn][m.group(1)] += 1
keys = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "SYNCS", "STL", "LDL", "MEMBAR",
        "FENCE", "RED", "ATOMG", "LDG", "STG", "BAR", "ELECT"]
print("| kernel | total | " + " | ".join(keys) + " |")
print("|---|---|" + "---|" * len(keys))
for f, c in sorted(hist.items(), key=lambda kv: -sum(kv[1].values())):
    name = subprocess.run(["c++filt", f], stdout=subprocess.PIPE, text=True).stdout.strip().split("(")[0]
    row = [str(sum(v for op, v in c.items() if op.startswith(k))) for k in keys]
    print("| `%s` | %d | %s |" % (name[:70], sum(c.values()), " | ".join(row)))
