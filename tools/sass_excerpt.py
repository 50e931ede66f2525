"""Per-kernel census of the Hopper-specific SASS in the built library (no GPU needed):

    python tools/sass_excerpt.py > sass.txt

wgmma -> HGMMA (its fences and waits -> WARPGROUP.*), TMA -> UTMALDG/UTMASTG (cluster multicast: UTMALDG.*.MULTICAST),
mbarrier -> SYNCS.  One example line per mnemonic is printed under the counts."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "vampnet_b200", "libvampnet_b200.so")
PAT = re.compile(r"\b(HGMMA\.\d+x\d+x\d+|WARPGROUP\.[A-Z]+|UTMALDG(?:\.\dD)?(?:\.MULTICAST)?|"
                 r"UTMASTG(?:\.\dD)?|UBLKCP|UTMAPF|SYNCS\.[A-Z.0-9]+|MUFU\.EX2|HMMA)\b")


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    demangle = lambda n: subprocess.run(["cu++filt", n], capture_output=True, text=True).stdout.strip() or n  # noqa: E731
    cur, per, example = None, collections.OrderedDict(), {}
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = demangle(m.group(1))
            per[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = PAT.search(line)
        if m:
            per[cur][m.group(1)] += 1
            if m.group(1).startswith("HGMMA") and re.search(r"HGMMA\S*\s+R\d+, R\d+, gdesc", line):
                per[cur]["(A operand from registers)"] += 1
            example.setdefault(m.group(1), re.sub(r"/\*[0-9a-f]+\*/", "", line).strip().rstrip(";").strip())
    print(f"# {os.path.relpath(LIB, ROOT)}: Hopper-specific SASS per kernel (cuobjdump -sass)")
    for name, c in per.items():
        if not c:
            continue
        short = name.split(">(")[0] + ">" if ">(" in name else re.sub(r"\(.*", "", name)
        print(f"\n{short}")
        print("   " + "  ".join(f"{k}:{v}" for k, v in sorted(c.items())))
    print("\n# one example per mnemonic")
    for k, v in sorted(example.items()):
        print(f"{k:28s} {v[:110]}")
    if any("HMMA" == k for c in per.values() for k in c):
        print("\n# WARNING: legacy HMMA (mma.sync) found", file=sys.stderr)


if __name__ == "__main__":
    main()
