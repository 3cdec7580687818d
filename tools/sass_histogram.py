"""SASS instruction histogram of libmi3d.so per kernel: the Hopper mnemonics (HGMMA = wgmma.mma_async, WARPGROUP = its fences,
UTMALDG/UTMASTG = TMA, SYNCS = mbarrier) that show which kernels run on the tensor cores, next to RED / ATOM / FFMA / loads / stores.
    python tools/sass_histogram.py        (no GPU needed: cuobjdump reads the cubin in the .so)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "make-it-3d_b200", "libmi3d.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "SYNCS", "RED", "ATOM", "HMMA", "FFMA", "LDG", "STG", "LDL", "STL", "MUFU"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    kern, hist = None, collections.OrderedDict()
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            kern = kern.replace("(anonymous namespace)::", "").replace("void ", "")
            kern = re.sub(r"\(.*$", "", kern)
            hist[kern] = collections.Counter()
            continue
        m = re.search(r"/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and kern:
            op = m.group(1)
            hist[kern]["_total"] += 1
            for w in WATCH:
                if op.startswith(w):
                    hist[kern][w] += 1
                    break
    print(f"# cuobjdump -sass {os.path.relpath(SO, ROOT)} : instruction counts per kernel (static SASS, sm_90a)")
    print(f"{'kernel':70s} {'total':>7s} " + " ".join(f"{w:>7s}" for w in WATCH))
    tot = collections.Counter()
    for k, c in hist.items():
        print(f"{k[:70]:70s} {c['_total']:7d} " + " ".join(f"{c[w]:7d}" for w in WATCH))
        tot.update(c)
    print(f"{'ALL KERNELS':70s} {tot['_total']:7d} " + " ".join(f"{tot[w]:7d}" for w in WATCH))


if __name__ == "__main__":
    sys.exit(main())
