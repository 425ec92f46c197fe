#!/usr/bin/env python
"""Compare the SASS of the 16 x 16 step kernels of two builds of libirbpp.so, ignoring symbol names.

    python tools/sass_compare.py OLD.so NEW.so [--diff]

Builds of the parent commit name the kernels without the grid parameter (irbpp_scan_kernel<false>); builds with the
32 x 32 grid name them Grid<2> (irbpp_scan_kernel<irbpp::Grid<2>, false>).  Prints, per kernel, the instruction counts
and whether the instruction streams are identical; --diff prints the differing instructions.  Exit code 0 when all are
identical.  Needs cuobjdump and c++filt (no GPU)."""
import re
import subprocess
import sys


def functions(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = re.sub(r"^void ", "", re.sub(r"irbpp::Grid<2>, |<irbpp::Grid<2> >", lambda g: "" if "," in g.group(0) else "", cur))
            out[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if cur is not None and m:
            out[cur].append(re.sub(r"\b_Z\w+", "SYM", m.group(1)))
    return out


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    names = ["irbpp::irbpp_scan_kernel<%s>(irbpp::Params)" % t for t in ("false", "true")]
    names += ["irbpp::irbpp_candidates_kernel<%d, %s>(irbpp::Params)" % (e, t) for e in (4, 8) for t in ("false", "true")]
    names += ["irbpp::irbpp_levels_kernel(irbpp::Params)", "irbpp::irbpp_heuristic_kernel(irbpp::Params)"]
    ok = True
    for n in names:
        a, b = old[n], new[n]
        diff = [(i, x, y) for i, (x, y) in enumerate(zip(a, b)) if x != y]
        same = not diff and len(a) == len(b)
        ok &= same
        print("%-55s %5d / %5d instructions  %s" % (n, len(a), len(b), "identical" if same else "%d differ" % len(diff)))
        if "--diff" in sys.argv:
            for i, x, y in diff:
                print("    [%5d] %-45s | %s" % (i, x, y))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
