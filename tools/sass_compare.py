#!/usr/bin/env python
"""Compare the SASS of every kernel of two builds of libirbpp.so, ignoring the names of called symbols.

    python tools/sass_compare.py OLD.so NEW.so [--diff]

Prints, per kernel, the instruction counts and whether the instruction streams are identical, the same instructions in
another order (possibly with other register numbers), or different.  The streams are aligned by difflib with branch
targets taken as the instructions they point at, so one inserted instruction counts as one difference and not as a
shift of every later address; a branch whose target does not align counts as a difference too.  --diff prints the
differing instructions.  A kernel that only one of the builds contains is reported as missing.  Exit code 0 when every
kernel is in both builds and identical.  Needs cuobjdump and c++filt (no GPU)."""
import difflib
import re
import subprocess
import sys

BRANCH = re.compile(r"(@!?U?P\w*\s+)?(BRA|BRX|BSSY|CALL|JMP|JMX|WARPSYNC\.COLLECTIVE)\b")     # instructions whose hex operand is a code address


def functions(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = re.sub(r"^void ", "", cur)
            out[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if cur is not None and m:
            out[cur].append(re.sub(r"\b_Z\w+", "SYM", m.group(1)))
    return out


def target(ins):
    """index of the instruction a branch points at (16 bytes per instruction), None for other instructions"""
    m = BRANCH.match(ins) and re.search(r"\b0x([0-9a-f]+)\b", ins)
    return int(m.group(1), 16) // 16 if m else None


def key(ins):
    """an instruction without its branch target, for the alignment"""
    return re.sub(r"\b0x[0-9a-f]+\b", "<target>", ins) if target(ins) is not None else ins


def unnumbered(ins):
    """an instruction with its register numbers dropped (R7 -> R, UR4 -> UR, P2 -> P, B1 -> B)"""
    return re.sub(r"\b(UR|R|UP|P|B)\d+\b", r"\1", ins)


def compare(a, b):
    """(old index or None, new index or None) of every difference of two instruction streams"""
    ka, kb = [key(x) for x in a], [key(x) for x in b]
    ops = difflib.SequenceMatcher(None, ka, kb, autojunk=False).get_opcodes()
    to_new = {i1 + k: j1 + k for tag, i1, i2, j1, j2 in ops if tag == "equal" for k in range(i2 - i1)}
    diff = []
    for tag, i1, i2, j1, j2 in ops:
        if tag == "equal":      # aligned branches must point at aligned instructions
            diff += [(i, to_new[i]) for i in range(i1, i2) if target(a[i]) is not None and to_new.get(target(a[i])) != target(b[to_new[i]])]
        else:
            diff += [(i1 + k if i1 + k < i2 else None, j1 + k if j1 + k < j2 else None) for k in range(max(i2 - i1, j2 - j1))]
    return sorted(diff, key=lambda d: d[0] if d[0] is not None else d[1])


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    ok = True
    for n in sorted(set(old) | set(new)):
        if n not in old or n not in new:
            ok = False
            print("%-76s missing from %s" % (n, "OLD" if n not in old else "NEW"))
            continue
        a, b = old[n], new[n]
        diff = compare(a, b)
        if not diff:
            verdict = "identical"
        else:
            ok = False
            ka, kb = sorted(map(key, a)), sorted(map(key, b))
            kind = "reordered" if ka == kb else \
                "reordered, registers renamed" if sorted(map(unnumbered, ka)) == sorted(map(unnumbered, kb)) else "changed"
            verdict = "%d differ (%s)" % (len(diff), kind)
        print("%-76s %5d / %5d instructions  %s" % (n, len(a), len(b), verdict))
        if "--diff" in sys.argv:
            for i, j in diff:                       # [old index|new index], blank where a side has none
                print("    [%5s|%5s] %-45s | %s" % ("" if i is None else i, "" if j is None else j,
                                                   "" if i is None else a[i], "" if j is None else b[j]))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
