"""Static SASS report for one kernel of a built library: total code bytes and every loop (backward branch) with its body size --
the partial-round loop of the Poseidon kernels must stay below the 32 KB L1.5 instruction cache -- and its opcode mix: wide
multiplies (IMAD.WIDE* + IMAD.HI*, the multiply-pipe work) and the other instructions by class.  For the Poseidon hash kernels the
partial-round loop, the full-round S-box body and the full-round row loop are the innermost loops; a loop's counts include the
loops nested in it.   usage: python tools/sass_loops.py <lib.so> <kernel-name-substring>"""
import collections
import re
import subprocess
import sys

CLASSES = ("IMAD.WIDE", "IMAD.HI", "IMAD.MOV", "IMAD.X", "IMAD.IADD", "IMAD", "IADD3.X", "IADD3", "SEL", "MOV", "HFMA2", "LOP3",
           "ISETP", "LDG", "LDS", "STL", "LDL", "BRA")


def kernels(lib, pat):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    cur, body = None, collections.defaultdict(list)
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and pat in cur:
            m = re.search(r"/\*([0-9a-f]{4,6})\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)([^;]*);", line)
            if m:
                body[cur].append((int(m.group(1), 16), m.group(3), m.group(4)))
    return body


def classify(op):
    for c in CLASSES:
        if op == c or op.startswith(c + "."):
            return c
    return "other"


def loops(ins):
    """(lo, hi) of every backward branch."""
    res = set()
    for addr, op, args in ins:
        b = re.search(r"(0x[0-9a-f]+)", args) if op.startswith("BRA") else None
        if b and int(b.group(1), 16) < addr:
            res.add((int(b.group(1), 16), addr))
    return sorted(res)


def mix(ins, lo, hi):
    c = collections.Counter(classify(op) if classify(op) != "other" else op for a, op, _ in ins if lo <= a <= hi)
    n = sum(c.values())
    wide = c["IMAD.WIDE"] + c["IMAD.HI"]
    return n, wide, c


def main():
    lib, pat = sys.argv[1], sys.argv[2]
    for fn, ins in kernels(lib, pat).items():
        total = max(a for a, _, _ in ins) + 16
        print(f"{fn}\n  code {total} B ({total / 1024:.1f} KB)")
        for what, (lo, hi) in [("kernel", (0, 1 << 30))] + [(f"loop {lo:#07x}..{hi:#07x} ({hi - lo + 16} B)", (lo, hi))
                                                           for lo, hi in loops(ins)]:
            n, wide, c = mix(ins, lo, hi)
            other = ", ".join(f"{k} {v}" for k, v in sorted(c.items(), key=lambda kv: -kv[1]) if k not in ("IMAD.WIDE", "IMAD.HI"))
            print(f"  {what}: {n} instructions, {wide} wide multiplies (IMAD.WIDE {c['IMAD.WIDE']}, IMAD.HI {c['IMAD.HI']}), "
                  f"{n - wide} other: {other}")


if __name__ == "__main__":
    main()
