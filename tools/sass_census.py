"""Static SASS census of the render kernels' loops: instruction count and opcode histogram of every loop body.

  python tools/sass_census.py [LIB] [--kernel REGEX ...] [--min-insts N] [--top K] [--ops OP,OP,...]

Runs `cuobjdump -sass` on the built library (default: the package's lib/libb200nerf.so) and, for every instance of the
selected kernels (default: nff_shade_lane_kernel and nff_sample_lane_kernel), finds each loop by its backward branch: a
BRA whose target lies at or before it spans the body [target, branch].  Per loop it prints the address range, the nesting
depth (loops inside other loops are indented), the instruction count, the counts of the opcodes named by --ops (always
shown, 0 included) and the K most frequent opcodes.  Opcodes are counted without their modifiers (HGMMA.64x32x8.F32.TF32
-> HGMMA).  Static counts say what the compiler emitted, not how often it executes or what it costs.
"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "neurad-studio_b200", "lib", "libb200nerf.so")
DEFAULT_KERNELS = ("nff_shade_lane_kernel", "nff_sample_lane_kernel")
DEFAULT_OPS = "HGMMA,R2UR,WARPGROUP.ARRIVE,WARPGROUP.DEPBAR,BAR,LDS,STS,LDL,STL"

_FUNC = re.compile(r"^\s*Function : (\S+)")
# /*0a10*/  @!P1 BRA 0xb00 ;   (predicate optional)
_INST = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)\s*([^;]*);")


def _tool(name):
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    return None


def parse_sass(text):
    """{mangled function name: [(address, full opcode, operands)]}"""
    funcs, cur = {}, None
    for line in text.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = _INST.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(3), m.group(4).strip()))
    return funcs


def base_op(op):
    # WARPGROUP.ARRIVE / WARPGROUP.DEPBAR are different instructions; everything else is named by its first field
    return ".".join(op.split(".")[:2]) if op.startswith("WARPGROUP.") else op.split(".")[0]


def find_loops(insts):
    """[(start address, branch address)] of every backward branch, outermost first"""
    loops = set()
    for addr, op, args in insts:
        if base_op(op) != "BRA":
            continue
        m = re.match(r"(?:`\()?\s*(0x[0-9a-f]+)", args)
        if m and int(m.group(1), 16) <= addr:
            loops.add((int(m.group(1), 16), addr))
    return sorted(loops, key=lambda se: (se[0], -se[1]))


def census(insts, lo, hi):
    return collections.Counter(base_op(op) for addr, op, _ in insts if lo <= addr <= hi)


def demangle(names):
    filt = _tool("cu++filt") or _tool("c++filt")
    if not filt or not names:
        return {n: n for n in names}
    out = subprocess.run([filt], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out)) if len(out) == len(names) else {n: n for n in names}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("lib", nargs="?", default=DEFAULT_LIB)
    ap.add_argument("--kernel", action="append", help="regex on the mangled name (repeatable)")
    ap.add_argument("--min-insts", type=int, default=32, help="hide loops with fewer instructions")
    ap.add_argument("--top", type=int, default=10, help="most frequent opcodes shown per loop")
    ap.add_argument("--ops", default=DEFAULT_OPS, help="opcodes always shown per loop (comma-separated)")
    a = ap.parse_args()
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        sys.exit("cuobjdump not found")
    res = subprocess.run([cuobjdump, "-sass", a.lib], capture_output=True, text=True)
    if res.returncode != 0:
        sys.exit(res.stderr)
    funcs = parse_sass(res.stdout)
    pats = [re.compile(k) for k in (a.kernel or DEFAULT_KERNELS)]
    names = sorted(n for n in funcs if any(p.search(n) for p in pats))
    if not names:
        sys.exit("no kernel matches " + ", ".join(p.pattern for p in pats))
    pretty = demangle(names)
    ops = [o for o in a.ops.split(",") if o]
    for name in names:
        insts = funcs[name]
        total = census(insts, 0, insts[-1][0] if insts else -1)
        print(f"{pretty[name]}  ({len(insts)} instructions; " + ", ".join(f"{o} {total[o]}" for o in ops) + ")")
        loops = find_loops(insts)
        for lo, hi in loops:
            c = census(insts, lo, hi)
            n = sum(c.values())
            if n < a.min_insts:
                continue
            depth = sum(1 for l2, h2 in loops if (l2, h2) != (lo, hi) and l2 <= lo and hi <= h2)
            fixed = ", ".join(f"{o} {c[o]}" for o in ops)
            top = ", ".join(f"{o} {k}" for o, k in c.most_common(a.top))
            print(f"  {'  ' * depth}loop {lo:#07x}-{hi:#07x}: {n} instructions | {fixed}")
            print(f"  {'  ' * depth}    top: {top}")
        print()
    return 0


if __name__ == "__main__":
    sys.exit(main())
