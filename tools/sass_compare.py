"""Compare the SASS of two builds of a CUDA library function by function (cuobjdump -sass), e.g. the library of a change against the
library of its parent, to show that a change left the existing kernels' instructions alone.

    python tools/sass_compare.py OLD.so NEW.so [--drop-template-arg N=VALUE ...] [--param-shift BYTES]

Functions are matched by their demangled names.  --drop-template-arg removes a trailing template argument that the new build added
with its default value (e.g. `false` for a new bool parameter) so that `f<true, false>` of the new build matches `f<true>` of the old
one.  --param-shift B: a kernel-parameter struct grew by B bytes, so the constant-bank offsets of the parameters behind it moved; every
c[0x0][X] in the NEW build's listing with X at or above the first moved offset of that kernel is compared as X - B (reported as such).
Prints one line per matched function (identical / differs) and the functions found in only one build."""
import argparse
import re
import subprocess
import sys


def sass_by_function(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        if cur is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*(/\*.*\*/)?\s*$", line)
        if m and m.group(1):
            funcs[cur].append(m.group(1).rstrip(" ;"))
    return funcs


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return dict(zip(names, r))


def normalise_name(name, drops):
    for d in drops:
        only = "<" + d + ">(" in name    # before the drop below, which turns f<false, false> into f<false> (not the only argument)
        name = name.replace(", " + d + ">", ">")
        if only:                         # the only template argument: f<false>(...) of a kernel that was not a template before
            name = re.sub(r"^void ", "", name.replace("<" + d + ">(", "("))
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--drop-template-arg", action="append", default=[], help="trailing template argument added with its default, e.g. false")
    ap.add_argument("--param-shift", type=int, default=0)
    ap.add_argument("--filter", default="", help="regular expression on the demangled name")
    a = ap.parse_args()
    old, new = sass_by_function(a.old), sass_by_function(a.new)
    dold, dnew = demangle(list(old)), demangle(list(new))
    by_old = {normalise_name(dold[k], []): k for k in old}
    flt = re.compile(a.filter)
    same = diff = 0
    seen = set()
    for k in sorted(new, key=lambda k: dnew[k]):
        name = normalise_name(dnew[k], a.drop_template_arg)
        if not flt.search(name) or name not in by_old:
            continue
        seen.add(name)
        o, n = old[by_old[name]], new[k]
        note = ""
        if o != n and a.param_shift and len(o) == len(n):
            # offsets that differ by exactly the shift, everything else equal
            def offs(s):
                return [int(x, 16) for x in re.findall(r"c\[0x0\]\[(0x[0-9a-f]+)\]", s)]
            ok = True
            for lo, ln in zip(o, n):
                if lo == ln:
                    continue
                if re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][*]", lo) != re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][*]", ln):
                    ok = False
                    break
                if any(y - x not in (0, a.param_shift) for x, y in zip(offs(lo), offs(ln))):
                    ok = False
                    break
            if ok:
                note = f" (identical but for parameter offsets moved by {a.param_shift} bytes)"
                o = n
        if o == n:
            same += 1
            print(f"identical{note}: {name[:150]} ({len(n)} instructions)")
        else:
            diff += 1
            print(f"DIFFERS: {name[:150]} ({len(o)} -> {len(n)} instructions)")
    only_old = [n for n in by_old if flt.search(n) and n not in seen]
    for n in sorted(only_old):
        print(f"only in old: {n[:150]}")
    for k in sorted(new, key=lambda k: dnew[k]):
        name = normalise_name(dnew[k], a.drop_template_arg)
        if flt.search(name) and name not in seen:
            print(f"only in new: {dnew[k][:150]}")
    print(f"{same} identical, {diff} differ")
    return 1 if diff else 0


if __name__ == "__main__":
    sys.exit(main())
