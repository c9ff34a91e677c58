#!/usr/bin/env python3
"""Compare the machine code of two builds of libabyssb200.so kernel by kernel: the SASS instruction stream (cuobjdump -sass,
addresses and encodings dropped) and the resources (cuobjdump -res-usage: registers, stack, shared and local memory).

    python scripts/compare_sass.py OLD.so NEW.so [--rename NEW=OLD ...]

Kernels are matched by demangled name.  A kernel that gained a template argument is matched through --rename, a plain text
substitution on the new demangled names (and on the symbols its instructions call).  The k > 192 change matches with

    --rename "k_hash_reads_tma<256>=k_hash_reads_tma" --rename "k_hash_segments<256>=k_hash_segments" \\
    --rename "k_kon_walk<false, 6u>=k_kon_walk<false>" --rename "k_kon_walk<true, 6u>=k_kon_walk<true>" \\
    --rename "k_kon_trim<6u>=k_kon_trim"

Prints one line per kernel of the old build (same / DIFFERENT / missing) and the kernels only the new build has; exits 1 when
a kernel of the old build is missing or differs."""
import argparse
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def demangle(names):
    if not names:
        return {}
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return dict(zip(names, out))


def sass(lib):
    """{mangled kernel name: [instruction text]}"""
    text = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\* 0x[0-9a-f]+ \*/", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def resources(lib):
    """{mangled name: 'REG:.. STACK:.. SHARED:.. LOCAL:..'}"""
    text = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            out[cur] = " ".join(x for x in line.split() if x.split(":")[0] in ("REG", "STACK", "SHARED", "LOCAL"))
            cur = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", action="append", default=[], help="NEW=OLD text substitution on the new build's names")
    a = ap.parse_args()
    renames = [r.split("=", 1) for r in a.rename]

    def rename(s):
        for new, old in renames:
            s = s.replace(new, old)
        return s

    builds = {}
    for tag, lib in (("old", a.old), ("new", a.new)):
        funcs, res = sass(lib), resources(lib)
        symbols = set(funcs) | {m for ins in funcs.values() for i in ins for m in re.findall(r"`\((\w+)\)", i)}
        dm = {m: re.sub(r"^void ", "", d) for m, d in demangle(sorted(symbols)).items()}  # a template's name carries its return type
        fix = (lambda s: rename(s)) if tag == "new" else (lambda s: s)
        builds[tag] = {fix(dm[f]): ([re.sub(r"`\((\w+)\)", lambda m: "`(" + fix(dm[m.group(1)]) + ")", i) for i in ins], res.get(f, ""))
                       for f, ins in funcs.items()}
    old, new = builds["old"], builds["new"]
    bad = 0
    for name in sorted(old):
        if name not in new:
            print(f"missing    {name}")
            bad += 1
        elif new[name] != old[name]:
            why = "instructions" if new[name][0] != old[name][0] else f"resources {old[name][1]} -> {new[name][1]}"
            print(f"DIFFERENT  {name}: {why}")
            bad += 1
        else:
            print(f"same       {name}  [{len(old[name][0])} instructions; {old[name][1]}]")
    for name in sorted(set(new) - set(old)):
        print(f"new only   {name}  [{len(new[name][0])} instructions; {new[name][1]}]")
    print(f"{len(old)} kernels in the old build: {len(old) - bad} identical, {bad} missing or different; "
          f"{len(set(new) - set(old))} only in the new build")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
