"""Compare the SASS of every kernel function of two builds of an object file or library, function by function.

    python scripts/compare_sass.py OLD.o NEW.o [--rename 'Lb0EEv=EEv' ...] [--demangle --rename ', c2v::ThreePass>=>']

A change that adds a kernel (a new template instantiation, a new mode behind `if constexpr`) should leave the code of
every existing kernel as it was.  Functions are matched by mangled name; --rename OLD=NEW rewrites substrings of the new
build's names first (e.g. a template parameter with a default value, appended to every instantiation: 'ELb0EEv=EEv').
--demangle matches demangled names (cu++filt) instead: a defaulted type argument shifts the substitution indices of the
mangled name, which a substring rewrite cannot undo.
Constant-bank addresses (kernel parameters move when a parameter is added) and line-info comments are normalised.
Exit status 1 when a function of the old build is missing from the new one or differs.  Needs cuobjdump (CUDA toolkit).
"""
import argparse
import re
import subprocess
import sys


def sass_functions(path):
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            name, body = m.group(1), []
            continue
        if name is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\*", line)
        if m:
            ins = re.sub(r"c\[0x[0-9a-f]+\]\[0x[0-9a-f]+\]", "c[.][.]", m.group(1))
            body.append(ins)
    if name:
        funcs[name] = body
    return funcs


def demangled(funcs):
    names = list(funcs)
    out = subprocess.run(["cu++filt"], input="\n".join(names), check=True, capture_output=True, text=True).stdout
    return {d: funcs[n] for n, d in zip(names, out.splitlines())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", action="append", default=[], help="OLD=NEW substring rewrite of the new build's names")
    ap.add_argument("--demangle", action="store_true", help="match demangled names")
    a = ap.parse_args()
    old, new = sass_functions(a.old), sass_functions(a.new)
    if a.demangle:
        old, new = demangled(old), demangled(new)
    renamed = {}
    for k, v in new.items():
        for r in a.rename:
            src, dst = r.split("=", 1)
            if k not in old:
                k = k.replace(src, dst)
        renamed[k] = v
    bad = 0
    for k, body in sorted(old.items()):
        if k not in renamed:
            print(f"MISSING  {k}")
            bad += 1
        elif renamed[k] != body:
            print(f"DIFFERS  {k} ({len(body)} -> {len(renamed[k])} instructions)")
            bad += 1
    added = sorted(set(renamed) - set(old))
    print(f"{len(old)} functions in the old build, {len(old) - bad} identical, {bad} missing or different; "
          f"{len(added)} new: {' '.join(added)}")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
