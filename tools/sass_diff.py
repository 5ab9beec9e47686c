"""Compare the SASS of two builds of libdprb.so kernel by kernel.

    python tools/sass_diff.py OLD/libdprb.so NEW/libdprb.so [--expect-changed SUBSTR ...]

Runs `cuobjdump -sass` on both libraries, splits the listings at `Function :` and compares each kernel's
instructions.  nvcc names a file's anonymous namespace `_GLOBAL__N__<hash>_<len>_<file>_cu_<hash2>`, and both hashes
change whenever the file's text changes, so the whole token is replaced by a fixed one first, and runs of whitespace
are collapsed.  A refactor that should not touch device code passes when every kernel is identical;
kernels that are meant to change are named with --expect-changed (a substring of the mangled name).  Exit code 1 when
a kernel is missing on one side or differs without being expected to.  No GPU is needed.
"""
import argparse
import difflib
import re
import subprocess
import sys

_ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_([0-9]+_\w+?_cu_)?[0-9a-f]{8}")


def kernels(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    out = _ANON.sub("_GLOBAL__N__ANON_", out)
    found = {}
    for part in out.split("Function : ")[1:]:
        name, _, body = part.partition("\n")
        # the function ends where the next ELF section starts
        body = body.split("\n\t\t..........")[0]
        # column padding depends on the longest line of the whole listing: compare whitespace-collapsed lines
        found[name.strip()] = [" ".join(line.split()) for line in body.splitlines() if line.strip()]
    return found


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--expect-changed", nargs="*", default=[], metavar="SUBSTR")
    ap.add_argument("--diff", action="store_true", help="print a unified diff of every changed kernel")
    args = ap.parse_args()
    old, new = kernels(args.old), kernels(args.new)
    bad = 0
    for name in sorted(set(old) | set(new)):
        if name not in old or name not in new:
            print(f"{'ONLY-OLD' if name in old else 'ONLY-NEW'}  {name}")
            bad += 1
            continue
        if old[name] == new[name]:
            print(f"same      {name}")
            continue
        expected = any(s in name for s in args.expect_changed)
        print(f"{'changed ' if expected else 'CHANGED '}  {name}  ({len(old[name])} -> {len(new[name])} lines)")
        bad += 0 if expected else 1
        if args.diff:
            sys.stdout.writelines(l + "\n" for l in difflib.unified_diff(old[name], new[name], "old", "new", lineterm=""))
    print(f"{len(old)} old / {len(new)} new kernels, {bad} unexpected difference(s)")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
