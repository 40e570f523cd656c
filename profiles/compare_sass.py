#!/usr/bin/env python3
"""Compare the kernels of two builds of csrc/ instruction by instruction.

    python3 profiles/compare_sass.py BUILD_A BUILD_B

Each argument is a directory holding the .o files of one `make -C staticmapping_b200/csrc`.  Every kernel of every
object is disassembled with `cuobjdump -sass`, matched across the two builds by demangled name (so a kernel that
moved to another translation unit still finds its partner), and its instruction stream compared with addresses and
encodings stripped.  Prints one JSON object: the kernels that differ, those found on one side only, and the number
that are identical.  No GPU involved; it reads the two directories and nothing else.
"""
import glob
import json
import os
import re
import subprocess
import sys


def kernels(build_dir):
    out = {}
    for obj in sorted(glob.glob(os.path.join(build_dir, "*.o"))):
        text = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
        name = None
        for line in text.splitlines():
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                name = m.group(1)
                out[name] = []
                continue
            if name is None:
                continue
            code = re.sub(r"/\*.*?\*/", "", line).strip()
            if code and not code.startswith("."):
                out[name].append(code)
    names = list(out)
    plain = subprocess.run(["cu++filt"] + names, check=True, capture_output=True, text=True).stdout.splitlines()
    return {p: out[n] for n, p in zip(names, plain)}


def main():
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    both = sorted(set(a) & set(b))
    print(json.dumps({
        "identical": sum(a[k] == b[k] for k in both),
        "differ": [{"kernel": k, "instructions": [len(a[k]), len(b[k])]} for k in both if a[k] != b[k]],
        "only_in_a": sorted(set(a) - set(b)),
        "only_in_b": sorted(set(b) - set(a)),
    }, indent=1))


if __name__ == "__main__":
    main()
