#!/usr/bin/env python
"""Is the built extension the code the evidence shows?  Compares the instruction stream of every kernel in
atomo_b200/_C*.so (cuobjdump -sass) with the committed manifest profiles/sass/kernels.json (instruction count and
SHA-256 of the normalised instruction text per kernel, taken from the sm_90a build that ran the GPU tests and the
benchmark on the H100).  Exit code 1 on any difference; run after touching a .cu file, and refresh the manifest
with `--update` when the change is intended."""
import glob
import hashlib
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MANIFEST = os.path.join(ROOT, "profiles", "sass", "kernels.json")


def kernel_key(mangled):
    """stable short name: v2 kernels are prefixed with 'v2_' (their namespace), e.g. v2_v2_ps_kernel"""
    m = re.match(r"_ZN5atomo(2v2)?(\d+)", mangled)
    if not m:
        return mangled
    name = mangled[m.end():m.end() + int(m.group(2))]
    return ("v2_" + name) if m.group(1) else name


def built_kernels(so):
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        head, _, body = part.partition("\n")
        ins = [re.sub(r"\s+", " ", m.group(1)).strip()
               for m in re.finditer(r"^\s*/\*[0-9a-f]{4,5}\*/\s+(.*?)\s*;", body, re.M)]
        funcs[kernel_key(head.strip())] = {"instructions": len(ins),
                                           "sha256": hashlib.sha256("\n".join(ins).encode()).hexdigest()}
    return funcs


def main():
    so = glob.glob(os.path.join(ROOT, "atomo_b200", "_C*.so"))
    if not so:
        print("no built extension (python setup.py build_ext --inplace)")
        return 2
    cur = built_kernels(so[0])
    if "--update" in sys.argv[1:]:
        os.makedirs(os.path.dirname(MANIFEST), exist_ok=True)
        with open(MANIFEST, "w") as f:
            json.dump(dict(sorted(cur.items())), f, indent=1)
            f.write("\n")
        print("wrote %d kernels to %s" % (len(cur), MANIFEST))
        return 0
    with open(MANIFEST) as f:
        ref = json.load(f)
    bad = 0
    for name, want in sorted(ref.items()):
        got = cur.get(name)
        if got is None:
            print("%-34s not in the binary" % name)
            bad += 1
        elif got != want:
            print("%-34s DIFFERS (%d committed, %d built instructions)" % (name, want["instructions"], got["instructions"]))
            bad += 1
        else:
            print("%-34s %5d instructions identical" % (name, want["instructions"]))
    for name in sorted(set(cur) - set(ref)):
        print("%-34s built but not in the manifest" % name)
        bad += 1
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
