#!/usr/bin/env python3
"""Per-kernel SASS comparison of two builds of libglim_b200.so (or of two .o / .cubin files): proves, without a GPU, that a
refactor of the sources left the generated code of every kernel unchanged.  Kernels are matched by mangled name with the
translation-unit hash of anonymous namespaces normalised; function order and trailing blank lines are ignored.

    python scripts/sass_identity.py old/libglim_b200.so glim_b200/libglim_b200.so

Used in round 2 when the per-point arithmetic moved into gb_vgicp_math.cuh (every kernel identical).  Measurement plumbing."""
import hashlib
import re
import subprocess
import sys


def kernels(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], text=True, capture_output=True, check=True).stdout
    txt = re.sub(r"_GLOBAL__N__[0-9a-f]+_[0-9]+_[A-Za-z_0-9]+_cu_[0-9a-f]+", "ANON", txt)
    txt = re.sub(r"_ZN\d+ANON", "_ZNxxANON", txt)
    out = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name, body = part.split("\n", 1)
        body = body.split("\nFatbin ", 1)[0]  # the last function of a cubin is followed by the next fatbin section's header
        # runs of blanks collapse: cuobjdump pads its columns to the widest instruction of the cubin, so a new kernel in the
        # same translation unit would otherwise change the text of every other kernel there
        body = "\n".join(" ".join(l.split()) for l in body.splitlines() if l.strip())
        out[name.strip()] = hashlib.sha256(body.encode()).hexdigest()
    return out


def main():
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    only_a, only_b = sorted(set(a) - set(b)), sorted(set(b) - set(a))
    diff = sorted(k for k in a if k in b and a[k] != b[k])
    print(f"{len(a)} / {len(b)} kernels; only in first: {len(only_a)}, only in second: {len(only_b)}, differing: {len(diff)}")
    for k in only_a + only_b + diff:
        print("  ", subprocess.run(["c++filt", k], text=True, capture_output=True).stdout.strip()[:160])
    return 1 if (only_a or only_b or diff) else 0


if __name__ == "__main__":
    sys.exit(main())
