"""Does a change leave existing kernels' machine code alone?  Compares the SASS of two builds of the same object, kernel by
kernel, with the names set aside (a new template parameter or a renumbered ScanMode renames an instantiation without
changing its code): every kernel body of OLD must appear, instruction for instruction, in NEW.  Kernels only NEW has are
counted as new.  Exit status 1 if some body of OLD is missing.  Needs cuobjdump (no GPU).

    git worktree add /tmp/parent HEAD~1 && (cd /tmp/parent && python -m nornicdb_b200.build)
    python -m nornicdb_b200.build
    for f in scan_simt scan_tensor scan_tensor_shadow; do
        python profiles/sass_unchanged.py /tmp/parent/nornicdb_b200/build/$f.o nornicdb_b200/build/$f.o
    done"""
from __future__ import annotations

import collections
import hashlib
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def kernel_bodies(obj: str) -> dict:
    """mangled name -> sha256 of its SASS instructions and their encodings (addresses dropped)"""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name and re.match(r"\s+(/\*[0-9a-f]{4,}\*/|/\* 0x[0-9a-f]+ \*/)", line):
            # instruction text and both 64-bit halves of its encoding (operands, scheduling and reuse bits), not its address
            funcs[name].append(re.sub(r"\s+", " ", re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)).strip())
    return {n: hashlib.sha256("\n".join(b).encode()).hexdigest() for n, b in funcs.items()}


def main() -> int:
    if len(sys.argv) != 3:
        print(__doc__)
        return 2
    old, new = kernel_bodies(sys.argv[1]), kernel_bodies(sys.argv[2])
    pool = collections.Counter(new.values())
    missing = []
    for name, h in old.items():
        if pool[h]:
            pool[h] -= 1
        else:
            missing.append(name)
    print(f"{os.path.basename(sys.argv[1])}: {len(old)} kernels, {len(old) - len(missing)} with unchanged SASS, "
          f"{len(missing)} changed; {sum(pool.values())} new")
    for name in missing:
        print("  changed:", name)
    return 1 if missing else 0


if __name__ == "__main__":
    sys.exit(main())
