"""Per-kernel digest of the SASS in libtloam_b200.so (cuobjdump -sass; no GPU needed).

A feature that adds kernels must leave the instructions of the existing ones alone; tests/golden/sass_digests.json holds
the digests of every kernel of the commit before the global map was added, and test_global_map.py compares against it.

    python tests/sass_digest.py > tests/golden/sass_digests.json      # regenerate (only when a kernel is meant to change)
"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tloam_b200", "libtloam_b200.so")


def cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


def digests(lib=LIB):
    """{mangled kernel name: sha256 of its instruction text}"""
    sass = subprocess.run([cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        ins = re.findall(r"^\s+/\*[0-9a-f]+\*/\s+([^;]*;)", block, flags=re.M)
        out[name] = hashlib.sha256("\n".join(i.strip() for i in ins).encode()).hexdigest()
    return out


if __name__ == "__main__":
    json.dump(digests(sys.argv[1] if len(sys.argv) > 1 else LIB), sys.stdout, indent=1, sort_keys=True)
    sys.stdout.write("\n")
