"""Per-kernel SHA-256 digests of the SASS instructions of the built extension (addresses and encodings stripped):

    python scripts/sass_digest.py [fms_fsdp_b200/_C.so] > tests/golden/sass_kernels.json

``tests/test_sass.py`` holds every kernel of ``_C.so`` to ``tests/golden/sass_kernels.json``.  A change that means to
change, add or remove kernels regenerates that file with this script in the same commit, so that the JSON diff names
every kernel whose instructions changed."""
import hashlib
import json
import os
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def parse(sass):
    """{kernel: [instruction text]} of a ``cuobjdump -sass`` listing, without addresses and encodings."""
    per, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            per[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)
        if name and m:
            per[name].append(m.group(1))
    return per


def digests(per):
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in sorted(per.items())}


if __name__ == "__main__":
    so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(__file__), "..", "fms_fsdp_b200", "_C.so")
    out = subprocess.run([CUOBJDUMP, "-sass", so], capture_output=True, text=True, check=True).stdout
    json.dump(digests(parse(out)), sys.stdout, indent=0, sort_keys=True)
    sys.stdout.write("\n")
