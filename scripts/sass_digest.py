"""Per-kernel SHA-256 digests of the SASS instructions of the built extension (addresses and encodings stripped):

    python scripts/sass_digest.py [fms_fsdp_b200/_C.so] > tests/golden/sass_before_qk_norm.json

A pull request that must leave existing kernels byte-identical compares these digests before and after
(``tests/test_qk_norm_gpu.py``)."""
import hashlib
import json
import os
import re
import subprocess
import sys


def digests(so):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    per, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            per[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)
        if name and m:
            per[name].append(m.group(1))
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in sorted(per.items())}


if __name__ == "__main__":
    so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(__file__), "..", "fms_fsdp_b200", "_C.so")
    json.dump(digests(so), sys.stdout, indent=0, sort_keys=True)
    sys.stdout.write("\n")
