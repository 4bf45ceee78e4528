#!/usr/bin/env python
"""Per-kernel SASS fingerprints of libepropnp_b200.so, and the check that the kernels which were validated on
hardware (the GPU parity suite) are still bit-identical in the current default build.

    python tools/sass_identity.py                 # compare the in-tree library with profiles/validated_sass.json
    python tools/sass_identity.py --write <lib>   # record a library's fingerprints as the validated set

Experiments live behind build options and new entry points get new kernels, so the validated kernels must not change
unless a GPU run re-validates them (then the manifest is rewritten in the same commit)."""
import hashlib
import json
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MANIFEST = os.path.join(REPO, "profiles", "validated_sass.json")
DEFAULT_LIB = os.path.join(REPO, "epro-pnp_b200", "lib", "libepropnp_b200.so")


def fingerprints(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_pnp_kernels_cu_[0-9a-f]{8}", "", part.split("\n")[0].strip())
        body = [re.sub(r"/\*[0-9a-fx ]+\*/", "", l).strip() for l in part.split("\n")[1:]
                if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
        out[name] = dict(instructions=len(body), sha1=hashlib.sha1("\n".join(body).encode()).hexdigest())
    return out


def compare(lib=DEFAULT_LIB):
    want = json.load(open(MANIFEST))["kernels"]
    have = fingerprints(lib)
    changed = sorted(k for k in want if have.get(k, {}).get("sha1") != want[k]["sha1"])
    added = sorted(k for k in have if k not in want)
    return changed, added


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--write":
        json.dump(dict(note="SASS fingerprints of the sm_90a kernels validated on an H100 (GPU parity suite green on "
                            "exactly this build)", kernels=fingerprints(sys.argv[2])),
                  open(MANIFEST, "w"), indent=1, sort_keys=True)
        print("wrote", MANIFEST)
    else:
        changed, added = compare(sys.argv[1] if len(sys.argv) > 1 else DEFAULT_LIB)
        print(json.dumps(dict(validated_kernels_changed=changed, kernels_without_hardware_validation=added), indent=1))
        sys.exit(1 if changed else 0)
