"""Write tests/golden/ref_pinned.json: for every case of tests/ref_cases.py, the digest of its inputs, of every cloud the
reference's own code published on them (oracle/_ref/libref_*.so, built by build() where the reference tree is present) and the q
it published with.  test_ref_pinned_cpu.py checks the file against the libraries wherever they are built; test_gpu_ref_pinned.py
checks the device against the file."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ref_cases as RC  # noqa: E402


def build_entries():
    return {c.id: RC.record(c.inputs, c.reference()) for c in RC.all_cases(RC.make_world_small())}


if __name__ == "__main__":
    cases = build_entries()
    with open(RC.GOLDEN, "w") as fh:      # one case per line
        fh.write('{"about": "SHA-256 of the reference\'s published clouds (NaNs canonical) per case of tests/ref_cases.py",\n')
        fh.write(' "cases": {\n')
        fh.write(",\n".join(f"  {json.dumps(k)}: {json.dumps(cases[k], sort_keys=True)}" for k in sorted(cases)))
        fh.write("\n }}\n")
    print(f"{len(cases)} cases -> {RC.GOLDEN}")
