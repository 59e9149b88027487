#!/usr/bin/env python
"""Regenerate tests/golden/tp_source_sha256.json (run from the repository root:
``python tests/golden/make_tp_source_hashes.py``).

The fixture holds the SHA-256 of the TP kernel source that ``codegen.generate`` emits for a set of signatures in both
layouts, leading comment block stripped; ``tests/test_presets.py::test_single_block_signatures_generate_the_same_source``
checks that the generator still emits exactly that source.  The committed file pins the signatures that were prebuilt
before the preset architectures (all with one fp32 channel block, so their work items are the plain
(path group, channel block) grid).  The script rewrites the hashes of the signatures already in the file; run it only
when a change to their generated kernels is intended, and say so in the change."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from nequip_b200 import known_signatures as ks  # noqa: E402
from nequip_b200.codegen import GenOptions, generate  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tp_source_sha256.json")


def body(src: str) -> str:
    """The generated source without its leading comment block (generator version, signature, decomposition)."""
    lines = src.split("\n")
    i = 0
    while lines[i].startswith("//"):
        i += 1
    return "\n".join(lines[i:])


def main():
    with open(OUT) as f:
        keys = sorted(json.load(f))
    known = {s.canonical(): s for s in ks.all_known()}
    out = {}
    for key in keys:
        layout, canon = key.split("|", 1)
        out[key] = hashlib.sha256(body(generate(known[canon], GenOptions(layout=layout))).encode()).hexdigest()
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} hashes -> {OUT}")


if __name__ == "__main__":
    main()
