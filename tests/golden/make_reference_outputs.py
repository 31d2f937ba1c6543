"""Generates tests/golden/reference_outputs.json: what the UNMODIFIED reference (oracle/_ref, built by
oracle/Makefile from the reference's sources) returns for every comparison the GPU tests, smoke() and
bench.py make, stored as exact digests (tests/zref.py: digest) so that those comparisons need no copy of
the reference where they run.  Each module below lists its own reference calls in reference_outputs(ref).
Run from the repository root after `make -C oracle all`:  python tests/golden/make_reference_outputs.py
With module names as arguments only those modules' calls are made, and their keys are merged into the
existing file (every other key is kept as it is):  python tests/golden/make_reference_outputs.py test_gpu_block_plan
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zref  # noqa: E402

MODULES = ["__graft_entry__", "bench", "test_gpu_parity", "test_gpu_parity_at_size", "test_gpu_integer_window",
           "test_gpu_multi", "test_gpu_block_plan", "test_gpu_large_range"]


def main(names):
    unknown = [n for n in names if n not in MODULES]
    assert not unknown, "not in MODULES: %s" % unknown
    ref = zref.Ref()
    out = {}
    for name in names or MODULES:
        mod = __import__(name)
        for key, value in mod.reference_outputs(ref):
            assert key not in out, key
            out[key] = zref.digest(value)
            print(key, flush=True)
    made = len(out)
    if names:
        with open(zref.REFERENCE_OUTPUTS) as f:
            old = json.load(f)
        out = dict(old, **out)
    with open(zref.REFERENCE_OUTPUTS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "entries,", made, "of them made now")


if __name__ == "__main__":
    main(sys.argv[1:])
