"""Generates tests/golden/random_step_reference_outputs.json: what the UNMODIFIED reference (oracle/_ref, built by
oracle/Makefile from the reference's sources) returns for the random-step and log-table cases of
tests/test_gpu_random_steps.py (inputs from tests/random_step_fixtures.py): store and stream digests
(tests/zref.py: digest) and every block's cost sequence, so that the GPU tests need no copy of the reference where
they run.
Run from the repository root after `make -C oracle all`:  python tests/golden/make_random_step_reference_outputs.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zref  # noqa: E402

OUTPUTS = os.path.join(ROOT, "tests", "golden", "random_step_reference_outputs.json")


def main():
    import test_gpu_random_steps
    ref = zref.Ref()
    out = {}
    for key, value in test_gpu_random_steps.reference_outputs(ref):
        assert key not in out, key
        out[key] = zref.digest(value)
        print(key, flush=True)
    with open(OUTPUTS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "entries")


if __name__ == "__main__":
    main()
