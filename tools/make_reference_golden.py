"""Stores what the reference's own code returns for the seeded cases of tests/test_alias_oracle.py and
tests/test_scene_pinning.py in tests/golden/reference_alias.npz and tests/golden/reference_scene.npz, so that those
tests compare against the reference without it. Needs oracle/_ref/libref_alias.so and libref_scene.so
(oracle/ref_alias/build.sh, oracle/ref_scene/build.sh: the reference tree must be present).

    python tools/make_reference_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import orc  # noqa: E402
from tests import test_alias_oracle, test_scene_pinning  # noqa: E402


def main():
    reflib = orc.load_ref()
    if reflib is None:
        raise SystemExit("oracle/_ref/libref_alias.so is missing: build it from the reference tree first")
    np.savez_compressed(test_alias_oracle.GOLDEN_REF, **test_alias_oracle.reference_alias_outputs(reflib))
    ref = orc.load_ref_scene()
    if ref is None:
        raise SystemExit("oracle/_ref/libref_scene.so is missing: build it from the reference tree first")
    np.savez_compressed(test_scene_pinning.GOLDEN, **test_scene_pinning.reference_scene_outputs(ref))
    for p in (test_alias_oracle.GOLDEN_REF, test_scene_pinning.GOLDEN):
        print("wrote", os.path.relpath(p, ROOT), os.path.getsize(p), "bytes")


if __name__ == "__main__":
    main()
