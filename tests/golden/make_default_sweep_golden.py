"""Generates tests/golden/default_sweep_reference_digests.npz from the UNMODIFIED reference: the default integer path
with the Manhattan spatial term (oracle/_ref/libfslic_ref.so, oracle/Makefile) and with the Euclidean one
(oracle_euclid/_ref/libfslic_ref_euclid.so, oracle_euclid/Makefile), each in both arch contexts.  With a checkout of
Algy/fast-slic at hand:

    FSLIC_REFERENCE=/path/to/fast-slic python tests/golden/make_default_sweep_golden.py

Inputs are seeded synthetic images (tests/default_sweep_cases.py), so only the SHA-256 of every array the reference
returns is stored, under "<arch>/<family>/<group>/<case>/<name>".
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from cases import digest  # noqa: E402
from default_sweep_cases import default_sweep_reference_outputs  # noqa: E402
from oracle.oracle import Ref  # noqa: E402
from oracle_euclid.euclid import Ref as EuclidRef  # noqa: E402


def main():
    keys, sha = [], []
    for prefix, outputs in default_sweep_reference_outputs(Ref(), EuclidRef()):
        for name, arr in outputs.items():
            keys.append("%s/%s" % (prefix, name))
            sha.append(np.frombuffer(digest(arr), np.uint8))
    path = os.path.join(HERE, "default_sweep_reference_digests.npz")
    np.savez_compressed(path, keys=np.array(keys), sha=np.stack(sha))
    print("wrote", len(keys), "digests,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
