"""Generates tests/golden/cca_reference_digests.npz from the UNMODIFIED reference's connectivity enforcement
(oracle/_ref/libfslic_ref.so, oracle/Makefile).  With a checkout of Algy/fast-slic at hand:

    FSLIC_REFERENCE=/path/to/fast-slic python tests/golden/make_cca_golden.py

Inputs are the seeded label maps of tests/cca_cases.py, so only the SHA-256 of every array the reference returns is
stored, under "cca_maps/<case>/labels" (tests/cca_cases.py::cca_reference_outputs).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from cases import digest  # noqa: E402
from cca_cases import cca_reference_outputs  # noqa: E402
from oracle.oracle import Ref  # noqa: E402


def main():
    keys, sha = [], []
    for prefix, outputs in cca_reference_outputs(Ref(), num_threads=2):
        for name, arr in outputs.items():
            keys.append("%s/%s" % (prefix, name))
            sha.append(np.frombuffer(digest(arr), np.uint8))
    path = os.path.join(HERE, "cca_reference_digests.npz")
    np.savez_compressed(path, keys=np.array(keys), sha=np.stack(sha))
    print("wrote", len(keys), "digests,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
