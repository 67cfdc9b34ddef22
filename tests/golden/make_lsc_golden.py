"""Generates tests/golden/lsc_reference_digests.npz from the UNMODIFIED reference's ContextLSC run with num_threads = 1
(oracle_lsc/_ref/libfslic_ref_lsc.so, oracle_lsc/Makefile).  With a checkout of Algy/fast-slic at hand:

    FSLIC_REFERENCE=/path/to/fast-slic python tests/golden/make_lsc_golden.py

Inputs are seeded synthetic images (tests/lsc_cases.py), so only the SHA-256 of every array the reference returns is
stored, under "lsc/<case>/<name>" (tests/lsc_cases.py::lsc_reference_outputs).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from cases import digest  # noqa: E402
from lsc_cases import lsc_reference_outputs  # noqa: E402
from oracle_lsc.lsc import Ref  # noqa: E402


def main():
    keys, sha = [], []
    for prefix, outputs in lsc_reference_outputs(Ref()):
        for name, arr in outputs.items():
            keys.append("%s/%s" % (prefix, name))
            sha.append(np.frombuffer(digest(arr), np.uint8))
    path = os.path.join(HERE, "lsc_reference_digests.npz")
    np.savez_compressed(path, keys=np.array(keys), sha=np.stack(sha))
    print("wrote", len(keys), "digests,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
