"""Generates tests/golden/crf_reference_digests.npz from the UNMODIFIED reference's SimpleCRF
(oracle_crf/_ref/libfslic_ref_crf.so, oracle_crf/Makefile) and glibc's expf.  With a checkout of Algy/fast-slic at hand:

    FSLIC_REFERENCE=/path/to/fast-slic python tests/golden/make_crf_golden.py

The cases are seeded scripts (tests/crf_cases.py), so only the SHA-256 of every array the reference returns is stored,
under "crf/<case>/<snapshot>/<frame>/<name>"; "expf/all" is the digest of glibc expf over all 2^32 float bit patterns
in order (float32, little endian).
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from cases import digest  # noqa: E402
from crf_cases import CRF_CASES, run_case  # noqa: E402
from oracle_crf.crf import Ref, glibc_expf_range  # noqa: E402


def expf_stream_digest(chunk_fn, chunk=1 << 26):
    h = hashlib.sha256()
    for first in range(0, 1 << 32, chunk):
        h.update(chunk_fn(first, chunk).tobytes())
    return h.digest()


def main():
    keys, sha = [], []
    for case in CRF_CASES:
        for name, arr in run_case(Ref(case[1], case[2]), case).items():
            keys.append("crf/%s/%s" % (case[0], name))
            sha.append(np.frombuffer(digest(arr), np.uint8))
    keys.append("expf/all")
    sha.append(np.frombuffer(expf_stream_digest(glibc_expf_range), np.uint8))
    path = os.path.join(HERE, "crf_reference_digests.npz")
    np.savez_compressed(path, keys=np.array(keys), sha=np.stack(sha))
    print("wrote", len(keys), "digests,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
