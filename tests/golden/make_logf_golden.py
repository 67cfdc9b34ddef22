"""Generates tests/golden/logf_reference_digests.npz from glibc's logf (oracle_crf/crf_oracle.c's orcl_logf_range):

    python tests/golden/make_logf_golden.py

"logf/all" is the SHA-256 of glibc logf over all 2^32 float bit patterns in order (float32, little endian), the
function the CRF's unary setters evaluate (fast_slic_b200/csrc/glibc_logf.cuh clones it).  About half a minute.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle_crf.crf import glibc_logf_range  # noqa: E402


def logf_stream_digest(chunk_fn, chunk=1 << 26):
    h = hashlib.sha256()
    for first in range(0, 1 << 32, chunk):
        h.update(chunk_fn(first, chunk).tobytes())
    return h.digest()


def main():
    path = os.path.join(HERE, "logf_reference_digests.npz")
    np.savez_compressed(path, keys=np.array(["logf/all"]),
                        sha=np.frombuffer(logf_stream_digest(glibc_logf_range), np.uint8)[None])
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
