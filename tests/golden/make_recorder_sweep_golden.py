"""Writes tests/golden/recorder_sweep_reference_digests.npz: name, SHA-256 and length of the compiled reference's
debug_mode report (recorder.h) for every case of tests/recorder_sweep_cases.py.

Needs oracle/_ref/libfslic_ref_recorder.so (make -C oracle -f recorder.mk ref REF=/path/to/fast-slic).  Also checks
that the reference's "standard" and "x64/avx2" contexts give byte-identical reports on every Slic case (preemptive
ones included), which is why one device path serves both Slic and SlicAvx2.

    python tests/golden/make_recorder_sweep_golden.py
"""
import hashlib
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.recorder import RecorderRef  # noqa: E402
from recorder_sweep_cases import CASES, reference_report  # noqa: E402

OUT = os.path.join(HERE, "recorder_sweep_reference_digests.npz")


def main():
    ref = RecorderRef()
    names, digests, lengths = [], [], []
    for case in CASES:
        t = time.time()
        rep = reference_report(case, ref)
        if case.cls == "Slic":
            assert reference_report(case, ref, kind="x64/avx2") == rep, case.name + ": standard and x64/avx2 differ"
        names.append(case.name)
        digests.append(hashlib.sha256(rep).hexdigest())
        lengths.append(len(rep))
        print("%-70s %10d bytes  %s  %.1f s" % (case.name, len(rep), digests[-1][:16], time.time() - t))
    np.savez(OUT, names=np.array(names), sha256=np.array(digests), length=np.array(lengths, np.int64))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
