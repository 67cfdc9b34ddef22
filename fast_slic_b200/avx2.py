"""Import compatibility with fast-slic/fast_slic/avx2.py:1-14: code written against ``fast_slic.avx2.SlicAvx2`` (the
reference's fastest arch, the one BASELINE quotes) switches to this package by changing the import only.  Same engine as
``fast_slic_b200.Slic``: the results are bit-identical to the reference's AVX2 context."""
from .base_slic import LSC, Slic


class SlicAvx2(Slic):
    """== fast_slic.avx2.SlicAvx2 (avx2.py:10-11), on the CUDA engine."""


class LSCAvx2(LSC):
    """== fast_slic.avx2.LSCAvx2 (avx2.py:13-14).  iterate() raises NotImplementedError: the reference's AVX2 LSC context
    normalises with _mm256_rcp_ps (arch/x64/avx2.h), an approximate reciprocal whose bits differ between CPU vendors,
    so there is no single result to reproduce.  LSC(num_threads=1) is the defined one."""

    def make_slic_model(self, num_components):
        model = super(LSCAvx2, self).make_slic_model(num_components)
        model.lsc_arch = "x64/avx2"
        return model
