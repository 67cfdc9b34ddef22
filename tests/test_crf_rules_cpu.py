"""SimpleCRF argument conversions that need no device: Cython's TypeError / OverflowError for the reference's size_t
arguments, and the 2^31 limits of the sizes."""
import pytest


def test_sizes_convert_like_cython_size_t():
    from fast_slic_b200.crf import SimpleCRF
    for bad in ((3.0, 4), (3, "4"), (None, 4)):
        with pytest.raises(TypeError):
            SimpleCRF(*bad)
    for bad in ((-1, 4), (3, -1), (2 ** 64, 1)):
        with pytest.raises(OverflowError):
            SimpleCRF(*bad)


def test_sizes_beyond_int32_are_refused_not_truncated():
    from fast_slic_b200.crf import SimpleCRF
    for bad in ((1, 2 ** 32 + 3), (0, 2 ** 40), (2 ** 16, 2 ** 16)):
        with pytest.raises(ValueError, match="2\\^31"):
            SimpleCRF(*bad)
