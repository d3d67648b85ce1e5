"""Feature element types without a GPU: the NULL handle and the wrapper's argument checks."""
import numpy as np
import pytest


def test_null_tracker_is_invalid():
    from similari_b200._lib import FEATURE_BF16, FEATURE_F16, FEATURE_F32, lib

    L = lib()
    for t in (FEATURE_F32, FEATURE_F16, FEATURE_BF16, 7):
        assert L.sb200_set_feature_type(None, t) == -1
    assert L.sb200_last_error()


def test_raw_columns_need_two_byte_elements():
    from similari_b200.engine import FEATURE_TYPES, _raw16

    assert FEATURE_TYPES == {"f32": 0, "f16": 1, "bf16": 2}
    bits = np.arange(16, dtype=np.uint16).reshape(2, 8)
    assert _raw16(bits, "bf16") is bits
    assert _raw16(bits[:, ::2], "f16").flags["C_CONTIGUOUS"]
    with pytest.raises(ValueError):
        _raw16(np.zeros((2, 8), np.float32), "bf16")
    with pytest.raises(ValueError):
        _raw16(bits, "f8")
