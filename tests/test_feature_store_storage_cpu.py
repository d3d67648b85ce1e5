"""CPU checks of the feature store's storage type (sb200_fstore_set_storage_type / _get_storage_type): the blob header
mirror carries storage_type, and the numpy rounding model the GPU tests compare stored rows with
(fstore_oracle.round_rows) equals numpy's float16 and torch's bfloat16 conversions bit for bit."""
import ctypes as C

import numpy as np
import pytest

import fstore_oracle as fo


def test_blob_header_carries_the_storage_type():
    from similari_b200 import _lib

    names = [n for n, _ in _lib.FstoreBlobHeader._fields_]
    assert "reserved" not in names
    assert names.index("storage_type") == names.index("feature_type") + 1
    assert _lib.FstoreBlobHeader.storage_type.offset == 52 and C.sizeof(_lib.FstoreBlobHeader) == 128
    assert _lib.FSTORE_BLOB_VERSION == 1   # an f32 store's blob is what it was; 0 there is SB200_FEATURE_F32
    assert _lib.FEATURE_F32 == 0


# ------------------------------------------------------------------------------------------------ the rounding model
def _np_f16(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def _torch_bf16(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def _same_or_nan(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    bad = np.flatnonzero(a.view(np.uint32)[~na] != b.view(np.uint32)[~nb])
    assert bad.size == 0, (a[~na][bad[:8]], b[~nb][bad[:8]])


def _all_f16():
    return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32)


def _all_bf16():
    return (np.arange(1 << 16, dtype=np.uint32) << 16).view(np.float32)


EDGES = np.array([
    0.0, -0.0, np.inf, -np.inf, np.nan,
    65504.0, -65504.0, 65519.99, -65519.99, 65520.0, -65520.0, 65536.0, 1e6,
    np.finfo(np.float32).max, -np.finfo(np.float32).max, np.finfo(np.float32).tiny, np.finfo(np.float32).smallest_subnormal,
    2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.0000001, 2.0 ** -26, 3 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -24,
    -(2.0 ** -24), -(2.0 ** -25), -(2.0 ** -26), 1023 * 2.0 ** -24,
    1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -9, 2049.0, 2051.0,
], np.float32)


def _ties():
    """Exact midpoints between neighbours of each type, and the f32 values one ulp either side of them."""
    f16 = _all_f16()
    f16 = f16[np.isfinite(f16)]
    f16 = np.unique(f16.astype(np.float64))
    mid16 = ((f16[:-1] + f16[1:]) / 2).astype(np.float32)
    bf = _all_bf16()
    bf = np.unique(bf[np.isfinite(bf)].astype(np.float64))
    midbf = ((bf[:-1] + bf[1:]) / 2).astype(np.float32)   # exact in f32: bfloat16 neighbours differ by 2^-8 relative
    out = []
    for m in (mid16, midbf):
        out += [m, np.nextafter(m, np.float32(np.inf)), np.nextafter(m, np.float32(-np.inf))]
    return np.concatenate(out)


def test_model_keeps_every_value_of_its_own_type():
    _same_or_nan(fo.round_rows(_all_f16(), "f16"), _all_f16())
    _same_or_nan(fo.round_rows(_all_bf16(), "bf16"), _all_bf16())
    x = np.random.default_rng(0).standard_normal(1000).astype(np.float32)
    assert np.array_equal(fo.round_rows(x, "f32").view(np.uint32), x.view(np.uint32))


@pytest.mark.parametrize("values", ["other_type", "edges", "ties", "random"])
def test_model_equals_numpy_float16(values):
    x = {"other_type": lambda: _all_bf16(), "edges": lambda: EDGES, "ties": _ties,
         "random": lambda: _random_f32(1)}[values]()
    _same_or_nan(fo.round_rows(x, "f16"), _np_f16(x))


@pytest.mark.parametrize("values", ["other_type", "edges", "ties", "random"])
def test_model_equals_torch_bfloat16(values):
    pytest.importorskip("torch")
    x = {"other_type": lambda: _all_f16(), "edges": lambda: EDGES, "ties": _ties,
         "random": lambda: _random_f32(2)}[values]()
    _same_or_nan(fo.round_rows(x, "bf16"), _torch_bf16(x))


def _random_f32(seed):
    """Random bit patterns over the whole f32 range, and values spread around the binary16 range."""
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 1 << 32, 200_000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    scaled = (rng.standard_normal(200_000) * np.exp2(rng.uniform(-30, 18, 200_000))).astype(np.float32)
    return np.concatenate([bits, scaled])


def test_model_edge_values():
    big = np.float32([65504.0, 65519.99, -65519.99, 65520.0, -65520.0])
    assert fo.round_rows(big, "f16").tolist() == [65504.0, 65504.0, -65504.0, np.inf, -np.inf]
    assert fo.round_rows(np.float32([2.0 ** -25, -(2.0 ** -25)]), "f16").view(np.uint32).tolist() == [0, 0x80000000]
    assert fo.round_rows(np.float32([3 * 2.0 ** -25]), "f16")[0] == 2.0 ** -23   # a tie between subnormals goes to even
    assert fo.round_rows(np.float32([np.finfo(np.float32).max]), "bf16")[0] == np.inf
    assert np.isnan(fo.round_rows(np.float32([np.nan]), "f16")[0])
