"""CPU checks of the batched NMS entry points: argument validation comes before anything else (so it holds with or
without a GPU), and without a GPU both entries fail loudly."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def _call(L, entry, n_sets, offsets, boxes, idx, counts):
    from similari_b200._lib import ptr

    args = [n_sets, ptr(offsets), ptr(boxes), None, 0.5, 0.0, 0, ptr(idx), ptr(counts), None, 0]
    if entry == "sb200_nms_batch_device":
        args.append(None)
    return getattr(L, entry)(*args)


@pytest.mark.parametrize("entry", ["sb200_nms_batch", "sb200_nms_batch_device"])
def test_no_cpu_fallback(L, entry):
    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present; the loud-failure path is for CPU-only machines")
    offsets = np.array([0, 2, 3], np.int32)
    boxes = np.ones((3, 6), np.float32)
    idx, counts = np.zeros(3, np.int32), np.zeros(2, np.int32)
    assert _call(L, entry, 2, offsets, boxes, idx, counts) == -2
    assert b"no CUDA device" in L.sb200_last_error()


@pytest.mark.parametrize("entry", ["sb200_nms_batch", "sb200_nms_batch_device"])
@pytest.mark.parametrize("n_sets,offsets", [
    (2, [0, 3, 2]),        # not monotone
    (3, [0, 2, 2, 1]),     # not monotone after an empty set
    (2, [1, 2, 3]),        # offsets[0] != 0
    (-1, [0]),             # n_sets < 0
])
def test_bad_offsets_are_invalid(L, entry, n_sets, offsets):
    offsets = np.array(offsets, np.int32)
    boxes = np.ones((4, 6), np.float32)
    idx = np.full(4, 7, np.int32)
    counts = np.full(4, 7, np.int32)
    assert _call(L, entry, n_sets, offsets, boxes, idx, counts) == -1
    assert L.sb200_last_error()
    assert np.all(idx == 7) and np.all(counts == 7)


@pytest.mark.parametrize("entry", ["sb200_nms_batch", "sb200_nms_batch_device"])
def test_missing_pointers_are_invalid(L, entry):
    offsets = np.array([0, 2], np.int32)
    boxes = np.ones((2, 6), np.float32)
    idx, counts = np.zeros(2, np.int32), np.zeros(1, np.int32)
    assert _call(L, entry, 1, offsets, None, idx, counts) == -1
    assert _call(L, entry, 1, offsets, boxes, None, counts) == -1
    assert _call(L, entry, 1, offsets, boxes, idx, None) == -1
    assert _call(L, entry, 1, None, boxes, idx, counts) == -1
    # an empty request needs no box or index buffer
    empty = np.array([0, 0], np.int32)
    if entry == "sb200_nms_batch_device" and L.sb200_device_count() > 0:
        # the device entry writes its counts on the device: give it device memory
        import torch

        from similari_b200._lib import ptr

        d_counts = torch.full((1,), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        rc = L.sb200_nms_batch_device(1, ptr(empty), None, None, 0.5, 0.0, 0, None, d_counts.data_ptr(), None, 0, None)
        torch.cuda.synchronize()
        assert rc == 0 and int(d_counts[0]) == 0
        return
    rc = _call(L, entry, 1, empty, None, None, counts)
    assert rc in (0, -2) and (rc == 0) == (L.sb200_device_count() > 0)


def test_engine_nms_batch_checks_offsets_against_boxes():
    import similari_b200.engine as eng

    boxes = np.ones((3, 6), np.float32)
    with pytest.raises(ValueError):
        eng.nms_batch(boxes, None, [0, 2], 0.5)
    with pytest.raises(ValueError):
        eng.nms_batch(boxes, None, [], 0.5)
    with pytest.raises(ValueError):
        eng.nms_batch(boxes, np.ones(2, np.float32), [0, 3], 0.5)


def test_api_exposes_nms_batch():
    import similari_b200.api as api

    assert callable(api.nms_batch) and "no PyO3 counterpart" in api.nms_batch.__doc__
