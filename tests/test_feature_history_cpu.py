"""Feature history entry points without a GPU: argument errors, the no-GPU failure, and the lazy conversion of the packed
arrays into WastedVisualSortTrack.observed_features."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    from similari_b200._lib import lib

    return lib()


def test_null_tracker_and_arguments_are_invalid(L):
    from similari_b200._lib import lib

    assert L.sb200_set_feature_history(None, 1) == -1
    assert L.sb200_feature_history_pool(None, None) == -1
    buf = np.zeros(8, np.float32)
    pres = np.zeros(8, np.uint8)
    assert L.sb200_wasted_visual(None, 1, None, None, None, None, None, None, 1, None, None, None,
                                 buf.ctypes.data_as(C.c_void_p), pres.ctypes.data_as(C.c_void_p)) == -1
    assert lib().sb200_last_error()


def test_no_gpu_failure(L):
    from similari_b200._lib import default_options

    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present; the loud-failure path is for CPU-only machines")
    o = default_options(kind=2, feature_dim=8)
    h = C.c_void_p()
    assert L.sb200_tracker_create(C.byref(o), C.byref(h)) == -2 and h.value is None


def test_api_visual_trackers_reach_the_device(L):
    """Without a GPU the API's visual trackers fail loudly at their first predict; there is no CPU path."""
    import similari_b200.api as sim
    from similari_b200._lib import Sb200Error

    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present")
    t = sim.VisualSort(1, sim.VisualSortOptions())
    assert t.wasted() == []   # nothing created yet
    s = sim.VisualSortObservationSet()
    s.add(sim.VisualSortObservation([0.1, 0.2], 0.9, sim.Universal2DBox(1.0, 2.0, None, 0.5, 10.0), None))
    with pytest.raises(Sb200Error):
        t.predict(s)


def test_observed_features_from_packed_rows():
    import similari_b200.api as sim

    b = sim.Universal2DBox(1.0, 2.0, None, 0.5, 10.0)
    rows = np.zeros((3, 8), np.float32)
    rows[0, :3] = [0.1, -0.0, 3.0]
    rows[2, :2] = [np.float32(1e-40), np.float32(2.5)]   # a subnormal survives as its f32 value
    present = np.array([True, False, True])
    w = sim.WastedVisualSortTrack(7, 3, b, b, 0, 3, [b, b, b], [b, b, b], rows, present)
    assert isinstance(w, sim.WastedSortTrack)
    feats = w.observed_features
    assert feats[1] is None
    assert feats[0] == [float(np.float32(0.1)), 0.0, 3.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    assert np.signbit(feats[0][1])   # -0.0 kept
    assert feats[2][0] == float(np.float32(1e-40)) and feats[2][1] == 2.5
    assert all(type(x) is float for x in feats[0])
    assert w.observed_features is feats   # converted once
    assert len(feats) == len(w.observed_boxes)
    empty = sim.WastedVisualSortTrack(8, 1, b, b, 0, 1)
    assert empty.observed_features == []
