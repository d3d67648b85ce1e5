"""State blob entry points without a GPU: NULL arguments are refused before any device call, and without a device the
four entries fail with SB200_ERR_CUDA -- there is no CPU path -- which the Python wrappers raise as Sb200Error."""
import ctypes as C

import numpy as np
import pytest

ERR_INVALID, ERR_CUDA = -1, -2


@pytest.fixture(scope="module")
def L():
    from similari_b200._lib import lib

    return lib()


@pytest.fixture()
def no_device(L):
    if L.sb200_device_count() > 0:
        pytest.skip("a CUDA device is present: these checks are about the library without one")


def test_null_arguments_are_invalid(L):
    n = C.c_size_t(0)
    h = C.c_void_p()
    blob = np.zeros(4096, np.uint8)
    sc = np.zeros(1, np.uint64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert L.sb200_tracker_save(None, None, 0, C.byref(n)) == ERR_INVALID
    assert L.sb200_tracker_load(None, 4096, 0, C.byref(h)) == ERR_INVALID
    assert L.sb200_tracker_load(vp(blob), 4096, 0, None) == ERR_INVALID
    assert L.sb200_scenes_export(None, 1, vp(sc), 0, None, 0, C.byref(n)) == ERR_INVALID
    assert L.sb200_scenes_import(None, vp(blob), 4096) == ERR_INVALID
    assert L.sb200_tracker_options(None, None, None) == ERR_INVALID


def test_entries_fail_without_a_device(L, no_device):
    n = C.c_size_t(0)
    h = C.c_void_p()
    fake = C.c_void_p(16)   # never dereferenced: the device check comes first
    blob = np.zeros(4096, np.uint8)
    sc = np.zeros(1, np.uint64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert L.sb200_tracker_save(fake, None, 0, C.byref(n)) == ERR_CUDA
    assert L.sb200_tracker_load(vp(blob), len(blob), 0, C.byref(h)) == ERR_CUDA
    assert not h.value
    assert L.sb200_scenes_export(fake, 1, vp(sc), 1, None, 0, C.byref(n)) == ERR_CUDA
    assert L.sb200_scenes_import(fake, vp(blob), len(blob)) == ERR_CUDA


def test_wrappers_raise_without_a_device(L, no_device):
    import similari_b200.api as api
    import similari_b200.engine as engine
    from similari_b200._lib import Sb200Error

    blob = np.zeros(4096, np.uint8)
    with pytest.raises(Sb200Error):
        engine.Tracker.load(blob)
    with pytest.raises(Sb200Error):
        api.load_state(blob)
    t = engine.Tracker.__new__(engine.Tracker)
    t._L, t._h = L, C.c_void_p(16)
    try:
        with pytest.raises(Sb200Error):
            t.save()
        with pytest.raises(Sb200Error):
            t.save_device(0, 0)
        with pytest.raises(Sb200Error):
            t.export_scenes([0], remove=True)
        with pytest.raises(Sb200Error):
            t.import_scenes(blob)
        s = api.BatchSort.__new__(api.BatchSort)
        s._t = t
        with pytest.raises(Sb200Error):
            s.save_state()
        with pytest.raises(Sb200Error):
            s.export_scenes([0])
    finally:
        t._h = None   # not a real tracker: nothing to destroy


def test_blob_options_reads_the_header_without_a_device():
    from similari_b200._lib import Options, Sb200Error
    from similari_b200.engine import blob_options

    o = Options()
    o.kind, o.feature_dim = 3, 96
    blob = np.zeros(1024, np.uint8)
    blob[24: 24 + C.sizeof(Options)] = np.frombuffer(bytes(o), np.uint8)
    got = blob_options(blob)
    assert got.kind == 3 and got.feature_dim == 96
    with pytest.raises(Sb200Error):
        blob_options(blob[:40])
