"""CPU checks of sb200_fstore_associate_wasted: NULL handles and bad arguments return SB200_ERR_INVALID without
touching a device; the Python wrapper validates its arguments before any call."""
import ctypes as C

import pytest



@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def _call(L, s, t, cap=1, history_cap=1):
    return L.sb200_fstore_associate_wasted(s, t, cap, 0, *([None] * 6), history_cap, *([None] * 10))


def test_null_handles_and_bad_arguments_without_a_device(L):
    fake = C.c_void_p(16)   # never dereferenced: the handles are checked first
    for s, t in ((None, None), (None, fake), (fake, None)):
        assert _call(L, s, t) == -1
        assert b"NULL" in L.sb200_last_error()
        assert _call(L, s, t, cap=-1, history_cap=-1) == -1


def test_python_wrapper_validates_its_arguments():
    from similari_b200 import engine

    s = engine.FeatureStore.__new__(engine.FeatureStore)   # no device: never reaches the library
    s._h, s.topn = None, 1
    t = engine.Tracker.__new__(engine.Tracker)
    t._h, t.opts = None, None
    with pytest.raises(TypeError):
        s.associate_wasted(object())
    with pytest.raises(ValueError):
        s.associate_wasted(t, cap=-1, history_cap=4)
    with pytest.raises(ValueError):
        s.associate_wasted(t, cap=4, history_cap=-1)
    for off in (-1, 1 << 64):
        with pytest.raises(ValueError):
            s.associate_wasted(t, cap=4, history_cap=4, id_offset=off)
