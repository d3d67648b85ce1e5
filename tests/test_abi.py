"""CPU checks of the drop-in boundary: the shared library loads, exports every symbol include/similari_b200.h
declares, struct layouts match, and compute entry points fail loudly (no CPU fallback) when there is no GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def test_exports_every_declared_symbol(L):
    from similari_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "similari_b200.h")).read()
    declared = set(re.findall(r"\b(sb200_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert getattr(L, name) is not None


def test_exports_only_declared_symbols(L):
    """The library's dynamic sb200_* symbols are exactly the header's declarations: nothing undeclared leaks out."""
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm is not installed")
    from similari_b200 import _build

    out = subprocess.run([nm, "-D", "--defined-only", _build.LIB], check=True, capture_output=True, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("sb200_")}
    hdr = open(os.path.join(ROOT, "include", "similari_b200.h")).read()
    declared = set(re.findall(r"\b(sb200_[a-z0-9_]+)\s*\(", hdr))
    assert exported == declared, exported ^ declared


def test_options_struct_layout_matches_oracle_mirror(L, oracle):
    from similari_b200 import _lib

    assert C.sizeof(_lib.Options) == C.sizeof(oracle.Options)
    a, b = _lib.Options(), oracle.Options()
    for (na, _), (nb, _) in zip(a._fields_, b._fields_):
        assert na == nb and getattr(_lib.Options, na).offset == getattr(oracle.Options, nb).offset
    o = _lib.default_options()
    # PySort / VisualMetricBuilder defaults (src/trackers/sort/simple_api.rs:461-470, metric/builder.rs:26-42)
    assert (o.kind, o.positional_kind, o.max_idle_epochs, o.history_length) == (0, 0, 5, 1)
    assert abs(o.iou_threshold - 0.3) < 1e-7 and abs(o.min_confidence - 0.05) < 1e-7
    assert abs(o.kalman_position_weight - 1 / 20) < 1e-7 and abs(o.kalman_velocity_weight - 1 / 160) < 1e-7
    assert (o.visual_max_observations, o.visual_min_votes, o.visual_minimal_track_length) == (5, 1, 3)


def test_no_cpu_fallback(L):
    """Without a CUDA device every compute entry point must fail loudly with SB200_ERR_CUDA."""
    from similari_b200 import _lib

    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present; the loud-failure path is for CPU-only machines")
    h = C.c_void_p()
    o = _lib.default_options()
    assert L.sb200_tracker_create(C.byref(o), C.byref(h)) == -2
    assert b"no CUDA device" in L.sb200_last_error()
    out = np.zeros((1, 1), np.float32)
    b = np.zeros((1, 6), np.float32)
    st = np.zeros((1, 30), np.float32)
    assert L.sb200_sort_cost_matrix(0, 0.3, 0.05, 0.05, 0.00625, _lib.ptr(b), 1, _lib.ptr(b), _lib.ptr(st), 1,
                                    _lib.ptr(out), 0) == -2
    idx = np.zeros(1, np.int32)
    assert L.sb200_nms(_lib.ptr(b), None, 1, 0.5, 0.0, 0, _lib.ptr(idx), 0) == -2
    with pytest.raises(_lib.Sb200Error):
        import similari_b200.engine as eng

        eng.Tracker(o)


def test_invalid_arguments_are_reported(L):
    from similari_b200 import _lib

    o = _lib.default_options(kind=7)
    h = C.c_void_p()
    rc = L.sb200_tracker_create(C.byref(o), C.byref(h))
    assert rc < 0 and h.value is None


def test_api_surface_names():
    """The PyO3 class / function names of src/lib.rs:122-159 that belong to the hot path exist in similari_b200.api."""
    import similari_b200.api as api

    for name in ["BoundingBox", "Universal2DBox", "SortTrack", "WastedSortTrack", "SortPredictionBatchRequest",
                 "SpatioTemporalConstraints", "Sort", "PositionalMetricType", "VisualSortMetricType", "VisualSortOptions",
                 "VisualSortObservation", "VisualSortObservationSet", "VisualSortPredictionBatchRequest",
                 "WastedVisualSortTrack", "VisualSort", "PredictionBatchResult", "BatchSort", "BatchVisualSort", "nms",
                 "version"]:
        assert hasattr(api, name), name
    b = api.BoundingBox(1.0, 2.0, 5.0, 5.0).as_xyaah()
    assert (float(b.xc), float(b.yc), b.angle, float(b.aspect), float(b.height)) == (3.5, 4.5, None, 1.0, 5.0)
    assert abs(api.BoundingBox(0, 0, 6, 8).as_xyaah().get_radius() - 5.0) < 1e-6
    c = api.SpatioTemporalConstraints()
    c.add_constraints([(1, 0.5), (2, 1.0), (3, 2.0), (4, 4.0)])
    c.add_constraints([(3, 2.5), (4, 4.5), (7, 8.5)])
    assert c.validate(1, 0.4) and not c.validate(1, 0.6) and c.validate(7, 8.5) and not c.validate(7, 8.7) and c.validate(9, 100.0)
