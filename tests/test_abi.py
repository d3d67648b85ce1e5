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
HEADER = os.path.join(ROOT, "include", "similari_b200.h")
# the header's return and scalar parameter types, as ctypes binds them
CTYPES = {"void": None, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
          "float": C.c_float, "size_t": C.c_size_t, "void*": C.c_void_p, "const char*": C.c_char_p}


@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def test_exports_every_declared_symbol(L):
    from similari_b200 import _lib

    hdr = open(HEADER).read()
    declared = set(re.findall(r"\b(sb200_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert getattr(L, name) is not None
    for name in _lib.EXPORTS:
        assert getattr(L, name).argtypes is not None, name


def test_bindings_match_the_declarations(L):
    """Each declared function is bound with the header's return type and one argtype per parameter: the scalar's own
    type, or a pointer type for a pointer."""
    hdr = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(HEADER).read(), flags=re.S)
    decls = re.findall(r"(\w[\w ]*\**)\s*\b(sb200_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr)
    assert len(decls) == len(set(n for _, n, _ in decls)) > 100
    for ret, name, params in decls:
        fn = getattr(L, name)
        assert fn.restype is CTYPES[" ".join(ret.split())], (name, ret, fn.restype)
        params = [] if params.strip() in ("", "void") else [" ".join(p.split()) for p in params.split(",")]
        assert len(fn.argtypes) == len(params), name
        for p, t in zip(params, fn.argtypes):
            typ = re.sub(r"\s*\b\w+$", "", p) if re.search(r"[\s*]\w+$", p) else p
            if typ.endswith("*"):
                assert t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer), (name, p, t)
            else:
                assert t is CTYPES[typ], (name, p, t)


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


def test_store_entry_points_fail_without_a_gpu(L):
    """Without a CUDA device every feature-store entry point fails loudly with SB200_ERR_CUDA, and the Python store
    refuses to be created or loaded."""
    from similari_b200 import _lib
    import similari_b200.engine as eng

    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present; the loud-failure path is for CPU-only machines")
    p = _lib.ptr
    o = _lib.FstoreOptions(0, 100.0, 3, 256, 1, 100.0, 1, 0)
    h = C.c_void_p()
    assert L.sb200_fstore_create(C.byref(o), C.byref(h)) == -2 and h.value is None
    ids = np.zeros(1, np.uint64)
    offs = np.array([0, 1], np.int32)
    f = np.zeros((1, 256), np.float32)
    cnt = np.zeros(1, np.int32)
    w = np.zeros(1, np.float64)
    m = np.zeros(1, np.uint8)
    t = np.zeros(1, np.int64)
    assert L.sb200_fstore_add(None, 1, p(ids), p(f)) == -2
    assert L.sb200_fstore_search(None, 1, p(ids), p(offs), p(f), p(cnt), p(ids), p(w)) == -2
    assert L.sb200_fstore_associate(None, 1, p(ids), p(offs), p(f), p(cnt), p(ids), p(w), p(ids), p(m)) == -2
    assert L.sb200_fstore_fetch(None, 1, p(ids), 0, p(cnt), p(f)) == -2
    assert L.sb200_fstore_size(None) == -2
    assert L.sb200_fstore_ids(None, 1, p(ids)) == -2
    assert L.sb200_fstore_last_stage_ms(None, p(f)) == -2
    L.sb200_fstore_destroy(None)
    assert L.sb200_fstore_set_feature_type(None, 1) == -2
    assert L.sb200_fstore_get_options(None, None, None) == -2
    assert L.sb200_fstore_add_device(None, 1, p(ids), None, None) == -2
    assert L.sb200_fstore_search_device(None, 1, p(ids), p(offs), None, p(cnt), p(ids), p(w), None) == -2
    assert L.sb200_fstore_associate_device(None, 1, p(ids), p(offs), None, p(cnt), p(ids), p(w), p(ids), p(m),
                                           None) == -2
    n = C.c_uint64(0)
    assert L.sb200_fstore_save(None, None, 0, C.byref(n)) == -2
    blob = np.zeros(1024, np.uint8)
    assert L.sb200_fstore_load(p(blob), len(blob), 0, C.byref(h)) == -2 and h.value is None
    assert b"no CUDA device" in L.sb200_last_error()
    assert L.sb200_fstore_search_owned(None, 1, p(ids), 0, p(cnt), p(ids), p(w)) == -2
    assert L.sb200_fstore_merge_owned(None, 1, p(ids), p(ids), 1) == -2
    assert b"no CUDA device" in L.sb200_last_error()
    st = C.c_int32(5)
    assert L.sb200_fstore_set_storage_type(None, 1) == -2
    assert L.sb200_fstore_get_storage_type(None, C.byref(st)) == -2 and st.value == 5
    assert b"no CUDA device" in L.sb200_last_error()
    assert L.sb200_fstore_set_gate(None, 1) == -2
    assert L.sb200_fstore_fetch_attr(None, 1, p(ids), p(ids), p(t), p(t)) == -2
    assert b"no CUDA device" in L.sb200_last_error()
    with pytest.raises(_lib.Sb200Error):
        eng.FeatureStore()
    with pytest.raises(_lib.Sb200Error, match="-2"):
        eng.FeatureStore.load(blob)
    with pytest.raises(_lib.Sb200Error, match="-2"):
        eng.FeatureStore(storage="f16")
    with pytest.raises(ValueError, match="storage"):
        eng.FeatureStore(storage="f8")


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
