"""Without a GPU: the constructions of tests/test_gpu_compat_gates.py hit the gate's boundaries (the f32 replica they are
built with is bit-equal to the product's box_radius / dist_in_2r, and the oracle gives every probe its expected
outcome), the oracle's epochs run past 2^32 in size_t, and the Python layer refuses the epoch values ctypes would
truncate."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest

import compat_gates_constructions as X

HERE = os.path.dirname(os.path.abspath(__file__))
F32MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "libshim_compat.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(HERE, "host_shim", "shim.cpp"), "-o", so])
    L = C.CDLL(so)
    f = C.c_float
    L.shim_box_radius.argtypes = [f, f]
    L.shim_box_radius.restype = f
    L.shim_dist_in_2r.argtypes = [f] * 6
    L.shim_dist_in_2r.restype = f
    return L


def scripts():
    out = [(f"pos-k{k}-{p}", X.positional_script(k, p, 0xC0417 + 4 * k + p), {}) for k in (0, 1) for p in (0, 1)]
    out += [(f"big-k{k}-{p}", X.positional_script(k, p, 0xB16 + 4 * k + p, big=True), {}) for k in (0, 1) for p in (0, 1)]
    for kind in (2, 3):
        for vis in (0, 1):
            for K in (1, 3):
                out.append((f"vis-k{kind}-{vis}-K{K}", X.visual_script(kind, vis, K, 0x6A7E + 16 * kind + 4 * vis + K), {}))
    for kind, vis in ((2, 0), (3, 1), (3, 0)):   # the NaN-centre scripts of the GPU file
        out.append((f"nan-k{kind}-{vis}", X.visual_script(kind, vis, 2, 0x7A7 + 4 * kind + vis, nan=True), {}))
    for vis in (0, 1):   # the dense request of the GPU file: a threshold that cuts nothing
        out.append((f"dense-{vis}", X.visual_script(3, vis, 2, 0xDE75 + vis),
                    dict(vis_threshold=F32MAX if vis == 0 else -1.0)))
    return out


SCRIPTS = scripts()


def same_bits(a, b):
    a, b = np.float32(a), np.float32(b)
    return a.view(np.uint32) == b.view(np.uint32) or (np.isnan(a) and np.isnan(b))


@pytest.mark.parametrize("name", [s[0] for s in SCRIPTS[:6]])
def test_replica_is_bit_equal_to_the_product(shim, oracle, name):
    """Every constructed pair: the numpy f32 replica's radius and dist_in_2r equal sb_math.cuh's (host build) and the
    oracle's bit for bit, and every tie sits exactly on its max_dist with its `above` partner strictly past it."""
    s = next(x[1] for x in SCRIPTS if x[0] == name)
    r = X.radius(s.boxes[:, 3], s.boxes[:, 4])
    for j in range(len(s.delta)):
        rj = shim.shim_box_radius(float(s.boxes[j, 3]), float(s.boxes[j, 4]))
        assert same_bits(rj, r[j]) and same_bits(oracle.radius(s.boxes[j]), r[j]), j
        c, t = s.cand[j], s.boxes[j]
        d = shim.shim_dist_in_2r(float(c[0]), float(c[1]), rj, float(t[0]), float(t[1]), rj)
        assert same_bits(d, s.dist[j]) and same_bits(oracle.dist_in_2r(c, t), s.dist[j]), j
    case = np.array(s.case)
    live = s.delta <= X.MAX_IDLE
    tie = (case == "tie") & live
    above = (case == "above") & live
    assert tie.sum() >= 4 and above.sum() >= 4
    assert np.all(s.dist[tie] == s.target[tie]) and np.all(s.dist[above] > s.target[above])
    # one ulp of the candidate centre below the `above` offset is the tie
    c = s.cand[above].copy()
    c[:, 1] = np.nextafter(c[:, 1], np.float32(0))
    rr = X.radius(c[:, 3], c[:, 4])
    assert np.all(X.dist_in_2r(c[:, 0], c[:, 1], rr, s.boxes[above, 0], s.boxes[above, 1], rr) == s.target[above])


@pytest.mark.parametrize("name", [s[0] for s in SCRIPTS])
def test_oracle_decides_every_probe_as_constructed(oracle, name):
    """The oracle continues exactly the tracks whose probe is compatible, over every delta 1 .. max_idle + 1 and every
    case; the tracks fed one box predict that box bit for bit (so the constructed centres and radii are the gate's)."""
    s, kw = next((x[1], x[2]) for x in SCRIPTS if x[0] == name)
    o = oracle.Tracker(oracle.make_options(**s.options(**kw)))
    boxes_in = []

    def check(fr, out):
        if fr < X.FRAMES:
            req = [st[1] for st in s.steps if st[0] == "frame"][fr]
            fin = ~np.isnan(req["boxes"][:, 0])
            assert np.array_equal(out["predicted"][fin].view(np.uint32), req["boxes"][fin].view(np.uint32)), fr
            boxes_in.append(fr)
        if fr == X.FRAMES - 1 and name.startswith("big"):   # past the culled scan's 4096 tracks at the probe
            assert len(o.scene_tracks(int(s.scene[0]))["ids"]) == 4100

    _, _, got = X.run(o, s, check=check)
    assert len(boxes_in) == X.FRAMES
    bad = np.flatnonzero(got != s.expect)
    assert len(bad) == 0, [(int(s.delta[j]), s.case[j], float(s.dist[j])) for j in bad]
    case = np.array(s.case)
    for dl in range(1, X.MAX_IDLE + 2):   # both outcomes, or the one the delta allows, at every delta
        sel = s.delta == dl
        if sel.any() and dl <= X.MAX_IDLE and X.applicable(s.constraints, dl) is not None:
            assert got[sel].any() and not got[sel].all(), dl
    assert not got[s.delta > X.MAX_IDLE].any() and got[(s.delta == X.MAX_IDLE) & (case == "free")].all()
    if s.kind >= 2:
        assert (case == "dup").sum() >= 2 and not got[case == "dup"].any()
    if name.startswith("nan"):   # NaN centres: cut under a constraint, a NaN track continued past every constraint epoch
        assert np.isin(case, ["nan_cand", "nan_track"]).sum() == 4
        assert not got[np.isin(case, ["nan_cand", "nan_track"]) & (s.delta == 2)].any()
        assert got[(case == "nan_track") & (s.delta == X.MAX_IDLE)].all()


def test_batch_scenes_are_at_different_epochs(oracle):
    s = next(x[1] for x in SCRIPTS if x[0] == "vis-k3-0-K1")
    o = oracle.Tracker(oracle.make_options(**s.options()))
    X.run(o, s)
    assert len({o.current_epoch(int(sid)) for sid in np.unique(s.scene)}) == 3


def test_oracle_epochs_past_2_32(oracle):
    """The oracle's epochs are size_t: two skips take a scene to 2^32 - 5, a track created at 2^32 - 4 is continued up
    to 2^32 - 1 and past it, and its epochs are reported modulo 2^32."""
    for max_idle in (5, 2**31 - 1):
        o = oracle.Tracker(oracle.make_options(kind=0, positional_kind=1, iou_threshold=0.3, max_idle_epochs=max_idle))
        o.skip_epochs(2**31 - 1)
        o.skip_epochs(2**32 - 5 - (2**31 - 1))
        assert o.current_epoch() == 2**32 - 5
        b = np.array([[100.0, 100.0, np.nan, 0.5, 60.0, 0.9]], np.float32)
        ids = []
        for k in range(6):
            out = o.predict_batch([0], [0, 1], b)
            ids.append(int(out["ids"][0]))
            assert int(out["epochs"][0]) == (2**32 - 4 + k) % 2**32 and int(out["lengths"][0]) == k + 1
        assert len(set(ids)) == 1 and o.current_epoch() == 2**32 + 1


# ------------------------------------------------------------------------------------------------ Python constraint rules
def test_constraints_reject_negative_epochs_and_saturate_for_trackers():
    """The object keeps the reference's list (sorted, the first entry of an epoch kept, any usize epoch), so validate()
    and later calls decide as the reference does; a tracker gets the list with epochs saturated at 2^31 - 1, which
    decides every delta up to max_idle_epochs <= 2^31 - 1 as the reference's list does."""
    from similari_b200 import api

    c = api.SpatioTemporalConstraints()
    c.add_constraints([(3, 0.9), (1, 0.25), (3, 2.0), (5, 1.5), (2, 0.5)])
    assert c.constraints == [(1, 0.25), (2, 0.5), (3, 0.9), (5, 1.5)]
    with pytest.raises(OverflowError):
        c.add_constraints([(4, 1.0), (-1, 1.0)])
    assert c.constraints == [(1, 0.25), (2, 0.5), (3, 0.9), (5, 1.5)]   # nothing of a refused call is kept
    # two calls: an epoch past int32 first, then 2^31 - 1
    c2 = api.SpatioTemporalConstraints()
    c2.add_constraints([(2**31, 6.0)])
    c2.add_constraints([(2**31 - 1, 9.0)])
    assert c2.constraints == [(2**31 - 1, 9.0), (2**31, 6.0)]
    assert c2.validate(2**31 - 1, 7.0) and not c2.validate(2**31, 7.0) and c2.validate(2**31 + 1, 7.0)
    assert c2._tracker_constraints() == [(2**31 - 1, 9.0)]
    c.add_constraints([(2**40, 7.0), (2**31, 6.0), (2**31 - 1 + 2**33, 8.0), (2**31 - 2, 3.0)])
    assert c.constraints[-4:] == [(2**31 - 2, 3.0), (2**31, 6.0), (2**33 + 2**31 - 1, 8.0), (2**40, 7.0)]
    t = c._tracker_constraints()
    assert t[-2:] == [(2**31 - 2, 3.0), (2**31 - 1, 6.0)] and all(0 <= e < 2**31 for e, _ in t)
    for cons in (c, c2):
        t = cons._tracker_constraints()
        for delta in (0, 1, 2, 4, 5, 6, 2**31 - 3, 2**31 - 2, 2**31 - 1):
            for dist in (0.2, 1.0, 2.5, 5.0, 6.5, 8.5, 9.5):
                assert cons.validate(delta, dist) == _validate_exact(t, delta, dist), (delta, dist)
    # what the trackers' options receive
    o = api._sort_options(0, 1, 2**31 - 1, None, 0.05, c2, 1 / 20, 1 / 160)
    assert o.n_constraints == 1 and o.constraint_epochs[0] == 2**31 - 1 and o.constraint_max_dist[0] == 9.0
    vo = api.VisualSortOptions()
    vo.spatio_temporal_constraints(c2)
    assert vo._constraints == [(2**31 - 1, 9.0)]


def _validate_exact(cons, delta, dist):
    for e, m in cons:
        if e >= delta:
            return dist <= m
    return True


def test_options_refuse_what_ctypes_would_truncate():
    from similari_b200 import _lib, engine

    assert C.c_int32(2**32 + 5).value == 5   # the truncation the checks stand in front of
    with pytest.raises(OverflowError):
        _lib.default_options(constraints=[(2**32 + 1, 1.0)])
    with pytest.raises(OverflowError):
        _lib.default_options(max_idle_epochs=2**32 + 5)
    o = _lib.default_options(constraints=[(2**31 - 1, 1.0)], max_idle_epochs=2**31 - 1)
    assert o.constraint_epochs[0] == 2**31 - 1 and o.max_idle_epochs == 2**31 - 1
    fake = types.SimpleNamespace(_L=None, _h=None)   # the count is checked before the library is called
    for n in (2**32 + 7, 2**31, -(2**31) - 1):
        with pytest.raises(OverflowError):
            engine.Tracker.skip_epochs(fake, n)
