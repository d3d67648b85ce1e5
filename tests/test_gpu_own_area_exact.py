"""Own-area shares on the GPU (kernels_own.cu) against the exact references of tests/own_area_exact.py: the warp kernel
and the CTA second pass on scenes dense in shared edge lines, at the list boundary (31 / 32 / 33 neighbours), in crowds
up to the second pass's cap of 2800 neighbours and one beyond it, and the visual trackers that derive the shares on the
device, with their thresholds placed exactly on a share.  Tolerances as in tests/test_own_area_exact_cpu.py."""
import numpy as np
import pytest

import own_area_exact as X
from test_own_area_exact_cpu import (assert_exact, edge_line_scenes, grid_scene, near_collinear_scene, px_scene,
                                     shifted)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the product has no CPU path")
    return e


def check_px(eng, name, rows, strict=True, idx=None):
    b, lt = px_scene(rows)
    got = eng.own_area_shares(b)
    assert_exact(name, b, eng.box_vertices(b), {"gpu": got if idx is None else got[idx]}, lt=lt, strict=strict, idx=idx)
    return got


def ring(k, far=0):
    """Box 0 (64 x 64) with k <= 34 4 x 4 boxes straddling its outline 7 pixels apart (each covers 8 pixels of box 0, no
    two of them meet), so that box 0 has exactly k neighbours and owns 4096 - 8 k; `far` boxes 10^4 pixels away."""
    rows = [(0, 0, 64, 64)]
    pos = [(7 * c + 1, -2) for c in range(9)] + [(62, 7 * c + 1) for c in range(1, 9)] + \
          [(7 * c + 1, 62) for c in range(9)] + [(-2, 7 * c + 1) for c in range(1, 9)]
    rows += [(x, y, 4, 4) for x, y in pos[:k]]
    rows += [(10000 + 8 * c, 10000, 4, 4) for c in range(far)]
    return rows


# ------------------------------------------------------------------------------------------------------- exactness
def test_exact_on_edge_line_scenes(eng):
    for name, rows in edge_line_scenes().items():
        check_px(eng, name, rows)
        check_px(eng, (name, 65536), shifted(rows, 65536.0), strict=False)


@pytest.mark.parametrize("off", [0.0, 65536.0])
def test_exact_on_grid_scenes(eng, off):
    r = np.random.default_rng(4321)
    for trial in range(30):
        check_px(eng, trial, shifted(grid_scene(r, int(r.integers(2, 32))), off), strict=(off == 0.0))


def test_near_collinear_oriented_scenes(eng):
    r = np.random.default_rng(98)
    for trial in range(10):
        b = near_collinear_scene(r, int(r.integers(3, 8)))
        assert_exact(trial, b, eng.box_vertices(b), {"gpu": eng.own_area_shares(b)})


@pytest.mark.parametrize("k", [31, 32, 33])
def test_list_boundary(eng, k):
    """31 and 32 neighbours fit the warp kernel's list; 33 spill to the second pass.  Far-away boxes change nothing."""
    b, lt = px_scene(ring(k))
    v = eng.box_vertices(b)
    assert len(X.neighbours(b, 0, v)) == k
    got = check_px(eng, k, ring(k))
    assert got[0] == X.expected_share(64 * 64 - 8 * k, 1.0, 64.0)
    got_far = check_px(eng, (k, "far"), ring(k, far=40))
    np.testing.assert_array_equal(got_far[: k + 1], got)


# ------------------------------------------------------------------------------------------------------ second pass
def test_second_pass_axis_aligned_crowds(eng):
    """Integer-pixel crowds where most boxes have 33-300 neighbours, against the cell count (every box)."""
    r = np.random.default_rng(78)
    for n in (60, 150, 301):
        rows = grid_scene(r, n, cell=2, span=12, hs=(8, 16))
        b, lt = px_scene(rows)
        v = eng.box_vertices(b)
        assert max(len(X.neighbours(b, i, v)) for i in range(n)) > 32
        check_px(eng, n, rows)


def test_second_pass_oriented_crowds(eng):
    """Oriented crowds, 40-150 neighbours: the f64 slab integral, within its bound plus the boundary sum's."""
    r = np.random.default_rng(79)
    for n, span in ((60, 90.0), (150, 150.0)):
        b = np.zeros((n, 6), np.float32)
        b[:, :2] = r.uniform(0, span, (n, 2))
        b[:, 2] = r.uniform(-1.5, 1.5, n)
        b[:, 3] = r.uniform(0.3, 0.8, n)
        b[:, 4] = r.uniform(40, 100, n)
        b[:, 5] = 1
        v = eng.box_vertices(b)
        got = eng.own_area_shares(b)
        crowd = [i for i in range(n) if len(X.neighbours(b, i, v)) > 32][:6]
        assert crowd
        for i in crowd:
            nb = X.neighbours(b, i, v)
            a64, bound = X.own_area_slabs_f64(v[i], v[nb])
            lo, hi = X.share_band(a64, bound + X.green_sum_bound(v[i], v[nb]), b[i, 3], b[i, 4])
            assert lo <= got[i] <= hi, (n, i, len(nb), a64, got[i])


def test_second_pass_reverse_ordered_row(eng):
    """Box 0 over 300 touching 2-pixel boxes listed against its edge direction: the walk grows its run one link per
    pass, serially in one thread (about 300 x 300 half-plane tests, well under a millisecond)."""
    check_px(eng, "row", [(0, 0, 600, 16)] + [(2 * c, 0, 2, 8) for c in range(299, -1, -1)], idx=[0])


def test_second_pass_grid_stride(eng):
    """300 detections overflow in one call (two stacks of 150 duplicates, half overlapping): more than the second
    pass's 132 CTAs, so its grid-stride loop takes a second round."""
    rows = [(0, 0, 16, 16)] * 150 + [(8, 0, 16, 16)] * 150
    got = check_px(eng, "stacks", rows)
    assert np.all(got <= X.FULL_COVER_RESIDUE)


def cap_grid(n):
    """Box 0 (256 x 256) with n <= 3136 2 x 2 boxes on a 4-pixel grid inside it: box 0 has n neighbours, none of the
    small boxes more than one."""
    return [(0, 0, 256, 256)] + [(16 + 4 * (c % 56), 16 + 4 * (c // 56), 2, 2) for c in range(n)]


def test_second_pass_at_its_capacity(eng):
    """2800 neighbours, the cap: exact.  Each of box 0's 11,204 edges walks 2800 boxes once (about 10 ms)."""
    got = check_px(eng, 2800, cap_grid(2800), idx=[0])
    assert got[0] == X.expected_share(256 * 256 - 4 * 2800, 1.0, 256.0)


def test_second_pass_beyond_its_capacity(eng):
    from similari_b200._lib import Sb200Error

    with pytest.raises(Sb200Error, match=r"status -3: more than 2800 boxes overlap one box"):
        eng.own_area_shares(px_scene(cap_grid(2801))[0])
    assert eng.own_area_shares(px_scene(cap_grid(16))[0])[0] > 0.99   # the next call is served


# ---------------------------------------------------------------------------------------------------- tracker path
F32_075_UP = float(np.nextafter(np.float32(0.75), np.float32(1)))


def tracker_groups(kind):
    """Integer-pixel groups (rows, exact shares 0.75 / 0 / 1 by construction):
      pair   A 16 x 16 and a 4 x 16 strip on its right quarter: A owns exactly 0.75, the strip 0;
      crowd  A 64 x 64, a 16 x 64 strip on its right quarter and 40 2 x 2 boxes inside the strip: A and the strip have
             41 neighbours (second pass), A owns exactly 0.75;
      free   a lone 16 x 16 box, share 1.
    kind 3: three scenes, two with a crowd beside clean groups and one clean; kind 2: one scene with a crowd."""
    pair = [(0, 0, 16, 16), (12, 0, 4, 16)]
    crowd = [(0, 0, 64, 64), (48, 0, 16, 64)] + [(49 + 3 * (c % 5), 2 + 8 * (c // 5), 2, 2) for c in range(40)]
    free = [(0, 0, 16, 16)]
    layout = [[crowd, pair, free, pair, free], [pair, free, pair, free], [crowd, pair, free]]
    if kind == 2:
        layout = layout[:1]
    scenes = []
    for groups in layout:
        rows = []
        for g, grp in enumerate(groups):
            rows += [(l + 200 * g, t, w, h) for l, t, w, h in grp]
        scenes.append(rows)
    return scenes


def exact_shares(rows):
    b, lt = px_scene(rows)
    v = np.array([[(l, t + h), (l + w, t + h), (l + w, t), (l, t)] for l, t, w, h in rows], np.float64)
    return np.array([X.expected_share(X.own_area_cells(lt, i, X.neighbours(b, i, v)), b[i, 3], b[i, 4])
                     for i in range(len(rows))], np.float32)


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("use,collect", [(0.75, F32_075_UP), (F32_075_UP, 0.75), (0.75, 0.75)])
def test_tracker_thresholds_on_an_exact_share(eng, oracle, kind, use, collect):
    """The tracker derives the shares on the device (crowds through the second pass, several scenes overflowing in one
    frame); the oracle gets the exact shares through own_area=.  Thresholds sit exactly on the exact share 0.75 or one
    f32 ulp above it, so a share computed as 0.74999994 would change ids, voting types or stored features.  The same
    run with those shares one ulp low must change something (the gates do bite)."""
    from similari_b200._lib import default_options

    kw = dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
              feature_dim=16, visual_max_observations=3, visual_min_votes=1, visual_minimal_track_length=1,
              visual_minimal_own_area_percentage_use=use, visual_minimal_own_area_percentage_collect=collect)
    g = eng.Tracker(default_options(**kw))
    o, lo = oracle.Tracker(oracle.make_options(**kw)), oracle.Tracker(oracle.make_options(**kw))
    scenes = tracker_groups(kind)
    n_sc = len(scenes)
    offs = np.cumsum([0] + [len(s) for s in scenes]).astype(np.int32)
    own = np.concatenate([exact_shares(s) for s in scenes])
    assert np.count_nonzero(own == np.float32(0.75)) == (3 if kind == 2 else 7)
    own_low = np.where(own == np.float32(0.75), np.nextafter(np.float32(0.75), np.float32(0)), own).astype(np.float32)
    r = np.random.default_rng(kind)
    cent = r.standard_normal((offs[-1], 16)).astype(np.float32)
    # the boxes stay put, so that every track is matched in every frame and none expires (the device store drops an
    # expired track at once, the oracle's scene_tracks still lists it)
    boxes = np.concatenate([px_scene(s)[0] for s in scenes])
    for s in range(n_sc):
        np.testing.assert_array_equal(eng.own_area_shares(boxes[offs[s]:offs[s + 1]]), own[offs[s]:offs[s + 1]])
    differs = False
    for fr in range(5):
        feats = cent + 0.01 * r.standard_normal(cent.shape).astype(np.float32)
        rg = g.predict_batch(np.arange(n_sc), offs, boxes, features=feats)
        ro = o.predict_batch(np.arange(n_sc), offs, boxes, features=feats, own_area=own)
        rl = lo.predict_batch(np.arange(n_sc), offs, boxes, features=feats, own_area=own_low)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
            differs = differs or not np.array_equal(ro[key], rl[key])
        for s in range(n_sc):
            fg, fo, fl = (t.scene_tracks(s)["feat_counts"] for t in (g, o, lo))
            assert np.array_equal(fg, fo), (fr, s)
            differs = differs or not np.array_equal(fo, fl)
    assert differs


def test_tracker_scene_beyond_the_cap(eng):
    """A scene in which one detection has 2801 neighbours (2802 detections), beside a clean scene.  The own-area second
    pass would report SB200_ERR_CAPACITY only after the frame had run, but a visual tracker never gets that far: a
    scene of 2802 detections is more than the on-chip assignment solver holds even with no stored tracks, and that
    bound refuses the request with SB200_ERR_CAPACITY before anything is committed.  The store is NOT advanced (the
    round-1 defect, "error after the store advanced", does not come back at 2801), and the next call is served as if
    the refused one had not been made."""
    from similari_b200._lib import Sb200Error, default_options
    from test_gpu_voting import smem_fits

    assert not smem_fits(2802, 0, viscap=8192)          # kDenseVoteCap: the visual trackers' voting list
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
              feature_dim=8, visual_max_observations=3, visual_min_votes=1, visual_minimal_track_length=1,
              visual_minimal_own_area_percentage_use=0.5, visual_minimal_own_area_percentage_collect=0.5)
    g, fresh = eng.Tracker(default_options(**kw)), eng.Tracker(default_options(**kw))
    big, _ = px_scene(cap_grid(2801))
    clean, _ = px_scene([(200 * c, 0, 16, 16) for c in range(4)])
    boxes = np.concatenate([clean, big])
    offs = np.array([0, len(clean), len(boxes)], np.int32)
    feats = np.random.default_rng(0).standard_normal((len(boxes), 8)).astype(np.float32)
    with pytest.raises(Sb200Error, match=r"status -3: scene too large for the on-chip assignment solver \(m=2802"):
        g.predict_batch(np.array([7, 8]), offs, boxes, features=feats)
    one = (np.array([7]), np.array([0, len(clean)], np.int32), clean)
    for _ in range(2):
        ra = g.predict_batch(*one, features=feats[: len(clean)])
        rb = fresh.predict_batch(*one, features=feats[: len(clean)])
        for key in ("ids", "epochs", "lengths", "voting_types"):
            np.testing.assert_array_equal(ra[key], rb[key], err_msg=key)


# -------------------------------------------------------------------------------------------------- degenerate boxes
def test_nan_centre_leaves_clean_neighbours_exact(eng):
    """A NaN-centre box covers nothing (the separating-axis gate drops it) and gets share 0 itself."""
    rows = edge_line_scenes()["one_line_both_directions"]
    b, lt = px_scene(rows)
    bad = b.copy()
    bad[2, 0] = np.nan
    got = eng.own_area_shares(bad)
    assert got[2] == 0.0 and not np.isnan(got).any()
    v = eng.box_vertices(bad)
    clean = [i for i in range(len(b)) if i != 2]
    assert_exact("nan", bad, v, {"gpu": got[clean]}, strict=True, idx=clean)


def test_zero_and_negative_sizes_do_not_poison_neighbours(eng):
    """The reference panics on aspect or height <= 0 (too_far asserts), so there is no share to match for those boxes:
    the call succeeds, no share is NaN, and zero-area boxes lying across clean boxes change no clean share.  (A
    negative aspect makes area_f32 negative, and with it the share: no positive threshold accepts it.)"""
    rows = [(0, 0, 32, 16), (16, 8, 32, 16), (60, 0, 16, 16)]
    b, lt = px_scene(rows)
    deg = np.array([[16.0, 8.0, np.nan, 0.0, 16.0, 1.0], [24.0, 8.0, np.nan, 1.0, 0.0, 1.0],
                    [20.0, 10.0, 0.3, 0.0, 8.0, 1.0], [300.0, 300.0, np.nan, -1.0, 16.0, 1.0],
                    [400.0, 300.0, np.nan, 1.0, -16.0, 1.0]], np.float32)
    allb = np.concatenate([b, deg])
    got = eng.own_area_shares(allb)
    assert not np.isnan(got).any() and np.all(got <= 1)
    np.testing.assert_array_equal(got[: len(b)], eng.own_area_shares(b))
    assert_exact("deg", b, eng.box_vertices(b), {"gpu": got[: len(b)]}, lt=lt, strict=True)
