"""The compatibility gate (compat_ok: idle limit, then the spatio-temporal constraints) on every cost path, against the
oracle frame by frame, with pairs on its boundaries (tests/compat_gates_constructions.py): dist_in_2r exactly on a
constraint's max_dist and one f32 past it, idle deltas of exactly each constraint epoch, of max_idle_epochs and one
more, NaN centres, and batch scenes at different epochs.  After the probe frame the device store is compared with the
oracle's as well (check_state), except in the NaN-centre cases.  Every case also asserts its expected outcome, so a
construction that missed its boundary fails instead of passing vacuously.

The visual scripts' first scene has more than 256 candidates and 256 feature columns with outcomes that vary by row
and column: both consumer warpgroups and both e4m3 halves of the screens, and more than one column tile.

The top of the epoch range: scenes skipped to just below 2^32 keep their tracks like the oracle, and a call that would
move an epoch past 2^32 - 1 is refused with nothing changed."""
import numpy as np
import pytest

import compat_gates_constructions as X
from test_gpu_track_observations import check_outputs, check_state, set_path

pytestmark = pytest.mark.gpu
F32MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def both(eng, oracle, opts):
    from similari_b200._lib import default_options

    return eng.Tracker(default_options(**opts)), oracle.Tracker(oracle.make_options(**opts))


def run_both(eng, oracle, script, opts, state=True, before_probe=None):
    """The oracle's run, then the device's compared with it frame by frame; before_probe(g) runs before the probe."""
    g, o = both(eng, oracle, opts)
    ro_all = []
    _, _, want = X.run(o, script, check=lambda fr, out: ro_all.append(out))
    scene_ids = np.unique(script.scene)

    frames = [st[1] for st in script.steps if st[0] == "frame"]

    def cmp(fr, rg):
        diff = np.flatnonzero(np.asarray(rg["ids"]) != ro_all[fr]["ids"])   # the first row names the case
        tr = frames[fr]["tracks"]
        assert len(diff) == 0, (fr, [(int(r), int(script.delta[tr[r]]), script.case[tr[r]]) if tr[r] >= 0 else (int(r), "filler")
                                     for r in diff[:4]])
        check_outputs(rg, ro_all[fr], fr)
        if before_probe and fr == X.FRAMES - 1:
            before_probe(g)

    _, _, got = X.run(g, script, check=cmp)
    for sid in scene_ids:
        assert g.current_epoch(int(sid)) == o.current_epoch(int(sid))
    if state:
        check_state(g, o, opts, scene_ids, "probe")
    assert np.array_equal(want, script.expect), np.flatnonzero(want != script.expect)
    assert np.array_equal(got, script.expect), [(int(script.delta[j]), script.case[j]) for j in np.flatnonzero(got != script.expect)]
    return g


POSITIONAL = [(kind, pos) for kind in (0, 1) for pos in (0, 1)]


@pytest.mark.parametrize("kind,pos", POSITIONAL, ids=[f"k{k}-{'iou' if p else 'maha'}" for k, p in POSITIONAL])
def test_positional_gate_boundaries(eng, oracle, kind, pos):
    """Sort and BatchSort, IoU and Mahalanobis, scenes of at most 4096 tracks: the culled positional scan."""
    s = X.positional_script(kind, pos, 0xC0417 + 4 * kind + pos)
    run_both(eng, oracle, s, s.options())


@pytest.mark.parametrize("kind,pos", POSITIONAL, ids=[f"k{k}-{'iou' if p else 'maha'}" for k, p in POSITIONAL])
def test_positional_gate_boundaries_past_4096_tracks(eng, oracle, kind, pos):
    """The same boundaries with one scene of 4100 tracks at the probe (filler tracks far away): the probe frame's
    positional cost runs in the dense tiled kernel (pos_cost_kernel).  BatchSort's other scenes, at other epochs, go
    through that kernel with it."""
    s = X.positional_script(kind, pos, 0xB16 + 4 * kind + pos, big=True)
    seen = []

    def big_scene(g):   # the tracks the probe frame's positional cost is computed against
        seen.append(int(g.scene_track_counts([int(s.scene[0])])[0]))

    run_both(eng, oracle, s, s.options(), before_probe=big_scene)
    assert seen == [4100], seen


VISUAL = [(kind, vis, K, path) for kind in (2, 3) for vis in (0, 1) for K in (1, 3) for path in ("simt", "tc16", "tc8")
          if (kind + vis + K) % 2 == 0 or path != "simt"]


@pytest.mark.parametrize("kind,vis,K,path", VISUAL,
                         ids=[f"k{k}-{'cos' if v else 'euclid'}-K{K}-{p}" for k, v, K, p in VISUAL])
def test_visual_gate_boundaries(eng, oracle, kind, vis, K, path, monkeypatch):
    """VisualSort and BatchVisualSort on the forced visual path: the SIMT kernel, or the BF16 / e4m3 screen's geo block
    (the exact refine then sees only the survivors)."""
    set_path(monkeypatch, path)
    s = X.visual_script(kind, vis, K, 0x6A7E + 16 * kind + 4 * vis + K)
    g = run_both(eng, oracle, s, s.options())
    wc, sc = g.work_counters(), g.screen_counters()
    assert wc["frames"] == X.FRAMES + 1 and wc["visual_dot_products"] > 0, wc
    if path == "simt":   # the visual stage ran every frame with tracks, and no screen did
        assert wc["tc_frames"] == 0 and wc["vis_screen_ms"] == 0.0 and wc["stage_ms"]["visual_cost"] > 0.0, wc
        assert sc["fp8_frames"] == 0 and sc["bf16_frames"] == 0, sc
    else:   # every frame with tracks, the probe included (the first frame has none), screened on the forced operands,
        # and no scene handed back to the exact SIMT kernel
        assert wc["tc_frames"] == X.FRAMES and wc["dense_fallback_scenes"] == 0, wc
        assert sc["fp8_frames" if path == "tc8" else "bf16_frames"] == X.FRAMES, sc
        assert sc["bf16_frames" if path == "tc8" else "fp8_frames"] == 0, sc


@pytest.mark.parametrize("kind,vis,path", [(2, 0, "tc8"), (3, 1, "tc16"), (3, 0, "simt")])
def test_nan_centres(eng, oracle, kind, vis, path, monkeypatch):
    """A NaN track or candidate centre: cut while a constraint applies (NaN <= d is false), compatible past every
    constraint epoch, where the NaN track is continued and the NaN candidate, whose feature is unusable (its Kalman box
    is NaN), starts a new track.  The outputs match the oracle frame by frame.  The device store is not compared: the
    device's per-block Kalman state of a NaN box is NaN in that box's blocks only, the oracle's 10 x 10 one everywhere."""
    set_path(monkeypatch, path)
    s = X.visual_script(kind, vis, 2, 0x7A7 + 4 * kind + vis, nan=True)
    run_both(eng, oracle, s, s.options(), state=False)


@pytest.mark.parametrize("vis", [0, 1])
def test_dense_request_with_constraints_goes_to_a_screen(eng, oracle, vis, monkeypatch):
    """SB200_VIS_KERNEL=dense and a threshold that cuts nothing: the dense path has no gate, so constrained frames are
    screened; every compatible probe still continues its own track (distance 0 beats every other pair)."""
    set_path(monkeypatch, "dense")
    s = X.visual_script(3, vis, 2, 0xDE75 + vis)
    g = run_both(eng, oracle, s, s.options(vis_threshold=F32MAX if vis == 0 else -1.0))
    wc, sc = g.work_counters(), g.screen_counters()
    assert wc["tc_frames"] == X.FRAMES and sc["fp8_frames"] + sc["bf16_frames"] == X.FRAMES, (wc, sc)


# ------------------------------------------------------------------------------------------------ top of the epoch range
TOP = 2**32 - 1


def box_at(x):
    return np.array([[x, 300.0, np.nan, 0.5, 60.0, 0.9]], np.float32)


def frame_both(g, o, sids, xs):
    offs = np.arange(len(sids) + 1, dtype=np.int32)
    b = np.concatenate([box_at(x) for x in xs])
    rg = g.predict_batch(np.array(sids, np.uint64), offs, b)
    ro = o.predict_batch(np.array(sids, np.uint64), offs, b)
    check_outputs(rg, ro, sids)
    for s in sids:
        assert g.current_epoch(s) == o.current_epoch(s)
    return rg


@pytest.mark.parametrize("max_idle", [5, 2**31 - 1])
def test_tracks_near_the_last_epoch(eng, oracle, max_idle):
    """Two skip_epochs calls take scene 1 to 2^32 - 5 (scene 0 stays low), and tracks are created, kept and continued up
    to epoch 2^32 - 1 exactly like the oracle's (the end-of-frame sweep used to compute epoch + max_idle in 32 bits
    and dropped them on creation).  With max_idle_epochs = 2^31 - 1 the same holds above 2^31, and a track idle for
    exactly 2^31 - 1 epochs is still continued."""
    opts = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=max_idle)
    g, o = both(eng, oracle, opts)
    frame_both(g, o, [0, 1], [100.0, 100.0])
    for t in (g, o):
        t.skip_epochs(2**31 - 1, 1)
        t.skip_epochs(2**32 - 5 - 1 - (2**31 - 1), 1)
    assert g.current_epoch(1) == o.current_epoch(1) == 2**32 - 5
    ids = []
    for k in range(4):   # epochs 2^32 - 4 .. 2^32 - 1
        ids.append(frame_both(g, o, [0, 1], [100.0 + k, 100.0 + k])["ids"])
    assert all(int(i[1]) == int(ids[0][1]) for i in ids), ids   # one track, continued
    assert g.current_epoch(1) == TOP
    check_state(g, o, opts, [0, 1], "top")
    if max_idle == 2**31 - 1:
        g2, o2 = both(eng, oracle, opts)
        first = frame_both(g2, o2, [7], [50.0])["ids"]
        for t in (g2, o2):
            t.skip_epochs(2**31 - 2, 7)   # the next frame is 2^31 - 1 epochs after the track's
        again = frame_both(g2, o2, [7], [50.0])["ids"]
        assert int(again[0]) == int(first[0]) and g2.current_epoch(7) == 2**31
        for t in (g2, o2):
            t.skip_epochs(2**31 - 2, 7)
        again = frame_both(g2, o2, [7], [50.0])["ids"]
        assert int(again[0]) == int(first[0]) and g2.current_epoch(7) == TOP


def test_epoch_overflow_is_refused(eng, oracle):
    """skip_epochs or a predict that would move any scene's epoch past 2^32 - 1 raises, and leaves every scene, track
    and frame in flight as it was."""
    from similari_b200._lib import Sb200Error, pinned_empty

    opts = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=5)
    g, o = both(eng, oracle, opts)
    frame_both(g, o, [0, 1], [100.0, 200.0])
    for t in (g, o):
        t.skip_epochs(2**31 - 1, 1)
        t.skip_epochs(2**31 - 2, 1)
    frame_both(g, o, [0, 1], [100.0, 200.0])   # scene 1 at 2^32 - 1
    assert g.current_epoch(1) == TOP
    before = {s: g.scene_tracks(s)["ids"].tolist() for s in (0, 1)}
    with pytest.raises(Sb200Error):
        g.skip_epochs(1, 1)
    with pytest.raises(Sb200Error):
        g.predict_batch(np.array([0, 1], np.uint64), np.array([0, 1, 2], np.int32), np.concatenate([box_at(1), box_at(2)]))
    g.skip_epochs(0, 1)   # zero epochs are always allowed
    # a frame in flight counts: scene 0 at 2^32 - 2 plus one queued frame is at the last epoch
    for t in (g, o):
        t.skip_epochs(2**31 - 1, 0)
        t.skip_epochs(2**31 - 3, 0)
    assert g.current_epoch(0) == TOP - 1
    out = {"ids": pinned_empty((1,), np.uint64), "epochs": pinned_empty((1,), np.uint32),
           "lengths": pinned_empty((1,), np.uint32), "voting_types": pinned_empty((1,), np.uint8)}
    g.predict_batch(np.array([0], np.uint64), np.array([0, 1], np.int32), box_at(100.0), out=out, wait=False)
    with pytest.raises(Sb200Error):
        g.predict_batch(np.array([0], np.uint64), np.array([0, 1], np.int32), box_at(100.0))
    g.sync()
    ro = o.predict_batch(np.array([0], np.uint64), np.array([0, 1], np.int32), box_at(100.0))
    check_outputs(out, ro, "in flight")
    assert g.current_epoch(0) == o.current_epoch(0) == TOP and g.current_epoch(1) == TOP
    assert g.scene_tracks(1)["ids"].tolist() == before[1]
    check_state(g, o, opts, [0, 1], "after refusals")


def test_negative_constraint_epoch_is_refused(eng):
    """The reference's constraint epochs are usize: the engine refuses a negative one when the tracker is made (compat_ok
    would compare it as a huge unsigned epoch, and the signed sort put it first, applied to every delta)."""
    from similari_b200._lib import Sb200Error, default_options

    for cons in ([(-1, 1.0)], [(2, 0.5), (-(2**31), 1.0)]):
        with pytest.raises(Sb200Error, match="constraint epochs"):
            eng.Tracker(default_options(kind=0, positional_kind=1, constraints=cons))
    eng.Tracker(default_options(kind=0, positional_kind=1, constraints=[(0, 1.0), (2**31 - 1, 2.0)])).close()
