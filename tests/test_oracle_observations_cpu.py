"""The oracle's per-track observation dump (Tracker.scene_observations) against the reference's merge rule, written out
here: one VisualSort track merged frame after frame with hand-picked qualities -- ties, a feature-less detection, a merge
below the collect threshold, one exactly on it -- for several visual_max_observations.  This pins the entry point the
device-state tests compare the GPU with, independently of the GPU."""
import numpy as np
import pytest

D = 12            # not a multiple of 8: the dump zero-pads every row to d8 = 16
D8 = 16
Q_COLLECT = 0.4
# (quality, has_feature) of detection 0 (the new track) and of every merge after it
SCRIPT = [(0.5, True), (0.5, True), (0.9, True), (0.5, True), (0.3, True), (0.9, True), (0.7, False), (0.5, True),
          (0.4, True), (np.nextafter(np.float32(0.4), np.float32(0)), True), (0.9, True), (0.5, True), (0.5, False),
          (0.5, True), (0.2, True), (0.9, True)]


def _norm2(row):
    """Squared norm in the order cosine accumulates it (distance.rs:36-44): per 8-lane block the reduce_add tree
    (lo + hi quads, then pairs, then the last two), blocks added one after the other, all in f32."""
    acc = np.float32(0)
    for b in range(len(row) // 8):
        t = row[8 * b: 8 * b + 8].astype(np.float32) ** 2
        q = t[:4] + t[4:]
        d = q[:2] + q[2:]
        acc = np.float32(acc + np.float32(d[0] + d[1]))
    return acc


def _merge(obs, new, K):
    """VisualMetric::optimize with is_merge (visual_sort/metric.rs:297-374, 129-154) on a list of (quality, feature or
    None): retain the featured entries, stable sort by quality descending, drop the last when len >= K, push the new
    observation, swap(0, last)."""
    obs = [o for o in obs if o[1] is not None]
    obs.sort(key=lambda o: -o[0])   # list.sort is stable
    if len(obs) >= K and obs:
        obs.pop()
    obs.append(new)
    obs[0], obs[-1] = obs[-1], obs[0]
    return obs


@pytest.mark.parametrize("K", [1, 2, 3, 5])
def test_scene_observations_follow_the_merge_rule(oracle, K):
    rng = np.random.default_rng(0x0B5E + K)
    o = oracle.Tracker(oracle.make_options(kind=oracle.KIND_VISUAL_SORT, positional_kind=oracle.POS_IOU,
                                           iou_threshold=0.3, max_idle_epochs=3, feature_dim=D,
                                           visual_max_observations=K, visual_minimal_track_length=1,
                                           visual_minimal_quality_collect=Q_COLLECT))
    box = oracle.box(100.0, 80.0, None, 0.5, 60.0, 0.9)
    want = []
    tid = None
    for i, (q, hf) in enumerate(SCRIPT):
        q = np.float32(q)
        feat = rng.standard_normal(D).astype(np.float32)
        r = o.predict_batch([0], [0, 1], box[None], features=feat[None], has_feature=[hf], quality=[q])
        if i == 0:
            tid = int(r["ids"][0])
            want = [(q, feat if hf else None)]
        else:
            assert int(r["ids"][0]) == tid, i           # every detection merges into the one track
            kept = feat if (hf and q >= np.float32(Q_COLLECT)) else None   # the collect gate of a merge
            want = _merge(want, (q, kept), K)
        got = o.scene_observations(0)
        assert got["n_obs"].tolist() == [len(want)], i
        assert got["feats"].shape == (1, K, D8)
        for k in range(K):
            if k < len(want):
                wq, wf = want[k]
                assert got["quality"][0, k].view(np.uint32) == np.float32(wq).view(np.uint32), (i, k)
                assert got["has_feat"][0, k] == (wf is not None), (i, k)
                row = np.zeros(D8, np.float32)
                if wf is not None:
                    row[:D] = wf
                assert np.array_equal(got["feats"][0, k], row), (i, k)
                assert got["norm2"][0, k].view(np.uint32) == (_norm2(row) if wf is not None else np.float32(0)).view(np.uint32), (i, k)
            else:
                assert got["has_feat"][0, k] == 0 and got["quality"][0, k] == 0 and not got["feats"][0, k].any()
        assert int(o.scene_tracks(0)["feat_counts"][0]) == sum(f is not None for _, f in want), i


def test_scene_observations_of_an_unknown_scene_are_empty(oracle):
    o = oracle.Tracker(oracle.make_options(kind=oracle.KIND_VISUAL_SORT, feature_dim=D, visual_max_observations=3))
    got = o.scene_observations(7)
    assert len(got["n_obs"]) == 0 and got["feats"].shape == (0, 3, D8)
