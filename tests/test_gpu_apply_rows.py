"""The apply stage runs by store row: every stored track is updated by the thread of its row, which finds its detection
through the inverse map the rank pass builds.  These frames send each scene's detections in the reverse of the store
order, with fresh objects in the middle, so that the map is anything but the identity, and compare the outputs and the
whole device store with the oracle frame after frame, for all four tracker kinds and K within and above kMaxObs."""
import numpy as np
import pytest

from test_gpu_track_observations import both, check_outputs, check_state, predict_both

pytestmark = pytest.mark.gpu

IOU = 1
FRAMES = 8


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


class ReversedScenes:
    """Objects on a grid, far enough apart that most keep their track.  Frame 0 creates the tracks in object order;
    later frames list each scene's known objects in the reverse of that order (the store order: new tracks are appended),
    with three fresh objects in the middle of the list."""

    def __init__(self, n_scenes, n_objects, d, seed):
        self.rng = np.random.default_rng(seed)
        self.S, self.d = n_scenes, d
        self.pos = [[(100.0 + 90.0 * (i % 14), 100.0 + 90.0 * (i // 14)) for i in range(n_objects)] for _ in range(n_scenes)]
        self.cent = [[self._unit(self.rng.standard_normal(d)) for _ in range(n_objects)] for _ in range(n_scenes)] if d else None
        self.frame = 0

    @staticmethod
    def _unit(v):
        return (v / np.linalg.norm(v)).astype(np.float32)

    def next_frame(self):
        r = self.rng
        boxes, feats, offs = [], [], [0]
        for s in range(self.S):
            order = list(range(len(self.pos[s])))
            if self.frame > 0:
                order = order[::-1]
                fresh = []
                for _ in range(3):
                    k = len(self.pos[s])
                    self.pos[s].append((100.0 + 90.0 * (k % 14), 100.0 + 90.0 * (k // 14)))
                    if self.d:
                        self.cent[s].append(self._unit(r.standard_normal(self.d)))
                    fresh.append(k)
                mid = len(order) // 2
                order = order[:mid] + fresh + order[mid:]
            for i in order:
                x, y = self.pos[s][i]
                x, y = x + float(r.normal(0, 1.0)), y + float(r.normal(0, 1.0))
                self.pos[s][i] = (x, y)
                boxes.append([x, y, np.nan, 0.5, 40.0 * float(r.uniform(0.98, 1.02)), float(r.uniform(0.3, 1.0))])
                if self.d:
                    feats.append(self._unit(self.cent[s][i] + 0.02 * r.standard_normal(self.d)))
            offs.append(len(boxes))
        self.frame += 1
        n = len(boxes)
        f = {"scene_ids": np.arange(self.S, dtype=np.uint64), "det_offsets": np.asarray(offs, np.int32),
             "boxes": np.asarray(boxes, np.float32)}
        if self.d:
            f["features"] = np.stack(feats).astype(np.float32)
            f["quality"] = r.choice(np.array([0.3, 0.6, 0.9, 0.9, 1.0], np.float32), n)
            f["has_feature"] = (r.random(n) >= 0.1).astype(np.uint8)
        return f


CASES = [(0, 3), (1, 3), (2, 3), (3, 3), (2, 25), (3, 25)]


@pytest.mark.parametrize("kind,K", CASES, ids=[f"kind{c[0]}-K{c[1]}" for c in CASES])
def test_reverse_store_order_matches_oracle(eng, oracle, kind, K):
    visual = kind >= 2
    d = 64 if visual else 0
    opts = dict(kind=kind, positional_kind=IOU, iou_threshold=0.3, max_idle_epochs=2, min_confidence=0.1)
    if visual:
        opts.update(visual_kind=0, visual_threshold=0.7, feature_dim=d, visual_max_observations=K,
                    visual_min_votes=min(2, K), visual_minimal_track_length=1, visual_minimal_quality_use=0.5,
                    visual_minimal_quality_collect=0.5)
    wl = ReversedScenes(1 if kind in (0, 2) else 3, 150, d, 0x5EEDB000 + 31 * kind + K)
    g, o = both(eng, oracle, **opts)
    for fr in range(FRAMES):
        f = wl.next_frame()
        rg, ro = predict_both(g, o, f)
        check_outputs(rg, ro, fr)
        check_state(g, o, opts, f["scene_ids"], fr)
        if fr > 0:   # most known objects merged: the map was mostly the reversed store order
            m = int(f["det_offsets"][1])
            assert int((np.asarray(rg["lengths"][:m]) > 1).sum()) >= 0.5 * m, fr
