"""Tensor-core visual screen against the CPU oracle at the shapes that select its work organisation.  D <= 512 runs the
A-stationary kernel over units of (scene, pair of 128-row candidate tiles, column range): column-split units when the
candidate-tile pairs are too few to give every cluster two units, whole scenes otherwise.  D > 512 runs the streaming
kernel over 256-column tiles."""
import numpy as np
import pytest

from test_gpu_parity import assert_bits_equal
from test_gpu_tracker import run_frames, small

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


# 300 candidates: the second candidate tile of the cluster is ragged (rows 256..299).  600 columns: five 128-column tiles
# split into units of two, two and one, so the last unit leaves one consumer warpgroup without a tile.  D = 512 fills the
# resident A; D = 640 takes the streaming kernel.
@pytest.mark.parametrize("kind", ["euclid", "cosine"])
@pytest.mark.parametrize("m,n,d", [(300, 600, 512), (300, 600, 640), (40, 1100, 200)])
def test_screen_operator_bit_exact(eng, oracle, kind, m, n, d, monkeypatch):
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    rng = np.random.default_rng(700 + d)
    cent = rng.standard_normal((n, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cf = cent[rng.integers(0, n, m)] + 0.02 * rng.standard_normal((m, d)).astype(np.float32)
    cf = (cf / np.linalg.norm(cf, axis=1, keepdims=True)).astype(np.float32)
    if kind == "euclid":
        ref = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, 1.2, cf, cent)
        got = eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, 1.2, cf, cent)
    else:
        ref = oracle.visual_cost_matrix(oracle.VIS_COSINE, 0.1, cf, cent)
        got = eng.visual_cost_matrix(eng._lib.VIS_COSINE, 0.1, cf, cent)
    assert_bits_equal(ref, got)
    assert np.isfinite(got).sum() >= m


@pytest.mark.parametrize("vis", [0, 1])
def test_screen_single_tile_units_match_oracle(eng, oracle, vis, monkeypatch):
    """140 scenes of 24 objects: more candidate-tile pairs than the H100 has SMs, so every unit is a whole scene, and a
    scene holds at most 72 feature rows, so every unit is ONE column tile: one consumer warpgroup has no tile in it and
    the producer stands in for it on the barrier that frees the resident A before the next unit's A is loaded."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cfg = small("cfg5", n_scenes=140, n_objects=24, oriented=False, canvas=(900.0, 600.0), feature_dim=512)
    run_frames(eng, oracle, cfg, 4,
               dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                    visual_threshold=0.7 if vis == 0 else 0.2, feature_dim=512, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))


@pytest.mark.parametrize("vis", [0, 1])
def test_screen_whole_scene_units_match_oracle(eng, oracle, vis, monkeypatch):
    """The benchmark's organisation: 140 scenes of 150 objects give more candidate-tile pairs than the H100 has SMs, so
    every unit is a whole scene and each cluster runs two or three units one after another.  From the second frame on a
    scene holds 150-205 tracks x 3 feature rows: units of four or five 128-column tiles, both consumer warpgroups working
    through several tiles on the same resident A before the last tile of each releases it for the next unit's load."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cfg = small("cfg5", n_scenes=140, n_objects=150, oriented=False, canvas=(1400.0, 900.0), feature_dim=128)
    run_frames(eng, oracle, cfg, 5,
               dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                    visual_threshold=0.7 if vis == 0 else 0.2, feature_dim=128, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))


@pytest.mark.parametrize("d", [512, 768])
def test_screen_column_split_units_match_oracle(eng, oracle, d, monkeypatch):
    """Two scenes of 300 candidates: four candidate-tile pairs, so the columns are split into units of two tiles; D = 768
    runs the same frames through the streaming kernel."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cfg = small("cfg5", n_scenes=2, n_objects=300, oriented=False, canvas=(2200.0, 1400.0), feature_dim=d)
    run_frames(eng, oracle, cfg, 4,
               dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0,
                    visual_threshold=0.7, feature_dim=d, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))
