"""Batched NMS (sb200_nms_batch / sb200_nms_batch_device) on the GPU: every set's result must equal oracle.nms on that
set alone, exactly."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 2, 63, 64, 65, 127, 500, 2049]
LOW_SET = SIZES.index(65)   # its scores all lie below the score threshold of the tests


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def clustered(rng, n, oriented, canvas=(1920.0, 1080.0), dup=5):
    """n boxes in clusters of `dup` near-duplicates (jitter 3 px / 0.03 rad), shuffled."""
    k = max(1, -(-n // dup))
    base = np.empty((k, 6), np.float32)
    base[:, 0] = rng.uniform(0, canvas[0], k)
    base[:, 1] = rng.uniform(0, canvas[1], k)
    base[:, 2] = rng.uniform(-1.5, 1.5, k) if oriented else np.nan
    base[:, 3] = rng.uniform(0.3, 0.8, k)
    base[:, 4] = rng.uniform(40, 160, k)
    base[:, 5] = 1.0
    b = np.repeat(base, dup, axis=0)[:n]
    b[:, :2] += rng.normal(0, 3, (n, 2)).astype(np.float32)
    if oriented:
        b[:, 2] += rng.normal(0, 0.03, n).astype(np.float32)
    return np.ascontiguousarray(b[rng.permutation(n)])


def offsets_of(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)


def assert_matches_oracle(oracle, got, boxes, scores, offsets, thr, score_threshold):
    assert len(got) == len(offsets) - 1
    for s in range(len(offsets) - 1):
        a, b = offsets[s], offsets[s + 1]
        ref = oracle.nms(boxes[a:b], None if scores is None else scores[a:b], thr, score_threshold)
        assert got[s].dtype == np.int32
        assert np.array_equal(got[s], ref), (s, b - a, len(got[s]), len(ref))


@pytest.mark.parametrize("oriented", [False, True])
@pytest.mark.parametrize("score_mode", ["given", "none", "partly_nan"])
@pytest.mark.parametrize("score_threshold", [None, 0.3])
def test_mixed_set_sizes_match_oracle(eng, oracle, oriented, score_mode, score_threshold):
    rng = np.random.default_rng(1000 + 10 * oriented + len(score_mode))
    boxes = np.concatenate([clustered(rng, n, oriented) for n in SIZES])
    offsets = offsets_of(SIZES)
    boxes[rng.random(len(boxes)) < 0.02, 4] = 0.0    # filtered: height 0
    boxes[rng.random(len(boxes)) < 0.02, 3] = -1.0   # filtered: aspect <= 0
    scores = rng.uniform(0, 1, len(boxes)).astype(np.float32)
    scores[offsets[LOW_SET]:offsets[LOW_SET + 1]] *= np.float32(0.25)
    if score_mode == "partly_nan":
        scores[rng.random(len(boxes)) < 0.3] = np.nan
    elif score_mode == "none":
        scores = None
    got = eng.nms_batch(boxes, scores, offsets, 0.6, score_threshold)
    assert_matches_oracle(oracle, got, boxes, scores, offsets, 0.6, score_threshold)
    if score_threshold is not None and score_mode == "given":
        assert len(got[LOW_SET]) == 0        # the threshold filters every box of the set
    assert sum(len(g) for g in got) < len(boxes) - 100   # suppression took place


def test_quantised_scores_stable_rank(eng, oracle):
    """Many equal ranks: the stable order (input order among ties) decides which duplicate survives."""
    rng = np.random.default_rng(77)
    sizes = [300, 64, 1000, 7]
    boxes = np.concatenate([clustered(rng, n, oriented=True, canvas=(800.0, 600.0)) for n in sizes])
    boxes[:, 4] = np.round(boxes[:, 4] / 40.0) * 40.0 + 40.0   # equal heights: ties among the None scores too
    scores = (np.round(rng.uniform(0, 1, len(boxes)) * 4) / 4).astype(np.float32)
    scores[rng.random(len(boxes)) < 0.2] = np.nan
    offsets = offsets_of(sizes)
    for thr, st in [(0.5, None), (0.3, 0.25)]:
        got = eng.nms_batch(boxes, scores, offsets, thr, st)
        assert_matches_oracle(oracle, got, boxes, scores, offsets, thr, st)


def bench_scenes(n_scenes=256, clusters=100, dup=5):
    """The tools/nms_bench.py --batch workload: 100 clusters x 5 near-duplicates per scene on 3840 x 2160."""
    parts, scs = [], []
    for s in range(n_scenes):
        rng = np.random.default_rng(0x5EED0000 + s)
        parts.append(clustered(rng, clusters * dup, oriented=True, canvas=(3840.0, 2160.0), dup=dup))
        scs.append(rng.uniform(0, 1, clusters * dup).astype(np.float32))
    return np.concatenate(parts), np.concatenate(scs), offsets_of([clusters * dup] * n_scenes)


def test_256_scenes_of_500_boxes_match_oracle_and_repeat(eng, oracle):
    boxes, scores, offsets = bench_scenes()
    got = eng.nms_batch(boxes, scores, offsets, 0.8)
    assert_matches_oracle(oracle, got, boxes, scores, offsets, 0.8, None)
    again = eng.nms_batch(boxes, scores, offsets, 0.8)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


def test_10k_set_between_small_sets(eng, oracle):
    rng = np.random.default_rng(5)
    sizes = [37, 10000, 100]
    boxes = np.concatenate([clustered(rng, n, oriented=True, canvas=(3840.0, 2160.0)) for n in sizes])
    scores = rng.uniform(0, 1, len(boxes)).astype(np.float32)
    offsets = offsets_of(sizes)
    got = eng.nms_batch(boxes, scores, offsets, 0.8)
    alone = eng.nms_indices(boxes[37:10037], scores[37:10037], 0.8)
    assert np.array_equal(got[1], alone) and 2000 <= len(alone) < 10000
    for s in (0, 2):
        a, b = offsets[s], offsets[s + 1]
        assert np.array_equal(got[s], oracle.nms(boxes[a:b], scores[a:b], 0.8))


def test_launch_count_does_not_depend_on_the_number_of_sets(eng):
    boxes, scores, offsets = bench_scenes()
    one = offsets[:2]
    eng.nms_batch(boxes[:500], scores[:500], one, 0.8)
    c0 = eng.launch_count()
    eng.nms_batch(boxes[:500], scores[:500], one, 0.8)
    c1 = eng.launch_count()
    eng.nms_batch(boxes, scores, offsets, 0.8)
    c2 = eng.launch_count()
    assert c1 - c0 == c2 - c1 > 0


@pytest.mark.parametrize("with_scores", [True, False])
def test_device_entry_on_a_side_stream_equals_host_entry(eng, with_scores):
    import torch

    from similari_b200._lib import lib, ptr

    rng = np.random.default_rng(31)
    sizes = [0, 500, 3, 64, 2049, 1]
    boxes = np.concatenate([clustered(rng, n, oriented=True) for n in sizes])
    scores = rng.uniform(0, 1, len(boxes)).astype(np.float32) if with_scores else None
    offsets = offsets_of(sizes)
    total, n_sets = len(boxes), len(sizes)
    h_idx, h_cnt, h_mask = np.zeros(total, np.int32), np.zeros(n_sets, np.int32), np.zeros(total, np.uint8)
    kept = lib().sb200_nms_batch(n_sets, ptr(offsets), ptr(boxes), ptr(scores), 0.6, 0.2, 1, ptr(h_idx), ptr(h_cnt),
                                 ptr(h_mask), 0)
    assert kept == h_cnt.sum()
    got = eng.nms_batch(boxes, scores, offsets, 0.6, 0.2)
    for s in range(n_sets):
        assert np.array_equal(h_idx[offsets[s]:offsets[s] + h_cnt[s]], got[s])

    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d_boxes = torch.from_numpy(boxes).cuda()
        d_scores = torch.from_numpy(scores).cuda() if with_scores else None
        d_idx = torch.full((total,), 12345, dtype=torch.int32, device="cuda")
        d_cnt = torch.full((n_sets,), 12345, dtype=torch.int32, device="cuda")
        d_mask = torch.full((total,), 7, dtype=torch.uint8, device="cuda")
    eng.nms_batch_device(offsets, d_boxes.data_ptr(), d_scores.data_ptr() if with_scores else 0, 0.6, 0.2,
                         d_idx.data_ptr(), d_cnt.data_ptr(), d_mask.data_ptr(), stream=side.cuda_stream)
    side.synchronize()
    idx, cnt, mask = d_idx.cpu().numpy(), d_cnt.cpu().numpy(), d_mask.cpu().numpy()
    assert np.array_equal(cnt, h_cnt) and np.array_equal(idx, h_idx) and np.array_equal(mask, h_mask)
    for s in range(n_sets):
        a, b, c = offsets[s], offsets[s + 1], cnt[s]
        assert np.all(idx[a + c:b] == -1)
        expect = np.zeros(b - a, np.uint8)
        expect[idx[a:a + c]] = 1
        assert np.array_equal(mask[a:b], expect)


def test_capacity_limit_leaves_outputs_untouched(eng):
    import torch

    from similari_b200._lib import lib, ptr

    L = lib()
    big = 64 * 25600 + 1     # ceil(n / 64) * 8 bytes just above the 200 KB sweep bitmap
    offsets = np.array([0, 5, 5 + big, 8 + big], np.int32)
    boxes = np.ones((8, 6), np.float32)     # never read: the check comes first
    idx, cnt = np.full(16, 9, np.int32), np.full(3, 9, np.int32)
    assert L.sb200_nms_batch(3, ptr(offsets), ptr(boxes), None, 0.5, 0.0, 0, ptr(idx), ptr(cnt), None, 0) == -3
    assert b"set 1" in L.sb200_last_error()
    assert np.all(idx == 9) and np.all(cnt == 9)
    assert L.sb200_nms(ptr(boxes), None, big, 0.5, 0.0, 0, ptr(idx), 0) == -3
    assert np.all(idx == 9)
    d_boxes = torch.ones((8, 6), dtype=torch.float32, device="cuda")
    d_idx = torch.full((16,), 9, dtype=torch.int32, device="cuda")
    d_cnt = torch.full((3,), 9, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(Exception, match="status -3"):
        eng.nms_batch_device(offsets, d_boxes.data_ptr(), 0, 0.5, None, d_idx.data_ptr(), d_cnt.data_ptr())
    torch.cuda.synchronize()
    assert bool((d_idx == 9).all()) and bool((d_cnt == 9).all())


def test_empty_requests(eng):
    assert eng.nms_batch(np.zeros((0, 6), np.float32), None, [0], 0.5) == []
    got = eng.nms_batch(np.zeros((0, 6), np.float32), None, [0, 0, 0], 0.5)
    assert len(got) == 2 and all(len(g) == 0 for g in got)


def test_api_nms_batch_equals_nms_per_scene():
    from similari_b200.api import Universal2DBox, nms, nms_batch

    rng = np.random.default_rng(12)
    scenes = {}
    for sid, n in [(7, 40), (3, 0), (11, 120), (2**40, 9)]:
        b = clustered(rng, n, oriented=bool(sid % 2), canvas=(500.0, 400.0))
        sc = rng.uniform(0, 1, n)
        scenes[sid] = [(Universal2DBox.new_with_confidence(*r[:5].tolist(), 1.0) if not np.isnan(r[2]) else
                        Universal2DBox.new_with_confidence(r[0], r[1], None, r[3], r[4], 1.0),
                        None if i % 5 == 0 else float(sc[i])) for i, r in enumerate(b)]
    got = nms_batch(scenes, 0.5, 0.1)
    assert list(got) == list(scenes)
    for sid, dets in scenes.items():
        assert got[sid] == nms(dets, 0.5, 0.1)
