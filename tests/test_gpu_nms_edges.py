"""Batched NMS on the GPU at its edges: the sweep's column-chunked path on detector-sized sets, the suppression test
at its threshold, the filters and ranks at theirs, degenerate boxes, and the refusal of a set whose mask cannot fit on
the device.  Every result equals oracle.nms on each set alone, exactly."""
import math

import numpy as np
import pytest

from test_gpu_nms_batch import clustered, eng, offsets_of  # noqa: F401  (eng: the module's fixture)

pytestmark = pytest.mark.gpu

F32 = np.float32
NAN = float("nan")
INF = float("inf")
SMALL_SETS = [0, 3, 64, 2049]


def below(x):
    """The f32 just below x: the largest threshold at which a metric of exactly x is suppressed."""
    return float(np.nextafter(F32(x), F32(-INF)))


# --------------------------------------------------------------------------- running both entries
def run_device(eng, boxes, scores, offsets, thr, st):
    """sb200_nms_batch_device with a keep mask: per set, the kept indices; checks the -1 fill and the mask."""
    import torch

    total, n_sets = len(boxes), len(offsets) - 1
    d_boxes = torch.from_numpy(np.ascontiguousarray(boxes, F32)).cuda()
    d_scores = torch.from_numpy(np.ascontiguousarray(scores, F32)).cuda() if scores is not None else None
    d_idx = torch.full((max(total, 1),), 12345, dtype=torch.int32, device="cuda")
    d_cnt = torch.full((n_sets,), 12345, dtype=torch.int32, device="cuda")
    d_mask = torch.full((max(total, 1),), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.nms_batch_device(offsets, d_boxes.data_ptr(), d_scores.data_ptr() if d_scores is not None else 0, thr, st,
                         d_idx.data_ptr(), d_cnt.data_ptr(), d_mask.data_ptr())
    torch.cuda.synchronize()
    idx, cnt, mask = d_idx.cpu().numpy(), d_cnt.cpu().numpy(), d_mask.cpu().numpy()
    out = []
    for s in range(n_sets):
        a, b, c = offsets[s], offsets[s + 1], cnt[s]
        assert 0 <= c <= b - a
        assert np.all(idx[a + c:b] == -1)
        expect = np.zeros(b - a, np.uint8)
        expect[idx[a:a + c]] = 1
        assert np.array_equal(mask[a:b], expect)
        out.append(idx[a:a + c])
    return out


def check(eng, oracle, boxes, scores, sizes, thr, st=None, refs=None, indices=False, device=True):
    """nms_batch (and the device entry, and nms_indices per set if asked) against oracle.nms on each set alone."""
    offsets = offsets_of(sizes)
    if refs is None:
        refs = [oracle.nms(boxes[a:b], None if scores is None else scores[a:b], thr, st)
                for a, b in zip(offsets[:-1], offsets[1:])]
    got = eng.nms_batch(boxes, scores, offsets, thr, st)
    for s, (g, r) in enumerate(zip(got, refs)):
        assert np.array_equal(g, r), ("nms_batch", s, sizes[s], first_difference(g, r))
    if device:
        for s, (g, r) in enumerate(zip(run_device(eng, boxes, scores, offsets, thr, st), refs)):
            assert np.array_equal(g, r), ("nms_batch_device", s, sizes[s], first_difference(g, r))
    if indices:
        for s, r in enumerate(refs):
            a, b = offsets[s], offsets[s + 1]
            g = eng.nms_indices(boxes[a:b], None if scores is None else scores[a:b], thr, st)
            assert np.array_equal(g, r), ("nms_indices", s, sizes[s], first_difference(g, r))
    return refs


def first_difference(got, ref):
    n = min(len(got), len(ref))
    k = next((i for i in range(n) if got[i] != ref[i]), n)
    return {"position": k, "got": got[k:k + 3].tolist(), "oracle": ref[k:k + 3].tolist(), "lengths": (len(got), len(ref))}


# --------------------------------------------------------------------------- the sweep's column chunks
def sweep_chunk(max_words):
    """nms_enqueue's column chunk for a request whose largest set has max_words mask words, on device 0."""
    import torch

    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    avail_words = (optin - 64) // 8 - max_words
    return max(1, min(max_words, avail_words // 128))


def block0_chunks(n):
    """Column chunks block 0 of a set of n boxes (all valid) takes when it is the largest set of its request."""
    w = (n + 63) // 64
    return -(-w // sweep_chunk(w)), sweep_chunk(w)


def chunk_sizes():
    """Set sizes whose block 0 takes 1, 2, 2, 3 and 5 chunks: the largest set the suite ran before, the smallest set
    that takes two (its second chunk one word wide), and the candidate boxes of YOLOv5 at 640 x 640 (25,200) and of
    YOLOv8 at 1280 x 1280 (33,600), and 60,000."""
    w = 1
    while sweep_chunk(w) >= w:
        w += 1
    first_two = 64 * (w - 1) + 1            # w words: the second chunk holds the last word only
    sizes = {"1": 10000, "2/1-word": first_two, "2": 25200, "3": 33600, "5": 60000}
    want = {"1": 1, "2/1-word": 2, "2": 2, "3": 3, "5": 5}
    got = {k: block0_chunks(n)[0] for k, n in sizes.items()}
    assert got == want, ("this device's shared memory gives other chunk counts", got)
    n = sizes["2/1-word"]
    assert (n + 63) // 64 - block0_chunks(n)[1] == 1
    return sizes


CHUNK_CASES = [
    ("1", False, "random"),
    ("2/1-word", False, "random"),
    ("2/1-word", True, "absent"),
    ("2/1-word", True, "quantised"),
    ("2", True, "absent"),
    ("3", False, "quantised"),
    ("5", True, "random"),
]


def scored(rng, n, mode):
    if mode == "absent":
        return None
    s = rng.uniform(0, 1, n).astype(F32)
    return (np.round(s * 4) / 4).astype(F32) if mode == "quantised" else s


@pytest.mark.parametrize("chunks,oriented,score_mode", CHUNK_CASES)
def test_chunked_sweep_matches_oracle(eng, oracle, chunks, oriented, score_mode):
    n = chunk_sizes()[chunks]
    rng = np.random.default_rng(n + 10 * oriented + len(score_mode))
    k = math.sqrt(n / 10000)     # the density of 10,000 boxes on 3840 x 2160
    big = clustered(rng, n, oriented, canvas=(3840.0 * k, 2160.0 * k))
    sc = scored(rng, n, score_mode)
    ref = check(eng, oracle, big, sc, [n], 0.5, indices=True)[0]
    assert 0.05 * n < len(ref) < 0.5 * n
    # next to small sets: the chunk comes from the largest set, so the small ones run with a chunk wider than they are
    small = [clustered(rng, m, oriented) for m in SMALL_SETS]
    sizes = SMALL_SETS[:2] + [n] + SMALL_SETS[2:]
    parts = small[:2] + [big] + small[2:]
    boxes = np.concatenate(parts)
    scores = None if sc is None else np.concatenate(
        [scored(rng, len(p), score_mode) if p is not big else sc for p in parts])
    refs = [oracle.nms(p, None if scores is None else scores[a:a + len(p)], 0.5) if p is not big else ref
            for p, a in zip(parts, offsets_of(sizes)[:-1])]
    check(eng, oracle, boxes, scores, sizes, 0.5, refs=refs)


def chain_set(n, wb, wc, rng):
    """n boxes ranked by score.  64 chains A_k -> B_k -> C_k of axis-aligned 100 x 100 boxes at x = 0, 30, 60 (the
    neighbours overlap 0.7, the outer pair 0.4): A_k at rank k, B_k at rank 64 wb + k, C_k at rank 64 wc + k.  Every
    other rank holds a box disjoint from all others.  Returns boxes and scores in shuffled input order, and the input
    indices greedy NMS at threshold 0.5 keeps, in rank order: everything but the B_k."""
    geo = np.empty((n, 6), F32)
    g = np.arange(n)
    geo[:, 0] = 200.0 * (g % 250)
    geo[:, 1] = 200.0 * (g // 250)
    geo[:, 2] = NAN
    geo[:, 3] = 1.0
    geo[:, 4] = 60.0
    geo[:, 5] = 1.0
    for k in range(64):
        x0 = 400.0 * k
        for w, dx in ((0, 0.0), (wb, 30.0), (wc, 60.0)):
            geo[64 * w + k] = [x0 + 50.0 + dx, -1000.0, NAN, 1.0, 100.0, 1.0]
    perm = rng.permutation(n)                        # rank r goes to input position perm[r]
    boxes = np.empty_like(geo)
    boxes[perm] = geo
    scores = np.empty(n, F32)
    scores[perm] = (n - np.arange(n)).astype(F32)    # distinct and exact: rank r has score n - r
    b_ranks = set(64 * wb + np.arange(64))
    expect = np.array([perm[r] for r in range(n) if r not in b_ranks], np.int32)
    return boxes, scores, expect


@pytest.mark.parametrize("layout", ["b_first_word_of_chunk_2", "b_last_word_of_chunk_2"])
def test_chains_across_chunks(eng, oracle, layout):
    """A keeps and removes B through a mask word past block 0's first chunk; C then survives, since its only
    suppressor B is gone.  If that word reached `removed` late or not at all, B would be kept and would remove C."""
    n = chunk_sizes()["3"]
    chunks, chunk = block0_chunks(n)
    nw = (n + 63) // 64
    assert chunks == 3
    if layout == "b_first_word_of_chunk_2":
        wb, wc = chunk, chunk + 1
    else:
        wb, wc = 2 * chunk - 1, nw - 1           # C in block 0's third chunk
    assert chunk <= wb < 2 * chunk and wb < wc < nw and wc - wb < chunk
    rng = np.random.default_rng(wb)
    boxes, scores, expect = chain_set(n, wb, wc, rng)
    a, b, c = (oracle.box(50.0 + dx, 0.0, None, 1.0, 100.0) for dx in (0.0, 30.0, 60.0))
    assert oracle.intersection(a, b) == 7000.0 and oracle.intersection(a, c) == 4000.0
    ref = check(eng, oracle, boxes, scores, [n], 0.5, indices=True)[0]
    assert np.array_equal(ref, expect)
    tail = oracle.nms(boxes[:3], scores[:3], 0.5)
    check(eng, oracle, np.concatenate([boxes, boxes[:3]]), np.concatenate([scores, scores[:3]]), [n, 3], 0.5,
          refs=[ref, tail])


@pytest.mark.parametrize("filtered_by", ["score", "geometry"])
def test_large_set_mostly_filtered(eng, oracle, filtered_by):
    """30,000 boxes of which about 100 pass the filters: a slab pitch of 469 words over 2 valid blocks."""
    rng = np.random.default_rng(3 + len(filtered_by))
    n = 30000
    boxes = clustered(rng, n, oriented=True, canvas=(800.0, 600.0))
    live = rng.permutation(n)[:100]
    if filtered_by == "score":
        scores = rng.uniform(0, 0.5, n).astype(F32)
        scores[live] = rng.uniform(0.6, 1.0, 100).astype(F32)
        st = 0.55
    else:
        scores, st = None, None
        dead = np.setdiff1d(np.arange(n), live)
        kinds = rng.integers(0, 4, len(dead))
        boxes[dead[kinds == 0], 4] = 0.0
        boxes[dead[kinds == 1], 4] = -5.0
        boxes[dead[kinds == 2], 3] = NAN
        boxes[dead[kinds == 3], 3] = 0.0
    ref = check(eng, oracle, boxes, scores, [n], 0.5, st, indices=True)[0]
    assert 0 < len(ref) <= 100
    small = clustered(rng, 64, oriented=True)
    sc2 = None if scores is None else np.concatenate([scores, rng.uniform(0.6, 1, 64).astype(F32)])
    check(eng, oracle, np.concatenate([boxes, small]), sc2, [n, 64], 0.5, st)


# --------------------------------------------------------------------------- the suppression test at its threshold
def square(x, y, side, aspect=1.0):
    return np.array([x, y, NAN, aspect, side, 1.0], F32)


EXACT_PAIRS = [   # (kept box, later box, intersection over the later box's area)
    (square(0, 0, 64), square(16, 0, 64), 0.75),
    (square(0, 0, 64), square(32, 0, 64), 0.5),
    (square(0, 0, 64), square(48, 0, 64), 0.25),
    (square(0, 0, 64), square(32, 32, 64), 0.25),
    (square(0, 0, 64, 2.0), square(64, 0, 64, 2.0), 0.5),
    (square(0, 0, 64), square(8, 8, 32), 1.0),        # small inside big, big first
    (square(8, 8, 32), square(0, 0, 64), 0.25),       # the same pair, small first
]


@pytest.mark.parametrize("at", ["threshold", "just_below"])
def test_metric_equal_to_threshold(eng, oracle, at):
    """The later box survives a metric equal to the threshold (the test is strict) and is removed one ulp below."""
    for cb, ob, m in EXACT_PAIRS:
        area = F32(ob[4]) * F32(ob[3]) * F32(ob[4])
        inter = oracle.intersection(cb, ob)
        assert inter == m * float(area) and F32(inter) / area == F32(m)     # exact in f64 and f32
        boxes = np.stack([cb, ob])
        scores = np.array([0.9, 0.8], F32)
        thr = m if at == "threshold" else below(m)
        ref = check(eng, oracle, boxes, scores, [2], thr)[0]
        assert ref.tolist() == ([0, 1] if at == "threshold" else [0])
    # all pairs in one request, with the sets in both orders of their boxes' scores
    boxes = np.concatenate([np.stack([cb, ob]) for cb, ob, _ in EXACT_PAIRS] * 2)
    scores = np.array([0.9, 0.8] * len(EXACT_PAIRS) + [0.8, 0.9] * len(EXACT_PAIRS), F32)
    for m in (0.25, 0.5, 0.75, 1.0):
        check(eng, oracle, boxes, scores, [2] * (2 * len(EXACT_PAIRS)), m if at == "threshold" else below(m))


@pytest.mark.parametrize("thr", [0.0, -0.1, NAN])
def test_thresholds_at_and_below_zero_and_nan(eng, oracle, thr):
    rng = np.random.default_rng(11)
    sizes = [500, 65, 2049]
    boxes = np.concatenate([clustered(rng, m, oriented=True, canvas=(3000.0, 2000.0)) for m in sizes])
    scores = rng.uniform(0, 1, len(boxes)).astype(F32)
    refs = check(eng, oracle, boxes, scores, sizes, thr, indices=True)
    offsets = offsets_of(sizes)
    for s, r in enumerate(refs):
        a, b = offsets[s], offsets[s + 1]
        if thr < 0:   # every later box goes, those behind the too_far gate (metric 0) included
            assert r.tolist() == [int(np.argmax(scores[a:b]))]
        elif thr != thr:   # nothing is ever suppressed: every box, in rank order
            assert r.tolist() == np.argsort(-scores[a:b], kind="stable").tolist()
        else:
            assert 1 < len(r) < b - a


@pytest.mark.parametrize("thr", [1.0, below(1.0)])
def test_identical_oriented_boxes_at_threshold_1(eng, oracle, thr):
    """The f64 clip of a box with itself over its f32 area can land on either side of 1."""
    rng = np.random.default_rng(21)
    m = 600
    base = np.empty((m, 6), F32)
    base[:, 0] = 1000.0 * (np.arange(m) % 30)
    base[:, 1] = 1000.0 * (np.arange(m) // 30)
    base[:, 2] = rng.uniform(-3.2, 3.2, m)
    base[:, 3] = rng.uniform(0.2, 3.0, m)
    base[:, 4] = rng.uniform(1.0, 300.0, m)
    base[:, 5] = 1.0
    boxes = np.repeat(base, 2, axis=0)
    scores = rng.uniform(0, 1, 2 * m).astype(F32)
    ref = check(eng, oracle, boxes, scores, [2 * m], thr, indices=True)[0]
    assert m <= len(ref) <= 2 * m
    check(eng, oracle, boxes, scores, [2] * m, thr)


# --------------------------------------------------------------------------- filters and ranks
def spread(n):
    """n axis-aligned 10 x 10 boxes, 100 apart: nothing suppresses anything, the output is the filter and the rank."""
    b = np.zeros((n, 6), F32)
    b[:, 0] = 100.0 * np.arange(n)
    b[:, 2] = NAN
    b[:, 3] = 1.0
    b[:, 4] = 10.0
    b[:, 5] = 1.0
    return b


@pytest.mark.parametrize("st", [None, 0.3, -INF, NAN])
def test_filters_and_ranks_at_their_edges(eng, oracle, st):
    sub = float(np.finfo(F32).smallest_subnormal)
    score_col = [0.3, 0.3, INF, -INF, -0.0, 0.0, -0.0, NAN, NAN, 0.5, 0.30000004, 0.29999998, 0.5, 0.5, 0.5, 0.5, 0.5,
                 0.5, 0.5, 0.5, 0.5, 0.5, NAN, NAN, INF, 1e-45]
    n = len(score_col)
    boxes = spread(n)
    scores = np.array(score_col, F32)
    # geometry filters on the boxes scored 0.5 from index 12 on; the NaN-scored ones rank by height
    for i, (col, v) in enumerate([(4, 0.0), (4, -1.0), (4, NAN), (4, sub), (3, 0.0), (3, -2.0), (3, NAN), (3, sub),
                                  (4, -0.0), (3, -0.0)]):
        boxes[12 + i, col] = v
    boxes[22, 4] = 2.0           # no score: ranks by its height, between the heights of 7, 8 and the scores
    boxes[23, 4] = sub           # no score, subnormal height: valid, ranks last among the valid
    ref = check(eng, oracle, boxes, scores, [n], 0.5, st, indices=True)[0]
    if st is not None and st != st:
        assert len(ref) == 0       # score > NaN is false, for the f32::MAX of boxes without a score as well
    if st == 0.3:
        assert 0 not in ref and 1 not in ref and 10 in ref and 11 not in ref   # a score equal to the threshold fails
    if st is None:
        assert ref[:5].tolist() == [2, 24, 7, 8, 22] and 3 not in ref   # +inf first, in input order; -inf fails
        pos = {int(i): k for k, i in enumerate(ref)}
        assert pos[4] < pos[5] < pos[6]                                # -0.0 and +0.0 tie: input order
    # the same set without scores: the filter is height and aspect only, the rank the height
    check(eng, oracle, boxes, None, [n], 0.5, st)


@pytest.mark.parametrize("with_scores", [True, False])
def test_identical_boxes_tie_across_rank_chunks(eng, oracle, with_scores):
    """2,049 identical boxes with equal ranks: ties across the rank kernel's 256-row chunks and the mask kernel's 64-row
    tiles.  The stable order keeps index 0 only."""
    n = 2049
    boxes = np.tile(np.array([[500.0, 400.0, 0.3, 0.5, 80.0, 1.0]], F32), (n, 1))
    scores = np.full(n, 0.7, F32) if with_scores else None
    ref = check(eng, oracle, boxes, scores, [n], 0.5, indices=True)[0]
    assert ref.tolist() == [0]
    check(eng, oracle, np.concatenate([boxes, boxes[:300]]),
          None if scores is None else np.concatenate([scores, scores[:300]]), [n, 300], 0.5)


# --------------------------------------------------------------------------- degenerate geometry
def degenerate_sets():
    """Small sets of degenerate boxes; each set is ranked by its scores (first highest)."""
    b = lambda x, y, a, asp, h: np.array([x, y, a, asp, h, 1.0], F32)   # noqa: E731
    tiny = 1e-23                   # area 1e-46: underflows to 0 in f32
    return {
        "nan_centre": [b(NAN, 0, NAN, 1, 10), b(0, 0, NAN, 1, 10), b(3, 0, NAN, 1, 10)],
        "inf_centres": [b(INF, 0, NAN, 1, 10), b(INF, 0, NAN, 1, 10), b(-INF, 5, NAN, 1, 10), b(0, INF, NAN, 1, 10),
                        b(0, 0, NAN, 1, 10)],
        "inf_angle": [b(0, 0, INF, 1, 10), b(1, 0, 0.2, 1, 10), b(0, 0, -INF, 1, 10), b(2, 0, NAN, 1, 10)],
        "area_underflow": [b(0, 0, NAN, 1, tiny), b(0, 0, NAN, 1, tiny), b(tiny / 2, 0, NAN, 1, tiny),
                           b(0, 0, 0.7, 1, tiny), b(0, 0, 0.7, 1, tiny)],
        "area_underflow_later": [b(0, 0, NAN, 1, 10), b(0, 0, NAN, 1, tiny), b(1, 1, 0.4, 1, tiny)],
        "area_overflow": [b(0, 0, NAN, 1, 1e20), b(0, 0, NAN, 1, 1e20), b(1e19, 0, NAN, 2, 1e20), b(0, 0, 0.3, 1, 1e20),
                          b(5, 5, NAN, 1, 10)],
        "far_coordinates": [b(1e7, 1e7, NAN, 1, 2), b(1e7 + 1, 1e7, NAN, 1, 2), b(1e7 + 2, 1e7 + 1, NAN, 1, 2),
                            b(1e7 + 3.5, 1e7, 0.5, 1, 2), b(1e7 + 1, 1e7 + 1, NAN, 1, 2)],
        "shared_edge": [b(0, 0, NAN, 1, 64), b(64, 0, NAN, 1, 64), b(0, 64, NAN, 1, 64), b(64, 64, NAN, 1, 64),
                        b(-64, 0, NAN, 2, 32)],
        "touching_circles": [b(0, 0, NAN, 0.75, 8), b(6, 8, NAN, 0.75, 8), b(-6, -8, NAN, 0.75, 8),
                             b(10, 0, math.pi / 2, 0.75, 8)],
    }


@pytest.mark.parametrize("thr", [0.5, 0.0, -0.1, NAN])
def test_degenerate_boxes_match_oracle(eng, oracle, thr):
    sets = degenerate_sets()
    # the touching circles touch exactly: the radius of a 6 x 8 box is 5, the centres are 10 apart
    t = sets["touching_circles"]
    assert oracle.radius(t[0]) == 5.0 and not oracle.too_far(t[0], t[1]) and not oracle.too_far(t[0], t[3])
    names = list(sets)
    boxes = np.concatenate([np.stack(sets[k]) for k in names])
    sizes = [len(sets[k]) for k in names]
    scores = np.concatenate([np.linspace(0.9, 0.1, m).astype(F32) for m in sizes])
    check(eng, oracle, boxes, scores, sizes, thr)
    check(eng, oracle, boxes, None, sizes, thr)
    if thr == 0.5:
        for k in names:   # each set alone, through the one-set entry
            i = names.index(k)
            a = int(offsets_of(sizes)[i])
            sb, ss = boxes[a:a + sizes[i]], scores[a:a + sizes[i]]
            assert np.array_equal(eng.nms_indices(sb, ss, thr), oracle.nms(sb, ss, thr)), k


# --------------------------------------------------------------------------- capacity
def test_set_whose_mask_exceeds_device_memory_is_refused(eng):
    """The largest set the sweep's 200 KB bitmap admits, 1,638,400 boxes, needs a 335 GB mask slab: every entry refuses
    it with SB200_ERR_CAPACITY before anything is enqueued, names the set, and leaves every output untouched."""
    import torch

    from similari_b200._lib import lib, ptr

    L = lib()
    big = 64 * 25600
    assert big * (big // 64) * 8 > torch.cuda.get_device_properties(0).total_memory
    offsets = np.array([0, 5, 5 + big, 8 + big], np.int32)
    total = 8 + big
    boxes = np.ones((total, 6), F32)     # full size, though the check reads nothing but the offsets
    idx, cnt, mask = np.full(total, 9, np.int32), np.full(3, 9, np.int32), np.full(total, 7, np.uint8)
    assert L.sb200_nms_batch(3, ptr(offsets), ptr(boxes), None, 0.5, 0.0, 0, ptr(idx), ptr(cnt), ptr(mask), 0) == -3
    err = L.sb200_last_error()
    assert b"set 1 " in err and b"1638400 boxes" in err
    assert np.all(idx == 9) and np.all(cnt == 9) and np.all(mask == 7)
    assert L.sb200_nms(ptr(boxes[5:5 + big]), None, big, 0.5, 0.0, 0, ptr(idx), 0) == -3
    assert b"set 0 " in L.sb200_last_error()
    assert np.all(idx == 9)
    d_boxes = torch.ones((total, 6), dtype=torch.float32, device="cuda")
    d_idx = torch.full((total,), 9, dtype=torch.int32, device="cuda")
    d_cnt = torch.full((3,), 9, dtype=torch.int32, device="cuda")
    d_mask = torch.full((total,), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(Exception, match="status -3"):
        eng.nms_batch_device(offsets, d_boxes.data_ptr(), 0, 0.5, None, d_idx.data_ptr(), d_cnt.data_ptr(),
                             d_mask.data_ptr())
    assert b"set 1 " in L.sb200_last_error()
    torch.cuda.synchronize()
    assert bool((d_idx == 9).all()) and bool((d_cnt == 9).all()) and bool((d_mask == 7).all())
