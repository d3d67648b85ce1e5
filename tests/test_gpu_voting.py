"""The voting kernels (kernels_assign.cu) against the oracle on adversarial cost matrices.

sb200_sort_voting / sb200_visual_voting compact their dense inputs into the tracker's entry lists and pick the kernel by
the tracker's rule; SB200_VOTE_KERNEL=dense|sparse|prepass forces one of them:
  dense    voting_kernel on the dense matrices (what a scene gets when one of its lists overflows);
  sparse   voting_sparse_kernel on the lists: the parallel fast path of Kuhn-Munkres, the CSR / CSC build, the first-seen
           column rank, BestFit's per-candidate buckets (or the whole-list bitonic sort above 160 entries of one candidate);
  prepass  (visual) the BestFit pre-pass writes decided / excl / pre_winner and the full pass reuses them, as in the
           tracker's lazy positional stage.
A forced sparse kernel the rule would not allow fails with SB200_ERR_CAPACITY, which the tests expect, so no case ever
tests the other kernel by accident.

Winners and voting types must equal the oracle's (its tie order is the reference's, DESIGN.md §2), every assignment must
be valid, and the Sort total must be the optimum scipy's linear_sum_assignment finds on the same i64 weight matrix.  The
scipy checks of the oracle itself need no GPU.

Thresholds whose weight (thr * 1e6f as i64) is 0 or negative are outside the reference's domain: SortVoting's "new
track" diagonal must outweigh an implicit zero column (similari_oracle.cpp, sort_voting), so they are not tested here.
"""
import zlib

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

NAN = np.float32(np.nan)
F32 = np.float32

# device limits (sb_engine.cuh, kernels_assign.cu)
VOTE_POS_CAP, VOTE_VIS_CAP, VOTING_SMEM_LIMIT, BUCKET_MAX = 3072, 4096, 220 * 1024, 160


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


# --------------------------------------------------------------------------------------------- numpy models
def weight_i64(v):
    """sb::weight_i64 / Rust `(v * 1e6f32) as i64`: f32 product, truncated; NaN -> 0."""
    w = np.asarray(v, F32) * F32(1e6)
    return np.where(np.isnan(w), 0, np.trunc(np.nan_to_num(w))).astype(np.int64)


def sort_weights(cost, thr):
    """SortVoting's i64 matrix: row i = candidate i, column i its "new track" diagonal (weight thr), columns m + j the
    tracks (None -> 0).  Column order does not change the optimum."""
    m, n = cost.shape
    w = np.zeros((m, m + n), np.int64)
    w[:, m:] = weight_i64(cost)
    w[np.arange(m), np.arange(m)] = weight_i64(thr)
    return w


def optimum(w):
    assert np.abs(w).max(initial=0) <= 10**9     # every sum below stays exact in f64
    if w.shape[0] == 0:
        return 0
    r, c = linear_sum_assignment(w.astype(np.float64), maximize=True)
    return int(w[r, c].sum())


def winners_total(winners, cost, thr):
    """Total weight of a Sort assignment: matched entries plus the unmatched candidates on their own diagonal."""
    wm, t = weight_i64(cost), int(weight_i64(thr))
    return sum(int(wm[i, j]) if j >= 0 else t for i, j in enumerate(winners))


def assert_valid(winners, cost):
    won = winners[winners >= 0]
    assert len(np.unique(won)) == len(won), "a track won twice"
    for i, j in enumerate(winners):
        if j >= 0:
            assert j < cost.shape[1] and not np.isnan(cost[i, j]), (i, j)


def smem_fits(m, n, viscap=VOTE_VIS_CAP):
    """launch_voting's shared-memory check: vote_smem_bytes and sparse_smem_bytes against kVotingSmemLimit."""
    ny = m + n
    dense = ny * 8 * 2 + m * 8 * 2 + ny * 4 * 3 + m * 4 * 5 + n * 4 * 2 + m * 2 + n + 64
    km = ny * 8 * 2 + m * 8 * 2 + ny * 4 * 3 + m * 4 * 4 + n * 4 * 3 + (m + 1) * 4 + (n + 1) * 4 + VOTE_POS_CAP * 12 + 64
    bf = viscap * 12 + m * 12 + n * 12 + (2 * m + 2) * 4 + 64
    sparse = max(km, bf) + m * 4 + m * 2 + n + 64
    return dense <= VOTING_SMEM_LIMIT and sparse <= VOTING_SMEM_LIMIT


def sparse_allowed(pos, vis=None):
    """The tracker's rule (scene_mode_kernel) with the list capacities of engine.cu."""
    m, n = pos.shape
    if m >= 65535 or n >= 65535:
        return False
    npos = int((~np.isnan(pos)).sum())
    if npos > min(m * 32, 2 * VOTE_POS_CAP) or npos > VOTE_POS_CAP:
        return False
    if vis is not None:
        nvis = int((~np.isnan(vis)).sum())
        if nvis > min(m * 64, 4 * VOTE_VIS_CAP) or nvis > VOTE_VIS_CAP:
            return False
    return True


def smallest_thr_of_weight_1():
    t = F32(1e-6)
    while weight_i64(t) >= 1:
        t = np.nextafter(t, F32(0))
    while weight_i64(t) < 1:
        t = np.nextafter(t, F32(1))
    return t


# --------------------------------------------------------------------------------------------- Sort cases
def _rand(rng, m, n, density, lo=0.0, hi=1.0):
    c = rng.uniform(lo, hi, (m, n)).astype(F32)
    c[rng.random((m, n)) >= density] = NAN
    return c


def _quantised(rng, m, n, density, levels):
    c = rng.choice(np.asarray(levels, F32), (m, n)).astype(F32)
    c[rng.random((m, n)) >= density] = NAN
    return c


def _staircase(rng, m=300):
    # every row prefers the columns of the rows before it: row i has its band i-3 .. i+1 with weights falling towards
    # its own column, so most roots displace their predecessors along long alternating paths
    c = np.full((m, m), NAN, F32)
    for i in range(m):
        for j in range(max(0, i - 3), min(m, i + 2)):
            c[i, j] = F32(0.5 + 0.1 * (i - j) + 0.01 * rng.integers(0, 3))
    return c


def _one_candidate_everywhere(rng):
    c = _quantised(rng, 50, 50, 0.08, [0.4, 0.6, 0.8])
    c[7, :] = F32(0.7)
    return c


def _one_track_wanted(rng):
    c = _quantised(rng, 50, 50, 0.08, [0.4, 0.6, 0.8])
    c[:, 11] = F32(0.9)
    return c


def _block_diagonal(rng, m=120, b=6):
    c = np.full((m, m), NAN, F32)
    for s in range(0, m, b):
        c[s:s + b, s:s + b] = _quantised(rng, b, b, 0.8, [0.35, 0.5, 0.65, 0.8, 0.95])
    return c[rng.permutation(m)][:, rng.permutation(m)]


def _taken_earlier(rng, m=200):
    # row r's tight column is its own, except every 10th row, which wants the column of row r - 7: taken either in the
    # same fast-path round (a lower row wants it) or in an earlier one, so the first failing root falls at many places
    # and fast-path rounds interleave with full searches
    c = np.full((m, m), NAN, F32)
    for r in range(m):
        c[r, r] = F32(0.8)
        if r % 10 == 0 and r >= 7:
            c[r, r - 7] = F32(0.9)
            c[r, r] = F32(0.7)
    extra = rng.random((m, m)) < 0.01
    c[extra & np.isnan(c)] = F32(0.5)
    return c


def _empty_rows_cols(rng):
    c = _rand(rng, 40, 40, 0.5)
    c[[3, 7, 8, 39], :] = NAN
    c[:, [0, 5, 9, 31]] = NAN
    return c


def _ulp_pairs(rng, thr):
    t = F32(thr)
    lv = [np.nextafter(t, F32(-1)), t, np.nextafter(t, F32(2)), F32(0.9)]
    return _quantised(rng, 50, 50, 0.5, lv)


def _capped(rng, m, n, count, levels=(0.4, 0.55, 0.7, 0.85, 1.0)):
    c = np.full((m, n), NAN, F32)
    idx = rng.choice(m * n, count, replace=False)
    c.flat[idx] = rng.choice(np.asarray(levels, F32), count)
    return c


THR_W1 = smallest_thr_of_weight_1()

SORT_CASES = {
    # ties
    "quantised_levels": lambda r: (_quantised(r, 60, 70, 0.4, [0.25, 0.5, 0.75, 1.0]), 0.3),
    "all_equal_square": lambda r: (np.full((30, 30), 0.5, F32), 0.3),
    "all_equal_wide": lambda r: (np.full((20, 32), 0.5, F32), 0.3),
    "all_equal_tall": lambda r: (np.full((60, 25), 0.5, F32), 0.3),
    "cost_equals_threshold": lambda r: (_quantised(r, 50, 50, 0.4, [0.3, 0.6]), 0.3),
    "ulp_around_0.3": lambda r: (_ulp_pairs(r, 0.3), 0.3),
    "ulp_around_1.0": lambda r: (_ulp_pairs(r, 1.0), 1.0),
    # shapes
    "1x1": lambda r: (np.full((1, 1), 0.5, F32), 0.3),
    "1xN": lambda r: (_rand(r, 1, 40, 0.6), 0.3),
    "Mx1": lambda r: (_rand(r, 40, 1, 0.6), 0.3),
    "3x1000": lambda r: (_capped(r, 3, 1000, 96, [0.5, 0.75, 1.0]), 0.3),
    "1000x3": lambda r: (_quantised(r, 1000, 3, 0.3, [0.5, 0.75, 1.0]), 0.3),
    "empty_rows_and_columns": lambda r: (_empty_rows_cols(r), 0.3),
    "all_nan": lambda r: (np.full((6, 9), NAN, F32), 0.3),
    "no_candidates": lambda r: (np.zeros((0, 5), F32), 0.3),
    "no_tracks": lambda r: (np.zeros((5, 0), F32), 0.3),
    # structures that defeat the fast path
    "staircase": lambda r: (_staircase(r), 0.3),
    "one_candidate_matches_every_track": lambda r: (_one_candidate_everywhere(r), 0.3),
    "one_track_every_candidate_wants": lambda r: (_one_track_wanted(r), 0.3),
    "permuted_block_diagonal": lambda r: (_block_diagonal(r), 0.3),
    "tight_column_taken_earlier": lambda r: (_taken_earlier(r), 0.3),
    # values
    "weights_1_to_1e8": lambda r: (np.where(r.random((80, 80)) < 0.3, 10.0 ** r.uniform(-6, 2, (80, 80)), np.nan).astype(F32), 0.3),
    "negative_costs": lambda r: (_rand(r, 60, 60, 0.4, -0.5, 1.0), 0.3),
    "threshold_1.0": lambda r: (_quantised(r, 60, 60, 0.4, [0.5, 1.0, 1.25, 1.5, 2.0]), 1.0),
    "threshold_of_weight_1": lambda r: (_quantised(r, 60, 60, 0.4, [0.0, THR_W1, F32(2e-6), F32(3e-6)]), THR_W1),
    # size
    "600x600_density_30pct": lambda r: (_rand(r, 600, 600, 0.3), 0.3),
    "1500x1500_3000_entries": lambda r: (_capped(r, 1500, 1500, 3000), 0.3),
}


def sort_case(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    cost, thr = SORT_CASES[name](rng)
    return np.ascontiguousarray(cost, F32), F32(thr)


# --------------------------------------------------------------------------------------------- oracle / device calls
# candidate ids and track ids share the oracle's id maps (as in the reference): keep the two ranges apart
CAND_BASE = 1 << 40


def sort_ents(cost):
    ii, jj = np.nonzero(~np.isnan(cost))
    return [(CAND_BASE + int(i), 1 + int(j), float(cost[i, j]), None) for i, j in zip(ii, jj)]


def oracle_sort(oracle, thr, cost):
    m, n = cost.shape
    w = oracle.sort_voting(float(thr), m, n, sort_ents(cost))
    out = np.full(m, -1, np.int32)
    for i in range(m):
        t = w.get(CAND_BASE + i)
        if t is not None and t[0] != CAND_BASE + i:
            out[i] = t[0] - 1
    return out


def vis_ents(pos, vis):
    m, n, k = vis.shape
    ents = []
    for i in range(m):
        for j in range(n):
            for kk in range(k):
                a = pos[i, j] if kk == 0 else NAN
                f = vis[i, j, kk]
                if not (np.isnan(a) and np.isnan(f)):
                    ents.append((CAND_BASE + i, 1 + j, None if np.isnan(a) else float(a), None if np.isnan(f) else float(f)))
    return ents


def oracle_visual(oracle, thr, min_votes, pos, vis):
    m = pos.shape[0]
    ref = oracle.visual_voting(float(thr), float(np.finfo(F32).max), min_votes, vis_ents(pos, vis))
    w, vt = np.full(m, -1, np.int32), np.ones(m, np.uint8)    # undecided: a new track, VotingType::Positional
    for i in range(m):
        r = ref.get(CAND_BASE + i)
        if r is not None:
            vt[i] = r[0][1]
            if r[0][0] != CAND_BASE + i:
                w[i] = r[0][0] - 1
    return w, vt


def device_call(monkeypatch, kernel, allowed, fn):
    """Runs fn() with SB200_VOTE_KERNEL=kernel; a sparse kernel the rule forbids must be refused, and None is returned."""
    from similari_b200._lib import Sb200Error

    monkeypatch.setenv("SB200_VOTE_KERNEL", kernel)
    try:
        if kernel != "dense" and not allowed:
            with pytest.raises(Sb200Error, match="status -3"):
                fn()
            return None
        return fn()
    finally:
        monkeypatch.delenv("SB200_VOTE_KERNEL")


def check_sort(eng, oracle, monkeypatch, kernel, cost, thr, ref=None):
    got = device_call(monkeypatch, kernel, sparse_allowed(cost), lambda: eng.sort_voting(float(thr), cost))
    if got is None:
        return None
    ref = oracle_sort(oracle, thr, cost) if ref is None else ref
    assert_valid(got, cost)
    assert np.array_equal(ref, got), np.nonzero(ref != got)[0][:10]
    assert winners_total(got, cost, thr) == optimum(sort_weights(cost, thr))
    return got


def check_visual(eng, oracle, monkeypatch, kernel, thr, min_votes, pos, vis):
    got = device_call(monkeypatch, kernel, sparse_allowed(pos, vis),
                      lambda: eng.visual_voting(float(thr), min_votes, pos, vis))
    if got is None:
        return None
    w, vt = got
    rw, rvt = oracle_visual(oracle, thr, min_votes, pos, vis)
    # a visual winner needs a valid distance, a positional one a valid positional entry
    has_vis = np.where(np.isnan(vis).all(axis=2), NAN, F32(0))
    assert_valid(w, np.where((vt == 0)[:, None], has_vis, pos))
    assert np.array_equal(rw, w), [(i, rw[i], w[i]) for i in np.nonzero(rw != w)[0][:10]]
    assert np.array_equal(rvt, vt), [(i, rvt[i], vt[i]) for i in np.nonzero(rvt != vt)[0][:10]]
    return w, vt


# --------------------------------------------------------------------------------------------- oracle vs scipy (no GPU)
@pytest.mark.parametrize("case", list(SORT_CASES))
def test_oracle_kuhn_munkres_reaches_the_optimum(oracle, case):
    """oracle.kuhn_munkres (pathfinding's algorithm, restated) and oracle.sort_voting reach scipy's optimum on every Sort
    case: the reference's own tests pin only small known answers."""
    cost, thr = sort_case(case)
    w = sort_weights(cost, thr)
    best = optimum(w)
    if w.shape[0]:
        total, xy = oracle.kuhn_munkres(w)
        assert total == best
        assert len(np.unique(xy)) == len(xy) and int(w[np.arange(len(xy)), xy].sum()) == best
    win = oracle_sort(oracle, thr, cost)
    assert_valid(win, cost)
    assert winners_total(win, cost, thr) == best


def test_numpy_weight_model():
    assert weight_i64(F32(0.3)) == 300000 and weight_i64(NAN) == 0 and weight_i64(F32(-0.5)) == -500000
    assert weight_i64(THR_W1) == 1 and weight_i64(np.nextafter(THR_W1, F32(0))) == 0
    assert weight_i64(F32(100.0)) == 10**8


# --------------------------------------------------------------------------------------------- Sort on the GPU
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["dense", "sparse"])
@pytest.mark.parametrize("case", list(SORT_CASES))
def test_sort_voting_adversarial(eng, oracle, monkeypatch, case, kernel):
    cost, thr = sort_case(case)
    got = check_sort(eng, oracle, monkeypatch, kernel, cost, thr)
    if kernel == "sparse" and case != "600x600_density_30pct":
        assert got is not None            # every other case fits the sparse kernel's lists
    if case == "600x600_density_30pct":
        assert (got is None) == (kernel == "sparse")


@pytest.mark.gpu
@pytest.mark.parametrize("count", [VOTE_POS_CAP, VOTE_POS_CAP + 1])
def test_sort_voting_positional_list_capacity(eng, oracle, monkeypatch, count):
    """Exactly kVotePosCap valid entries vote on the lists under the tracker's rule; one more goes to the dense kernel, and
    forcing the sparse kernel onto it is refused."""
    cost = _capped(np.random.default_rng(count), 128, 128, count)
    ref = oracle_sort(oracle, F32(0.3), cost)
    for kernel in ("dense", "sparse"):
        got = check_sort(eng, oracle, monkeypatch, kernel, cost, F32(0.3), ref)
        assert (got is None) == (kernel == "sparse" and count > VOTE_POS_CAP)
    assert np.array_equal(eng.sort_voting(0.3, cost), ref)     # the rule's own choice


def largest_square():
    s = 1
    while smem_fits(s + 1, s + 1):
        s += 1
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["square", "one_row_more", "one_column_more"])
def test_sort_voting_largest_scene(eng, oracle, monkeypatch, shape):
    """The largest square scene launch_voting accepts (from the shared-memory formulas of both kernels) votes on both
    kernels; one row or column more is refused with SB200_ERR_CAPACITY when the formulas say it does not fit."""
    from similari_b200._lib import Sb200Error

    s = largest_square()
    assert not smem_fits(s + 1, s + 1)
    m, n = {"square": (s, s), "one_row_more": (s + 1, s), "one_column_more": (s, s + 1)}[shape]
    cost = _capped(np.random.default_rng(s), m, n, 3000)
    if smem_fits(m, n):
        ref = oracle_sort(oracle, F32(0.3), cost)
        for kernel in ("dense", "sparse"):
            assert check_sort(eng, oracle, monkeypatch, kernel, cost, F32(0.3), ref) is not None
    else:
        for kernel in (None, "dense", "sparse"):
            if kernel:
                monkeypatch.setenv("SB200_VOTE_KERNEL", kernel)
            with pytest.raises(Sb200Error, match="status -3"):
                eng.sort_voting(0.3, cost)
            monkeypatch.delenv("SB200_VOTE_KERNEL", raising=False)
    if shape == "square":
        assert smem_fits(m, n)


def test_largest_scene_formula():
    s = largest_square()
    assert smem_fits(s, s) and not smem_fits(s + 1, s + 1) and 1000 < s < 2200


@pytest.mark.gpu
def test_vote_kernel_hook_rejects_unknown_values(eng, monkeypatch):
    from similari_b200._lib import Sb200Error

    cost = np.full((2, 2), 0.5, F32)
    monkeypatch.setenv("SB200_VOTE_KERNEL", "fast")
    with pytest.raises(Sb200Error, match="status -1"):
        eng.sort_voting(0.3, cost)
    monkeypatch.setenv("SB200_VOTE_KERNEL", "prepass")   # the BestFit pre-pass exists for visual voting only
    with pytest.raises(Sb200Error, match="status -1"):
        eng.sort_voting(0.3, cost)


# --------------------------------------------------------------------------------------------- visual voting on the GPU
VIS_KERNELS = ["dense", "sparse", "prepass"]


def _visual_scene(rng, m, n, k, tracks_per_cand=5, obs_density=0.7, pos_density=0.15, levels=8):
    """A tracking-like scene: each candidate sees a few tracks visually, distances quantised to 1/levels (f64 weight
    ties), positional costs on a sparse random subset."""
    vis = np.full((m, n, k), NAN, F32)
    for i in range(m):
        for j in rng.choice(n, min(n, tracks_per_cand), replace=False):
            d = (np.round(rng.uniform(0.0, 0.7, k) * levels) / levels).astype(F32)
            d[rng.random(k) >= obs_density] = NAN
            vis[i, j] = d
    pos = _quantised(rng, m, n, pos_density, [0.35, 0.5, 0.65, 0.8])
    return pos, vis


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
@pytest.mark.parametrize("k", range(1, 9))
def test_visual_voting_observations_and_votes(eng, oracle, monkeypatch, k, kernel):
    """K = 1..8 observations, min_votes 1..K and K + 1 (which no candidate reaches: everything falls through to the
    positional stage)."""
    rng = np.random.default_rng(100 + k)
    pos, vis = _visual_scene(rng, 40, 30, k)
    assert sparse_allowed(pos, vis)
    for mv in range(1, k + 2):
        w, vt = check_visual(eng, oracle, monkeypatch, kernel, 0.3, mv, pos, vis)
        if mv == k + 1:
            assert (vt == 1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
def test_visual_voting_f64_weight_ties(eng, oracle, monkeypatch, kernel):
    """Exactly equal f64 BestFit weights: two candidates with identical distance vectors for one track (the lower row
    wins it), and one candidate tied between two tracks (it takes the lower column)."""
    m, n, k = 6, 6, 3
    pos = np.full((m, n), NAN, F32)
    vis = np.full((m, n, k), NAN, F32)
    vis[4, 2] = vis[1, 2] = [0.1, 0.2, NAN]          # rows 1 and 4 tie on track 2
    vis[3, 5] = vis[3, 4] = [0.3, NAN, 0.1]          # row 3 ties between tracks 4 and 5
    vis[0, 0] = [0.6, 0.6, 0.6]                      # sets max_dist
    pos[4, 1] = F32(0.8)                             # row 4 was decided visually: never positional
    pos[5, 3] = F32(0.7)
    w, vt = check_visual(eng, oracle, monkeypatch, kernel, 0.3, 1, pos, vis)
    assert w[1] == 2 and w[4] == -1 and vt[4] == 0
    assert w[3] == 4 and vt[3] == 0
    assert w[5] == 3 and vt[5] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
@pytest.mark.parametrize("total", [256, 300])
@pytest.mark.parametrize("count0", [BUCKET_MAX, BUCKET_MAX + 1])
def test_visual_voting_bucket_boundary(eng, oracle, monkeypatch, count0, total, kernel):
    """One candidate with exactly 160 valid visual entries (per-candidate buckets) or 161 (whole-list bitonic sort), in a
    list of a power-of-two and of a non-power-of-two length."""
    rng = np.random.default_rng(count0 * 7 + total)
    m, n, k = 8, 30, 8
    vis = np.full((m, n, k), NAN, F32)
    flat0 = rng.choice(n * k, count0, replace=False)
    vis[0].reshape(-1)[flat0] = (np.round(rng.uniform(0, 0.7, count0) * 4) / 4).astype(F32)
    rows = rng.integers(1, m, total - count0)
    free = [np.nonzero(np.isnan(vis[i].reshape(-1)))[0] for i in range(m)]
    used = {i: 0 for i in range(m)}
    for i in rows:
        vis[i].reshape(-1)[free[i][used[i]]] = F32(np.round(rng.uniform(0, 0.7) * 4) / 4)
        used[i] += 1
    assert int((~np.isnan(vis)).sum()) == total and int((~np.isnan(vis[0])).sum()) == count0
    pos = _quantised(rng, m, n, 0.3, [0.4, 0.7])
    for mv in (1, 2):
        check_visual(eng, oracle, monkeypatch, kernel, 0.3, mv, pos, vis)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
@pytest.mark.parametrize("count", [VOTE_VIS_CAP, VOTE_VIS_CAP + 1])
def test_visual_voting_list_capacity(eng, oracle, monkeypatch, count, kernel):
    """kVoteVisCap valid visual entries vote on the lists; one more sends the scene to the dense kernel."""
    rng = np.random.default_rng(count)
    m, n, k = 80, 64, 4
    vis = np.full((m, n, k), NAN, F32)
    idx = rng.choice(m * n * k, count, replace=False)
    vis.reshape(-1)[idx] = (np.round(rng.uniform(0, 0.7, count) * 8) / 8).astype(F32)
    pos = _quantised(rng, m, n, 0.1, [0.4, 0.6, 0.8])
    got = check_visual(eng, oracle, monkeypatch, kernel, 0.3, 2, pos, vis)
    assert (got is None) == (kernel != "dense" and count > VOTE_VIS_CAP)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
def test_visual_voting_cascade(eng, oracle, monkeypatch, kernel):
    """VisualVoting's cascade: a candidate BestFit sends to "self" stays out of the positional stage, a track BestFit
    claimed is excluded from it, and candidates below min_votes fall through to Kuhn-Munkres."""
    m, n, k = 6, 5, 3
    pos = np.full((m, n), NAN, F32)
    vis = np.full((m, n, k), NAN, F32)
    vis[0, 0] = [0.1, 0.1, 0.1]      # row 0 wins track 0
    vis[1, 0] = [0.2, 0.2, 0.2]      # row 1 also wants track 0 most: sent to self
    pos[1, 1] = F32(0.9)             # ... and must not take track 1 positionally
    pos[2, 0] = F32(0.95)            # track 0 is claimed: row 2 must take track 2
    pos[2, 2] = F32(0.5)
    vis[3, 3] = [0.1, NAN, NAN]      # one vote < min_votes 2: row 3 is positional
    pos[3, 3] = F32(0.6)
    pos[4, 1] = F32(0.7)
    vis[5, 4] = [0.6, 0.6, 0.6]      # max_dist 0.6: row 5's weight is 0 yet it wins track 4
    w, vt = check_visual(eng, oracle, monkeypatch, kernel, 0.3, 2, pos, vis)
    assert list(w) == [0, -1, 2, 3, 1, 4]
    assert list(vt) == [0, 0, 1, 1, 1, 0]
    rng = np.random.default_rng(77)
    for _ in range(4):
        pos, vis = _visual_scene(rng, 60, 40, 3, tracks_per_cand=3, pos_density=0.2, levels=4)
        check_visual(eng, oracle, monkeypatch, kernel, 0.3, 2, pos, vis)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", VIS_KERNELS)
@pytest.mark.parametrize("case", ["below_minus_one", "all_at_the_maximum"])
def test_visual_voting_distance_extremes(eng, oracle, monkeypatch, case, kernel):
    """Distances below -1, the initial max_dist (so max_dist stays -1), and a scene whose distances all equal the
    maximum, so every BestFit weight is exactly 0."""
    rng = np.random.default_rng(5)
    pos, vis = _visual_scene(rng, 30, 20, 3, levels=4)
    if case == "below_minus_one":
        vis = (vis - F32(2.5)).astype(F32)
    else:
        vis = np.where(np.isnan(vis), vis, F32(0.42)).astype(F32)
    for mv in (1, 2):
        check_visual(eng, oracle, monkeypatch, kernel, 0.3, mv, pos, vis)


# --------------------------------------------------------------------------------------------- trackers with real ties
def _grid_frame(rng, scene_sizes, shift, drop=0.15):
    boxes, offs = [], [0]
    for s, side in enumerate(scene_sizes):
        xs, ys = np.meshgrid(np.arange(side) * 6.0, np.arange(side) * 6.0)
        b = np.zeros((side * side, 6), F32)
        b[:, 0] = xs.ravel() + 1000.0 * s + shift
        b[:, 1] = ys.ravel()
        b[:, 2] = NAN
        b[:, 3] = 1.0
        b[:, 4] = 10.0
        b[:, 5] = 1.0
        b = b[rng.random(len(b)) >= drop]
        boxes.append(b)
        offs.append(offs[-1] + len(b))
    return np.concatenate(boxes), np.asarray(offs, np.int32)


@pytest.mark.gpu
def test_batch_sort_iou_grid_ties(eng, oracle):
    """BatchSort, IoU metric: equal axis-aligned boxes on an integer grid, half-cell shifts between frames, so a
    detection overlaps two tracks with exactly equal IoU; three scenes of different sizes in one batch."""
    from similari_b200._lib import default_options

    kw = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3)
    g, o = eng.Tracker(default_options(**kw)), oracle.Tracker(oracle.make_options(**kw))
    rng = np.random.default_rng(3)
    for fr in range(6):
        boxes, offs = _grid_frame(rng, (4, 9, 14), shift=3.0 * (fr % 2))
        rg = g.predict_batch([0, 1, 2], offs, boxes)
        ro = o.predict_batch([0, 1, 2], offs, boxes)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)


@pytest.mark.gpu
def test_batch_visual_sort_duplicated_features(eng, oracle, monkeypatch):
    """BatchVisualSort on the tensor-core path with exactly duplicated features: a handful of feature vectors shared by
    many tracks, so the BestFit pre-pass, the lazy positional scan and the sparse voting kernel see exact ties in the
    tracker's own lists."""
    from similari_b200._lib import default_options

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    d = 64
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
              feature_dim=d, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1,
              min_confidence=0.1)
    g, o = eng.Tracker(default_options(**kw)), oracle.Tracker(oracle.make_options(**kw))
    rng = np.random.default_rng(4)
    pool = rng.normal(size=(4, d)).astype(F32)
    pool /= np.linalg.norm(pool, axis=1, keepdims=True)
    for fr in range(6):
        boxes, offs = _grid_frame(rng, (5, 8), shift=3.0 * (fr % 2), drop=0.1)
        feats = pool[(np.arange(len(boxes)) // 3) % len(pool)].copy()
        rg = g.predict_batch([0, 1], offs, boxes, features=feats)
        ro = o.predict_batch([0, 1], offs, boxes, features=feats)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
    assert g.work_counters()["tc_frames"] >= 4
