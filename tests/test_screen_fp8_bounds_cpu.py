"""CPU checks of the constructions that put the e4m3 screen at the edge of its bound (screen_fp8_constructions.py): each
spends a stated share of screen_rel_err_fp8 (compiled for the host from sb_engine.cuh), always in the direction that
lowers dot~, and never more than the bound."""
import numpy as np
import pytest

from screen_fp8_constructions import (ACC_PLACES, KINDS, NORM_EDGES, SCALE_EDGE_MANTISSAS, acc_pair, acc_pair_cases,
                                      accumulation_error, fp8_pair, model_error, norm_edge_pair, operand_error,
                                      rel_err_fp8, row_scale, scale_edge_pair, scaled_e4m3, subnormal_pair, wgmma_model)
from test_screen_fp8_cpu import e4m3_rne, probe  # noqa: F401  (probe: the nvcc host build of sb_engine.cuh)

FP8_D = [64, 136, 200, 250, 256, 512]
NORMS = [2.0 ** -10, 1.0, 2.0 ** 10]
# the least share of ||a|| ||b|| the operand pair spends, per column type (2u / (1 + u) squared out is 0.1142)
OPERAND_FLOOR = {"f32": 0.113, "f16": 0.105, "bf16": 0.100}
COLS = ["f32", "f16", "bf16"]


def pair_seed(d):
    return 4000 + d


def test_bound_matches_the_host_build(probe):  # noqa: F811
    got = probe([f"e {d}" for d in FP8_D])
    for d, e in zip(FP8_D, got):
        assert rel_err_fp8(d)[0] <= e <= rel_err_fp8(d)[0] * (1 + 2.0 ** -18)


def test_row_scale_mirror_matches_the_host_build(probe):  # noqa: F811
    amax = [224.0, 0.875, float(np.float32(0.87499994)), 272.0, 2.0 ** -35, 2.0 ** 30, 3.0e-39, 7.5]
    got = probe([f"s {float(np.float32(a)).hex()}" for a in amax])
    assert got == [row_scale(a) for a in amax]


@pytest.mark.parametrize("col", COLS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", FP8_D + [500])
def test_operand_pair_reaches_the_operand_bound(probe, d, kind, col):  # noqa: F811
    """Every scaled component rounds by almost u / (1 + u), all in the direction that lowers dot~."""
    e = probe([f"e {d}"])[0]
    for norm in NORMS if col == "f32" else [1.0]:
        a, b = fp8_pair(pair_seed(d), d, norm, kind, col)
        if col == "f16":
            assert np.array_equal(a.astype(np.float16).astype(np.float32), a)
            assert np.array_equal(b.astype(np.float16).astype(np.float32), b)
        elif col == "bf16":
            assert np.array_equal(a.view(np.uint32) & 0xFFFF, np.zeros(d, np.uint32))
            assert np.array_equal(b.view(np.uint32) & 0xFFFF, np.zeros(d, np.uint32))
        assert np.all(np.sign(a) == (-np.sign(b) if kind == "cos-" else np.sign(b)))
        assert not np.array_equal(a, b if kind != "cos-" else -b)   # a Euclidean threshold above zero
        qa, sa = scaled_e4m3(a)
        assert 256.0 < np.max(np.abs(a.astype(np.float64) * sa)) < 288.0   # the row maximum scales to ~272
        assert np.min(np.abs(qa)) >= 4.0                            # every scaled component is a normal e4m3 value
        err = operand_error(a, b)
        assert OPERAND_FLOOR[col] <= err <= rel_err_fp8(d)[1]
        assert err < e
        assert 0.5 * norm <= np.linalg.norm(a.astype(np.float64)) <= 2.0 * norm


@pytest.mark.parametrize("mant", SCALE_EDGE_MANTISSAS)
@pytest.mark.parametrize("kind", KINDS)
def test_scale_edge_rows(probe, mant, kind):  # noqa: F811
    """The row maximum scales to 224 (mantissa 0.875) or to 447.99997, which rounds to 448, the largest finite value."""
    a, b = scale_edge_pair(pair_seed(512), 512, kind, mant)
    for x in (a, b):
        amax = float(np.max(np.abs(x)))
        assert np.frexp(amax)[0] == np.float32(mant)
        s = probe([f"s {amax.hex()}"])[0]
        assert s == row_scale(amax)
        top = amax * s
        q = e4m3_rne(top)
        assert (top, q) == ((224.0, 224.0) if mant == 0.875 else (float(np.float32(447.99997)), 448.0))
    assert 0.105 <= operand_error(a, b) < rel_err_fp8(512)[1]


@pytest.mark.parametrize("edge", list(NORM_EDGES))
def test_norm_edge_rows(edge):
    """Squared norms in f32 land on the intended side of [2^-60, 2^60] with room for the device's rounding."""
    for kind in KINDS:
        for x in norm_edge_pair(pair_seed(512), 512, kind, NORM_EDGES[edge]):
            n2 = float(np.float32(np.sum(x.astype(np.float64) ** 2)))
            inside = 2.0 ** -60 <= n2 <= 2.0 ** 60
            assert inside == edge.startswith("in")
            assert abs(n2 / NORM_EDGES[edge] - 1) < 2.0 ** -12
            assert np.all(np.isfinite(x)) and np.min(np.abs(x)) > np.finfo(np.float32).tiny


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", [64, 136, 512])
def test_subnormal_floor_errs_one_way(kind, d):
    """a's small lanes encode to e4m3 subnormals (or flush to zero) with errors of almost 2^-10 each, every one against a
    partner of 256 and lowering dot~: 0.4 of the subnormal term, inside the bound."""
    a, b = subnormal_pair(pair_seed(d), d, 1.0, kind)
    qa, sa = scaled_e4m3(a)
    qb, sb = scaled_e4m3(b)
    x = a.astype(np.float64) * sa
    assert np.max(np.abs(x)) == 256.0 and np.all(np.abs(qb) == 256.0)
    small = np.abs(x) < 2.0 ** -6
    assert small.sum() == d - 1
    # below the midpoints the lowest lanes flush to zero; above them the top lanes reach the smallest normal value
    assert np.any(np.abs(qa[small]) == 2.0 ** -6) if kind == "cos-" else np.any(qa[small] == 0.0)
    lane = (x - qa) * qb   # each small lane's contribution to dot - dot~, in scaled units
    assert np.all(lane[small] > 0.999 * 2.0 ** -10 * 256.0)
    err = operand_error(a, b)
    total, _, sub, _ = rel_err_fp8(d)
    assert 0.38 * sub <= err < sub < total


def test_accumulator_model_exact_on_small_integers():
    rng = np.random.default_rng(1)
    for _ in range(50):
        a = rng.integers(-2, 3, 512).astype(np.float64)
        b = rng.integers(-2, 3, 512).astype(np.float64)
        assert wgmma_model(a, b) == a @ b


# share of the accumulation term the construction spends, at the least, per placement of its large step
ACC_FLOOR = {("first", False): 0.55, ("middle", False): 0.14, ("last", False): 0.02, ("first", True): 0.45}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", FP8_D)
def test_accumulator_constructions_use_the_accumulation_term(d, kind):
    """With the large product in the accumulator, the model drops every small product that follows: the 'first' rows
    spend 0.56 - 0.67 of the accumulation term (32 of its 34 truncations per step), in the direction that lowers dot~.
    With operand midpoints as well, the total error exceeds either term alone.  All stay inside the bound."""
    total, rnd, sub, acc = rel_err_fp8(d)
    for where, mid in acc_pair_cases(d):
        for norm in NORMS:
            a, b = acc_pair(pair_seed(d), d, norm, kind, where, mid)
            e_acc, e_all = accumulation_error(a, b), model_error(a, b)
            assert ACC_FLOOR[(where, mid)] * acc <= e_acc <= acc, (where, mid, e_acc / acc)
            assert 0 < e_all < total
            if mid:
                assert e_all > max(acc * 0.5 + rnd * 0.5, e_acc)
                assert operand_error(a, b) > 0


def test_accumulator_places_cover_every_step():
    for d in FP8_D:
        lanes = {w: acc_pair(1, d, 1.0, "cos+", w)[0] for w in ACC_PLACES}
        steps = {w: int(np.argmax(np.abs(x))) // 32 for w, x in lanes.items()}
        assert steps["first"] == 0 and steps["last"] == (d - 1) // 32
        assert 0 < steps["middle"] < steps["last"] or d <= 64


def test_e4m3_encoder_matches_torch():
    """The bytes the accumulator probe sends are the e4m3 codes of its values (every finite code but -0)."""
    torch = pytest.importorskip("torch")
    from screen_fp8_constructions import e4m3_bits

    codes = np.arange(256, dtype=np.uint8)
    vals = torch.from_numpy(codes).view(torch.float8_e4m3fn).float().numpy().astype(np.float64)
    keep = np.isfinite(vals) & ((vals != 0) | (codes == 0))
    assert keep.sum() == 253
    assert np.array_equal(e4m3_bits(vals[keep]), codes[keep])
    assert np.array_equal(e4m3_rne(vals[keep]), vals[keep])
