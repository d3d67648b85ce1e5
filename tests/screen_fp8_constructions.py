"""Host constructions that put the e4m3 visual screen at the edge of its bound (screen_rel_err_fp8, sb_engine.cuh).

The screen stores each row as x~ = e4m3(2^k x), with 2^k the power of two that puts max|x| in [224, 448), and drops a
pair only when the tensor-core dot product of the copies is below the threshold by more than E = screen_rel_err_fp8(d)
times ||a|| ||b||.  E has three parts: operand rounding (2u + u^2, u = 2^-4), the subnormal floor of the scaled copies,
and the FP8 accumulation of the tensor cores.  Each construction below spends one or more of those parts in the
direction that lowers dot~, and the CPU tests (test_screen_fp8_bounds_cpu.py) state how much of each it spends, measured
with the numpy e4m3 model and a numpy emulation of the accumulator model.  The GPU tests (test_gpu_screen_fp8_bounds.py)
put the exact value of such a pair on the threshold and check that the screen keeps it.
"""
import numpy as np

from test_screen_fp8_cpu import e4m3_rne

U4 = 2.0 ** -4
KINDS = ["euclid", "cos+", "cos-"]
# offsets from an e4m3 rounding midpoint that every column type holds exactly (the row's mantissa keeps its value in it)
STEP = {"f32": 2.0 ** -20, "f16": 2.0 ** -10, "bf16": 2.0 ** -7}


def row_scale(amax):
    """numpy mirror of fp8_row_scale: 2^k with amax 2^k in [224, 448), 1 for a row without a usable maximum."""
    amax = float(np.float32(amax))
    if not (2.0 ** -100 <= amax <= 2.0 ** 100):
        return 1.0
    m, e = np.frexp(amax)
    return float(np.ldexp(1.0, (8 if m >= 0.875 else 9) - int(e)))


def scaled_e4m3(x):
    """(x~ = e4m3(2^k x) as f64, 2^k) of one f32 row, as the writers of the e4m3 copies store it."""
    x = np.asarray(x, np.float32).astype(np.float64)
    s = row_scale(np.max(np.abs(x)))
    return e4m3_rne(x * s), s


def e4m3_bits(v):
    """The e4m3 byte (sign, 4-bit exponent of bias 7, 3-bit mantissa) of values that e4m3 holds exactly."""
    v = np.asarray(v, np.float64)
    a = np.abs(v)
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    normal = a >= 2.0 ** -6
    mant = np.where(normal, (a / np.exp2(e) - 1.0) * 8.0, a * 2.0 ** 9)
    expf = np.where(normal, e + 7, 0)
    assert np.all(mant == np.round(mant)) and np.all(mant < 8) and np.all(expf <= 15)
    return ((np.signbit(v).astype(np.uint32) << 7) | (expf.astype(np.uint32) << 3) | mant.astype(np.uint32)).astype(np.uint8)


def rel_err_fp8(d):
    """screen_rel_err_fp8 and its three terms (rounding, subnormal floor, accumulation), in f64."""
    rnd = 2 * U4 + U4 * U4
    sub = 2 * (1 + U4) * np.sqrt(d) * 2.0 ** -10 / 224.0 + d * 2.0 ** -20 / 224.0 ** 2
    acc = -(-d // 32) * 34 * 2.0 ** -12 * (1 + U4) ** 2 * 1.01
    return rnd + sub + acc, rnd, sub, acc


def operand_error(a, b):
    """(dot - dot~) / (||a|| ||b||) with dot~ the exact dot product of the scaled e4m3 copies, unscaled: how much of the
    bound the operand rounding (normal and subnormal) spends, positive when it lowers dot~."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    qa, sa = scaled_e4m3(a)
    qb, sb = scaled_e4m3(b)
    return (a64 @ b64 - (qa @ qb) / (sa * sb)) / (np.linalg.norm(a64) * np.linalg.norm(b64))


def wgmma_model(qa, qb):
    """The accumulator model of screen_rel_err_fp8 on one pair of scaled e4m3 rows (f64, exact products): per k32 step,
    the 32 products and the accumulator are aligned to the largest of them and truncated to 13 significant bits, then
    their sum is rounded to fp32."""
    qa, qb = np.asarray(qa, np.float64), np.asarray(qb, np.float64)
    acc = 0.0
    for s in range(0, len(qa), 32):
        t = np.append(qa[s:s + 32] * qb[s:s + 32], acc)
        mx = np.max(np.abs(t))
        if mx == 0.0:
            continue
        q = 2.0 ** (np.floor(np.log2(mx)) - 12)
        acc = float(np.float32(np.sum(np.trunc(t / q) * q)))   # the truncated sum is exact in f64
    return acc


def model_error(a, b):
    """(dot - dot~) / (||a|| ||b||) with dot~ the modelled accumulator of the scaled copies: operand rounding and
    accumulation together."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    qa, sa = scaled_e4m3(a)
    qb, sb = scaled_e4m3(b)
    return (a64 @ b64 - wgmma_model(qa, qb) / (sa * sb)) / (np.linalg.norm(a64) * np.linalg.norm(b64))


def accumulation_error(a, b):
    """The accumulator's share alone: (exact dot of the copies - modelled accumulator) / (||a|| ||b||), unscaled."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    qa, sa = scaled_e4m3(a)
    qb, sb = scaled_e4m3(b)
    return (qa @ qb - wgmma_model(qa, qb)) / (sa * sb) / (np.linalg.norm(a64) * np.linalg.norm(b64))


def _to_norm(a, b, norm):
    """Both rows times the power of two that brings ||a|| nearest to `norm` (exact: every mantissa is kept)."""
    s = np.exp2(np.round(np.log2(norm / np.linalg.norm(np.asarray(a, np.float64)))))
    return (np.asarray(a, np.float64) * s).astype(np.float32), (np.asarray(b, np.float64) * s).astype(np.float32)


# ------------------------------------------------------------------------------------------------------- operand pair
def fp8_pair(seed, d, norm, kind, col="f32"):
    """The e4m3 analogue of screen_pair (test_gpu_visual_bounds.py).  Components sgn 2^e (1 + 2^-4 -/+ k step): just below
    (above, for 'cos-') the e4m3 rounding midpoint of their binade, same exponents and signs in a and b, so every scaled
    component rounds down (up) by almost 2^-4 / (1 + 2^-4) relative.  Exponents span -3..3: the row maximum scales to
    272 (288 above) and every scaled component stays a normal e4m3 value (>= 4.25).  'euclid' and 'cos+' give dot~ below
    dot; 'cos-' returns (a, -b), whose dot~ is more negative than dot.  `step` keeps every value exact in the column
    type `col`; in bf16 it leaves one value below the midpoint (k = 1), so b takes k = 2 on one component in 16 to stay
    distinct from a."""
    rng = np.random.default_rng(seed)
    exps = rng.integers(-3, 4, d).astype(np.float64)
    signs = rng.choice([-1.0, 1.0], d)
    step = STEP[col]
    if col == "bf16":
        ka = np.ones(d)
        kb = np.where(rng.random(d) < 1.0 / 16, 2.0, 1.0)
    else:
        ka = rng.integers(1, 9, d).astype(np.float64)
        kb = rng.integers(1, 9, d).astype(np.float64)
    sgn = 1.0 if kind == "cos-" else -1.0
    a = signs * (1.0 + U4 + sgn * ka * step) * np.exp2(exps)
    b = signs * (1.0 + U4 + sgn * kb * step) * np.exp2(exps)
    a, b = _to_norm(a, b, norm)
    return (a, -b) if kind == "cos-" else (a, b)


SCALE_EDGE_MANTISSAS = [0.875, float(np.float32(0.87499994))]   # scaled maximum 224; 447.99997, which rounds to 448


def scale_edge_pair(seed, d, kind, mant):
    """fp8_pair at norm 1 whose largest component (the same lane in a and b) is replaced by mant * 2^(E + 1) > every other
    component: frexp of the row maximum is exactly `mant`.  0.875 scales it to 224, the bottom of the scaled range;
    0.87499994, the f32 just below, takes the other power of two and scales it to 447.99997, which rounds to 448, the
    largest finite e4m3 value (no saturation)."""
    a, b = fp8_pair(seed, d, 1.0, kind)
    i = int(np.argmax(np.abs(a)))
    e = np.floor(np.log2(np.abs(float(a[i]))))
    v = np.float32(mant) * np.float32(2.0 ** (e + 1))
    a[i], b[i] = np.sign(a[i]) * v, np.sign(b[i]) * v
    return a, b


# squared norms just inside and just outside [2^-60, 2^60] (fp8_norm_ok), by 2^-6 relative: far more than the f32
# rounding of the norm on the device
NORM_EDGES = {"in_hi": 2.0 ** 60 * (1 - 2.0 ** -6), "in_lo": 2.0 ** -60 * (1 + 2.0 ** -6),
              "out_hi": 2.0 ** 60 * (1 + 2.0 ** -6), "out_lo": 2.0 ** -60 * (1 - 2.0 ** -6)}


def norm_edge_pair(seed, d, kind, n2):
    """fp8_pair with both rows scaled (by a non-power of two) to squared norm n2."""
    a, b = fp8_pair(seed, d, 1.0, kind)
    out = []
    for x in (a, b):
        x64 = x.astype(np.float64)
        out.append((x64 * np.sqrt(n2 / (x64 @ x64))).astype(np.float32))
    return out[0], out[1]


# ------------------------------------------------------------------------------------------------- the subnormal floor
def subnormal_pair(seed, d, norm, kind):
    """a: one component of 256 (scaled units) fixes the row's scale; the other d - 1 sit 2^-20 below (above, 'cos-') the
    e4m3 subnormal midpoints (k + 1/2) 2^-9, k = 0..7, so they encode to k 2^-9 (k = 0: flush to zero) or, above, to
    (k + 1) 2^-9 -- the top one to 2^-6, the smallest normal value.  b: 256 in every lane with a's sign ('cos-': the
    opposite sign), exact in e4m3.  Every rounding error of a meets a partner of 256 and lowers dot~: the largest
    weight the floor can get, since ||a|| is as small as the scale allows."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 8, d).astype(np.float64)
    signs = rng.choice([-1.0, 1.0], d)
    off = 2.0 ** -20 if kind == "cos-" else -2.0 ** -20
    a = signs * ((k + 0.5) * 2.0 ** -9 + off)
    a[0] = signs[0] * 256.0
    b = signs * 256.0
    a, b = _to_norm(a, b, norm)
    if kind == "cos-":
        b = -b
    # b's norm is sqrt(d) times a's; keep it where it lands (the fillers of each side take that side's norm)
    return a, b


# ------------------------------------------------------------------------------------------------------ the accumulator
ACC_PLACES = ["first", "middle", "last"]


def acc_big_lane(d, where):
    steps = -(-d // 32)
    return {"first": 0, "middle": 32 * (steps // 2), "last": 32 * (steps - 1)}[where]


def acc_pair(seed, d, norm, kind, where="first", midpoints=False):
    """Rows for the accumulator term, in scaled units: one large lane of 256 x 256 = 2^16 (in the k32 step `where`), and
    d - 1 small lanes of 3.25 .. 3.75 whose products (< 16 = 2^(16 - 12)) lie just below the truncation quantum of an
    accumulator that holds 2^16: the model drops every one of them once the large product is in the accumulator (from
    the first step on for 'first', half-way for 'middle', only in the last step for 'last').  The small products are
    positive; 'cos-' makes the large one negative (b's large lane is -256), so that dropping them lowers dot~ there too.
    `midpoints` puts every lane 2^-20 relative below its e4m3 rounding midpoint as well (272 -> 256, 3.625 -> 3.5), and the
    large lane of 'cos-' above it (272 -> 288): operand rounding and accumulation then both lower dot~."""
    rng = np.random.default_rng(seed)
    signs = rng.choice([-1.0, 1.0], d)
    big = acc_big_lane(d, where)
    if midpoints:
        lo = 3.625 - 2.0 ** -21 * rng.integers(1, 9, d)
        a, b = lo.copy(), 3.625 - 2.0 ** -21 * rng.integers(1, 9, d)
        up = kind == "cos-"
        a[big] = 272.0 + (1.0 if up else -1.0) * 2.0 ** -12 * rng.integers(1, 9)
        b[big] = 272.0 + (1.0 if up else -1.0) * 2.0 ** -12 * rng.integers(1, 9)
    else:
        a = rng.choice([3.75, 3.75, 3.75, 3.5], d)
        b = rng.choice([3.75, 3.75, 3.75, 3.25], d)
        a[big] = b[big] = 256.0
    a, b = a * signs, b * signs
    if kind == "cos-":
        b[big] = -b[big]
    return _to_norm(a, b, norm)


def acc_pair_cases(d):
    """(where, midpoints) of the accumulator constructions a test runs at width d."""
    return [(w, False) for w in ACC_PLACES] + [("first", True)]
