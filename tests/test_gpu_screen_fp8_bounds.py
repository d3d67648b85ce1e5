"""The e4m3 screen at the edge of its bound, in the operator, on the tensor cores themselves, and in the tracker's own
e4m3 rows.

The e4m3 screen is the tracker's default for features of up to 512 lanes.  It only filters, so it is correct exactly
while screen_rel_err_fp8 (sb_engine.cuh) bounds dot - dot~.  The pairs of screen_fp8_constructions.py spend the bound's
operand, subnormal and accumulation terms in the direction that lowers dot~; here the threshold sits exactly at the
oracle's value for such a pair (kept, with zero margin in the oracle) and one ulp past it (cut), and every output is
compared bit for bit with the oracle.  The accumulator probe measures what the bound's accumulation term models.
"""
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from screen_fp8_constructions import (KINDS, NORM_EDGES, SCALE_EDGE_MANTISSAS, acc_pair, acc_pair_cases, e4m3_bits,
                                      fp8_pair, norm_edge_pair, scale_edge_pair, scaled_e4m3, subnormal_pair,
                                      wgmma_model)
from test_gpu_visual_bounds import A_ROWS, B_COLS, VIS_KW, _far_box, _frame, _grid_boxes

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FP8_D = [64, 136, 200, 250, 256, 512]   # 136 and 200: padded fp8_pitch rows; 250: zero-padded d8
NORMS = [2.0 ** -10, 1.0, 2.0 ** 10]


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def pair_seed(d):
    return 4000 + d


# ----------------------------------------------------------------------------------------- operator at the threshold
def pair_matrix(seed, a, b):
    """300 x 600 features: the pair (a, b) at every (A_ROWS, B_COLS) crossing, random fillers of a's norm (candidates)
    and b's norm (tracks) elsewhere."""
    rng = np.random.default_rng(seed)
    d = len(a)
    cand = rng.standard_normal((300, d))
    trk = rng.standard_normal((600, d))
    cand *= np.linalg.norm(a.astype(np.float64)) / np.linalg.norm(cand, axis=1, keepdims=True)
    trk *= np.linalg.norm(b.astype(np.float64)) / np.linalg.norm(trk, axis=1, keepdims=True)
    cand, trk = cand.astype(np.float32), trk.astype(np.float32)
    cand[A_ROWS] = a
    trk[B_COLS] = b
    return cand, trk


def _fp8_at_threshold(eng, oracle, a, b, kind, seed, monkeypatch):
    from test_gpu_parity import assert_bits_equal

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    cand, trk = pair_matrix(seed, a, b)
    # room for every pair in the survivor list: fillers near a cosine threshold below zero, and rows outside
    # fp8_norm_ok, pass the screen wholesale
    monkeypatch.setenv("SB200_VIS_PAIR_CAP", str(cand.shape[0] * trk.shape[0]))
    if kind == "euclid":
        vk_o, vk_g = oracle.VIS_EUCLIDEAN, eng._lib.VIS_EUCLIDEAN
        thr = np.float32(oracle.euclidean(a, b))
        cut = np.nextafter(thr, np.float32(0))
        assert thr > 0
    else:
        vk_o, vk_g = oracle.VIS_COSINE, eng._lib.VIS_COSINE
        thr = np.float32(oracle.cosine(a, b))
        cut = np.nextafter(thr, np.float32(2))
    for t, kept in ((thr, True), (cut, False)):
        ref = oracle.visual_cost_matrix(vk_o, float(t), cand, trk, threads=os.cpu_count() or 1)
        got = eng.visual_cost_matrix(vk_g, float(t), cand, trk)
        pairs = ref[np.ix_(A_ROWS, B_COLS)]
        assert np.isfinite(pairs).all() if kept else np.isnan(pairs).all()   # the oracle's decision has zero margin
        assert_bits_equal(ref, got)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", FP8_D)
@pytest.mark.parametrize("norm", NORMS)
def test_fp8_screen_keeps_operand_pairs_on_the_threshold(eng, oracle, d, norm, kind, monkeypatch):
    """Every scaled component rounds by almost 2^-4 / (1 + 2^-4) against dot~: 0.114 (0.121 for 'cos-') of ||a|| ||b||."""
    a, b = fp8_pair(pair_seed(d), d, norm, kind)
    _fp8_at_threshold(eng, oracle, a, b, kind, pair_seed(d), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mant", SCALE_EDGE_MANTISSAS)
@pytest.mark.parametrize("d", [250, 512])
def test_fp8_screen_scale_edges(eng, oracle, d, mant, kind, monkeypatch):
    """Row maxima that scale to 224 and to 447.99997 (rounded to 448, the largest finite e4m3 value)."""
    a, b = scale_edge_pair(pair_seed(d), d, kind, mant)
    _fp8_at_threshold(eng, oracle, a, b, kind, pair_seed(d), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("edge", list(NORM_EDGES))
def test_fp8_screen_norm_edges(eng, oracle, edge, kind, monkeypatch):
    """Squared norms just inside [2^-60, 2^60] (the folded constants at their extremes) and just outside it (the rows
    keep every pair, the exact pass decides)."""
    a, b = norm_edge_pair(pair_seed(512), 512, kind, NORM_EDGES[edge])
    _fp8_at_threshold(eng, oracle, a, b, kind, pair_seed(512), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", [136, 512])
def test_fp8_screen_subnormal_floor(eng, oracle, d, kind, monkeypatch):
    """Lanes that encode to e4m3 subnormals or flush to zero, all erring against a partner of 256 and against dot~."""
    a, b = subnormal_pair(pair_seed(d), d, 1.0, kind)
    _fp8_at_threshold(eng, oracle, a, b, kind, pair_seed(d), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("where,mid", acc_pair_cases(512))
@pytest.mark.parametrize("d", [64, 250, 512])
def test_fp8_screen_accumulator_rows(eng, oracle, d, where, mid, kind, monkeypatch):
    """A product of 2^16 in the accumulator and small products just below its truncation quantum, the large step first,
    in the middle or last, alone or with every lane at an e4m3 rounding midpoint."""
    a, b = acc_pair(pair_seed(d), d, 1.0, kind, where, mid)
    _fp8_at_threshold(eng, oracle, a, b, kind, pair_seed(d), monkeypatch)


# ------------------------------------------------------------------------------------------- the FP8 accumulator probe
def _probe_exe(tmp):
    from similari_b200._build import nvcc

    src = os.path.join(HERE, "gpu_probe", "fp8_wgmma_probe.cu")
    exe = os.path.join(tmp, "fp8_wgmma_probe")
    subprocess.check_call([nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", os.path.join(HERE, "..", "similari_b200", "csrc"), src, "-o", exe],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return exe


def _run_probe(exe, cases):
    """cases: (steps, A [64, 512] e4m3 values, B [128, 512] e4m3 values) -> the [64, 128] accumulators of each."""
    buf = [struct.pack("<i", len(cases))]
    for steps, a, b in cases:
        assert a.shape == (64, 512) and b.shape == (128, 512)
        buf += [struct.pack("<i", steps), e4m3_bits(a).tobytes(), e4m3_bits(b).tobytes()]
    out = subprocess.run([exe], input=b"".join(buf), capture_output=True, check=True, timeout=300).stdout
    return np.frombuffer(out, np.float32).reshape(len(cases), 64, 128).astype(np.float64)


def _step_maxima(qa, qb, steps):
    """Per k32 step, the largest of its 32 products and the exact running sum in front of it."""
    p = qa * qb
    run, out = 0.0, []
    for s in range(steps):
        t = p[32 * s: 32 * s + 32]
        out.append(max(np.max(np.abs(t)), abs(run)))
        run += t.sum()
    return np.array(out)


PROBE_D = [64, 136, 250, 512]


def test_fp8_wgmma_accumulator_within_the_model(eng):
    """Stage 1: integer operands whose sums are exact (|acc| < 2^12) must come out exact at every (row, column), over 1,
    5 and 16 k32 steps: the swizzled layout, the descriptor advance and the accumulator mapping are right.  Stage 2: the
    accumulator constructions (every pair of their rows) against the exact sum of the decoded products: the error stays
    within ceil(d / 32) * 34 * 2^-12 * sum|a~ b~|, the accumulation term of screen_rel_err_fp8."""
    rng = np.random.default_rng(90)
    layout = []
    for steps in (16, 5, 1):
        a = rng.integers(-2, 3, (64, 512)).astype(np.float64)
        b = rng.integers(-2, 3, (128, 512)).astype(np.float64)
        layout.append((steps, a, b))
    rows = {}
    measure = []
    for d in PROBE_D:
        a = np.zeros((64, 512))
        b = np.zeros((128, 512))
        names = []
        for kind in KINDS:
            for where, mid in acc_pair_cases(d):
                x, y = acc_pair(pair_seed(d), d, 1.0, kind, where, mid)
                a[len(names), :d] = scaled_e4m3(x)[0]
                b[len(names), :d] = scaled_e4m3(y)[0]
                names.append((kind, where, mid))
        # resolution rows: 2^16 in the first step, then one product of 2^j (j = 0..5) in the second
        r0 = len(names)
        for j in range(6):
            a[r0 + j, 0], a[r0 + j, 32] = 256.0, 2.0 ** j
        b[r0, 0], b[r0, 32] = 256.0, 1.0
        rows[d] = (names, r0)
        measure.append((-(-d // 32), a, b))
    with tempfile.TemporaryDirectory() as tmp:
        got = _run_probe(_probe_exe(tmp), layout + measure)
    for (steps, a, b), g in zip(layout, got[:3]):
        k = 32 * steps
        assert np.array_equal(g, a[:, :k] @ b[:, :k].T), steps

    worst_units, worst_per_step, model_gap = 0.0, 0.0, 0.0
    for d, (steps, a, b), g in zip(PROBE_D, measure, got[3:]):
        names, r0 = rows[d]
        k = 32 * steps
        exact = a[:, :k] @ b[:, :k].T
        bound = steps * 34 * 2.0 ** -12 * (np.abs(a[:, :k]) @ np.abs(b[:, :k]).T)
        n = len(names)
        err = np.abs(g - exact)[:n, :n]
        assert np.all(err <= bound[:n, :n]), (d, np.unravel_index(np.argmax(err / bound[:n, :n]), err.shape))
        for i in range(n):
            for j in range(n):
                m = _step_maxima(a[i, :k], b[j, :k], steps)
                worst_units = max(worst_units, err[i, j] / (2.0 ** -12 * m.max()))
                worst_per_step = max(worst_per_step, err[i, j] / (2.0 ** -12 * m.sum()))
                model_gap = max(model_gap, abs(g[i, j] - wgmma_model(a[i, :k], b[j, :k])) / (2.0 ** -12 * m.max()))
        kept = [g[r0 + j, r0] - 65536.0 for j in range(6)]
        print(f"\nfp8 wgmma probe d={d}: 2^16 + 2^j (j = 0..5) in the next step keeps {kept}")
    print(f"fp8 wgmma probe: largest error {worst_units:.3f} x 2^-12 of the largest step maximum, "
          f"{worst_per_step:.3f} x 2^-12 per step (the model allows 34); largest distance from the model "
          f"{model_gap:.3f} x 2^-12")
    assert worst_per_step <= 34.0


# ---------------------------------------------------------------------------------- the tracker's own e4m3 rows
TRACKER_SLOTS = [0, 63, 64, 129]   # the adversarial detection's row inside each of the four scenes
TRACKER_N = 130


def _narrow(feats, col):
    """(the column as sent, its exact f32 widening)."""
    if col == "f32":
        return feats, feats
    from test_gpu_feature_types import _narrow as narrow

    return narrow(feats, col)


def _tracker_frames(a, b, d, col):
    """Four scenes of 130 detections; in frames 0-2 each holds b at its slot, in frame 3 a far from b's track.  The
    fillers are rounded to the column type, so the oracle's f32 rows are the widened column."""
    rng = np.random.default_rng(5)
    fill = []
    for _ in TRACKER_SLOTS:
        f = rng.standard_normal((TRACKER_N, d)).astype(np.float32)
        fill.append(_narrow(f / np.linalg.norm(f, axis=1, keepdims=True), col)[1])
    frames = []
    for fr in range(4):
        scenes = []
        for s, slot in enumerate(TRACKER_SLOTS):
            boxes, feats = _grid_boxes(TRACKER_N), fill[s].copy()
            feats[slot] = b
            if fr == 3:
                boxes[slot] = _far_box(s)
                feats[slot] = a
            scenes.append((boxes, feats))
        frames.append(_frame(scenes))
    return frames


def _predict_device(t, frame, col):
    import torch

    sid, offs, boxes, feats = frame
    total = len(boxes)
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[col]
    db = torch.from_numpy(boxes).cuda()
    df = torch.from_numpy(feats).cuda().to(tdt).contiguous()
    out = {k: torch.zeros(total, dtype=dt, device="cuda") for k, dt in
           (("ids", torch.int64), ("epochs", torch.int32), ("lengths", torch.int32), ("voting_types", torch.uint8))}
    torch.cuda.synchronize()
    t.predict_batch_device(sid, offs, db.data_ptr(), df.data_ptr(), d_ids=out["ids"].data_ptr(),
                           d_epochs=out["epochs"].data_ptr(), d_lengths=out["lengths"].data_ptr(),
                           d_voting_types=out["voting_types"].data_ptr(), feature_type=col)
    t.sync()
    return {"ids": out["ids"].cpu().numpy().view(np.uint64), "epochs": out["epochs"].cpu().numpy().view(np.uint32),
            "lengths": out["lengths"].cpu().numpy().view(np.uint32), "voting_types": out["voting_types"].cpu().numpy()}


def _predict(t, frame, col, device):
    if device:
        return _predict_device(t, frame, col)
    sid, offs, boxes, feats = frame
    return t.predict_batch(sid, offs, boxes, features=_narrow(feats, col)[0], feature_type=col)


def _assert_e4m3_decided(t, frames):
    sc = t.screen_counters()
    assert sc["fp8_frames"] >= frames and sc["bf16_frames"] == 0 and sc["survivors"] > 0, sc


TRACKER_CASES = ([(col, d, kobs, "host") for col in ("f32", "f16", "bf16") for d in (512, 500) for kobs in (3, 1)] +
                 [(col, d, 3, mode) for mode in ("device", "load", "transfer") for col in ("f32", "f16", "bf16")
                  for d in (512, 500)])


@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("col,d,kobs,mode", TRACKER_CASES)
def test_tracker_fp8_rows_keep_pairs_on_the_threshold(eng, oracle, col, d, kobs, mode, vis, monkeypatch):
    """The tracker writes its own e4m3 rows: cand_norm_kernel the candidates', feat_store_kernel the arena's (D = 512
    with f32 and 2-byte columns: the vector writers; D = 500: the scalar ones), and regen_fp8 both after a load or a
    scene transfer.  b is stored for three frames (K = 3 or 1 observations) and a arrives far from its track: with the
    threshold at the oracle's value for (a, b) only a visual match keeps the id, and the e4m3 screen must pass it."""
    from similari_b200._lib import default_options
    from test_gpu_tracker import both

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    a, b = fp8_pair(77 + vis, d, 1.0, "euclid" if vis == 0 else "cos+", col)
    thr = float(oracle.euclidean(a, b)) if vis == 0 else float(oracle.cosine(a, b))
    frames = _tracker_frames(a, b, d, col)
    kw = dict(kind=3, visual_kind=vis, visual_threshold=thr, feature_dim=d, visual_max_observations=kobs,
              visual_min_votes=1, **VIS_KW)
    g, o = both(eng, oracle, **kw)
    for fr, frame in enumerate(frames):
        if fr == 3 and mode == "load":
            _assert_e4m3_decided(g, 2)
            g = eng.Tracker.load(g.save())
        elif fr == 3 and mode == "transfer":
            _assert_e4m3_decided(g, 2)
            g2 = eng.Tracker(default_options(**kw))
            g2.import_scenes(g.export_scenes(frame[0], remove=True))
            g = g2
        rg = _predict(g, frame, col, mode == "device")
        sid, offs, boxes, feats = frame
        ro = o.predict_batch(sid, offs, boxes, features=feats)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(np.asarray(rg[key]), np.asarray(ro[key])), (fr, key)
    _assert_e4m3_decided(g, 1 if mode in ("load", "transfer") else 3)
    assert g.active_tracks() == o.active_tracks()
