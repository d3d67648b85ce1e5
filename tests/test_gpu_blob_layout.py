"""The v1 state blob format, pinned: the section table of Tracker.save() and export_scenes() blobs against a restatement
of the layout of DESIGN §3b, written out here column by column.  A column added, dropped, resized or moved in the engine
changes the format, and blobs saved by an earlier build would no longer load; this test says so."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAHA, IOU = 0, 1
MAX_SECTIONS = 48
ALIGN = 256
KST_BYTES = 4 * 32   # Kalman state row: 30 floats padded to 128 bytes


def _blob_header():
    from similari_b200._lib import Options

    class BlobHeader(C.Structure):
        _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("type", C.c_uint32), ("n_sections", C.c_uint32),
                    ("total_bytes", C.c_uint64), ("opts", Options),
                    ("feature_history", C.c_int32), ("hist_len", C.c_int32), ("d8", C.c_int32), ("n_scenes", C.c_int32),
                    ("seen_features", C.c_int32), ("adapt_dense", C.c_int32), ("auto_waste_counter", C.c_int32),
                    ("auto_waste_periodicity", C.c_int32), ("scene_cap", C.c_int32), ("track_cap", C.c_int32),
                    ("pad0", C.c_int32), ("pad1", C.c_int32),
                    ("live_total", C.c_int64), ("blk_total", C.c_int64), ("free_total", C.c_int64),
                    ("wasted_count", C.c_int64), ("revealed", C.c_int64), ("hpool_top", C.c_int64),
                    ("hpool_free", C.c_int64), ("hpool_cap", C.c_int64), ("id_counter", C.c_uint64),
                    ("sec_off", C.c_uint64 * MAX_SECTIONS), ("sec_bytes", C.c_uint64 * MAX_SECTIONS)]

    return BlobHeader


class BlobScene(C.Structure):
    _fields_ = [("scene_id", C.c_uint64), ("epoch", C.c_uint32), ("n_tracks", C.c_int32), ("n_hidden", C.c_int32),
                ("arena_top", C.c_int32)]


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _align(n):
    return (n + ALIGN - 1) // ALIGN * ALIGN


def _expected_sections(kind, pos, H, fh, D, K, tracker_blob, n_scenes, live, blk, fre, wasted, top, hfree):
    """Section sizes in blob order, from DESIGN §3b."""
    visual = kind >= 2
    d8 = (D + 7) // 8 * 8
    sec = [n_scenes * C.sizeof(BlobScene)]
    # per live track: id, epoch, length, custom id, voting type, predicted box, observed box, radius, Kalman state
    per_track = [8, 4, 4, 8, 1, 24, 24, 4, KST_BYTES]
    if pos == IOU:
        per_track.append(64)                    # vertex cache
    if H > 1:
        per_track += [24 * H, 24 * H]           # predicted / observed box rings
    if visual:
        per_track += [K, K, 4 * K, 1, 1, 4]     # obs_phys, obs_hasf, obs_q, obs_n, feat_cnt, fblk
        if fh and tracker_blob:
            per_track.append(4)                 # hblk
    sec += [live * w for w in per_track]
    if visual:
        sec += [blk * w for w in (4 * K * d8, 2 * K * d8, 4 * K, 4)]   # f32 rows, BF16 rows, fnorm2, blk_owner
        sec.append(fre * 4)                                          # free list
    if tracker_blob:
        rec = [8, 8, 4, 4, 24, 24] + ([24 * H, 24 * H] if H > 1 else []) + ([4] if fh else [])
        sec += [wasted * w for w in rec]
        if fh:
            sec += [top * H * d8 * 4, top * H, hfree * 4]             # pool rows, present bytes, free stack
    elif fh:
        sec += [live * H * d8 * 4, live * H]                          # history block of each live track
    return sec


def _check(blob, case, tracker_blob):
    kind, pos, H, fh, D, K = case
    BlobHeader = _blob_header()
    assert C.sizeof(BlobHeader) == 24 + 160 + 12 * 4 + 8 * 8 + 8 + 2 * 8 * MAX_SECTIONS
    h = BlobHeader.from_buffer_copy(np.ascontiguousarray(blob)[: C.sizeof(BlobHeader)].tobytes())
    assert (h.magic, h.version, h.type) == (0x42534253, 1, 1 if tracker_blob else 2)
    assert (h.feature_history, h.hist_len) == (int(fh), H)
    if kind >= 2:
        assert h.d8 == (D + 7) // 8 * 8
    assert h.total_bytes == len(blob)
    # the counts in the header are the scene table's
    table = (BlobScene * h.n_scenes).from_buffer_copy(blob[h.sec_off[0]: h.sec_off[0] + h.n_scenes * C.sizeof(BlobScene)].tobytes())
    live = sum(s.n_tracks for s in table)
    blk = sum(s.arena_top for s in table)
    assert (h.live_total, h.blk_total, h.free_total) == (live, blk, blk - live if kind >= 2 else 0)
    assert live > 0
    if tracker_blob:
        assert h.wasted_count > 0
        if fh:
            assert h.hpool_top > 0
    else:
        assert h.wasted_count == h.hpool_top == h.hpool_free == 0
    want = _expected_sections(kind, pos, H, fh, D, K, tracker_blob, h.n_scenes, live, blk, h.free_total, h.wasted_count,
                              h.hpool_top, h.hpool_free)
    assert h.n_sections == len(want)
    assert list(h.sec_bytes[: h.n_sections]) == want
    off = _align(C.sizeof(BlobHeader))
    for i, b in enumerate(want):
        assert h.sec_off[i] == off, i
        off += _align(b)
    assert h.total_bytes == off


# kind, positional metric, history_length, feature history, D, K
CASES = [
    (0, IOU, 1, False, 0, 1),
    (1, MAHA, 5, False, 0, 1),
    (2, IOU, 5, True, 30, 3),
    (2, MAHA, 1, False, 30, 2),
    (3, MAHA, 1, False, 512, 2),
    (3, IOU, 5, True, 512, 3),
    (3, MAHA, 5, True, 600, 2),
    (3, IOU, 1, False, 600, 3),
]


def _case_id(c):
    return f"k{c[0]}-{'iou' if c[1] else 'maha'}-h{c[2]}-{'fh' if c[3] else 'nofh'}-D{c[4]}-K{c[5]}"


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_blob_sections_follow_the_v1_layout(eng, case):
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload

    kind, pos, H, fh, D, K = case
    kw = dict(kind=kind, positional_kind=pos, iou_threshold=0.2, max_idle_epochs=2, history_length=H)
    if kind >= 2:
        kw.update(visual_kind=0, visual_threshold=0.7, feature_dim=D, visual_max_observations=K, visual_min_votes=1,
                  visual_minimal_track_length=1)
    g = eng.Tracker(default_options(**kw))
    if fh:
        g.set_feature_history(True)
    n_scenes = 3 if kind in (1, 3) else 1
    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=40, feature_dim=D, oriented=False,
                              canvas=(900.0, 600.0), drop_frac=0.25, fresh_frac=0.15, feat_noise=0.05,
                              seed=0x5EED9000 + 31 * kind + 7 * H + D + K)
    wl = Workload(cfg)
    for _ in range(12):
        f = wl.next_frame()
        g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
    _check(g.save(), case, True)
    _check(g.export_scenes(list(range(n_scenes))), case, False)
