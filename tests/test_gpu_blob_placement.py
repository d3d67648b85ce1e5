"""Device blobs at any address.  The tracker blob (save_device), the scene blob of a tracker with the feature history on
(export_scenes with d_ptr: its history sections go through xfer_hist_kernel's 16-byte accesses) and the store blob of an
f32 and a bf16 store (FeatureStore.save_device) are written into, and read from, a device buffer at byte offsets 0 and
16, where the library works on the blob in place, and 4 and 8, where it goes through a device copy.  At every offset the
bytes are those of the host blob, the bytes around the blob are untouched, and what is loaded from that address
continues exactly as a copy loaded from the host blob."""
import numpy as np
import pytest

import test_gpu_feature_store_storage as fss
from fstore_checks import same_results
import test_gpu_state_transfer as tst
from test_gpu_state_transfer import eng  # noqa: F401  (the module's fixture)

pytestmark = pytest.mark.gpu

OFFSETS = [0, 16, 4, 8]
SENTINEL = 0xAB


def _placed(write, blob, off):
    """A device buffer into which `write(d_ptr, cap)` has put the blob at byte offset `off`; checks the bytes and the
    sentinel around them."""
    import torch

    n = len(blob)
    buf = torch.full((off + n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 256 == 0   # `off` is the blob's alignment
    torch.cuda.synchronize()
    assert write(buf.data_ptr() + off, n) == n
    got = buf.cpu().numpy()
    assert np.array_equal(got[off:off + n], blob)
    assert (got[:off] == SENTINEL).all() and (got[off + n:] == SENTINEL).all()
    return buf


def _visual_tracker(eng, dim):
    t = eng.Tracker(tst._opts(3, tst.IOU, 5, dim, 3))
    t.set_feature_history(True)
    return t


@pytest.mark.parametrize("off", OFFSETS)
def test_tracker_blob_at_any_offset(eng, off):
    dim = 64
    wl = tst._cfg(3, 40, dim, False, seed=0x5EED8100 + off)
    frames = [wl.next_frame() for _ in range(16)]
    g = _visual_tracker(eng, dim)
    for f in frames[:8]:
        tst._predict(g, f)
    blob = g.save()
    buf = _placed(g.save_device, blob, off)
    dev, host = eng.Tracker.load(buf.data_ptr() + off, len(blob)), eng.Tracker.load(blob)
    for i, f in enumerate(frames[8:]):
        tst._same(tst._predict(dev, f), tst._predict(host, f), f"frame {i}")
    tst._same(tst._collect(dev, True), tst._collect(host, True), "wasted")


@pytest.mark.parametrize("off", OFFSETS)
def test_scene_blob_with_the_feature_history_at_any_offset(eng, off):
    dim = 64
    wl = tst._cfg(4, 40, dim, False, seed=0x5EED8200 + off)
    frames = [wl.next_frame() for _ in range(16)]
    src = _visual_tracker(eng, dim)
    for f in frames[:8]:
        tst._predict(src, f)
    moved = [1, 2]
    blob = src.export_scenes(moved)
    buf = _placed(lambda p, n: src.export_scenes(moved, d_ptr=p, cap=n), blob, off)
    dev, host = _visual_tracker(eng, dim), _visual_tracker(eng, dim)
    dev.import_scenes(buf.data_ptr() + off, len(blob))
    host.import_scenes(blob)
    live, _ = dev.scene_live_counts(moved)
    assert live.sum() > 0
    assert np.array_equal(dev.export_scenes(moved), blob) and np.array_equal(host.export_scenes(moved), blob)
    for i, f in enumerate(frames[8:]):
        part, _ = tst._split(f, set(moved))
        tst._same(tst._predict(dev, part), tst._predict(host, part), f"frame {i}")
    tst._same(tst._collect(dev, True), tst._collect(host, True), "wasted")


@pytest.mark.parametrize("storage", ["f32", "bf16"])
@pytest.mark.parametrize("off", OFFSETS)
def test_store_blob_at_any_offset(off, storage):
    import similari_b200.engine as e

    K = 3
    s, raw = fss._worn(storage, storage, K=K)
    blob = s.save()
    buf = _placed(s.save_device, blob, off)
    dev, host = e.FeatureStore.load(buf.data_ptr() + off, len(blob)), e.FeatureStore.load(blob)
    steps = fss._script(K, 96)
    for st in steps:   # fresh ids: the script's query ids must not be stored yet
        if st[0] in ("search", "associate"):
            st[1][:] += 5000
    same_results(fss._run(dev, steps, raw), fss._run(host, steps, raw))
