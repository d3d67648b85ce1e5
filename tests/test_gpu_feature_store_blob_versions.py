"""Feature store blobs of every version written by an earlier build (tests/golden/fstore_blobs.npz, from the seeded
scripts of tests/golden/make_fstore_blobs.py): each loads into the state the writing store held, saves back byte for
byte, and the same script run on a fresh store saves to the same bytes."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def _scripts():
    spec = importlib.util.spec_from_file_location("make_fstore_blobs", os.path.join(GOLDEN, "make_fstore_blobs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MK = _scripts()
FIXTURE = np.load(os.path.join(GOLDEN, "fstore_blobs.npz"))


@pytest.mark.gpu
@pytest.mark.parametrize("script", MK.SCRIPTS, ids=lambda f: f.__name__)
def test_blob_of_an_earlier_build_loads_and_saves_unchanged(script):
    import similari_b200.engine as eng

    name = script.__name__
    blob = FIXTURE[f"{name}/blob"]
    want = {k.split("/", 1)[1]: FIXTURE[k] for k in FIXTURE.files if k.startswith(name + "/") and k != f"{name}/blob"}
    s = eng.FeatureStore.load(blob)
    got = MK.state(s)
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        assert got[k].dtype == v.dtype and np.array_equal(got[k], v), (name, k)
    assert np.array_equal(s.save(), blob)
    s.close()
    fresh = MK.run(eng, script)
    assert np.array_equal(fresh.save(), blob)
    fresh.close()
