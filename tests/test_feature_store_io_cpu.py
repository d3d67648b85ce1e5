"""CPU checks of the feature store's I/O additions (typed and device-resident feature columns, the store blob): the blob
header that Python mirrors is the one the C header declares, the blob's section plan is the header's layout, and the
host-side row table behind fs_stage_kernel (the newest K rows of each query) matches a numpy restatement."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "similari_b200.h")
CTYPES = {"uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float}


def test_blob_header_mirror_matches_the_c_header():
    from similari_b200 import _lib

    hdr = open(HEADER).read()
    defs = dict(re.findall(r"#define (SB200_FSTORE_BLOB_[A-Z]+) (\w+)", hdr))
    val = lambda k: int(defs["SB200_FSTORE_BLOB_" + k].rstrip("u"), 0)  # noqa: E731
    assert (val("MAGIC"), val("VERSION"), val("ALIGN"), val("SECTIONS")) == \
        (_lib.FSTORE_BLOB_MAGIC, _lib.FSTORE_BLOB_VERSION, _lib.FSTORE_BLOB_ALIGN, _lib.FSTORE_BLOB_SECTIONS)
    assert _lib.FSTORE_BLOB_MAGIC.to_bytes(4, "little") == b"SBFS"
    body = re.search(r"typedef struct \{([^}]*)\} sb200_fstore_blob_header;", hdr).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    declared = []
    for typ, name, dim in re.findall(r"(\w+)\s+(\w+)(?:\[(\w+)\])?;", body):
        declared.append((name, CTYPES[typ] * val(dim.replace("SB200_FSTORE_BLOB_", "")) if dim else CTYPES[typ]))
    mirror = [(n, t) for n, t in _lib.FstoreBlobHeader._fields_]
    assert [n for n, _ in declared] == [n for n, _ in mirror]
    for (n, a), (_, b) in zip(declared, mirror):
        assert C.sizeof(a) == C.sizeof(b) and a._type_ == b._type_, n
    assert C.sizeof(_lib.FstoreBlobHeader) == 128 <= _lib.FSTORE_BLOB_ALIGN
    # every options field but the device travels in the blob
    opts = [n for n, _ in _lib.FstoreOptions._fields_ if n != "device"]
    assert [n for n, _ in mirror][3:3 + len(opts)] == opts


@pytest.fixture(scope="module")
def rows_shim(tmp_path_factory):
    from similari_b200 import _build

    so = str(tmp_path_factory.mktemp("fstore_shim") / "libfstore_rows.so")
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(_build.nvcc()))), "include")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", inc,
                           os.path.join(ROOT, "tests", "host_shim", "fstore_rows_shim.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.shim_fs_row_table.restype = C.c_int
    lib.shim_fs_row_table.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return lib


@pytest.mark.parametrize("K", [1, 3, 5, 64])
def test_row_table_takes_the_newest_k_rows_of_each_query(rows_shim, K):
    rng = np.random.default_rng(K)
    for Q in (1, 2, 17, 300):
        lens = rng.integers(1, 2 * K + 3, Q)
        lens[0] = K   # exactly K, one more and one fewer are all present
        if Q > 2:
            lens[1], lens[2] = K + 1, max(1, K - 1)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        row_src = np.full(int(offs[-1]), -1, np.int32)
        qoff = np.full(Q + 1, -1, np.int32)
        R = rows_shim.shim_fs_row_table(Q, offs.ctypes.data, K, row_src.ctypes.data, qoff.ctypes.data)
        want = [np.arange(offs[q], offs[q + 1])[-K:] for q in range(Q)]
        assert R == sum(len(x) for x in want)
        assert np.array_equal(row_src[:R], np.concatenate(want))
        assert np.array_equal(qoff, np.concatenate([[0], np.cumsum([len(x) for x in want])]))


@pytest.fixture(scope="module")
def plan_shim(tmp_path_factory):
    from similari_b200 import _build

    so = str(tmp_path_factory.mktemp("fstore_plan") / "libfstore_plan.so")
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(_build.nvcc()))), "include")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", inc,
                           os.path.join(ROOT, "tests", "host_shim", "fstore_plan_shim.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.shim_fs_blob_sections.restype = C.c_int
    lib.shim_fs_blob_sections.argtypes = [C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                          C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _header_layout(version, live, K, stype, gate, keep, dims, hist_total):
    """The sections of a blob as include/similari_b200.h states them: (name, bytes, class index), in blob order."""
    elem = 4 if stype == 0 else 2
    feat = [live * K * ((d + 7) // 8 * 8) * elem for d in dims]
    g = 8 * live if gate else 0
    if version == 1:
        return [("ids", 8 * live, 0), ("cnt", 4 * live, 0), ("start", 4 * live, 0), ("feat", feat[0], 0)]
    if version == 2:
        return _header_layout(1, live, K, stype, gate, keep, dims, 0) + \
            [("source", g, 0), ("t_start", g, 0), ("t_end", g, 0)]
    if version == 3:
        return _header_layout(2, live, K, stype, gate, keep, dims, 0) + \
            [("quality", 4 * live * K, 0), ("history_length", 4 * live, 0), ("history", 8 * hist_total, 0)]
    out = [("ids", 8 * live, 0), ("source", g, 0), ("t_start", g, 0), ("t_end", g, 0),
           ("history_length", 4 * live if keep else 0, 0), ("history", 8 * hist_total if keep else 0, 0),
           ("class_ids", 8 * len(dims), 0), ("class_dims", 4 * len(dims), 0)]
    for k in range(len(dims)):
        out += [("cnt", 4 * live, k), ("start", 4 * live, k), ("feat", feat[k], k),
                ("quality", 4 * live * K if keep else 0, k)]
    return out


# the sections' roles (sb::kFsSec*), in enum order
_ROLES = ["ids", "source", "t_start", "t_end", "history_length", "history", "class_ids", "class_dims", "cnt", "start",
          "feat", "quality"]
# version: the gate rules and retention rules its blobs carry (include/similari_b200.h)
_BLOB_RULES = {1: ([0], [0]), 2: ([1, 2], [0]), 3: ([0, 1, 2], [1]), 4: ([0, 1, 2], [0, 1])}


@pytest.mark.parametrize("version", [1, 2, 3, 4])
def test_blob_section_plan_is_the_header_layout(plan_shim, version):
    gates, keeps = _BLOB_RULES[version]
    counts = {1: 4, 2: 7, 3: 10}
    for gate in gates:
        for keep in keeps:
            for stype in (0, 1, 2):   # SB200_FEATURE_F32, _F16, _BF16
                for live, K, dims, hist_total in ((0, 1, [20], 0), (5, 3, [20], 9), (7, 64, [8193 - 1], 7),
                                                  (3, 4, [8, 13, 1], 5), (2, 2, [3] * 16, 4)):
                    if version < 4 and len(dims) > 1:
                        continue
                    want = _header_layout(version, live, K, stype, gate, keep, dims, hist_total)
                    cap = 8 + 4 * 16
                    names = C.create_string_buffer(32 * cap)
                    nbytes, role, cls = np.zeros(cap, np.uint64), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
                    d = np.array(dims, np.int32)
                    n = plan_shim.shim_fs_blob_sections(version, live, K, stype, gate, keep, len(dims), d.ctypes.data,
                                                        hist_total, cap, names, nbytes.ctypes.data, role.ctypes.data,
                                                        cls.ctypes.data)
                    assert n == len(want) == counts.get(version, 8 + 4 * len(dims))
                    got = [(names.raw[32 * i: 32 * i + 32].split(b"\0")[0].decode(), int(nbytes[i]), int(cls[i]))
                           for i in range(n)]
                    assert got == want, (version, gate, keep, stype, live, K, dims)
                    assert [_ROLES[r] for r in role[:n]] == [w[0] for w in want]
