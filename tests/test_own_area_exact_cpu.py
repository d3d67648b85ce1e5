"""Own-area shares against an exact reference that shares nothing with their formulation (tests/own_area_exact.py:
rational slabs and half-pixel cell counts instead of Green's theorem with tie rules).  Checked here, without a GPU:
the oracle, own_area_share_seq (the warp kernel's arithmetic, <= 32 neighbours) and own_edge_term_big (the second
pass's arithmetic, any number of neighbours), on scenes dense in shared edge lines, on near-collinear oriented scenes
and on translates by powers of two.

Tolerance: a share equals the correctly rounded share of the exact own area (expected_share), or lies in the band of
own areas within green_sum_bound of it -- the error the f64 boundary sum can make.  On integer-pixel scenes near the
origin that band is a single value unless a box is covered completely, where the residue is at most 2^-40."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import own_area_exact as X
from test_own_area_cpu import ie_share

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "libshim_own.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(HERE, "host_shim", "shim.cpp"), "-o", so])
    L = C.CDLL(so)
    f32p, f64p = C.POINTER(C.c_float), C.POINTER(C.c_double)
    L.shim_vertices.argtypes = [f32p, f64p]
    L.shim_own_area_shares.argtypes = [f32p, C.c_int, f32p]
    L.shim_own_area_share_big.argtypes = [f32p, C.c_int, C.c_int]
    L.shim_own_area_share_big.restype = C.c_float

    class Shim:
        @staticmethod
        def verts(b):
            b = X.f32_rows(b)
            out = np.zeros((len(b), 4, 2), np.float64)
            for i in range(len(b)):
                L.shim_vertices(b[i].ctypes.data_as(f32p), out[i].ctypes.data_as(f64p))
            return out

        @staticmethod
        def seq(b):
            b = X.f32_rows(b)
            out = np.zeros(len(b), np.float32)
            L.shim_own_area_shares(b.ctypes.data_as(f32p), len(b), out.ctypes.data_as(f32p))
            return out

        @staticmethod
        def big(b, idx=None):
            b = X.f32_rows(b)
            idx = range(len(b)) if idx is None else idx
            return np.array([L.shim_own_area_share_big(b.ctypes.data_as(f32p), len(b), int(i)) for i in idx], np.float32)

    return Shim


# ------------------------------------------------------------------------------------------------------ scene families
def px_scene(rows):
    """(product rows, l t w h array) of integer-pixel / half-pixel boxes with power-of-two heights (exact f32 aspect)."""
    lt = np.asarray(rows, np.float64).reshape(-1, 4)
    assert all(float(h) in (2.0 ** np.arange(0, 12)).tolist() for h in lt[:, 3])
    return X.f32_rows([X.ltwh(*r) for r in lt]), lt


def edge_line_scenes():
    """Hand-built integer-pixel scenes, each dense in one kind of shared edge line."""
    S = {}
    S["duplicates"] = [(0, 0, 24, 16)] * 4 + [(12, 0, 24, 16), (12, 0, 24, 16), (0, 8, 24, 16)]
    S["t_junctions"] = [(0, 0, 40, 16), (10, 16, 8, 16), (18, 8, 6, 32), (24, 0, 16, 8), (0, 8, 10, 8)]
    S["nested"] = [(0, 0, 64, 64), (8, 8, 48, 32), (16, 16, 32, 16), (16, 16, 32, 16), (0, 0, 64, 32), (24, 40, 8, 8)]
    # box 0 is tiled by 2 x 4 tiles, two of them overhanging the outline, plus one more stack on a tile line
    tiles = [(0, 0, 48, 32)] + [(12 * c - (4 if c == 0 else 0), 16 * r, 12 + (4 if c == 0 else 0), 16)
                               for r in range(2) for c in range(4)]
    S["tiling"] = tiles + [(12, 0, 12, 32)]
    S["tiling_reversed"] = [tiles[0]] + tiles[:0:-1]
    # one horizontal line y = 16 carrying edges of six boxes in both directions, indices interleaved
    S["one_line_both_directions"] = [(0, 0, 40, 16), (0, 16, 40, 16), (5, 0, 10, 16), (10, 16, 20, 16), (20, 0, 20, 16),
                                     (0, 16, 8, 16), (30, 8, 10, 8)]
    # three or more boxes on one vertical line x = 20, same and opposite directions
    S["one_vertical_line"] = [(0, 0, 20, 32), (20, 0, 20, 32), (20, 8, 8, 16), (12, 4, 8, 8), (20, 0, 4, 32),
                              (4, 16, 16, 16), (20, 16, 12, 16)]
    S["half_pixel"] = [(0.5, 0, 10.5, 16), (5, 0, 11, 16), (5.5, 8, 5, 8), (0.5, 8, 4.5, 8), (0, 0, 16, 16)]
    S["reference_case"] = [(0, 0, 10, 8), (5, 4, 10, 8), (10, 8, 10, 8)]
    return S


def grid_scene(r, n, cell=4, span=12, hs=(4, 8, 16)):
    """n boxes on a coarse grid: every edge lies on one of few lines, duplicates and tilings occur by themselves."""
    rows = [(cell * int(r.integers(0, span)), cell * int(r.integers(0, span)), cell * int(r.integers(1, 6)),
             int(r.choice(hs))) for _ in range(n)]
    return rows


def shifted(rows, off):
    return [(l + off, t + off, w, h) for l, t, w, h in rows]


def near_collinear_scene(r, n):
    """Oriented boxes whose edges are nearly collinear with box 0's: the same angle plus 0, 1e-7 or 1e-4 rad, centres
    moved along and across box 0's axes by whole and tiny amounts."""
    a0 = float(r.uniform(-1.5, 1.5))
    c, s = np.cos(a0), np.sin(a0)
    rows = [[50.0, 50.0, a0, 0.5, 32.0, 1.0]]
    for _ in range(n - 1):
        da = float(r.choice([0.0, 1e-7, -1e-7, 1e-4]))
        u = float(r.choice([-8.0, 0.0, 8.0, 16.0])) + float(r.choice([0.0, 1e-5]))
        v = float(r.choice([-16.0, 0.0, 16.0, 32.0])) + float(r.choice([0.0, 1e-5]))
        rows.append([50.0 + u * c - v * s, 50.0 + u * s + v * c, a0 + da, float(r.choice([0.25, 0.5, 1.0])),
                     float(r.choice([16.0, 32.0])), 1.0])
    return X.f32_rows(rows)


# ---------------------------------------------------------------------------------------------------------- checking
def exact_case(boxes, verts, i, lt=None):
    """(exact own area, bound of the f64 boundary sum, neighbour count) of box i."""
    nb = X.neighbours(boxes, i, verts)
    own = X.own_area_cells(lt, i, nb) if lt is not None else X.own_area_rational(verts[i], verts[nb])
    return own, X.green_sum_bound(verts[i], verts[nb]), len(nb)


def assert_exact(name, boxes, verts, shares, lt=None, strict=False, idx=None):
    """Every implementation's share of box i is in share_band(exact, green_sum_bound); strict: equal to the correctly
    rounded share, or within FULL_COVER_RESIDUE above 0 when box i is covered completely."""
    b = X.f32_rows(boxes)
    idx = range(len(b)) if idx is None else idx
    for n_i, i in enumerate(idx):
        own, delta, k = exact_case(b, verts, i, lt)
        want = X.expected_share(own, b[i, 3], b[i, 4])
        lo, hi = X.share_band(own, delta, b[i, 3], b[i, 4])
        for impl, got in shares.items():
            g = np.float32(got[n_i])
            ctx = (name, impl, i, k, float(own), float(want), float(g))
            assert lo <= g <= hi, ctx
            if strict:
                if own == 0:
                    assert 0.0 <= g <= X.FULL_COVER_RESIDUE, ctx
                else:
                    assert g == want, ctx


def all_impls(oracle, shim, b, with_big=True):
    out = {"oracle": oracle.own_area_shares(b), "seq": shim.seq(b)}
    if with_big:
        out["big"] = shim.big(b)
    return out


# ------------------------------------------------------------------------------------------------- the reference itself
def test_reference_known_answer():
    """bbox_own_areas.rs:50-79: three 10 x 10 boxes stepped by (5, 5) own 75 / 50 / 75 of 100."""
    b = X.f32_rows([X.ltwh(0, 0, 10, 10), X.ltwh(5, 5, 10, 10), X.ltwh(10, 10, 10, 10)])
    lt = [(0, 0, 10, 10), (5, 5, 10, 10), (10, 10, 10, 10)]
    v = np.array([[(x, y) for x, y in ((l, t + 10), (l + 10, t + 10), (l + 10, t), (l, t))] for l, t, _, _ in lt], float)
    for i, want in enumerate((75, 50, 75)):
        nb = X.neighbours(b, i, v)
        assert X.own_area_cells(lt, i, nb) == want
        assert X.own_area_rational(v[i], v[nb]) == want


def test_reference_matches_inclusion_exclusion(shim):
    """The slab reference against the inclusion-exclusion evaluation of test_own_area_cpu.py on small random scenes,
    half of them oriented (that evaluation clips in f64: agreement to 1e-9 of the area)."""
    r = np.random.default_rng(7)
    for trial in range(24):
        n = int(r.integers(2, 6))
        b = np.zeros((n, 6), np.float32)
        b[:, :2] = r.uniform(0, 80, (n, 2))
        b[:, 2] = r.uniform(-1.5, 1.5, n) if trial % 2 else np.nan
        b[:, 3] = r.uniform(0.3, 0.8, n)
        b[:, 4] = r.uniform(30, 90, n)
        b[:, 5] = 1
        v = shim.verts(b)
        for i in range(n):
            nb = X.neighbours(b, i, v)
            own = float(X.own_area_rational(v[i], v[nb]))
            # ie_share divides by its own f32 rounding of aspect * h * h: compare the own areas it implies
            den = float(np.float32(float(b[i, 3]) * float(b[i, 4]) * float(b[i, 4]))) + 1e-5
            want = ie_share(b.astype(np.float64), i) * den
            assert abs(min(own, den) - want) < 1e-9 * den, (trial, i, own, want)


def test_reference_coincident_outline_cases(shim):
    """The hand cases of test_own_area_cpu.test_coincident_outlines, from the cell count and from the rational slabs."""
    cases = {
        "identical": ([(0, 0, 10, 8), (0, 0, 10, 8)], [0, 0]),
        "triple duplicate": ([(0, 0, 10, 8)] * 3, [0, 0, 0]),
        "nested": ([(0, 0, 10, 8), (2, 2, 4, 4)], [64, 0]),
        "adjacent (shared edge, outside)": ([(0, 0, 10, 8), (10, 0, 10, 8)], [80, 80]),
        "duplicate cover of one half": ([(0, 0, 10, 8), (5, 0, 10, 8), (5, 0, 10, 8)], [40, 0, 0]),
        "two halves tile the box": ([(0, 0, 10, 8), (0, 0, 5, 8), (5, 0, 5, 8)], [0, 0, 0]),
        "cross": ([(0, 3, 10, 2), (4, 0, 2, 8)], [16, 12]),
        "far apart": ([(0, 0, 10, 8), (500, 500, 10, 8)], [80, 80]),
        "single": ([(0, 0, 10, 8)], [80]),
    }
    for name, (rows, want) in cases.items():
        b, lt = px_scene(rows)
        v = shim.verts(b)
        for i, w in enumerate(want):
            nb = X.neighbours(b, i, v)
            assert X.own_area_cells(lt, i, nb) == w, (name, i)
            assert X.own_area_rational(v[i], v[nb]) == w, (name, i)


def test_f64_slabs_within_their_bound(shim):
    """own_area_slabs_f64 against own_area_rational on oriented scenes of up to a dozen boxes: inside its stated bound,
    and the bound far below one f32 ulp of the share (so the f64 reference decides the rounded share)."""
    r = np.random.default_rng(17)
    for trial in range(6):
        n = 12
        b = np.zeros((n, 6), np.float32)
        b[:, :2] = r.uniform(0, 60, (n, 2))
        b[:, 2] = r.uniform(-1.5, 1.5, n)
        b[:, 3] = r.uniform(0.3, 0.8, n)
        b[:, 4] = r.uniform(30, 60, n)
        b[:, 5] = 1
        v = shim.verts(b)
        for i in range(0, n, 3):
            nb = X.neighbours(b, i, v)
            exact = X.own_area_rational(v[i], v[nb])
            a64, bound = X.own_area_slabs_f64(v[i], v[nb])
            assert abs(Fraction(a64) - exact) <= Fraction(bound), (trial, i, a64, float(exact), bound)
            assert bound < 1e-4 * 2.0 ** -24 * float(X.area_f32(b[i, 3], b[i, 4]))


# ------------------------------------------------------------------------------------- oracle and product vs exact
@pytest.mark.parametrize("name", sorted(edge_line_scenes()))
def test_shared_edge_line_scenes_are_exact(oracle, shim, name):
    rows = edge_line_scenes()[name]
    b, lt = px_scene(rows)
    v = shim.verts(b)
    assert_exact(name, b, v, all_impls(oracle, shim, b), lt=lt, strict=True)
    for off in (65536.0, 2.0 ** 20):       # exact coordinates far from the origin: px dy - py dx grows with them
        b2, lt2 = px_scene(shifted(rows, off))
        v2 = shim.verts(b2)
        assert_exact((name, off), b2, v2, all_impls(oracle, shim, b2), lt=lt2)


@pytest.mark.parametrize("off", [0.0, 65536.0])
def test_grid_scenes_are_exact(oracle, shim, off):
    """Random boxes on a 4-pixel grid (every edge on one of a few lines; duplicates, nesting and tilings by chance),
    2-31 boxes, so that both the warp arithmetic and the second pass's cover every box."""
    r = np.random.default_rng(1234)
    full = 0
    for trial in range(40):
        rows = shifted(grid_scene(r, int(r.integers(2, 32))), off)
        b, lt = px_scene(rows)
        v = shim.verts(b)
        sh = all_impls(oracle, shim, b)
        assert_exact(trial, b, v, sh, lt=lt, strict=(off == 0.0))
        full += int((sh["oracle"] < 1e-6).sum())
    assert full > 20          # covered boxes, the residue case, do occur


def test_near_collinear_oriented_scenes(oracle, shim):
    r = np.random.default_rng(99)
    for trial in range(10):
        b = near_collinear_scene(r, int(r.integers(3, 8)))
        v = shim.verts(b)
        assert_exact(trial, b, v, all_impls(oracle, shim, b))


def test_big_walk_equals_warp_list_bit_for_bit(shim):
    """Up to 32 neighbours both product functions apply: own_edge_term_big walks the same runs as own_edge_term's
    sorted merge, so the shares must be identical, on edge-line scenes (touching intervals) and random oriented ones."""
    r = np.random.default_rng(5)
    scenes = [px_scene(rows)[0] for rows in edge_line_scenes().values()]
    scenes += [px_scene(grid_scene(r, int(r.integers(2, 33))))[0] for _ in range(20)]
    for _ in range(20):
        n = int(r.integers(2, 32))
        b = np.zeros((n, 6), np.float32)
        b[:, :2] = r.uniform(0, 100, (n, 2))
        b[:, 2] = r.uniform(-1.5, 1.5, n) if _ % 2 else np.nan
        b[:, 3] = r.uniform(0.3, 0.8, n)
        b[:, 4] = r.uniform(40, 160, n)
        b[:, 5] = 1
        scenes.append(b)
    for b in scenes:
        seq = shim.seq(b)
        assert np.all(seq >= 0)
        np.testing.assert_array_equal(shim.big(b).view(np.uint32), seq.view(np.uint32))


def test_big_walk_in_crowds_is_exact(oracle, shim):
    """Beyond 32 neighbours only the second pass's arithmetic applies (own_area_share_seq returns -1): integer-pixel
    crowds of 40-300 boxes against the cell count, including a row of touching boxes ordered against the edge."""
    r = np.random.default_rng(77)
    scenes = []
    for n in (60, 120, 300):
        scenes.append(grid_scene(r, n, cell=2, span=12, hs=(8, 16)))
    # box 0 over a row of 120 touching 2-pixel boxes on its top edge, in descending x: the run grows one box per pass
    scenes.append([(0, 0, 240, 16)] + [(2 * c, 0, 2, 8) for c in range(119, -1, -1)])
    for s, rows in enumerate(scenes):
        b, lt = px_scene(rows)
        v = shim.verts(b)
        idx = np.flatnonzero(shim.seq(b) == -1.0)[:12]     # more than 32 boxes overlap these
        assert len(idx) and min(len(X.neighbours(b, i, v)) for i in idx) > 32, s
        got = {"big": shim.big(b, idx), "oracle": oracle.own_area_shares(b)[idx]}
        assert_exact(s, b, v, got, lt=lt, strict=True, idx=idx)


def test_zero_area_boxes_cover_nothing(oracle, shim):
    """A box of aspect or height 0 (the reference panics on it) has its edges in coincident pairs of opposite
    direction; lying on another box's edge line, such a pair once took area from box_i.  It covers nothing."""
    rows = [(0, 0, 32, 16), (16, 8, 32, 16), (60, 0, 16, 16)]
    b, lt = px_scene(rows)
    deg = np.array([[16.0, 8.0, np.nan, 0.0, 16.0, 1.0], [32.0, 8.0, np.nan, 1.0, 0.0, 1.0],
                    [20.0, 10.0, 0.3, 0.0, 8.0, 1.0]], np.float32)
    allb = np.concatenate([b, deg])
    sh = all_impls(oracle, shim, allb)
    for impl, got in sh.items():
        assert not np.isnan(got).any(), impl
        np.testing.assert_array_equal(got[len(b):], 0.0, err_msg=impl)
    assert_exact("zero area", b, shim.verts(b), {k: v[: len(b)] for k, v in sh.items()}, lt=lt, strict=True)


def test_big_walk_capacity_boundary(shim):
    """kOwnBigNb = 2800 neighbours is the largest crowd the second pass takes; 2801 are refused (-1, the kernel's
    SB200_ERR_CAPACITY).  The 2800 case is a stack of duplicates: one run per edge (about 1 s of host time)."""
    b2800, lt = px_scene([(0, 0, 16, 16)] + [(0, 0, 16, 16)] * 2800)
    b2801, _ = px_scene([(0, 0, 16, 16)] + [(0, 0, 16, 16)] * 2801)
    assert shim.big(b2801, [0])[0] == -1.0
    got = shim.big(b2800, [0])[0]
    assert 0.0 <= got <= X.FULL_COVER_RESIDUE
