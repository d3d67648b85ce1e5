"""Independent references for the own-area shares (exclusively_owned_areas_normalized_shares,
src/utils/clipping/bbox_own_areas.rs:8-46), for the tests of sb_own_area.cuh / kernels_own.cu and of the oracle.

share_i = min(1, area(box_i minus the union of box_j) / (area_f32(box_i) + EPS)), over the boxes j that are not too_far
from box_i.  The product and the oracle integrate the boundary of that difference (Green's theorem, one interval union
per edge, tie rules for coincident edges).  Nothing here does: the covered area is integrated over vertical slabs, or
counted in half-pixel cells, so a wrong tie rule or a lost interval in the product cannot be repeated here.

  * `neighbours`: which boxes take part -- too_far on the f32 radii (bbox.rs:452-462, sb_math.cuh), box i itself and
    boxes whose vertices are not finite excluded (a box with a NaN coordinate covers nothing: the product's
    separating-axis gate drops it, and the reference's polygon would be empty).
  * `own_area_rational`: exact, fractions.Fraction, for any convex quadrilaterals given by their f64 vertices.
  * `own_area_cells`: exact, integer arithmetic, for axis-aligned boxes on the half-pixel grid; scales to the
    2,800-neighbour cap.
  * `own_area_slabs_f64`: the slab integral in f64 for oriented crowds beyond the rational range, with a stated bound.
  * `expected_share` / `share_band`: the share rounded exactly as own_share (sb_own_area.cuh) rounds.

The vertices are the product's (shim_vertices on the host, engine.box_vertices on the GPU), so sin/cos is not part of
the question; for axis-aligned boxes on the half-pixel grid with a power-of-two height they are exact anyway."""
from fractions import Fraction

import numpy as np

F32 = np.float32
EPS = F32(1e-5)
U64 = 2.0 ** -53          # unit roundoff of f64
FULL_COVER_RESIDUE = 2.0 ** -40   # largest share a fully covered box may return instead of 0 (see green_sum_bound)


def ltwh(l, t, w, h, angle=np.nan):
    """A box given by left, top, width, height (the reference's from_ltwh), as a product row [xc, yc, angle, aspect, h, 1]."""
    return [l + w / 2, t + h / 2, angle, w / h, h, 1.0]


def f32_rows(boxes):
    return np.ascontiguousarray(np.asarray(boxes, np.float32).reshape(-1, 6))


def radii(b):
    """Universal2DBox::get_radius in f32 (sb_math.cuh box_radius)."""
    hw = (b[:, 3] * b[:, 4]) / F32(2)
    hh = b[:, 4] / F32(2)
    return np.sqrt(hw * hw + hh * hh)


def neighbours(boxes, i, verts):
    """Indices j != i of the boxes that box i's share is taken against: not too_far in f32 (bbox.rs:452-462) and with
    finite vertices.  verts: [n][4][2] f64 vertices of the rows."""
    b = f32_rows(boxes)
    with np.errstate(invalid="ignore", over="ignore"):
        r = radii(b)
        md = r[i] + r
        x = b[i, 0] - b[:, 0]
        y = b[i, 1] - b[:, 1]
        far = x * x + y * y > md * md
    fin = np.isfinite(np.asarray(verts, np.float64).reshape(len(b), 8)).all(axis=1)
    return [j for j in range(len(b)) if j != i and not far[j] and fin[j]]


def area_f32(aspect, height):
    """Universal2DBox::area in f32 (sb_math.cuh box_area)."""
    return F32(F32(F32(height) * F32(aspect)) * F32(height))


def _share_of(q, denom):
    """own_share's rounding of a non-negative exact quotient q = own / denom: to f64 (correctly rounded), then to f32,
    then clamped at 1 -- what sb_own_area.cuh:159-164 does to its f64 quotient."""
    e = F32(float(q))
    return F32(1.0) if e >= F32(1.0) else e


def expected_share(own, aspect, height):
    """own_share(own, aspect, height) for an exact own area (Fraction or int)."""
    denom = Fraction(float(area_f32(aspect, height) + EPS))
    own = Fraction(own)
    return _share_of(max(own, Fraction(0)) / denom, denom)


def share_band(own, delta, aspect, height):
    """[lo, hi]: every share own_share can return for an own area within `delta` of the exact `own` (own_share is
    monotone, so the ends are those of own - delta and own + delta)."""
    own, delta = Fraction(own), Fraction(delta)
    return expected_share(own - delta, aspect, height), expected_share(own + delta, aspect, height)


# ---------------------------------------------------------------------------------------------------- exact, rational
def _quad(v):
    return [(Fraction(float(v[a][0])), Fraction(float(v[a][1]))) for a in range(4)]


def _edges(q):
    return [(q[a], q[(a + 1) % 4]) for a in range(4)]


def _yspan(edges, x):
    """The vertical extent [lo, hi] of a convex quadrilateral on the line at x (x not a vertex abscissa), or None."""
    ys = []
    for (x0, y0), (x1, y1) in edges:
        if x0 == x1 or not (min(x0, x1) < x < max(x0, x1)):
            continue
        ys.append(y0 + (y1 - y0) * (x - x0) / (x1 - x0))
    return (min(ys), max(ys)) if len(ys) >= 2 else None


def _crossing_x(e, f):
    """x of the single crossing point of segments e and f (None when parallel or disjoint)."""
    (px, py), (qx, qy) = e
    (ax, ay), (bx, by) = f
    rx, ry, sx, sy = qx - px, qy - py, bx - ax, by - ay
    den = rx * sy - ry * sx
    if den == 0:
        return None
    wx, wy = ax - px, ay - py
    t = (wx * sy - wy * sx) / den
    u = (wx * ry - wy * rx) / den
    if 0 <= t <= 1 and 0 <= u <= 1:
        return px + t * rx
    return None


def own_area_rational(vi, covers):
    """Exact area(box_i) - area(box_i ∩ ∪ covers) of convex quadrilaterals (f64 vertices [4][2], any orientation), as a
    Fraction.  Between two consecutive event abscissae -- every vertex x and every crossing x of two edges -- each
    quadrilateral meets the vertical line in one interval whose ends move linearly, and no two ends cross, so the
    uncovered length of box_i is linear in x and the slab's area is its width times the length at the midpoint."""
    qi = _quad(vi)
    xlo, xhi = min(p[0] for p in qi), max(p[0] for p in qi)
    ei = _edges(qi)
    cq = []
    for v in covers:
        q = _quad(v)
        if max(p[0] for p in q) > xlo and min(p[0] for p in q) < xhi:
            cq.append(_edges(q))
    events = {xlo, xhi}
    alle = ei + [e for es in cq for e in es]
    boxes = [(min(e[0][0], e[1][0]), max(e[0][0], e[1][0]), min(e[0][1], e[1][1]), max(e[0][1], e[1][1])) for e in alle]
    for a, e in enumerate(alle):
        for x in (e[0][0], e[1][0]):
            if xlo < x < xhi:
                events.add(x)
        ba = boxes[a]
        for c in range(a + 1, len(alle)):
            bc = boxes[c]
            if ba[1] < bc[0] or bc[1] < ba[0] or ba[3] < bc[2] or bc[3] < ba[2]:
                continue
            x = _crossing_x(e, alle[c])
            if x is not None and xlo < x < xhi:
                events.add(x)
    xs = sorted(events)
    area = Fraction(0)
    for x0, x1 in zip(xs[:-1], xs[1:]):
        m = (x0 + x1) / 2
        si = _yspan(ei, m)
        if si is None:
            continue
        lo_i, hi_i = si
        iv = []
        for es in cq:
            s = _yspan(es, m)
            if s is not None and s[0] < hi_i and s[1] > lo_i:
                iv.append((max(s[0], lo_i), min(s[1], hi_i)))
        iv.sort()
        covered, top = Fraction(0), lo_i
        for a, b in iv:
            if b > top:
                covered += b - max(a, top)
                top = b
        area += (x1 - x0) * ((hi_i - lo_i) - covered)
    return area


# ---------------------------------------------------------------------------------------------- exact, half-pixel cells
def own_area_cells(lt_wh, i, nb):
    """Exact own area of axis-aligned box i among the boxes nb, all given as [n][4] (l, t, w, h) on the half-pixel grid:
    the covered half-pixel cells of box i counted with a 2-D difference array (integers only).  Returns a Fraction."""
    g = np.asarray(lt_wh, np.float64) * 2
    if not np.array_equal(g, np.round(g)):
        raise ValueError("coordinates must lie on the half-pixel grid")
    g = g.astype(np.int64)
    l0, t0, w0, h0 = g[i]
    d = np.zeros((h0 + 1, w0 + 1), np.int64)
    if len(nb):
        o = g[np.asarray(nb, np.int64)]
        x0 = np.clip(o[:, 0] - l0, 0, w0)
        x1 = np.clip(o[:, 0] + o[:, 2] - l0, 0, w0)
        y0 = np.clip(o[:, 1] - t0, 0, h0)
        y1 = np.clip(o[:, 1] + o[:, 3] - t0, 0, h0)
        k = (x0 < x1) & (y0 < y1)
        x0, x1, y0, y1 = x0[k], x1[k], y0[k], y1[k]
        np.add.at(d, (y0, x0), 1)
        np.add.at(d, (y0, x1), -1)
        np.add.at(d, (y1, x0), -1)
        np.add.at(d, (y1, x1), 1)
    cov = np.cumsum(np.cumsum(d, axis=0), axis=1)[:h0, :w0]
    return Fraction(int((cov == 0).sum()), 4)


# ------------------------------------------------------------------------------------------------- f64 slab integral
def own_area_slabs_f64(vi, covers):
    """The slab integral of own_area_rational in f64, vectorised, for crowds of a few hundred oriented boxes.
    Returns (area, bound) with |area - exact| <= bound.

    Bound: in each slab, the 2 (k + 1) interval ends are line evaluations y0 + (y1 - y0) (m - x0) / (x1 - x0) of f64
    vertices with |coordinates| <= R, each within 8 u R of the ends at the computed midpoint, and the union takes at most
    two ends per interval: the uncovered length is within 32 (k + 1) u R of the exact one at that abscissa; over box_i's
    width W that is 32 (k + 1) u R W.  The computed event abscissae (f64 crossings, within u R of the exact ones only
    for crossing angles that are not tiny) and the midpoint's rounding move the sample point inside a slab where the
    length has slope at most 2 (k + 1) H / w_slab (H: box_i's height): a further 2 (k + 1) u R H per slab.  The final sum
    of N slab areas adds N u area(box_i)."""
    vi = np.asarray(vi, np.float64)
    cv = np.asarray(covers, np.float64).reshape(-1, 4, 2)
    xlo, xhi = vi[:, 0].min(), vi[:, 0].max()
    keep = (cv[:, :, 0].max(axis=1) > xlo) & (cv[:, :, 0].min(axis=1) < xhi)
    cv = cv[keep]
    quads = np.concatenate([vi[None], cv], axis=0)                       # [k + 1][4][2]
    p = quads.reshape(-1, 2)
    q = np.roll(quads, -1, axis=1).reshape(-1, 2)                          # edge a: p[a] -> q[a]
    r = q - p
    ev = [xlo, xhi, *p[:, 0][(p[:, 0] > xlo) & (p[:, 0] < xhi)]]
    for a0 in range(0, len(p), 256):                                       # pairwise crossings, in blocks
        pa, ra = p[a0:a0 + 256, None, :], r[a0:a0 + 256, None, :]
        w = p[None, :, :] - pa
        den = ra[..., 0] * r[None, :, 1] - ra[..., 1] * r[None, :, 0]
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (w[..., 0] * r[None, :, 1] - w[..., 1] * r[None, :, 0]) / den
            u = (w[..., 0] * ra[..., 1] - w[..., 1] * ra[..., 0]) / den
            x = pa[..., 0] + t * ra[..., 0]
        ok = (den != 0) & (t >= 0) & (t <= 1) & (u >= 0) & (u <= 1) & (x > xlo) & (x < xhi)
        ev.extend(x[ok].tolist())
    xs = np.unique(np.asarray(ev, np.float64))
    area = 0.0
    n_slabs = len(xs) - 1
    for s0 in range(0, n_slabs, 2048):
        x0 = xs[s0:min(s0 + 2048, n_slabs)]
        x1 = xs[s0 + 1:s0 + 1 + len(x0)]
        m = (x0 + x1) / 2
        ex0, ex1 = p[:, 0], q[:, 0]
        lo_e, hi_e = np.minimum(ex0, ex1), np.maximum(ex0, ex1)
        on = (lo_e[None, :] < m[:, None]) & (m[:, None] < hi_e[None, :])
        with np.errstate(divide="ignore", invalid="ignore"):
            y = p[None, :, 1] + r[None, :, 1] * ((m[:, None] - p[None, :, 0]) / r[None, :, 0])
        y = y.reshape(len(m), -1, 4)
        on = on.reshape(len(m), -1, 4)
        ylo = np.where(on, y, np.inf).min(axis=2)
        yhi = np.where(on, y, -np.inf).max(axis=2)
        lo_i, hi_i = ylo[:, 0], yhi[:, 0]
        a = np.maximum(ylo[:, 1:], lo_i[:, None])
        b = np.minimum(yhi[:, 1:], hi_i[:, None])
        valid = a < b
        a = np.where(valid, a, np.inf)
        b = np.where(valid, b, -np.inf)
        order = np.argsort(a, axis=1)
        a = np.take_along_axis(a, order, axis=1)
        b = np.take_along_axis(b, order, axis=1)
        top = np.maximum.accumulate(b, axis=1)
        prev = np.concatenate([np.full((len(m), 1), -np.inf), top[:, :-1]], axis=1)
        add = np.where(np.isfinite(a), np.maximum(0.0, b - np.maximum(a, prev)), 0.0)
        own = np.where(hi_i > lo_i, (hi_i - lo_i) - add.sum(axis=1), 0.0)
        area += float(((x1 - x0) * own).sum())
    k = len(cv)
    R = float(np.abs(quads).max())
    W, H = xhi - xlo, vi[:, 1].max() - vi[:, 1].min()
    bound = U64 * (32 * (k + 1) * R * W + 2 * (k + 1) * R * H * n_slabs + n_slabs * W * H)
    return area, bound


# ------------------------------------------------------------------------------------- the product's f64 Green's sum
def green_sum_bound(vi, covers):
    """A bound on how far the product's (and the oracle's) f64 boundary sum can be from the exact own area, for inputs
    whose interval ends are well conditioned (edges that meet at a right angle or not at all, or cross at angles far
    from 0): the sum has 4 (k + 1) terms ((wb - wa) - covered) * (px dy - py dx).  Each clipped parameter t in [0, 1] is
    one quotient of exact or once-rounded differences (error <= 4 u); a term's covered length merges at most k intervals
    (<= (2 k + 2) * 4 u + k u); |px dy - py dx| is found within 3 u of itself from exact vertices; and the sum of 4 (k + 1)
    terms adds 4 (k + 1) u times the sum of their magnitudes.  Altogether, with G = sum over edges of |px dy| + |py dx|,
    |2 area - sum| <= (16 k + 20) u G, and the area is within (8 k + 10) u G.

    For a box that other boxes cover completely this is the largest residue own_share can see; for integer-pixel boxes
    of a few hundred pixels near the origin it is below 2^-40 of the box's area (FULL_COVER_RESIDUE)."""
    quads = np.concatenate([np.asarray(vi, np.float64)[None], np.asarray(covers, np.float64).reshape(-1, 4, 2)])
    p = quads
    d = np.roll(quads, -1, axis=1) - quads
    G = float((np.abs(p[..., 0] * d[..., 1]) + np.abs(p[..., 1] * d[..., 0])).sum())
    k = len(quads) - 1
    return (8 * k + 10) * U64 * G
