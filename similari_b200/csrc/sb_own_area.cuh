// sb_own_area.cuh -- exclusively owned area shares of the detections of a scene.
//
// Reference: exclusively_owned_areas + exclusively_owned_areas_normalized_shares
// (src/utils/clipping/bbox_own_areas.rs:8-46), called by the visual trackers when
// visual_minimal_own_area_percentage_{use,collect} > 0 (src/trackers/visual_sort/simple_api.rs:110-127,
// visual_sort/batch_api.rs:236-249): for every box, the part of it that no other (not too_far) box covers, as a share
// of its own area:  share_i = min(1, area(box_i \ U_j box_j) / (area_f32(box_i) + EPS)).
//
// The reference builds the difference with geo's BooleanOps (a general polygon clipper, third-party, not under
// /root/reference).  Here the same quantity is computed in closed form for convex quadrilaterals by Green's theorem on
// the boundary of the difference region D = box_i \ U_j box_j, which consists of
//   * the parts of box_i's edges outside every other box, in box_i's direction, and
//   * the parts of every other box's edges inside box_i and outside all remaining boxes, in the reverse direction.
// For a convex box the part of a segment inside it is ONE parameter interval (four half-planes), so each edge needs an
// interval union and nothing else -- no polygon clipping, no intermediate polygons.
// Coincident boundaries (common with axis-aligned detections that share coordinates; exact zeros in f64 then): a segment
// lying on an edge line of another box counts as inside that box iff both run in the same direction -- and, between two
// covering boxes, only if the other one has the lower index, so that a doubly covered boundary is integrated once.
// "Inside box_i" (for the edges of the covering boxes) is open: a covering box's edge on box_i's outline never borders D.
//
// `__host__ __device__` like sb_math.cuh: the CPU suite checks these functions (tests/host_shim) against the oracle and
// against an exact reference that does not use this formulation (tests/own_area_exact.py) without a GPU.
#pragma once
#include "sb_math.cuh"

namespace sb {

constexpr int kOwnMaxNb = 32;     // boxes overlapping one box the warp-per-detection kernel keeps on chip
constexpr int kOwnBigNb = 2800;   // ... and the CTA-per-detection second pass (more: SB200_ERR_CAPACITY); 64 B each

// signed shoelace area of a quadrilateral (x0,y0,...,x3,y3), coordinates shifted by the first vertex like geo
SB_HD double quad_area_signed(const double* q) {
  double tmp = 0.0, pax = 0.0, pay = 0.0;
  for (int j = 1; j <= 4; ++j) {
    const int jj = (j == 4) ? 0 : j;
    const double qx = q[2 * jj] - q[0], qy = q[2 * jj + 1] - q[1];
    tmp += pax * qy - pay * qx;
    pax = qx; pay = qy;
  }
  return tmp / 2.0;
}

// Whether box j (vertices vj) can take area from box i (vi) and so joins box i's list.  Certainly disjoint boxes remove
// nothing (separating-axis gate; it also drops boxes with a NaN vertex).  Nor do boxes of zero area (aspect or height
// 0): their edges come in coincident pairs of opposite direction, which the tie rules for coincident edges do not
// cancel where the pair lies on another box's edge line.
SB_HD bool own_can_cover(const double* vi, const double* vj) {
  return quad_area_signed(vj) != 0.0 && rect_overlap_bound(vi, vj) != 0.0;
}

// Parameter interval [t0, t1] of the segment P + t d (t in [0, 1]) inside the convex quadrilateral q whose vertices run
// with orientation sign s (+1 counter-clockwise, -1 clockwise).  on_edge_same_dir_inside: what a segment lying exactly on
// one of q's edge lines and running in that edge's direction counts as (opposite direction: always outside).
SB_HD bool seg_inside_quad(double px, double py, double dx, double dy, const double* q, double s,
                           bool on_edge_same_dir_inside, double* t0, double* t1) {
  double lo = 0.0, hi = 1.0;
  for (int a = 0; a < 4; ++a) {
    const int b = (a + 1) & 3;
    const double ax = q[2 * a], ay = q[2 * a + 1];
    const double ex = q[2 * b] - ax, ey = q[2 * b + 1] - ay;
    const double f0 = s * (ex * (py - ay) - ey * (px - ax));
    const double f1 = s * (ex * dy - ey * dx);
    if (f1 > 0.0) {
      const double t = -f0 / f1;
      if (t > lo) lo = t;
    } else if (f1 < 0.0) {
      const double t = -f0 / f1;
      if (t < hi) hi = t;
    } else {
      if (f0 < 0.0) return false;
      if (f0 == 0.0 && !(on_edge_same_dir_inside && (ex * dx + ey * dy) > 0.0)) return false;
    }
    if (!(lo < hi)) return false;
  }
  *t0 = lo; *t1 = hi;
  return true;
}

// Boundary term of edge e of quadrilateral js of the list `quads` ([k + 1][8]; quads[0] = box_i, 1..k = the boxes that
// overlap it): the measure of the edge's part that borders D times the Green integrand, signed for D's orientation.
// The terms of all 4 * (k + 1) edges add up to 2 * s * area(D).
SB_HD double own_edge_term(const double* quads, int k, int js, int e, double s) {
  const double* q = quads + js * 8;
  const int e2 = (e + 1) & 3;
  const double px = q[2 * e], py = q[2 * e + 1];
  const double dx = q[2 * e2] - px, dy = q[2 * e2 + 1] - py;
  if (dx == 0.0 && dy == 0.0) return 0.0;
  double wa = 0.0, wb = 1.0;   // window of the edge that can border D at all
  if (js != 0 && !seg_inside_quad(px, py, dx, dy, quads, s, /*on_edge_same_dir_inside=*/false, &wa, &wb)) return 0.0;
  double ia[kOwnMaxNb], ib[kOwnMaxNb];
  int cnt = 0;
  for (int l = 1; l <= k; ++l) {
    if (l == js) continue;
    double t0, t1;
    // box_i's own edge: any covering box on the same line and direction covers it; between covering boxes: lower index
    if (!seg_inside_quad(px, py, dx, dy, quads + l * 8, s, js == 0 || l < js, &t0, &t1)) continue;
    if (t0 < wa) t0 = wa;
    if (t1 > wb) t1 = wb;
    if (!(t0 < t1)) continue;
    int qn = cnt++;   // insertion by start
    while (qn > 0 && ia[qn - 1] > t0) { ia[qn] = ia[qn - 1]; ib[qn] = ib[qn - 1]; --qn; }
    ia[qn] = t0; ib[qn] = t1;
  }
  double covered = 0.0, cur_a = 0.0, cur_b = -1.0;
  for (int qn = 0; qn < cnt; ++qn) {
    if (cur_b < cur_a) { cur_a = ia[qn]; cur_b = ib[qn]; }
    else if (ia[qn] <= cur_b) { if (ib[qn] > cur_b) cur_b = ib[qn]; }
    else { covered += cur_b - cur_a; cur_a = ia[qn]; cur_b = ib[qn]; }
  }
  if (cur_b >= cur_a) covered += cur_b - cur_a;
  const double term = ((wb - wa) - covered) * (px * dy - py * dx);
  return js == 0 ? term : -term;
}

// The same term without per-thread interval storage, for a box that more than kOwnMaxNb boxes overlap (second pass of
// own_area_kernel).  The union of the covering intervals inside the window [wa, wb] is walked run by run: a run starts at
// the smallest interval start beyond the previous run and grows while some interval starts inside it and ends beyond it.
// The runs -- and therefore the partial sums -- are exactly those of the sorted merge above; cost O(k) per step.
SB_HD double own_edge_term_big(const double* quads, int k, int js, int e, double s) {
  const double* q = quads + js * 8;
  const int e2 = (e + 1) & 3;
  const double px = q[2 * e], py = q[2 * e + 1];
  const double dx = q[2 * e2] - px, dy = q[2 * e2 + 1] - py;
  if (dx == 0.0 && dy == 0.0) return 0.0;
  double wa = 0.0, wb = 1.0;
  if (js != 0 && !seg_inside_quad(px, py, dx, dy, quads, s, false, &wa, &wb)) return 0.0;
  double covered = 0.0;
  double done = -1.0;      // everything up to `done` is accounted for
  bool first = true;
  for (;;) {
    // next run: the smallest clipped start that is >= wa and lies beyond `done` (first run: any start)
    double ra = 0.0, rb = -1.0;
    bool found = false;
    for (int l = 1; l <= k; ++l) {
      if (l == js) continue;
      double t0, t1;
      if (!seg_inside_quad(px, py, dx, dy, quads + l * 8, s, js == 0 || l < js, &t0, &t1)) continue;
      if (t0 < wa) t0 = wa;
      if (t1 > wb) t1 = wb;
      if (!(t0 < t1)) continue;
      if (!first && !(t0 > done)) continue;            // starts inside what is already merged
      if (!found || t0 < ra || (t0 == ra && t1 > rb)) { ra = t0; rb = t1; found = true; }
    }
    if (!found) break;
    // grow the run
    for (bool grown = true; grown;) {
      grown = false;
      for (int l = 1; l <= k; ++l) {
        if (l == js) continue;
        double t0, t1;
        if (!seg_inside_quad(px, py, dx, dy, quads + l * 8, s, js == 0 || l < js, &t0, &t1)) continue;
        if (t0 < wa) t0 = wa;
        if (t1 > wb) t1 = wb;
        if (!(t0 < t1)) continue;
        if (t0 <= rb && t0 >= ra && t1 > rb) { rb = t1; grown = true; }
      }
    }
    covered += rb - ra;
    done = rb;
    first = false;
  }
  const double term = ((wb - wa) - covered) * (px * dy - py * dx);
  return js == 0 ? term : -term;
}

// share from the owned area: (own / (area_f32 + EPS) as f64) as f32, clamped to 1 (bbox_own_areas.rs:36-46)
SB_HD float own_share(double own, float aspect, float height) {
  if (!(own > 0.0)) own = 0.0;
  const float denom = box_area(aspect, height) + kEps;
  const float e = (float)(own / (double)denom);
  return e >= 1.0f ? 1.0f : e;
}

// Whole computation for box i of a list (sequential form used by the host shim; the kernel spreads the same steps over
// a warp).  boxes: [n][6] raw boxes.  Returns the share, or -1 when more than kOwnMaxNb boxes overlap box i.
SB_HD float own_area_share_seq(const float* boxes, int n, int i) {
  const float* bi = boxes + (size_t)i * 6;
  double quads[(kOwnMaxNb + 1) * 8];
  box_vertices(bi[0], bi[1], bi[2], bi[3], bi[4], quads);
  const double s = quad_area_signed(quads) < 0.0 ? -1.0 : 1.0;
  const float ri = box_radius(bi[3], bi[4]);
  int k = 0;
  for (int j = 0; j < n; ++j) {
    if (j == i) continue;
    const float* bj = boxes + (size_t)j * 6;
    if (too_far(bi[0], bi[1], ri, bj[0], bj[1], box_radius(bj[3], bj[4]))) continue;   // bbox_own_areas.rs:12-14
    double vj[8];
    box_vertices(bj[0], bj[1], bj[2], bj[3], bj[4], vj);
    if (!own_can_cover(quads, vj)) continue;
    if (k >= kOwnMaxNb) return -1.0f;
    ++k;
    for (int q = 0; q < 8; ++q) quads[k * 8 + q] = vj[q];
  }
  double sum = 0.0;
  for (int js = 0; js <= k; ++js)
    for (int e = 0; e < 4; ++e) sum += own_edge_term(quads, k, js, e, s);
  return own_share(s * sum / 2.0, bi[3], bi[4]);   // 2 s area(D); rounding below zero clamps to 0
}

}  // namespace sb
