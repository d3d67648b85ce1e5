/*
 * similari_oracle.cpp -- CPU ORACLE (test infrastructure, see similari_oracle.h).
 *
 * Every function restates one reference function operation-for-operation (same precision,
 * same evaluation order, no FMA: build with -ffp-contract=off) and cites the reference
 * file:line (paths relative to /root/reference).  Third-party crates that are not vendored
 * in the reference tree are restated from their published algorithms:
 *   pathfinding 4.x  kuhn_munkres        (Cargo.toml:34, call site src/trackers/sort/voting.rs:86)
 *   nalgebra 0.32    SMatrix gemm / cholesky / solve_lower_triangular (Cargo.toml:33)
 *   geo 0.27         Area::unsigned_area (Cargo.toml:35, call site src/utils/bbox.rs:507)
 *   wide/ultraviolet f32x8 reduce_add    (Cargo.toml:29, call sites src/distance.rs:12-44)
 */
#include "similari_oracle.h"

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <set>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace {

constexpr float EPS = 0.00001f;                 // src/lib.rs:80
constexpr float F32_U64_MULT = 1000000.0f;      // src/trackers/sort/voting.rs:9
constexpr float CHI2_UPPER_BOUND = 100.0f;      // src/utils/kalman.rs:16
constexpr float CHI2INV95_4 = 11.070f;          // src/utils/kalman.rs:18 (index 4)
constexpr float MAHALANOBIS_NEW_TRACK_THRESHOLD = 1.0f;  // src/trackers/sort.rs:379
constexpr int DEFAULT_AUTO_WASTE_PERIODICITY = 100;      // src/trackers/sort.rs:378
constexpr int64_t NONE_ID = INT64_MIN;

struct Box {
  float xc, yc, angle, aspect, height, conf;  // angle NaN == None
};
inline Box load_box(const float* p) { return Box{p[0], p[1], p[2], p[3], p[4], p[5]}; }
inline void store_box(const Box& b, float* p) {
  p[0] = b.xc; p[1] = b.yc; p[2] = b.angle; p[3] = b.aspect; p[4] = b.height; p[5] = b.conf;
}
inline bool has_angle(const Box& b) { return !std::isnan(b.angle); }
inline float angle_or0(const Box& b) { return has_angle(b) ? b.angle : 0.0f; }

// ---------------------------------------------------------------- geometry
// Universal2DBox::get_radius, src/utils/bbox.rs:157-161
float radius(const Box& b) {
  float hw = b.aspect * b.height / 2.0f;
  float hh = b.height / 2.0f;
  return std::sqrt(hw * hw + hh * hh);
}
// Universal2DBox::area, src/utils/bbox.rs:163-166
float area(const Box& b) {
  float w = b.height * b.aspect;
  return w * b.height;
}
// Universal2DBox::too_far, src/utils/bbox.rs:452-462
bool too_far(const Box& l, const Box& r) {
  float max_distance = radius(l) + radius(r);
  float x = l.xc - r.xc;
  float y = l.yc - r.yc;
  return x * x + y * y > max_distance * max_distance;
}
// Universal2DBox::dist_in_2r, src/utils/bbox.rs:464-474
float dist_in_2r(const Box& l, const Box& r) {
  float radial_distance = radius(l) + radius(r);
  float x = l.xc - r.xc;
  float y = l.yc - r.yc;
  return std::sqrt(x * x + y * y) / std::sqrt(radial_distance * radial_distance + EPS);
}

struct P2 { double x, y; };

// From<&Universal2DBox> for Polygon<f64>, src/utils/bbox.rs:287-330
void vertices(const Box& b, P2 out[4]) {
  double angle = (double)angle_or0(b);
  double height = (double)b.height;
  double aspect = (double)b.aspect;
  double c = std::cos(angle);
  double s = std::sin(angle);
  double half_width = height * aspect / 2.0;
  double half_height = height / 2.0;
  double r1x = -half_width * c - half_height * s;
  double r1y = -half_width * s + half_height * c;
  double r2x = half_width * c - half_height * s;
  double r2y = half_width * s + half_height * c;
  double x = (double)b.xc;
  double y = (double)b.yc;
  out[0] = {x + r1x, y + r1y};
  out[1] = {x + r2x, y + r2y};
  out[2] = {x - r1x, y - r1y};
  out[3] = {x - r2x, y - r2y};
}

// is_inside, src/utils/clipping.rs:12-15
inline bool is_inside(const P2& q, const P2& p1, const P2& p2) {
  double r = (p2.x - p1.x) * (q.y - p1.y) - (p2.y - p1.y) * (q.x - p1.x);
  return r <= 0.0;
}
// compute_intersection, src/utils/clipping.rs:17-38
inline P2 compute_intersection(const P2& cp1, const P2& cp2, const P2& s, const P2& e) {
  P2 dc{cp1.x - cp2.x, cp1.y - cp2.y};
  P2 dp{s.x - e.x, s.y - e.y};
  double n1 = cp1.x * cp2.y - cp1.y * cp2.x;
  double n2 = s.x * e.y - s.y * e.x;
  double n3 = 1.0 / (dc.x * dp.y - dc.y * dp.x);
  return P2{(n1 * dp.x - n2 * dc.x) * n3, (n1 * dp.y - n2 * dc.y) * n3};
}
// sutherland_hodgman_clip, src/utils/clipping.rs:40-91
std::vector<P2> sh_clip(const std::vector<P2>& subject, const std::vector<P2>& clipping) {
  std::vector<P2> final_polygon = subject;
  for (size_t i = 0; i < clipping.size(); ++i) {
    std::vector<P2> next_polygon;
    next_polygon.swap(final_polygon);
    size_t i_i = (i == 0) ? clipping.size() - 1 : i - 1;
    const P2& c_edge_start = clipping[i_i];
    const P2& c_edge_end = clipping[i];
    for (size_t j = 0; j < next_polygon.size(); ++j) {
      size_t j_i = (j == 0) ? next_polygon.size() - 1 : j - 1;
      const P2& s_edge_start = next_polygon[j_i];
      const P2& s_edge_end = next_polygon[j];
      if (is_inside(s_edge_end, c_edge_start, c_edge_end)) {
        if (!is_inside(s_edge_start, c_edge_start, c_edge_end)) {
          final_polygon.push_back(compute_intersection(s_edge_start, s_edge_end, c_edge_start, c_edge_end));
        }
        final_polygon.push_back(s_edge_end);
      } else if (is_inside(s_edge_start, c_edge_start, c_edge_end)) {
        final_polygon.push_back(compute_intersection(s_edge_start, s_edge_end, c_edge_start, c_edge_end));
      }
    }
  }
  return final_polygon;
}
// geo 0.27 Area::unsigned_area for a Polygon without holes == |signed ring area|.
// geo's get_linestring_area: ring must have >= 3 coords and be closed (Polygon::new closes it);
// coordinates are shifted by the first coordinate, then tmp += line.determinant() over the ring's
// lines ((a.x*b.y - a.y*b.x) with a,b shifted), result tmp / 2.
double polygon_area(const std::vector<P2>& poly) {
  if (poly.size() < 3) return 0.0;  // closed ring of < 3 distinct-coords: area 0 (geo: < 3 coords => 0)
  std::vector<P2> ring = poly;
  if (ring.front().x != ring.back().x || ring.front().y != ring.back().y) ring.push_back(ring.front());
  const P2 shift = ring[0];
  double tmp = 0.0;
  for (size_t i = 0; i + 1 < ring.size(); ++i) {
    P2 a{ring[i].x - shift.x, ring[i].y - shift.y};
    P2 b{ring[i + 1].x - shift.x, ring[i + 1].y - shift.y};
    tmp += a.x * b.y - a.y * b.x;
  }
  return std::fabs(tmp / 2.0);
}
// Universal2DBox::intersection, src/utils/bbox.rs:476-509
double intersection(const Box& l, const Box& r) {
  if (too_far(l, r)) return 0.0;
  P2 pl[4], pr[4];
  vertices(l, pl);
  vertices(r, pr);
  std::vector<P2> s(pl, pl + 4), c(pr, pr + 4);
  return polygon_area(sh_clip(s, c));
}
// Universal2DBox::calculate_metric_object, src/utils/bbox.rs:512-535
bool iou(const Box& l, const Box& r, float* out) {
  double inter = intersection(l, r);
  if (inter == 0.0) return false;
  double uni = (double)(l.height * l.height * l.aspect + r.height * r.height * r.aspect) - inter;
  double res = inter / uni;
  *out = (float)res;
  return true;
}

// ---------------------------------------------------------------- exclusively owned areas
// exclusively_owned_areas + exclusively_owned_areas_normalized_shares, src/utils/clipping/bbox_own_areas.rs:8-46:
//   share_i = min(1, area(box_i \ U_{j: !too_far(i, j)} box_j) / (box_i.area() + EPS)).
// The reference takes the difference with geo::BooleanOps (geo = "0.27", Cargo.toml:35; not under /root/reference).  Its
// published algorithm is a general polygon clipper; for convex quadrilaterals the same area is the Green's-theorem
// integral over the boundary of the difference region: box_i's edges where no other box covers them, plus -- reversed --
// the other boxes' edges where they run inside box_i outside every remaining box.  A segment meets a convex box in one
// parameter interval, so each edge needs an interval union only.  Coincident outlines (exact zeros): a segment on an
// edge line of another box is inside it iff both run the same way (between two covering boxes: only the lower index
// covers), and never counts as inside box_i itself.  Pinned by the reference's own test (bbox_own_areas.rs:50-79:
// 75 / 50 / 75) and cross-checked against inclusion-exclusion (tests/test_own_area_cpu.py) and an exact slab / cell
// reference (tests/test_own_area_exact_cpu.py);
// parity with geo's floating-point pipeline beyond that is unpinned (expected agreement ~1e-12 relative).
namespace own {
bool inside_interval(const P2& p, const P2& d, const P2 q[4], double s, bool on_edge_same_dir_inside, double* t0, double* t1) {
  double lo = 0.0, hi = 1.0;
  for (int a = 0; a < 4; ++a) {
    const P2& A = q[a];
    const P2& B = q[(a + 1) % 4];
    const double ex = B.x - A.x, ey = B.y - A.y;
    const double f0 = s * (ex * (p.y - A.y) - ey * (p.x - A.x));
    const double f1 = s * (ex * d.y - ey * d.x);
    if (f1 > 0.0) lo = std::max(lo, -f0 / f1);
    else if (f1 < 0.0) hi = std::min(hi, -f0 / f1);
    else {
      if (f0 < 0.0) return false;
      if (f0 == 0.0 && !(on_edge_same_dir_inside && (ex * d.x + ey * d.y) > 0.0)) return false;
    }
    if (!(lo < hi)) return false;
  }
  *t0 = lo; *t1 = hi;
  return true;
}
// certain separation of two quadrilaterals on their edge directions (same margin as the product's pre-gate)
bool apart(const P2 a[4], const P2 b[4]) {
  double scale = 0.0;
  for (int i = 0; i < 4; ++i) {
    scale = std::max(scale, std::max(std::fabs(a[i].x), std::fabs(a[i].y)));
    scale = std::max(scale, std::max(std::fabs(b[i].x), std::fabs(b[i].y)));
  }
  for (int pass = 0; pass < 2; ++pass) {
    const P2* q = pass == 0 ? a : b;
    for (int e = 0; e < 2; ++e) {
      const double ux = q[e + 1].x - q[e].x, uy = q[e + 1].y - q[e].y;
      double amin = 1e300, amax = -1e300, bmin = 1e300, bmax = -1e300;
      for (int v = 0; v < 4; ++v) {
        const double pa = a[v].x * ux + a[v].y * uy, pb = b[v].x * ux + b[v].y * uy;
        amin = std::min(amin, pa); amax = std::max(amax, pa);
        bmin = std::min(bmin, pb); bmax = std::max(bmax, pb);
      }
      const double tol = 1e-7 * (std::fabs(ux) + std::fabs(uy)) * (scale + 1.0);
      if (bmin - amax > tol || amin - bmax > tol) return true;
    }
  }
  return false;
}
// a box of zero area: its edges come in coincident pairs of opposite direction, which the coincident-edge rules above do
// not cancel on another box's edge line
bool zero_area(const P2 q[4]) {
  double a = 0.0;
  for (int v = 1; v < 3; ++v) {
    const double ux = q[v].x - q[0].x, uy = q[v].y - q[0].y, wx = q[v + 1].x - q[0].x, wy = q[v + 1].y - q[0].y;
    a += ux * wy - uy * wx;
  }
  return a == 0.0;
}
}  // namespace own

std::vector<float> own_area_shares(const std::vector<Box>& boxes) {
  const int n = (int)boxes.size();
  std::vector<float> out(n, 1.0f);
  std::vector<std::array<P2, 4>> quad(n);
  for (int i = 0; i < n; ++i) vertices(boxes[i], quad[i].data());
  for (int i = 0; i < n; ++i) {
    std::vector<const P2*> qs;   // qs[0] = box_i, then the boxes that can cover part of it
    qs.push_back(quad[i].data());
    for (int j = 0; j < n; ++j) {
      if (j == i || too_far(boxes[i], boxes[j])) continue;          // bbox_own_areas.rs:10-15
      if (own::apart(quad[i].data(), quad[j].data())) continue;      // disjoint: the difference removes nothing
      if (own::zero_area(quad[j].data())) continue;                   // aspect or height 0: covers nothing
      qs.push_back(quad[j].data());
    }
    std::vector<P2> ring(quad[i].begin(), quad[i].end());
    double signed_area = 0.0;
    {
      const P2 sh = ring[0];
      for (int a = 0; a < 4; ++a) {
        const P2 u{ring[a].x - sh.x, ring[a].y - sh.y}, v{ring[(a + 1) % 4].x - sh.x, ring[(a + 1) % 4].y - sh.y};
        signed_area += u.x * v.y - u.y * v.x;
      }
    }
    const double s = signed_area < 0.0 ? -1.0 : 1.0;
    const int k = (int)qs.size() - 1;
    double sum = 0.0;
    for (int js = 0; js <= k; ++js) {
      for (int e = 0; e < 4; ++e) {
        const P2 p = qs[js][e];
        const P2 d{qs[js][(e + 1) % 4].x - p.x, qs[js][(e + 1) % 4].y - p.y};
        if (d.x == 0.0 && d.y == 0.0) continue;
        double wa = 0.0, wb = 1.0;
        if (js != 0 && !own::inside_interval(p, d, qs[0], s, false, &wa, &wb)) continue;
        std::vector<std::pair<double, double>> iv;
        for (int l = 1; l <= k; ++l) {
          if (l == js) continue;
          double t0, t1;
          if (!own::inside_interval(p, d, qs[l], s, js == 0 || l < js, &t0, &t1)) continue;
          t0 = std::max(t0, wa); t1 = std::min(t1, wb);
          if (t0 < t1) iv.emplace_back(t0, t1);
        }
        std::stable_sort(iv.begin(), iv.end(), [](const std::pair<double, double>& x, const std::pair<double, double>& y) { return x.first < y.first; });
        double covered = 0.0, ca = 0.0, cb = -1.0;
        for (const auto& t : iv) {
          if (cb < ca) { ca = t.first; cb = t.second; }
          else if (t.first <= cb) cb = std::max(cb, t.second);
          else { covered += cb - ca; ca = t.first; cb = t.second; }
        }
        if (cb >= ca) covered += cb - ca;
        const double term = ((wb - wa) - covered) * (p.x * d.y - p.y * d.x);
        sum += js == 0 ? term : -term;
      }
    }
    double own_area = s * sum / 2.0;
    if (!(own_area > 0.0)) own_area = 0.0;
    const float e = (float)(own_area / (double)(area(boxes[i]) + EPS));   // bbox_own_areas.rs:42-45
    out[i] = e >= 1.0f ? 1.0f : e;
  }
  return out;
}

// ---------------------------------------------------------------- Kalman (nalgebra-order f32 arithmetic)
constexpr int D5 = 5, D10 = 10;
struct KState {
  float mean[D10];
  float cov[D10][D10];
};
struct M1010 { float a[D10][D10]; };

// nalgebra gemm for statically sized matrices: C[i][j] = sum_k A[i][k]*B[k][j], k ascending,
// first term assigned, later terms added (no FMA).
template <int R, int K, int C>
void matmul(const float (*A)[K], const float (*B)[C], float (*out)[C]) {
  for (int j = 0; j < C; ++j)
    for (int i = 0; i < R; ++i) {
      float acc = A[i][0] * B[0][j];
      for (int k = 1; k < K; ++k) acc = A[i][k] * B[k][j] + acc;
      out[i][j] = acc;
    }
}

struct Filter {
  float motion[D10][D10];
  float update_m[D5][D10];
  float pw, vw;
  // Universal2DBoxKalmanFilter::new, src/utils/kalman/kalman_2d_box.rs:31-44
  Filter(float position_weight, float velocity_weight) : pw(position_weight), vw(velocity_weight) {
    std::memset(motion, 0, sizeof(motion));
    std::memset(update_m, 0, sizeof(update_m));
    for (int i = 0; i < D10; ++i) motion[i][i] = 1.0f;
    for (int i = 0; i < D5; ++i) motion[i][D5 + i] = 1.0f;  // DT as f32
    for (int i = 0; i < D5; ++i) update_m[i][i] = 1.0f;
  }
  // std_position / std_velocity, :46-54
  void std_position(float k, float cnst, float p, float out[D5]) const {
    float w = k * pw * p;
    out[0] = w; out[1] = w; out[2] = w; out[3] = cnst; out[4] = w;
  }
  void std_velocity(float k, float cnst, float p, float out[D5]) const {
    float w = k * vw * p;
    out[0] = w; out[1] = w; out[2] = w; out[3] = cnst; out[4] = w;
  }
  // initiate, :58-84
  KState initiate(const Box& b) const {
    KState s;
    std::memset(&s, 0, sizeof(s));
    s.mean[0] = b.xc; s.mean[1] = b.yc; s.mean[2] = angle_or0(b); s.mean[3] = b.aspect; s.mean[4] = b.height;
    float sp[D5], sv[D5];
    std_position(2.0f, 1e-2f, b.height, sp);
    std_velocity(10.0f, 1e-5f, b.height, sv);
    for (int i = 0; i < D5; ++i) {
      s.cov[i][i] = sp[i] * sp[i];
      s.cov[D5 + i][D5 + i] = sv[i] * sv[i];
    }
    return s;
  }
  // predict, :86-102
  KState predict(const KState& st) const {
    float sp[D5], sv[D5];
    std_position(1.0f, 1e-2f, st.mean[4], sp);
    std_velocity(1.0f, 1e-5f, st.mean[4], sv);
    float stdv[D10];
    for (int i = 0; i < D5; ++i) { stdv[i] = sp[i] * sp[i]; stdv[D5 + i] = sv[i] * sv[i]; }
    KState out;
    // mean = motion_matrix * mean
    for (int i = 0; i < D10; ++i) {
      float acc = motion[i][0] * st.mean[0];
      for (int k = 1; k < D10; ++k) acc = motion[i][k] * st.mean[k] + acc;
      out.mean[i] = acc;
    }
    // covariance = motion * cov * motion^T + motion_cov
    float t1[D10][D10], mt[D10][D10], t2[D10][D10];
    matmul<D10, D10, D10>(motion, st.cov, t1);
    for (int i = 0; i < D10; ++i) for (int j = 0; j < D10; ++j) mt[i][j] = motion[j][i];
    matmul<D10, D10, D10>(t1, mt, t2);
    for (int i = 0; i < D10; ++i)
      for (int j = 0; j < D10; ++j) out.cov[i][j] = t2[i][j] + (i == j ? stdv[i] : 0.0f);
    return out;
  }
  // project, :104-120
  void project(const float mean[D10], const float cov[D10][D10], float pmean[D5], float pcov[D5][D5]) const {
    float sp[D5];
    std_position(1.0f, 1e-1f, mean[4], sp);
    float stdv[D5];
    for (int i = 0; i < D5; ++i) stdv[i] = sp[i] * sp[i];
    for (int i = 0; i < D5; ++i) {
      float acc = update_m[i][0] * mean[0];
      for (int k = 1; k < D10; ++k) acc = update_m[i][k] * mean[k] + acc;
      pmean[i] = acc;
    }
    float t1[D5][D10], ut[D10][D5], t2[D5][D5];
    matmul<D5, D10, D10>(update_m, cov, t1);
    for (int i = 0; i < D10; ++i) for (int j = 0; j < D5; ++j) ut[i][j] = update_m[j][i];
    matmul<D5, D10, D5>(t1, ut, t2);
    for (int i = 0; i < D5; ++i)
      for (int j = 0; j < D5; ++j) pcov[i][j] = t2[i][j] + (i == j ? stdv[i] : 0.0f);
  }
  // nalgebra solve_lower_triangular (forward substitution on the LOWER triangle of `m`, whatever
  // is stored above the diagonal is ignored), applied column by column to b (5 x C) in place.
  template <int C>
  static void solve_lower_triangular(const float m[D5][D5], float b[D5][C]) {
    for (int col = 0; col < C; ++col) {
      for (int i = 0; i < D5; ++i) {
        float diag = m[i][i];
        float coeff = b[i][col] / diag;
        b[i][col] = coeff;
        for (int r = i + 1; r < D5; ++r) b[r][col] = (-coeff) * m[r][i] + b[r][col];
      }
    }
  }
  // update, :124-148
  KState update(const KState& st, const Box& meas) const {
    float pmean[D5], pcov[D5][D5];
    project(st.mean, st.cov, pmean, pcov);
    // b = (covariance * update_matrix^T)^T   (5 x 10)
    float ut[D10][D5], cu[D10][D5], b[D5][D10];
    for (int i = 0; i < D10; ++i) for (int j = 0; j < D5; ++j) ut[i][j] = update_m[j][i];
    matmul<D10, D10, D5>(st.cov, ut, cu);
    for (int i = 0; i < D5; ++i) for (int j = 0; j < D10; ++j) b[i][j] = cu[j][i];
    // kalman_gain = projected_cov.solve_lower_triangular(&b)
    solve_lower_triangular<D10>(pcov, b);  // b now holds kalman_gain (5 x 10)
    float innov[D5] = {meas.xc - pmean[0], meas.yc - pmean[1], angle_or0(meas) - pmean[2],
                       meas.aspect - pmean[3], meas.height - pmean[4]};
    KState out;
    // mean = mean + (innovation(1x5) * kalman_gain(5x10))^T
    for (int j = 0; j < D10; ++j) {
      float acc = innov[0] * b[0][j];
      for (int k = 1; k < D5; ++k) acc = innov[k] * b[k][j] + acc;
      out.mean[j] = st.mean[j] + acc;
    }
    // covariance = covariance - kalman_gain^T * projected_cov * kalman_gain
    float kt[D10][D5], t1[D10][D5], t2[D10][D10];
    for (int i = 0; i < D10; ++i) for (int j = 0; j < D5; ++j) kt[i][j] = b[j][i];
    matmul<D10, D5, D5>(kt, pcov, t1);
    matmul<D10, D5, D10>(t1, b, t2);
    for (int i = 0; i < D10; ++i) for (int j = 0; j < D10; ++j) out.cov[i][j] = st.cov[i][j] - t2[i][j];
    return out;
  }
  // distance, :150-170  (nalgebra Cholesky::new + l() + solve_lower_triangular + component_mul + sum)
  float distance(const KState& st, const Box& meas) const {
    float pmean[D5], pcov[D5][D5];
    project(st.mean, st.cov, pmean, pcov);
    float r[D5][1] = {{meas.xc - pmean[0]}, {meas.yc - pmean[1]}, {angle_or0(meas) - pmean[2]},
                      {meas.aspect - pmean[3]}, {meas.height - pmean[4]}};
    float m[D5][D5];
    std::memcpy(m, pcov, sizeof(m));
    for (int j = 0; j < D5; ++j) {
      for (int k = 0; k < j; ++k) {
        float factor = -m[j][k];
        for (int row = j; row < D5; ++row) m[row][j] = factor * m[row][k] + m[row][j];
      }
      float diag = m[j][j];
      float denom = std::sqrt(diag);  // reference unwraps: a non-SPD matrix panics there
      m[j][j] = denom;
      for (int row = j + 1; row < D5; ++row) m[row][j] = m[row][j] / denom;
    }
    solve_lower_triangular<1>(m, r);
    float sum = 0.0f;
    for (int i = 0; i < D5; ++i) sum = sum + r[i][0] * r[i][0];
    return sum;
  }
};
// calculate_cost, :172-184
float calculate_cost(float distance, bool inverted) {
  if (!inverted) return distance > CHI2INV95_4 ? CHI2_UPPER_BOUND : distance;
  return distance > CHI2INV95_4 ? 0.0f : CHI2_UPPER_BOUND - distance;
}
// TryFrom<KalmanState> for Universal2DBox, src/utils/kalman.rs:72-92 (confidence 1.0 by ::new)
Box state_box(const KState& s) {
  Box b;
  b.xc = s.mean[0]; b.yc = s.mean[1];
  b.angle = (s.mean[2] == 0.0f) ? std::numeric_limits<float>::quiet_NaN() : s.mean[2];
  b.aspect = s.mean[3]; b.height = s.mean[4]; b.conf = 1.0f;
  return b;
}
// TrackAttributesKalmanPrediction::make_prediction, src/trackers/kalman_prediction.rs:13-32
Box make_prediction(bool has_state, KState& state, float pw, float vw, const Box& observation) {
  Filter f(pw, vw);
  KState current = has_state ? state : f.initiate(observation);
  KState prediction = f.predict(current);
  KState ns = f.update(prediction, observation);
  state = ns;
  Box res = state_box(ns);
  res.conf = observation.conf;
  return res;
}

// ---------------------------------------------------------------- features
// Feature::from_vec zero-pads to a multiple of 8 lanes, src/track/utils.rs:45-71
std::vector<float> pad8(const float* v, int d) {
  int blocks = d / 8 + (d % 8 > 0 ? 1 : 0);
  std::vector<float> out((size_t)blocks * 8, 0.0f);
  std::memcpy(out.data(), v, sizeof(float) * (size_t)d);
  return out;
}
// wide::f32x8::reduce_add (AVX path): lo+hi quads, then dual, then single.
inline float reduce_add8(const float l[8]) {
  float q0 = l[0] + l[4], q1 = l[1] + l[5], q2 = l[2] + l[6], q3 = l[3] + l[7];
  float d0 = q0 + q2, d1 = q1 + q3;
  return d0 + d1;
}
// The reference computes these with 8-lane SIMD vectors (ultraviolet / wide f32x8, src/distance.rs:9-47).  The scalar
// loops below restate the arithmetic lane by lane; on x86-64 hosts with AVX2 the same operations are issued as 8-lane
// vector instructions (sub / mul per lane, the reduce_add tree lo+hi -> pairs -> single, blocks accumulated one after the
// other), which is bit-identical (every operation is the same IEEE f32 operation on the same operands; no FMA) and lets
// the timed CPU baseline run at the speed a SIMD build of the reference would.  ORACLE_NO_SIMD=1 forces the scalar loops;
// tests/test_oracle_simd.py checks both paths bit for bit.
float euclidean_scalar(const float* a, const float* b, int blocks) {
  float acc = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    float blk[8];
    for (int l = 0; l < 8; ++l) {
      float t = a[i * 8 + l] - b[i * 8 + l];
      blk[l] = t * t;
    }
    acc += reduce_add8(blk);
  }
  return std::sqrt(acc);
}
float cosine_scalar(const float* a, const float* b, int blocks) {
  float divided = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    float blk[8];
    for (int l = 0; l < 8; ++l) blk[l] = a[i * 8 + l] * b[i * 8 + l];
    divided += reduce_add8(blk);
  }
  float f1 = 0.0f, f2 = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    float blk[8];
    for (int l = 0; l < 8; ++l) blk[l] = a[i * 8 + l] * a[i * 8 + l];
    f1 = f1 + reduce_add8(blk);
  }
  for (int i = 0; i < blocks; ++i) {
    float blk[8];
    for (int l = 0; l < 8; ++l) blk[l] = b[i * 8 + l] * b[i * 8 + l];
    f2 = f2 + reduce_add8(blk);
  }
  return divided / std::sqrt(f1 * f2);
}

#if defined(__x86_64__) && defined(__GNUC__)
#define ORC_HAVE_AVX2_PATH 1
}  // namespace (intrinsics header must be included at file scope)
#include <immintrin.h>
namespace {
// wide::f32x8::reduce_add on a vector register: (lo + hi) -> q0..q3; (q0 + q2, q1 + q3); d0 + d1
__attribute__((target("avx2"))) inline float reduce_add8_v(__m256 t) {
  const __m128 q = _mm_add_ps(_mm256_castps256_ps128(t), _mm256_extractf128_ps(t, 1));
  const __m128 d = _mm_add_ps(q, _mm_movehl_ps(q, q));
  return _mm_cvtss_f32(_mm_add_ss(d, _mm_shuffle_ps(d, d, 0x55)));
}
__attribute__((target("avx2"))) float euclidean_avx2(const float* a, const float* b, int blocks) {
  float acc = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    const __m256 t = _mm256_sub_ps(_mm256_loadu_ps(a + i * 8), _mm256_loadu_ps(b + i * 8));
    acc += reduce_add8_v(_mm256_mul_ps(t, t));
  }
  return std::sqrt(acc);
}
__attribute__((target("avx2"))) float cosine_avx2(const float* a, const float* b, int blocks) {
  float divided = 0.0f, f1 = 0.0f, f2 = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    const __m256 va = _mm256_loadu_ps(a + i * 8), vb = _mm256_loadu_ps(b + i * 8);
    divided += reduce_add8_v(_mm256_mul_ps(va, vb));
    f1 = f1 + reduce_add8_v(_mm256_mul_ps(va, va));
    f2 = f2 + reduce_add8_v(_mm256_mul_ps(vb, vb));
  }
  return divided / std::sqrt(f1 * f2);
}
inline bool use_avx2() {
  static const bool ok = __builtin_cpu_supports("avx2") && std::getenv("ORACLE_NO_SIMD") == nullptr;
  return ok;
}
#else
inline bool use_avx2() { return false; }
#endif

// squared norm of one padded feature, the f1 / f2 accumulation of cosine (src/distance.rs:36-44): per-block reduce_add
// of the lane squares, blocks added in order (the same operations on both paths)
float norm2_p(const float* a, int blocks) {
  float acc = 0.0f;
  for (int i = 0; i < blocks; ++i) {
    float blk[8];
    for (int l = 0; l < 8; ++l) blk[l] = a[i * 8 + l] * a[i * 8 + l];
    acc = acc + reduce_add8(blk);
  }
  return acc;
}

// euclidean, src/distance.rs:9-19
float euclidean_p(const float* a, const float* b, int blocks) {
#ifdef ORC_HAVE_AVX2_PATH
  if (use_avx2()) return euclidean_avx2(a, b, blocks);
#endif
  return euclidean_scalar(a, b, blocks);
}
// cosine, src/distance.rs:26-47
float cosine_p(const float* a, const float* b, int blocks) {
#ifdef ORC_HAVE_AVX2_PATH
  if (use_avx2()) return cosine_avx2(a, b, blocks);
#endif
  return cosine_scalar(a, b, blocks);
}

// ---------------------------------------------------------------- voting
struct Ent {
  uint64_t from, to;
  float attr;  // NaN none
  float feat;  // NaN none
};

// Rust `f32 as i64`: saturating, NaN -> 0
inline int64_t f32_as_i64(float v) {
  if (std::isnan(v)) return 0;
  if (v >= 9223372036854775807.0f) return INT64_MAX;
  if (v <= -9223372036854775808.0f) return INT64_MIN;
  return (int64_t)v;
}

// pathfinding 4.x kuhn_munkres (maximum weight perfect matching on rows <= cols), restated.
int64_t kuhn_munkres(const int64_t* w, int nx, int ny, std::vector<int>& xy_out) {
  auto at = [&](int r, int c) { return w[(size_t)r * ny + c]; };
  std::vector<int> xy(nx, -1), yx(ny, -1);
  std::vector<int64_t> lx(nx), ly(ny, 0);
  for (int row = 0; row < nx; ++row) {
    int64_t mx = at(row, 0);
    for (int col = 1; col < ny; ++col) mx = std::max(mx, at(row, col));
    lx[row] = mx;
  }
  std::vector<char> s(nx, 0);
  std::vector<int> alternating(ny, -1);
  std::vector<int64_t> slack(ny, 0);
  std::vector<int> slackx(ny, 0);
  for (int root = 0; root < nx; ++root) {
    std::fill(alternating.begin(), alternating.end(), -1);
    std::fill(s.begin(), s.end(), 0);
    s[root] = 1;
    for (int y = 0; y < ny; ++y) slack[y] = lx[root] + ly[y] - at(root, y);
    std::fill(slackx.begin(), slackx.end(), root);
    int y_end;
    for (;;) {
      int64_t delta = INT64_MAX;
      int x = 0, y = 0;
      for (int yy = 0; yy < ny; ++yy) {
        if (alternating[yy] < 0 && slack[yy] < delta) {
          delta = slack[yy];
          x = slackx[yy];
          y = yy;
        }
      }
      if (delta > 0) {
        for (int xx = 0; xx < nx; ++xx)
          if (s[xx]) lx[xx] -= delta;
        for (int yy = 0; yy < ny; ++yy) {
          if (alternating[yy] >= 0) ly[yy] += delta;
          else slack[yy] -= delta;
        }
      }
      alternating[y] = x;
      if (yx[y] < 0) { y_end = y; break; }
      int x2 = yx[y];
      s[x2] = 1;
      for (int yy = 0; yy < ny; ++yy) {
        if (alternating[yy] < 0) {
          int64_t alt = lx[x2] + ly[yy] - at(x2, yy);
          if (slack[yy] > alt) { slack[yy] = alt; slackx[yy] = x2; }
        }
      }
    }
    int y = y_end;
    while (y >= 0) {
      int x = alternating[y];
      int prec = xy[x];
      yx[y] = x;
      xy[x] = y;
      y = prec;
    }
  }
  int64_t total = 0;
  for (auto v : lx) total += v;
  for (auto v : ly) total += v;
  xy_out = xy;
  return total;
}

// SortVoting::winners, src/trackers/sort/voting.rs:30-100. Output: (from, to) pairs in row order.
std::vector<std::pair<uint64_t, uint64_t>> sort_voting(float threshold_f, size_t candidate_num, size_t track_num,
                                                        const std::vector<Ent>& distances) {
  std::vector<std::pair<uint64_t, uint64_t>> out;
  const int64_t threshold = f32_as_i64(threshold_f * F32_U64_MULT);
  if (track_num == 0) return out;
  size_t candidates_index = 0;
  std::vector<uint64_t> tracks_index(candidate_num, 0);
  std::unordered_map<uint64_t, size_t> tracks_r_index;
  const size_t cols = candidate_num + track_num;
  std::vector<int64_t> cost((size_t)candidate_num * cols, 0);
  for (const Ent& e : distances) {
    int64_t weight = f32_as_i64((std::isnan(e.attr) ? 0.0f : e.attr) * F32_U64_MULT);
    size_t row, col;
    auto it = tracks_r_index.find(e.from);
    if (it != tracks_r_index.end()) row = it->second;
    else {
      row = candidates_index++;
      tracks_index[row] = e.from;
      tracks_r_index[e.from] = row;
    }
    it = tracks_r_index.find(e.to);
    if (it != tracks_r_index.end()) col = it->second;
    else {
      col = tracks_index.size();
      tracks_index.push_back(e.to);
      tracks_r_index[e.to] = col;
    }
    cost[row * cols + col] = weight;
  }
  for (size_t i = 0; i < candidate_num; ++i) cost[i * cols + i] = threshold;
  std::vector<int> sol;
  kuhn_munkres(cost.data(), (int)candidate_num, (int)cols, sol);
  for (size_t i = 0; i < sol.size(); ++i) {
    size_t e = (size_t)sol[i];
    uint64_t from = tracks_index[i];
    uint64_t to = e < tracks_index.size() ? tracks_index[e] : 0;  // reference would panic (cannot occur, thr > 0)
    if (from > 0 && to > 0) out.emplace_back(from, to);
  }
  return out;
}

struct TopNElt { uint64_t query_track, winner_track; double weight; };

// BestFitVoting::winners, src/track/voting/best.rs:52-128.
// Returns per query (first-appearance order) its elements in sorted order.
std::vector<std::pair<uint64_t, std::vector<TopNElt>>> bestfit_voting(float max_distance, size_t min_votes,
                                                                       const std::vector<Ent>& distances) {
  float max_dist = -1.0f;
  // into_group_map: HashMap<(from,to), Vec<f32>>; iteration order is arbitrary in the reference,
  // here: first-appearance order (documented tie rule).
  std::vector<std::pair<std::pair<uint64_t, uint64_t>, std::vector<float>>> groups;
  std::map<std::pair<uint64_t, uint64_t>, size_t> gidx;
  for (const Ent& e : distances) {
    if (std::isnan(e.feat)) continue;
    if (max_dist < e.feat) max_dist = e.feat;
    if (!(e.feat <= max_distance)) continue;
    auto key = std::make_pair(e.from, e.to);
    auto it = gidx.find(key);
    if (it == gidx.end()) {
      gidx[key] = groups.size();
      groups.push_back({key, {e.feat}});
    } else groups[it->second].second.push_back(e.feat);
  }
  std::vector<TopNElt> cands;
  for (auto& g : groups) {
    if (g.second.size() < min_votes) continue;
    double weight = 0.0;
    for (float d : g.second) weight += (double)(max_dist - d);
    cands.push_back({g.first.first, g.first.second, weight});
  }
  std::stable_sort(cands.begin(), cands.end(), [](const TopNElt& a, const TopNElt& b) { return a.weight > b.weight; });
  std::unordered_set<uint64_t> results;
  for (auto& c : cands) {
    if (results.count(c.winner_track)) c.winner_track = c.query_track;
    else results.insert(c.winner_track);
  }
  std::vector<std::pair<uint64_t, std::vector<TopNElt>>> res;
  std::unordered_map<uint64_t, size_t> qidx;
  for (auto& c : cands) {
    auto it = qidx.find(c.query_track);
    if (it == qidx.end()) {
      qidx[c.query_track] = res.size();
      res.push_back({c.query_track, {c}});
    } else res[it->second].second.push_back(c);
  }
  return res;
}

struct Winner { uint64_t from, to; int type; };

// VisualVoting::winners, src/trackers/visual_sort/voting.rs:45-100
std::vector<Winner> visual_voting(float positional_threshold, float max_allowed_feature_distance, size_t min_votes,
                                  const std::vector<Ent>& distances) {
  auto fw = bestfit_voting(max_allowed_feature_distance, min_votes, distances);
  std::unordered_set<uint64_t> excluded_tracks;
  std::unordered_set<uint64_t> feature_winner_keys;
  std::vector<Winner> out;
  for (auto& q : fw) {
    uint64_t winner_track = q.second[0].winner_track;
    excluded_tracks.insert(winner_track);
    feature_winner_keys.insert(q.first);
    out.push_back({q.first, winner_track, ORC_VOTING_VISUAL});
  }
  std::unordered_set<uint64_t> remaining_candidates, remaining_tracks;
  std::vector<Ent> remaining;
  for (const Ent& e : distances) {
    if (!(feature_winner_keys.count(e.from) || excluded_tracks.count(e.to)) && !std::isnan(e.attr)) {
      remaining_candidates.insert(e.from);
      remaining_tracks.insert(e.to);
      remaining.push_back(e);
    }
  }
  auto pw = sort_voting(positional_threshold, remaining_candidates.size(), remaining_tracks.size(), remaining);
  for (auto& p : pw) out.push_back({p.first, p.second, ORC_VOTING_POSITIONAL});
  return out;
}

// ---------------------------------------------------------------- metrics
struct Opts {
  orc_options o;
  std::vector<std::pair<size_t, float>> constraints;  // sorted + dedup, spatio_temporal_constraints.rs:36-46
  explicit Opts(const orc_options& in) : o(in) {
    for (int i = 0; i < in.n_constraints && i < ORC_MAX_CONSTRAINTS; ++i)
      constraints.emplace_back((size_t)in.constraint_epochs[i], in.constraint_max_dist[i]);
    std::stable_sort(constraints.begin(), constraints.end(),
                     [](const std::pair<size_t, float>& a, const std::pair<size_t, float>& b) { return a.first < b.first; });
    constraints.erase(std::unique(constraints.begin(), constraints.end(),
                                  [](const std::pair<size_t, float>& a, const std::pair<size_t, float>& b) { return a.first == b.first; }),
                      constraints.end());
  }
  // SpatioTemporalConstraints::validate, spatio_temporal_constraints.rs:48-59
  bool validate(size_t epoch_delta, float dist) const {
    for (auto& c : constraints)
      if (c.first >= epoch_delta) return dist <= c.second;
    return true;
  }
  bool is_visual() const { return o.kind == ORC_KIND_VISUAL_SORT || o.kind == ORC_KIND_BATCH_VISUAL_SORT; }
  bool is_batch() const { return o.kind == ORC_KIND_BATCH_SORT || o.kind == ORC_KIND_BATCH_VISUAL_SORT; }
};

// positional part shared by SortMetric::metric (sort/metric.rs:38-77) and
// VisualMetric::positional_metric (visual_sort/metric.rs:156-198). NaN == None.
float positional_metric(int positional_kind, float iou_threshold, float min_confidence, float pw, float vw,
                        const Box& cand, const Box& track_box, const KState* track_state) {
  const float nan = std::numeric_limits<float>::quiet_NaN();
  float conf = cand.conf < min_confidence ? min_confidence : cand.conf;
  if (too_far(cand, track_box)) return nan;
  if (positional_kind == ORC_POS_MAHA) {
    Filter f(pw, vw);
    float dist = f.distance(*track_state, cand);
    return calculate_cost(dist, true) / conf;
  }
  float v;
  if (!iou(cand, track_box, &v)) return nan;
  v = v * conf;
  return v >= iou_threshold ? v : nan;
}

// ---------------------------------------------------------------- tracker
struct Obs {
  bool has_box = false;
  Box box{};
  float quality = 1.0f;
  bool has_own = false;
  float own = 0.0f;
  bool has_feat = false;
  std::vector<float> feat;  // padded x8
};
struct Track {
  uint64_t id = 0, scene = 0;
  int64_t custom = NONE_ID;
  size_t epoch = 0, length = 0;
  int voting_type = -1;  // None
  bool has_state = false;
  KState st{};
  Box last_pred{}, last_obs{};
  std::vector<Obs> obs;
  size_t feat_count = 0;
};

void parallel_for(int n, int threads, const std::function<void(int, int)>& fn) {
  if (threads <= 1 || n <= 1) { fn(0, n); return; }
  threads = std::min(threads, n);
  std::vector<std::thread> th;
  int chunk = (n + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    int b = t * chunk, e = std::min(n, b + chunk);
    if (b >= e) break;
    th.emplace_back(fn, b, e);
  }
  for (auto& x : th) x.join();
}

}  // namespace

struct orc_tracker {
  Opts opts;
  int threads = 1;
  std::map<uint64_t, size_t> epoch_db;              // epoch_db.rs
  std::map<uint64_t, std::vector<Track>> store;     // per-scene dense store (store order == insertion order)
  std::vector<Track> wasted;
  uint64_t track_id = 0;
  int auto_waste_counter = DEFAULT_AUTO_WASTE_PERIODICITY;
  int auto_waste_periodicity = DEFAULT_AUTO_WASTE_PERIODICITY;
  std::map<uint64_t, std::vector<float>> last_costs;
  std::map<uint64_t, std::pair<int, int>> last_shape;
  explicit orc_tracker(const orc_options& o) : opts(o) {}

  size_t current_epoch(uint64_t scene) const {
    auto it = epoch_db.find(scene);
    return it == epoch_db.end() ? 0 : it->second;
  }
  // EpochDb::baked, epoch_db.rs:51-66 ; TrackerAPI::auto_waste, tracker_api.rs:70-88
  void auto_waste() {
    for (auto& kv : store) {
      size_t cur = current_epoch(kv.first);
      std::vector<Track> keep;
      for (auto& t : kv.second) {
        if (t.epoch + (size_t)opts.o.max_idle_epochs < cur) wasted.push_back(std::move(t));
        else keep.push_back(std::move(t));
      }
      kv.second.swap(keep);
    }
  }

  // VisualMetric::feature_can_be_used, visual_sort/metric.rs:227-249
  bool feature_can_be_used(const Box& bbox, float q, float min_q, bool has_own, float own, float min_own) const {
    bool quality_is_ok = q >= min_q;
    bool percentage_is_ok = has_own ? own >= min_own : true;
    bool bbox_is_ok = area(bbox) >= opts.o.visual_minimal_area;
    return bbox_is_ok && quality_is_ok && percentage_is_ok;
  }

  // Builds the candidate track for one detection: SortMetric::optimize / VisualMetric::optimize with
  // is_merge == false on a fresh track (sort/metric.rs:79-105, visual_sort/metric.rs:297-374).
  Track make_candidate(uint64_t scene, size_t epoch, const Box& det, int64_t custom, const float* feat,
                       bool has_feat, float quality, bool has_own, float own) const {
    Track t;
    t.scene = scene; t.epoch = epoch; t.custom = custom;
    t.has_state = false;
    Box pred = make_prediction(false, t.st, opts.o.kalman_position_weight, opts.o.kalman_velocity_weight, det);
    t.has_state = true;
    t.length = 1;
    t.last_obs = det;
    t.last_pred = pred;
    Obs o;
    o.has_box = true; o.box = pred; o.quality = quality; o.has_own = has_own; o.own = own;
    if (opts.is_visual() && has_feat) {
      o.has_feat = true;
      o.feat = pad8(feat, opts.o.feature_dim);
    }
    t.obs.push_back(std::move(o));
    t.feat_count = t.obs[0].has_feat ? 1 : 0;
    return t;
  }

  // SortAttributes::compatible / VisualAttributes::compatible, sort.rs:250-270
  bool compatible(const Track& c, const Track& t) const {
    if (c.scene != t.scene) return false;
    size_t d = c.epoch > t.epoch ? c.epoch - t.epoch : t.epoch - c.epoch;
    float center_dist = dist_in_2r(c.last_pred, t.last_pred);
    return (size_t)opts.o.max_idle_epochs >= d && opts.validate(d, center_dist);
  }

  // Track::merge + metric.optimize(is_merge = true), track.rs:522-588
  void merge(Track& dst, const Track& cand) {
    dst.epoch = cand.epoch;
    dst.custom = cand.custom;
    const Obs& co = cand.obs[0];
    const Box& observation_bbox = co.box;
    Box pred = make_prediction(dst.has_state, dst.st, opts.o.kalman_position_weight, opts.o.kalman_velocity_weight,
                               observation_bbox);
    dst.has_state = true;
    dst.length += 1;
    dst.last_obs = observation_bbox;
    dst.last_pred = pred;
    if (!opts.is_visual()) {
      dst.obs.clear();
      Obs o; o.has_box = true; o.box = pred;
      dst.obs.push_back(o);
      return;
    }
    dst.voting_type = cand.voting_type;
    Obs o = co;
    if (!feature_can_be_used(observation_bbox, co.quality, opts.o.visual_minimal_quality_collect, co.has_own, co.own,
                             opts.o.visual_minimal_own_area_percentage_collect)) {
      o.has_feat = false;
      o.feat.clear();
    }
    o.has_box = true;
    o.box = pred;
    // optimize_observations, visual_sort/metric.rs:129-154
    std::vector<Obs>& obs = dst.obs;
    obs.erase(std::remove_if(obs.begin(), obs.end(), [](const Obs& x) { return !x.has_feat; }), obs.end());
    for (auto& x : obs) x.has_box = false;
    std::stable_sort(obs.begin(), obs.end(), [](const Obs& a, const Obs& b) { return a.quality > b.quality; });
    if (obs.size() >= (size_t)opts.o.visual_max_observations && !obs.empty()) obs.pop_back();
    obs.push_back(std::move(o));
    std::swap(obs[0], obs[obs.size() - 1]);
    size_t cnt = 0;
    for (auto& x : obs) cnt += x.has_feat ? 1 : 0;
    dst.feat_count = cnt;
  }

  void emit(const Track& t, size_t idx, uint64_t* out_ids, uint32_t* out_epochs, uint32_t* out_lengths,
            uint8_t* out_vt, float* out_pred, float* out_obs) const {
    if (out_ids) out_ids[idx] = t.id;
    if (out_epochs) out_epochs[idx] = (uint32_t)t.epoch;
    if (out_lengths) out_lengths[idx] = (uint32_t)t.length;
    // SortTrack::from: Sort => Positional; VisualSort => voting_type.unwrap_or(Positional)
    if (out_vt) out_vt[idx] = (uint8_t)(t.voting_type < 0 ? ORC_VOTING_POSITIONAL : t.voting_type);
    if (out_pred) store_box(t.last_pred, out_pred + idx * 6);
    if (out_obs) store_box(t.last_obs, out_obs + idx * 6);
  }

  struct SceneWork {
    uint64_t scene = 0;
    int m = 0;
    size_t base = 0;
    std::vector<Track> cands;
    std::unordered_map<uint64_t, std::pair<uint64_t, int>> winners;
    std::vector<float> pos;
    int n = 0;
  };

  // distance pass + voting of one scene (read-only on the scene's store: scenes can run on separate threads,
  // like the reference's distance shards + voting threads)
  void scene_vote(SceneWork& w, size_t epoch, const float* boxes, const float* features, const uint8_t* has_feature,
                  const float* quality, const int64_t* custom_ids, const float* own_area, int inner_threads) {
    const uint64_t scene = w.scene;
    const int m = w.m;
    const size_t base = w.base;
    const int threads = inner_threads;
    const orc_options& o = opts.o;
    std::vector<Track>& tracks = store.find(scene)->second;
    const int n = (int)tracks.size();
    const bool visual = opts.is_visual();
    std::vector<Track>& cands = w.cands;
    cands.reserve(m);
    const bool use_own = visual && (o.visual_minimal_own_area_percentage_collect + o.visual_minimal_own_area_percentage_use > 0.0f);
    // visual_sort/simple_api.rs:110-127: the shares are computed from the scene's observation boxes unless the caller
    // supplied them
    std::vector<float> own_local;
    if (use_own && own_area == nullptr) {
      std::vector<Box> obs_boxes(m);
      for (int i = 0; i < m; ++i) obs_boxes[i] = load_box(boxes + (base + i) * 6);
      own_local = own_area_shares(obs_boxes);
    }
    for (int i = 0; i < m; ++i) {
      Box det = load_box(boxes + (base + i) * 6);
      bool hf = visual && features != nullptr && (has_feature == nullptr || has_feature[base + i]);
      float q = quality ? quality[base + i] : 1.0f;
      bool ho = use_own;
      Track c = make_candidate(scene, epoch, det, custom_ids ? custom_ids[base + i] : NONE_ID,
                               features ? features + (base + i) * (size_t)o.feature_dim : nullptr, hf, q, ho,
                               ho ? (own_area != nullptr ? own_area[base + i] : own_local[i]) : 0.0f);
      c.id = UINT64_MAX - (uint64_t)i;  // stand-in for rng.gen(): unique, never collides with real ids
      cands.push_back(std::move(c));
    }
    // ---- distance pass: TrackStore::foreign_track_distances -> Track::distances (track.rs:604-652)
    const int kmax = visual ? std::max(1, o.visual_max_observations) : 1;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    std::vector<float> pos((size_t)m * n, nan);
    std::vector<float> vis(visual ? (size_t)m * n * kmax : 0, nan);
    std::vector<uint8_t> pair_ok((size_t)m * n, 0);
    const int blocks = (o.feature_dim + 7) / 8;
    parallel_for(m, threads, [&](int b, int e) {
      for (int i = b; i < e; ++i) {
        const Track& c = cands[i];
        const Obs& co = c.obs[0];
        for (int j = 0; j < n; ++j) {
          const Track& t = tracks[j];
          if (!compatible(c, t)) continue;
          pair_ok[(size_t)i * n + j] = 1;
          if (!visual) {
            pos[(size_t)i * n + j] = positional_metric(o.positional_kind, o.iou_threshold, o.min_confidence,
                                                       o.kalman_position_weight, o.kalman_velocity_weight, co.box,
                                                       t.obs[0].box, &t.st);
            continue;
          }
          bool can_use = feature_can_be_used(co.box, co.quality, o.visual_minimal_quality_use, co.has_own, co.own,
                                             o.visual_minimal_own_area_percentage_use);
          for (size_t k = 0; k < t.obs.size() && (int)k < kmax; ++k) {
            const Obs& to = t.obs[k];
            if (to.has_box && k == 0)
              pos[(size_t)i * n + j] = positional_metric(o.positional_kind, o.iou_threshold, o.min_confidence,
                                                         o.kalman_position_weight, o.kalman_velocity_weight, co.box,
                                                         to.box, &t.st);
            if (can_use && co.has_feat && to.has_feat && t.feat_count >= (size_t)o.visual_minimal_track_length) {
              float d = o.visual_kind == ORC_VIS_EUCLIDEAN ? euclidean_p(co.feat.data(), to.feat.data(), blocks)
                                                           : cosine_p(co.feat.data(), to.feat.data(), blocks);
              bool ok = o.visual_kind == ORC_VIS_EUCLIDEAN ? d <= o.visual_threshold : d >= o.visual_threshold;
              if (ok) vis[((size_t)i * n + j) * kmax + k] = o.visual_kind == ORC_VIS_EUCLIDEAN ? d : 1.0f - d;
            }
          }
        }
      }
    });
    w.pos = pos;
    w.n = n;
    // ---- COO stream in (candidate, track, observation) order; postprocess_distances filters
    std::vector<Ent> ents;
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < n; ++j) {
        if (!pair_ok[(size_t)i * n + j]) continue;
        if (!visual) {
          float a = pos[(size_t)i * n + j];
          if (!std::isnan(a)) ents.push_back({cands[i].id, tracks[j].id, a, nan});
        } else {
          for (size_t k = 0; k < tracks[j].obs.size() && (int)k < kmax; ++k) {
            float a = k == 0 ? pos[(size_t)i * n + j] : nan;
            float f = vis[((size_t)i * n + j) * kmax + k];
            if (!std::isnan(a) || !std::isnan(f)) ents.push_back({cands[i].id, tracks[j].id, a, f});
          }
        }
      }
    // ---- voting
    float thr = o.positional_kind == ORC_POS_MAHA ? MAHALANOBIS_NEW_TRACK_THRESHOLD : o.iou_threshold;
    std::unordered_map<uint64_t, std::pair<uint64_t, int>>& winners = w.winners;
    if (!visual) {
      for (auto& p : sort_voting(thr, (size_t)m, (size_t)n, ents)) winners[p.first] = {p.second, ORC_VOTING_POSITIONAL};
    } else {
      for (auto& w : visual_voting(thr, std::numeric_limits<float>::max(), (size_t)o.visual_min_votes, ents))
        winners[w.from] = {w.to, w.type};
    }
  }

  // ---- apply in candidate order (sort/simple_api.rs:165-187, batch_api.rs:98-139); sequential over scenes
  void scene_apply(SceneWork& w, uint64_t* out_ids, uint32_t* out_epochs, uint32_t* out_lengths, uint8_t* out_vt,
                   float* out_pred, float* out_obs) {
    const bool visual = opts.is_visual();
    const int m = w.m;
    const size_t base = w.base;
    std::vector<Track>& tracks = store.find(w.scene)->second;
    std::vector<Track>& cands = w.cands;
    auto& winners = w.winners;
    last_costs[w.scene] = w.pos;
    last_shape[w.scene] = {m, w.n};
    std::unordered_map<uint64_t, size_t> by_id;
    for (size_t j = 0; j < tracks.size(); ++j) by_id[tracks[j].id] = j;
    for (int i = 0; i < m; ++i) {
      Track& c = cands[i];
      uint64_t tid = 0;
      if (opts.is_batch()) tid = ++track_id;  // one id consumed per candidate
      auto it = winners.find(c.id);
      bool is_new = it == winners.end() || it->second.first == c.id;
      if (is_new) {
        if (!opts.is_batch()) tid = ++track_id;
        c.id = tid;
        tracks.push_back(c);
        emit(tracks.back(), base + i, out_ids, out_epochs, out_lengths, out_vt, out_pred, out_obs);
      } else {
        if (visual) c.voting_type = it->second.second;
        Track& dst = tracks[by_id[it->second.first]];
        merge(dst, c);
        emit(dst, base + i, out_ids, out_epochs, out_lengths, out_vt, out_pred, out_obs);
      }
    }
  }
};

// ================================================================== C API
extern "C" {

float orc_radius(const float* box) { return radius(load_box(box)); }
int orc_too_far(const float* l, const float* r) { return too_far(load_box(l), load_box(r)) ? 1 : 0; }
float orc_dist_in_2r(const float* l, const float* r) { return dist_in_2r(load_box(l), load_box(r)); }
void orc_vertices(const float* box, double* out8) {
  P2 v[4];
  vertices(load_box(box), v);
  for (int i = 0; i < 4; ++i) { out8[2 * i] = v[i].x; out8[2 * i + 1] = v[i].y; }
}
int orc_sutherland_hodgman_clip(const double* subject, int ns, const double* clip, int nc, double* out) {
  std::vector<P2> s(ns), c(nc);
  for (int i = 0; i < ns; ++i) s[i] = {subject[2 * i], subject[2 * i + 1]};
  for (int i = 0; i < nc; ++i) c[i] = {clip[2 * i], clip[2 * i + 1]};
  auto r = sh_clip(s, c);
  for (size_t i = 0; i < r.size(); ++i) { out[2 * i] = r[i].x; out[2 * i + 1] = r[i].y; }
  return (int)r.size();
}
double orc_polygon_area(const double* poly, int n) {
  std::vector<P2> p(n);
  for (int i = 0; i < n; ++i) p[i] = {poly[2 * i], poly[2 * i + 1]};
  return polygon_area(p);
}
double orc_intersection(const float* l, const float* r) { return intersection(load_box(l), load_box(r)); }
int orc_iou(const float* l, const float* r, float* out) { return iou(load_box(l), load_box(r), out) ? 1 : 0; }

static KState load_state(const float* p) {
  KState s;
  std::memcpy(s.mean, p, sizeof(float) * 10);
  std::memcpy(s.cov, p + 10, sizeof(float) * 100);
  return s;
}
static void store_state(const KState& s, float* p) {
  std::memcpy(p, s.mean, sizeof(float) * 10);
  std::memcpy(p + 10, s.cov, sizeof(float) * 100);
}
void orc_kalman_initiate(float pw, float vw, const float* box, float* st) { store_state(Filter(pw, vw).initiate(load_box(box)), st); }
void orc_kalman_predict(float pw, float vw, const float* in, float* out) { store_state(Filter(pw, vw).predict(load_state(in)), out); }
void orc_kalman_update(float pw, float vw, const float* in, const float* box, float* out) {
  store_state(Filter(pw, vw).update(load_state(in), load_box(box)), out);
}
float orc_kalman_distance(float pw, float vw, const float* st, const float* box) {
  return Filter(pw, vw).distance(load_state(st), load_box(box));
}
float orc_kalman_calculate_cost(float d, int inverted) { return calculate_cost(d, inverted != 0); }
void orc_kalman_state_box(const float* st, float* box6) { store_box(state_box(load_state(st)), box6); }

float orc_euclidean(const float* a, const float* b, int d) {
  auto pa = pad8(a, d), pb = pad8(b, d);
  return euclidean_p(pa.data(), pb.data(), (int)pa.size() / 8);
}
float orc_cosine(const float* a, const float* b, int d) {
  auto pa = pad8(a, d), pb = pad8(b, d);
  return cosine_p(pa.data(), pb.data(), (int)pa.size() / 8);
}

void orc_sort_cost_matrix(int positional_kind, float iou_threshold, float min_confidence, float pw, float vw,
                          const float* cand_boxes, int m, const float* track_boxes, const float* track_states110,
                          int n, float* out_mn, int threads) {
  parallel_for(m, threads, [&](int b, int e) {
    for (int i = b; i < e; ++i) {
      Box c = load_box(cand_boxes + (size_t)i * 6);
      for (int j = 0; j < n; ++j) {
        Box t = load_box(track_boxes + (size_t)j * 6);
        KState st;
        if (positional_kind == ORC_POS_MAHA) st = load_state(track_states110 + (size_t)j * 110);
        out_mn[(size_t)i * n + j] = positional_metric(positional_kind, iou_threshold, min_confidence, pw, vw, c, t,
                                                      positional_kind == ORC_POS_MAHA ? &st : nullptr);
      }
    }
  });
}

void orc_visual_cost_matrix(int visual_kind, float threshold, const float* cand_feats, int m, const float* track_feats,
                            int n, int d, float* out_mn, int threads) {
  const int blocks = (d + 7) / 8;
  std::vector<float> cp((size_t)m * blocks * 8, 0.0f), tp((size_t)n * blocks * 8, 0.0f);
  for (int i = 0; i < m; ++i) std::memcpy(&cp[(size_t)i * blocks * 8], cand_feats + (size_t)i * d, sizeof(float) * d);
  for (int j = 0; j < n; ++j) std::memcpy(&tp[(size_t)j * blocks * 8], track_feats + (size_t)j * d, sizeof(float) * d);
  const float nan = std::numeric_limits<float>::quiet_NaN();
  parallel_for(m, threads, [&](int b, int e) {
    for (int i = b; i < e; ++i)
      for (int j = 0; j < n; ++j) {
        const float* a = &cp[(size_t)i * blocks * 8];
        const float* t = &tp[(size_t)j * blocks * 8];
        float dd = visual_kind == ORC_VIS_EUCLIDEAN ? euclidean_p(a, t, blocks) : cosine_p(a, t, blocks);
        bool ok = visual_kind == ORC_VIS_EUCLIDEAN ? dd <= threshold : dd >= threshold;
        out_mn[(size_t)i * n + j] = ok ? (visual_kind == ORC_VIS_EUCLIDEAN ? dd : 1.0f - dd) : nan;
      }
  });
}

int64_t orc_kuhn_munkres(const int64_t* w, int rows, int cols, int32_t* out) {
  std::vector<int> xy;
  int64_t total = kuhn_munkres(w, rows, cols, xy);
  for (int i = 0; i < rows; ++i) out[i] = xy[i];
  return total;
}

static std::vector<Ent> load_ents(int n, const uint64_t* from, const uint64_t* to, const float* attr, const float* feat) {
  const float nan = std::numeric_limits<float>::quiet_NaN();
  std::vector<Ent> e(n);
  for (int i = 0; i < n; ++i) e[i] = {from[i], to[i], attr ? attr[i] : nan, feat ? feat[i] : nan};
  return e;
}
int orc_sort_voting(float threshold, int candidates_num, int tracks_num, int n_ent, const uint64_t* from,
                    const uint64_t* to, const float* attr, uint64_t* out_from, uint64_t* out_to) {
  auto r = sort_voting(threshold, candidates_num, tracks_num, load_ents(n_ent, from, to, attr, nullptr));
  for (size_t i = 0; i < r.size(); ++i) { out_from[i] = r[i].first; out_to[i] = r[i].second; }
  return (int)r.size();
}
int orc_bestfit_voting(float max_distance, int min_votes, int n_ent, const uint64_t* from, const uint64_t* to,
                       const float* feat, uint64_t* out_query, uint64_t* out_winner, double* out_weight) {
  auto r = bestfit_voting(max_distance, min_votes, load_ents(n_ent, from, to, nullptr, feat));
  int k = 0;
  for (auto& q : r)
    for (auto& e : q.second) { out_query[k] = e.query_track; out_winner[k] = e.winner_track; out_weight[k] = e.weight; ++k; }
  return k;
}
int orc_visual_voting(float positional_threshold, float max_allowed_feature_distance, int min_votes, int n_ent,
                      const uint64_t* from, const uint64_t* to, const float* attr, const float* feat,
                      uint64_t* out_from, uint64_t* out_to, int32_t* out_type) {
  auto r = visual_voting(positional_threshold, max_allowed_feature_distance, min_votes, load_ents(n_ent, from, to, attr, feat));
  for (size_t i = 0; i < r.size(); ++i) { out_from[i] = r[i].from; out_to[i] = r[i].to; out_type[i] = r[i].type; }
  return (int)r.size();
}

// nms, src/utils/nms.rs:32-72
// test hooks: the scalar and (when compiled and supported) the AVX2 restatement of the feature distances
float orc_euclidean_scalar(const float* a, const float* b, int blocks) { return euclidean_scalar(a, b, blocks); }
float orc_cosine_scalar(const float* a, const float* b, int blocks) { return cosine_scalar(a, b, blocks); }
int orc_simd_active(void) { return use_avx2() ? 1 : 0; }
float orc_euclidean_blocks(const float* a, const float* b, int blocks) { return euclidean_p(a, b, blocks); }
float orc_cosine_blocks(const float* a, const float* b, int blocks) { return cosine_p(a, b, blocks); }

int orc_own_area_shares(const float* boxes, int n, float* out) {
  std::vector<Box> b(n);
  for (int i = 0; i < n; ++i) b[i] = load_box(boxes + (size_t)i * 6);
  std::vector<float> r = own_area_shares(b);
  for (int i = 0; i < n; ++i) out[i] = r[i];
  return 0;
}

int orc_nms(const float* boxes, const float* scores, int n, float nms_threshold, float score_threshold,
            int has_score_threshold, int32_t* out_idx) {
  struct Cand { int src; float rank; int index; };
  float st = has_score_threshold ? score_threshold : std::numeric_limits<float>::lowest();  // f32::MIN
  std::vector<Cand> c;
  int index = 0;
  for (int i = 0; i < n; ++i) {
    Box b = load_box(boxes + (size_t)i * 6);
    bool has_score = scores && !std::isnan(scores[i]);
    float s = has_score ? scores[i] : std::numeric_limits<float>::max();
    if (s > st && b.height > 0.0f && b.aspect > 0.0f) {
      c.push_back({i, has_score ? scores[i] : b.height, index});
      ++index;
    }
  }
  std::stable_sort(c.begin(), c.end(), [](const Cand& a, const Cand& b) { return a.rank > b.rank; });
  std::vector<char> excluded(c.size(), 0);
  for (size_t i = 0; i < c.size(); ++i) {
    if (excluded[c[i].index]) continue;
    Box cb = load_box(boxes + (size_t)c[i].src * 6);
    for (size_t j = i + 1; j < c.size(); ++j) {
      if (excluded[c[j].index]) continue;
      Box ob = load_box(boxes + (size_t)c[j].src * 6);
      float metric = (float)intersection(cb, ob) / area(ob);
      if (metric > nms_threshold) excluded[c[j].index] = 1;
    }
  }
  int k = 0;
  for (auto& e : c)
    if (!excluded[e.index]) out_idx[k++] = e.src;
  return k;
}

orc_tracker* orc_tracker_create(const orc_options* o) { return new orc_tracker(*o); }
void orc_tracker_destroy(orc_tracker* t) { delete t; }
void orc_tracker_set_threads(orc_tracker* t, int threads) { t->threads = threads < 1 ? 1 : threads; }

int orc_tracker_predict_batch(orc_tracker* t, int n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                              const float* boxes, const float* features, const uint8_t* has_feature,
                              const float* quality, const int64_t* custom_ids, const float* own_area,
                              uint64_t* out_ids, uint32_t* out_epochs, uint32_t* out_lengths,
                              uint8_t* out_voting_types, float* out_predicted, float* out_observed) {
  // auto-waste tick, sort/simple_api.rs:115-120
  if (t->auto_waste_counter == 0) {
    t->auto_waste();
    t->auto_waste_counter = t->auto_waste_periodicity;
  } else t->auto_waste_counter -= 1;
  std::vector<orc_tracker::SceneWork> work(n_scenes);
  std::vector<size_t> epochs(n_scenes);
  for (int s = 0; s < n_scenes; ++s) {
    work[s].scene = scene_ids[s];
    work[s].base = (size_t)det_offsets[s];
    work[s].m = det_offsets[s + 1] - det_offsets[s];
    epochs[s] = ++t->epoch_db[scene_ids[s]];  // next_epoch, epoch_db.rs:35-49
    t->store[scene_ids[s]];                    // make sure the scene's store exists before threads read the map
  }
  const bool scene_parallel = t->threads > 1 && n_scenes > 1;
  parallel_for(n_scenes, scene_parallel ? t->threads : 1, [&](int b, int e) {
    for (int s = b; s < e; ++s)
      t->scene_vote(work[s], epochs[s], boxes, features, has_feature, quality, custom_ids, own_area,
                    scene_parallel ? 1 : t->threads);
  });
  for (int s = 0; s < n_scenes; ++s)
    t->scene_apply(work[s], out_ids, out_epochs, out_lengths, out_voting_types, out_predicted, out_observed);
  return 0;
}
// TrackerAPI::skip_epochs_for_scene, tracker_api.rs:48-51
void orc_tracker_skip_epochs(orc_tracker* t, uint64_t scene_id, int n) {
  t->epoch_db[scene_id] += (size_t)n;
  t->auto_waste();
}
int64_t orc_tracker_current_epoch(orc_tracker* t, uint64_t scene_id) { return (int64_t)t->current_epoch(scene_id); }
int orc_tracker_active_tracks(orc_tracker* t) {
  size_t n = 0;
  for (auto& kv : t->store) n += kv.second.size();
  return (int)n;
}
static void emit_track(const Track& tr, int i, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs, uint32_t* lengths,
                       float* predicted, float* observed) {
  if (ids) ids[i] = tr.id;
  if (scene_ids) scene_ids[i] = tr.scene;
  if (epochs) epochs[i] = (uint32_t)tr.epoch;
  if (lengths) lengths[i] = (uint32_t)tr.length;
  if (predicted) store_box(tr.last_pred, predicted + (size_t)i * 6);
  if (observed) store_box(tr.last_obs, observed + (size_t)i * 6);
}
// TrackerAPI::wasted, tracker_api.rs:90-100
int orc_tracker_wasted(orc_tracker* t, int cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                       uint32_t* lengths, float* predicted, float* observed) {
  t->auto_waste();
  int n = (int)std::min((size_t)cap, t->wasted.size());
  for (int i = 0; i < n; ++i) emit_track(t->wasted[i], i, ids, scene_ids, epochs, lengths, predicted, observed);
  t->wasted.erase(t->wasted.begin(), t->wasted.begin() + n);
  return n;
}
// SortLookup::IdleLookup, sort.rs:190-208
int orc_tracker_idle_tracks(orc_tracker* t, uint64_t scene_id, int cap, uint64_t* ids, uint32_t* epochs,
                            uint32_t* lengths, float* predicted, float* observed) {
  auto it = t->store.find(scene_id);
  if (it == t->store.end()) return 0;
  size_t cur = t->current_epoch(scene_id);
  int k = 0;
  for (auto& tr : it->second)
    if (tr.epoch != cur && k < cap) { emit_track(tr, k, ids, nullptr, epochs, lengths, predicted, observed); ++k; }
  return k;
}
void orc_tracker_clear_wasted(orc_tracker* t) { t->wasted.clear(); }
int orc_tracker_scene_tracks(orc_tracker* t, uint64_t scene_id, int cap, uint64_t* ids, float* boxes6,
                             float* states110, int32_t* feat_counts) {
  auto it = t->store.find(scene_id);
  if (it == t->store.end()) return 0;
  int k = 0;
  for (auto& tr : it->second) {
    if (k >= cap) break;
    if (ids) ids[k] = tr.id;
    if (boxes6) store_box(tr.last_pred, boxes6 + (size_t)k * 6);
    if (states110) store_state(tr.st, states110 + (size_t)k * 110);
    if (feat_counts) feat_counts[k] = (int32_t)tr.feat_count;
    ++k;
  }
  return k;
}
int orc_tracker_scene_observations(orc_tracker* t, uint64_t scene_id, int cap, int K, int d8, int32_t* n_obs,
                                   uint8_t* has_feat, float* quality, float* feats, float* norm2) {
  auto it = t->store.find(scene_id);
  if (it == t->store.end()) return 0;
  const int blocks = d8 / 8;
  int k = 0;
  for (auto& tr : it->second) {
    if (k >= cap) break;
    const int n = (int)std::min(tr.obs.size(), (size_t)K);
    n_obs[k] = n;
    for (int j = 0; j < K; ++j) {
      const size_t e = (size_t)k * K + j;
      const Obs* o = j < n ? &tr.obs[j] : nullptr;
      const bool f = o && o->has_feat;
      has_feat[e] = f ? 1 : 0;
      quality[e] = o ? o->quality : 0.0f;
      float* row = feats + e * d8;
      std::memset(row, 0, sizeof(float) * (size_t)d8);
      if (f) std::memcpy(row, o->feat.data(), sizeof(float) * std::min((size_t)d8, o->feat.size()));
      norm2[e] = f ? norm2_p(row, blocks) : 0.0f;
    }
    ++k;
  }
  return k;
}
int orc_tracker_last_costs(orc_tracker* t, uint64_t scene_id, int cap, float* out, int32_t* m, int32_t* n) {
  auto it = t->last_costs.find(scene_id);
  if (it == t->last_costs.end()) return 0;
  auto sh = t->last_shape[scene_id];
  *m = sh.first; *n = sh.second;
  size_t cnt = std::min((size_t)cap, it->second.size());
  std::memcpy(out, it->second.data(), cnt * sizeof(float));
  return (int)cnt;
}

}  // extern "C"
