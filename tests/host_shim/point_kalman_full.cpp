// Full-matrix restatement of Point2DKalmanFilter (src/utils/kalman/kalman_2d_point.rs) in nalgebra's f32 operation
// order: state = mean[4] + cov[4][4] (row-major), the same shape and arithmetic order as the oracle's box filter
// (oracle/similari_oracle.cpp, Filter).  It is what the product's 12-float block form is checked against, so it keeps
// every 0 * x term of the products.  TEST INFRASTRUCTURE: compiled with -ffp-contract=off, never linked by the product.
#include <cmath>
#include <cstring>

namespace {
constexpr int D2 = 2, D4 = 4;
constexpr float kChi2Inv95[9] = {3.8415f, 5.9915f, 7.8147f, 9.4877f, 11.070f, 12.592f, 14.067f, 15.507f, 16.919f};
constexpr float kChi2Upper = 100.0f;  // src/utils/kalman.rs:16-20

struct PState {
  float mean[D4];
  float cov[D4][D4];
};

// C[i][j] = sum_k A[i][k] * B[k][j], k ascending, first term assigned, later terms added (no FMA)
template <int R, int K, int C>
void matmul(const float (*A)[K], const float (*B)[C], float (*out)[C]) {
  for (int j = 0; j < C; ++j)
    for (int i = 0; i < R; ++i) {
      float acc = A[i][0] * B[0][j];
      for (int k = 1; k < K; ++k) acc = A[i][k] * B[k][j] + acc;
      out[i][j] = acc;
    }
}

// nalgebra solve_lower_triangular: forward substitution on the lower triangle of m, column by column, in place
template <int C>
void solve_lower_triangular(const float m[D2][D2], float b[D2][C]) {
  for (int col = 0; col < C; ++col)
    for (int i = 0; i < D2; ++i) {
      const float coeff = b[i][col] / m[i][i];
      b[i][col] = coeff;
      for (int r = i + 1; r < D2; ++r) b[r][col] = (-coeff) * m[r][i] + b[r][col];
    }
}

struct PFilter {
  float motion[D4][D4];
  float update_m[D2][D4];
  float pw, vw;
  // Point2DKalmanFilter::new, :26-39
  PFilter(float position_weight, float velocity_weight) : pw(position_weight), vw(velocity_weight) {
    std::memset(motion, 0, sizeof(motion));
    std::memset(update_m, 0, sizeof(update_m));
    for (int i = 0; i < D4; ++i) motion[i][i] = 1.0f;
    for (int i = 0; i < D2; ++i) motion[i][D2 + i] = 1.0f;  // DT as f32
    for (int i = 0; i < D2; ++i) update_m[i][i] = 1.0f;
  }
  // std_position / std_velocity, :41-49
  float std_position(float k) const { return k * pw; }
  float std_velocity(float k) const { return k * vw; }
  // initiate, :51-65
  PState initiate(float x, float y) const {
    PState s;
    std::memset(&s, 0, sizeof(s));
    s.mean[0] = x; s.mean[1] = y; s.mean[2] = 0.0f; s.mean[3] = 0.0f;
    const float sp = std_position(2.0f), sv = std_velocity(10.0f);
    const float stdv[D4] = {sp * sp, sp * sp, sv * sv, sv * sv};
    for (int i = 0; i < D4; ++i) s.cov[i][i] = stdv[i];
    return s;
  }
  // predict, :67-84
  PState predict(const PState& st) const {
    const float sp = std_position(1.0f), sv = std_velocity(1.0f);
    const float stdv[D4] = {sp * sp, sp * sp, sv * sv, sv * sv};
    PState out;
    for (int i = 0; i < D4; ++i) {
      float acc = motion[i][0] * st.mean[0];
      for (int k = 1; k < D4; ++k) acc = motion[i][k] * st.mean[k] + acc;
      out.mean[i] = acc;
    }
    float t1[D4][D4], mt[D4][D4], t2[D4][D4];
    matmul<D4, D4, D4>(motion, st.cov, t1);
    for (int i = 0; i < D4; ++i) for (int j = 0; j < D4; ++j) mt[i][j] = motion[j][i];
    matmul<D4, D4, D4>(t1, mt, t2);
    for (int i = 0; i < D4; ++i)
      for (int j = 0; j < D4; ++j) out.cov[i][j] = t2[i][j] + (i == j ? stdv[i] : 0.0f);
    return out;
  }
  // project, :86-101
  void project(const PState& st, float pmean[D2], float pcov[D2][D2]) const {
    const float sp = std_position(1.0f);
    const float stdv[D2] = {sp * sp, sp * sp};
    for (int i = 0; i < D2; ++i) {
      float acc = update_m[i][0] * st.mean[0];
      for (int k = 1; k < D4; ++k) acc = update_m[i][k] * st.mean[k] + acc;
      pmean[i] = acc;
    }
    float t1[D2][D4], ut[D4][D2], t2[D2][D2];
    matmul<D2, D4, D4>(update_m, st.cov, t1);
    for (int i = 0; i < D4; ++i) for (int j = 0; j < D2; ++j) ut[i][j] = update_m[j][i];
    matmul<D2, D4, D2>(t1, ut, t2);
    for (int i = 0; i < D2; ++i)
      for (int j = 0; j < D2; ++j) pcov[i][j] = t2[i][j] + (i == j ? stdv[i] : 0.0f);
  }
  // update, :103-121
  PState update(const PState& st, float x, float y) const {
    float pmean[D2], pcov[D2][D2];
    project(st, pmean, pcov);
    float ut[D4][D2], cu[D4][D2], b[D2][D4];
    for (int i = 0; i < D4; ++i) for (int j = 0; j < D2; ++j) ut[i][j] = update_m[j][i];
    matmul<D4, D4, D2>(st.cov, ut, cu);
    for (int i = 0; i < D2; ++i) for (int j = 0; j < D4; ++j) b[i][j] = cu[j][i];
    solve_lower_triangular<D4>(pcov, b);  // kalman_gain (2 x 4)
    const float innov[D2] = {x - pmean[0], y - pmean[1]};
    PState out;
    for (int j = 0; j < D4; ++j) {
      float acc = innov[0] * b[0][j];
      for (int k = 1; k < D2; ++k) acc = innov[k] * b[k][j] + acc;
      out.mean[j] = st.mean[j] + acc;
    }
    float kt[D4][D2], t1[D4][D2], t2[D4][D4];
    for (int i = 0; i < D4; ++i) for (int j = 0; j < D2; ++j) kt[i][j] = b[j][i];
    matmul<D4, D2, D2>(kt, pcov, t1);
    matmul<D4, D2, D4>(t1, b, t2);
    for (int i = 0; i < D4; ++i) for (int j = 0; j < D4; ++j) out.cov[i][j] = st.cov[i][j] - t2[i][j];
    return out;
  }
  // distance, :123-137 (Cholesky factor of S, forward substitution, sum of squares)
  float distance(const PState& st, float x, float y) const {
    float pmean[D2], m[D2][D2];
    project(st, pmean, m);
    float r[D2][1] = {{x - pmean[0]}, {y - pmean[1]}};
    for (int j = 0; j < D2; ++j) {
      for (int k = 0; k < j; ++k) {
        const float factor = -m[j][k];
        for (int row = j; row < D2; ++row) m[row][j] = factor * m[row][k] + m[row][j];
      }
      const float denom = std::sqrt(m[j][j]);
      m[j][j] = denom;
      for (int row = j + 1; row < D2; ++row) m[row][j] = m[row][j] / denom;
    }
    solve_lower_triangular<1>(m, r);
    float sum = 0.0f;
    for (int i = 0; i < D2; ++i) sum = sum + r[i][0] * r[i][0];
    return sum;
  }
};

PState load(const float* p) {
  PState s;
  std::memcpy(s.mean, p, sizeof(float) * D4);
  std::memcpy(s.cov, p + D4, sizeof(float) * D4 * D4);
  return s;
}
void store(const PState& s, float* p) {
  std::memcpy(p, s.mean, sizeof(float) * D4);
  std::memcpy(p + D4, s.cov, sizeof(float) * D4 * D4);
}
}  // namespace

extern "C" {
void pref_initiate(float pw, float vw, float x, float y, float* st20) { store(PFilter(pw, vw).initiate(x, y), st20); }
void pref_predict(float pw, float vw, const float* in20, float* out20) { store(PFilter(pw, vw).predict(load(in20)), out20); }
void pref_update(float pw, float vw, const float* in20, float x, float y, float* out20) {
  store(PFilter(pw, vw).update(load(in20), x, y), out20);
}
float pref_distance(float pw, float vw, const float* st20, float x, float y) {
  return PFilter(pw, vw).distance(load(st20), x, y);
}
// calculate_cost, :139-151: the non-inverted branch compares with CHI2INV95[1], the inverted one with CHI2INV95[4]
float pref_calculate_cost(float distance, int inverted) {
  if (!inverted) return distance > kChi2Inv95[1] ? kChi2Upper : distance;
  return distance > kChi2Inv95[4] ? 0.0f : kChi2Upper - distance;
}
}
