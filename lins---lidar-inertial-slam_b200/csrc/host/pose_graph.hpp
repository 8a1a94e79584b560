// pose_graph.hpp — the mapping node's key-pose graph (lidar_mapping_node.cpp: the prior on key 0 and the chain factors of
// saveKeyFramesAndFactor :1673-1705, the loop factors of performLoopClosure :1156-1183) and its solve, in f64 on the host.
//
// The reference keeps the graph in gtsam's iSAM2 (relinearizeThreshold 0.01, relinearizeSkip 1, two update() calls per
// event); this header replaces it by Gauss-Newton to convergence on the whole graph, i.e. the fixed point iSAM2 moves
// towards.  How far iSAM2 lags behind that fixed point after its two updates cannot be measured without gtsam.
// gtsam 4's default-build conventions are taken on trust (no gtsam source is at hand): Pose3 = (R, t) acting as
// R p + t, between(a, b) = a^-1 b, local coordinates Logmap(a^-1 b) and retraction a Expmap(xi) with GTSAM_POSE3_EXPMAP
// on, tangent order (rotation, translation), a factor's error the local coordinates of its measurement to the
// prediction, and Diagonal::Variances(v) weighting component k by 1 / v[k].
//
// The graph is a chain plus a few loop edges, so the normal equations are solved by a block-envelope (skyline)
// Cholesky in natural key order: row r keeps the 6x6 blocks from its lowest connected key to the diagonal, and the
// factor's fill stays inside that envelope.  The Jacobians are central differences of each factor's error in the
// variable's right retraction (h = 1e-6: their error, ~1e-10, moves the fixed point by ~1e-10 of a residual).
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <vector>

namespace lins_pg {

// gtsam Rot3::RzRyRx(x, y, z) (the matrix representation) and Rot3::xyz() through RQ; ypr = (z, y, x):
// roll() = x, pitch() = y, yaw() = z
inline void rot3_rzryrx(double x, double y, double z, double R[3][3]) {
  const double cx = std::cos(x), sx = std::sin(x), cy = std::cos(y), sy = std::sin(y), cz = std::cos(z), sz = std::sin(z);
  const double ss_ = sx * sy, cs_ = cx * sy, sc_ = sx * cy, cc_ = cx * cy, c_s = cx * sz, s_s = sx * sz, _cs = cy * sz, _cc = cy * cz,
               s_c = sx * cz, c_c = cx * cz, ssc = ss_ * cz, csc = cs_ * cz, sss = ss_ * sz, css = cs_ * sz;
  const double M[3][3] = {{_cc, -c_s + ssc, s_s + csc}, {_cs, c_c + sss, -s_c + css}, {-sy, sc_, cc_}};
  std::memcpy(R, M, sizeof(M));
}
inline void mat_mul3(const double A[3][3], const double B[3][3], double C[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i][j] = A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j];
}
inline void rot3_xyz(const double A[3][3], double xyz[3]) {
  const double x = -std::atan2(-A[2][1], A[2][2]);
  const double cqx = std::cos(-x), sqx = std::sin(-x);
  const double Qx[3][3] = {{1, 0, 0}, {0, cqx, -sqx}, {0, sqx, cqx}};
  double B[3][3];
  mat_mul3(A, Qx, B);
  const double y = -std::atan2(B[2][0], B[2][2]);
  const double cqy = std::cos(-y), sqy = std::sin(-y);
  const double Qy[3][3] = {{cqy, 0, sqy}, {0, 1, 0}, {-sqy, 0, cqy}};
  double Cm[3][3];
  mat_mul3(B, Qy, Cm);
  const double z = -std::atan2(-Cm[1][0], Cm[1][1]);
  xyz[0] = x; xyz[1] = y; xyz[2] = z;
}

struct Pose3 { double R[3][3]; double t[3]; };
using Vec6 = std::array<double, 6>;
using Blk = std::array<double, 36>;  // row-major 6x6

inline Pose3 compose(const Pose3& a, const Pose3& b) {
  Pose3 c;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) c.R[i][j] = a.R[i][0] * b.R[0][j] + a.R[i][1] * b.R[1][j] + a.R[i][2] * b.R[2][j];
    c.t[i] = a.R[i][0] * b.t[0] + a.R[i][1] * b.t[1] + a.R[i][2] * b.t[2] + a.t[i];
  }
  return c;
}
inline Pose3 inverse(const Pose3& a) {
  Pose3 c;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c.R[i][j] = a.R[j][i];
  for (int i = 0; i < 3; ++i) c.t[i] = -(c.R[i][0] * a.t[0] + c.R[i][1] * a.t[1] + c.R[i][2] * a.t[2]);
  return c;
}
inline Pose3 between(const Pose3& a, const Pose3& b) { return compose(inverse(a), b); }

// SO(3) / SE(3) exponential and logarithm (gtsam Rot3::Expmap / Logmap, Pose3::Expmap / Logmap)
inline void skew(const double w[3], double W[3][3]) {
  W[0][0] = 0; W[0][1] = -w[2]; W[0][2] = w[1];
  W[1][0] = w[2]; W[1][1] = 0; W[1][2] = -w[0];
  W[2][0] = -w[1]; W[2][1] = w[0]; W[2][2] = 0;
}
inline Pose3 expmap(const double xi[6]) {
  const double* w = xi;
  const double* v = xi + 3;
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = std::sqrt(th2);
  double W[3][3], W2[3][3];
  skew(w, W);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) W2[i][j] = W[i][0] * W[0][j] + W[i][1] * W[1][j] + W[i][2] * W[2][j];
  const double A = th2 > 1e-20 ? std::sin(th) / th : 1.0 - th2 / 6.0;
  const double B = th2 > 1e-20 ? (1.0 - std::cos(th)) / th2 : 0.5 - th2 / 24.0;
  const double Cc = th2 > 1e-20 ? (th - std::sin(th)) / (th2 * th) : 1.0 / 6.0 - th2 / 120.0;
  Pose3 p;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) p.R[i][j] = (i == j) + A * W[i][j] + B * W2[i][j];
  for (int i = 0; i < 3; ++i) {  // t = V v, V = I + B W + C W^2
    p.t[i] = v[i];
    for (int j = 0; j < 3; ++j) p.t[i] += (B * W[i][j] + Cc * W2[i][j]) * v[j];
  }
  return p;
}
inline void logmap(const Pose3& p, double xi[6]) {
  const double tr = p.R[0][0] + p.R[1][1] + p.R[2][2];
  const double c = std::max(-1.0, std::min(1.0, 0.5 * (tr - 1.0)));
  const double th = std::acos(c);
  const double vee[3] = {p.R[2][1] - p.R[1][2], p.R[0][2] - p.R[2][0], p.R[1][0] - p.R[0][1]};
  const double s = std::sin(th);
  const double f = th < 1e-8 ? 0.5 + th * th / 12.0 : 0.5 * th / s;  // (factor errors stay far from theta = pi)
  double w[3] = {f * vee[0], f * vee[1], f * vee[2]};
  std::memcpy(xi, w, sizeof(w));
  double W[3][3];
  skew(w, W);
  double WT[3], WWT[3];
  for (int i = 0; i < 3; ++i) WT[i] = W[i][0] * p.t[0] + W[i][1] * p.t[1] + W[i][2] * p.t[2];
  for (int i = 0; i < 3; ++i) WWT[i] = W[i][0] * WT[0] + W[i][1] * WT[1] + W[i][2] * WT[2];
  // V^-1 t = t - W t / 2 + (1 - th sin / (2 (1 - cos))) / th^2 W^2 t
  const double k = th < 1e-8 ? 1.0 / 12.0 : (1.0 - th * s / (2.0 * (1.0 - std::cos(th)))) / (th * th);
  for (int i = 0; i < 3; ++i) xi[3 + i] = p.t[i] - 0.5 * WT[i] + k * WWT[i];
}
inline Pose3 retract(const Pose3& x, const double d[6]) { return compose(x, expmap(d)); }

// one factor: a prior (b < 0) on key a, or a between factor from key a to key b; variances per tangent component
struct Factor { int a, b; Pose3 z; Vec6 var; };

inline void factor_error(const Factor& f, const Pose3& xa, const Pose3* xb, double e[6]) {
  logmap(f.b < 0 ? between(f.z, xa) : between(f.z, between(xa, *xb)), e);
}

// Gauss-Newton on keys x (initial values in, the fixed point out); returns the iterations run
inline int solve(const std::vector<Factor>& fs, std::vector<Pose3>& x, int max_iter = 100, double tol = 1e-10) {
  const int n = (int)x.size();
  std::vector<int> first(n);
  for (int r = 0; r < n; ++r) first[r] = r;
  for (const Factor& f : fs)
    if (f.b >= 0) { const int lo = std::min(f.a, f.b), hi = std::max(f.a, f.b); first[hi] = std::min(first[hi], lo); }
  std::vector<size_t> base(n + 1, 0);  // row r's blocks (first[r] .. r) at base[r]
  for (int r = 0; r < n; ++r) base[r + 1] = base[r] + (size_t)(r - first[r] + 1);
  std::vector<Blk> L(base[n]);
  std::vector<double> g(6 * (size_t)n);
  auto blk = [&](int r, int c) -> Blk& { return L[base[r] + (size_t)(c - first[r])]; };
  const double h = 1e-6;
  int it = 0;
  for (; it < max_iter; ++it) {
    std::fill(L.begin(), L.end(), Blk{});
    std::fill(g.begin(), g.end(), 0.0);
    for (const Factor& f : fs) {
      const int nv = f.b < 0 ? 1 : 2;
      const int key[2] = {f.a, f.b};
      double e[6], J[2][6][6];
      factor_error(f, x[f.a], f.b < 0 ? nullptr : &x[f.b], e);
      for (int v = 0; v < nv; ++v)
        for (int k = 0; k < 6; ++k) {
          double d[6] = {0, 0, 0, 0, 0, 0}, ep[6], em[6];
          Pose3 xa = x[f.a], xb = f.b < 0 ? x[f.a] : x[f.b];
          Pose3& xv = v == 0 ? xa : xb;
          const Pose3 x0 = xv;
          d[k] = h; xv = retract(x0, d); factor_error(f, xa, f.b < 0 ? nullptr : &xb, ep);
          d[k] = -h; xv = retract(x0, d); factor_error(f, xa, f.b < 0 ? nullptr : &xb, em);
          for (int i = 0; i < 6; ++i) J[v][i][k] = (ep[i] - em[i]) / (2 * h);
        }
      for (int u = 0; u < nv; ++u) {
        for (int k = 0; k < 6; ++k)
          for (int i = 0; i < 6; ++i) g[6 * (size_t)key[u] + k] += J[u][i][k] * e[i] / f.var[i];
        for (int v = 0; v < nv; ++v) {
          if (key[v] > key[u]) continue;  // the lower triangle: block (key[u], key[v]) with key[v] <= key[u]
          Blk& B = blk(key[u], key[v]);
          for (int k = 0; k < 6; ++k)
            for (int l = 0; l < 6; ++l) {
              double s = 0;
              for (int i = 0; i < 6; ++i) s += J[u][i][k] * J[v][i][l] / f.var[i];
              B[6 * k + l] += s;
            }
        }
      }
    }
    // envelope Cholesky H = L L^T in place
    for (int r = 0; r < n; ++r) {
      for (int c = first[r]; c <= r; ++c) {
        Blk S = blk(r, c);
        for (int k = std::max(first[r], first[c]); k < c; ++k) {
          const Blk &A = blk(r, k), &Bk = blk(c, k);
          for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 6; ++j) {
              double s = 0;
              for (int m = 0; m < 6; ++m) s += A[6 * i + m] * Bk[6 * j + m];
              S[6 * i + j] -= s;
            }
        }
        Blk& out = blk(r, c);
        if (c < r) {  // out = S L_cc^-T: row i solves out_i L_cc^T = S_i
          const Blk& D = blk(c, c);
          for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 6; ++j) {
              double s = S[6 * i + j];
              for (int m = 0; m < j; ++m) s -= out[6 * i + m] * D[6 * j + m];
              out[6 * i + j] = s / D[6 * j + j];
            }
        } else {  // dense 6x6 Cholesky of S
          Blk Lc{};
          for (int j = 0; j < 6; ++j) {
            double d = S[6 * j + j];
            for (int m = 0; m < j; ++m) d -= Lc[6 * j + m] * Lc[6 * j + m];
            Lc[6 * j + j] = std::sqrt(d);
            for (int i = j + 1; i < 6; ++i) {
              double s = S[6 * i + j];
              for (int m = 0; m < j; ++m) s -= Lc[6 * i + m] * Lc[6 * j + m];
              Lc[6 * i + j] = s / Lc[6 * j + j];
            }
          }
          out = Lc;
        }
      }
    }
    // L y = -g, then L^T d = y
    std::vector<double> y(6 * (size_t)n);
    for (int r = 0; r < n; ++r)
      for (int i = 0; i < 6; ++i) {
        double s = -g[6 * (size_t)r + i];
        for (int c = first[r]; c <= r; ++c) {
          const Blk& B = blk(r, c);
          const int mmax = c == r ? i : 6;
          for (int m = 0; m < mmax; ++m) s -= B[6 * i + m] * y[6 * (size_t)c + m];
        }
        y[6 * (size_t)r + i] = s / blk(r, r)[6 * i + i];
      }
    for (int r = n - 1; r >= 0; --r) {  // column r of L^T: the diagonal block, then its blocks in the rows c < r
      double* d = &y[6 * (size_t)r];
      const Blk& D = blk(r, r);
      for (int i = 5; i >= 0; --i) {
        double s = d[i];
        for (int m = i + 1; m < 6; ++m) s -= D[6 * m + i] * d[m];
        d[i] = s / D[6 * i + i];
      }
      for (int c = first[r]; c < r; ++c) {
        const Blk& B = blk(r, c);
        for (int j = 0; j < 6; ++j)
          for (int i = 0; i < 6; ++i) y[6 * (size_t)c + j] -= B[6 * i + j] * d[i];
      }
    }
    double dmax = 0;
    for (int r = 0; r < n; ++r) {
      for (int i = 0; i < 6; ++i) dmax = std::max(dmax, std::fabs(y[6 * (size_t)r + i]));
      x[r] = retract(x[r], &y[6 * (size_t)r]);
    }
    if (!(dmax >= tol)) { ++it; break; }
  }
  return it;
}

}  // namespace lins_pg
