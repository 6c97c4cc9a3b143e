// malio_posegraph.cpp — malio_pose_graph_optimize (include/malio_b200.h): an odometry chain plus loop edges, Gauss-Newton on
// the host.  The normal matrix is the chain's block tridiagonal T plus V V^T, one 6-column block of V per loop edge (its
// Jacobians times a square root of its information); H^-1 g = T^-1 (g - V C^-1 V^T T^-1 g) with the capacitance
// C = I + V^T T^-1 V (Woodbury), so the solve is exact and direct: one block Cholesky of T, m + 2 block-tridiagonal solves
// (the m in parallel) and one dense Cholesky of C.  Built with -ffp-contract=off, as the match's host part.
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "malio_b200.h"
#include "malio_se3.h"

namespace {

struct Pose { double q[4], p[3]; };

void to_T(const Pose& x, double T[16]) {
  double R[9];
  malio_se3::q_to_R(x.q, R);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[4 * i + j] = R[3 * i + j];
    T[4 * i + 3] = x.p[i];
  }
  T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}

// T <- T exp_se3(delta) as malio_scan_store_match's pose update
void right_update(Pose& x, const double delta[6]) {
  double E[16];
  malio_se3::exp_se3(delta, E);
  const double Rm[9] = {E[0], E[1], E[2], E[4], E[5], E[6], E[8], E[9], E[10]};
  double qd[4], qn[4], dp[3];
  malio_se3::quat_from_R(Rm, qd);
  malio_se3::q_mul(x.q, qd, qn);
  const double td[3] = {E[3], E[7], E[11]};
  malio_se3::q_rot(x.q, td, dp);
  const double nrm = std::sqrt(((qn[0] * qn[0] + qn[1] * qn[1]) + qn[2] * qn[2]) + qn[3] * qn[3]);
  for (int i = 0; i < 4; ++i) x.q[i] = qn[i] / nrm;
  for (int i = 0; i < 3; ++i) x.p[i] = x.p[i] + dp[i];
}

struct Edge {
  uint64_t a, b;
  double Zi[16];   // Z^-1
  double W[36];    // Omega
};

// e = log_se3(Z^-1 T_a^-1 T_b) and, with Ja != NULL, J_a = -Ad(T_b^-1 T_a) (row-major 6 x 6, order [dtheta, dt])
void residual(const Edge& e, const double Ta[16], const double Tb[16], double r[6], double* Ja) {
  double Tai[16], M[16], E[16];
  malio_se3::inv_se3(Ta, Tai);
  malio_se3::mul4(e.Zi, Tai, M);
  malio_se3::mul4(M, Tb, E);
  malio_se3::log_se3(E, r);
  if (!Ja) return;
  double Tbi[16], N[16];
  malio_se3::inv_se3(Tb, Tbi);
  malio_se3::mul4(Tbi, Ta, N);
  const double R[9] = {N[0], N[1], N[2], N[4], N[5], N[6], N[8], N[9], N[10]};
  const double t[3] = {N[3], N[7], N[11]};
  const double tx[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
  double TR[9];
  malio_se3::mul3(tx, R, TR);
  for (int i = 0; i < 36; ++i) Ja[i] = 0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      Ja[6 * i + j] = -R[3 * i + j];
      Ja[6 * (i + 3) + j] = -TR[3 * i + j];
      Ja[6 * (i + 3) + j + 3] = -R[3 * i + j];
    }
}

double quad(const double r[6], const double W[36]) {
  double s = 0;
  for (int i = 0; i < 6; ++i) {
    double t = 0;
    for (int j = 0; j < 6; ++j) t += W[6 * i + j] * r[j];
    s += r[i] * t;
  }
  return s;
}

// C = A^T B (6 x 6); C = A B; y = A^T x
void mtm(const double* A, const double* B, double* C) {
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += A[6 * k + i] * B[6 * k + j];
      C[6 * i + j] = s;
    }
}
void mm(const double* A, const double* B, double* C) {
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += A[6 * i + k] * B[6 * k + j];
      C[6 * i + j] = s;
    }
}
void mtv(const double* A, const double* x, double* y) {
  for (int i = 0; i < 6; ++i) {
    double s = 0;
    for (int k = 0; k < 6; ++k) s += A[6 * k + i] * x[k];
    y[i] = s;
  }
}

// in-place lower Cholesky of an n x n SPD matrix (row-major, leading dimension n); false on a pivot <= 0
bool chol(double* A, int n) {
  for (int j = 0; j < n; ++j) {
    double s = A[(size_t)j * n + j];
    for (int k = 0; k < j; ++k) s -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
    if (!(s > 0)) return false;
    const double d = std::sqrt(s);
    A[(size_t)j * n + j] = d;
#pragma omp parallel for schedule(static) if (n - j > 256)
    for (int i = j + 1; i < n; ++i) {
      double t = A[(size_t)i * n + j];
      const double* ri = A + (size_t)i * n;
      const double* rj = A + (size_t)j * n;
      for (int k = 0; k < j; ++k) t -= ri[k] * rj[k];
      A[(size_t)i * n + j] = t / d;
    }
  }
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j) A[(size_t)i * n + j] = 0;
  return true;
}
// L y = b then L^T x = y for the lower L of chol (n x n), k right-hand sides stored as n x k
void chol_solve(const double* L, int n, double* B, int k) {
  for (int c = 0; c < k; ++c) {
    for (int i = 0; i < n; ++i) {
      double t = B[(size_t)i * k + c];
      for (int j = 0; j < i; ++j) t -= L[(size_t)i * n + j] * B[(size_t)j * k + c];
      B[(size_t)i * k + c] = t / L[(size_t)i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
      double t = B[(size_t)i * k + c];
      for (int j = i + 1; j < n; ++j) t -= L[(size_t)j * n + i] * B[(size_t)j * k + c];
      B[(size_t)i * k + c] = t / L[(size_t)i * n + i];
    }
  }
}

// The block Cholesky of the chain's block-tridiagonal T over the free nodes 1..n-1 (index i = node - 1): diag blocks Dg[i],
// off-diagonal B[i] = T(i, i + 1).  Lii[i] lower, Lsub[i] = L(i, i - 1).
struct Chain {
  size_t N;
  std::vector<double> Lii, Lsub;
  bool factor(const std::vector<double>& Dg, const std::vector<double>& B) {
    Lii.assign(N * 36, 0);
    Lsub.assign(N * 36, 0);
    for (size_t i = 0; i < N; ++i) {
      double S[36];
      std::memcpy(S, &Dg[i * 36], sizeof(S));
      if (i > 0) {
        // Lsub[i] = B[i-1]^T L[i-1]^-T: row r solves L[i-1] x = B[i-1]^T's row r transposed
        const double* Lp = &Lii[(i - 1) * 36];
        double* Ls = &Lsub[i * 36];
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) {
            double t = B[(i - 1) * 36 + 6 * c + r];
            for (int k = 0; k < c; ++k) t -= Ls[6 * r + k] * Lp[6 * c + k];
            Ls[6 * r + c] = t / Lp[6 * c + c];
          }
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) {
            double t = 0;
            for (int k = 0; k < 6; ++k) t += Ls[6 * r + k] * Ls[6 * c + k];
            S[6 * r + c] -= t;
          }
      }
      if (!chol(S, 6)) return false;
      std::memcpy(&Lii[i * 36], S, sizeof(S));
    }
    return true;
  }
  // T^-1 applied to X (N x 6 blocks of k columns, row-major N*6 x k), in place
  void solve(double* X, int k) const {
    for (size_t i = 0; i < N; ++i) {
      double* xi = X + i * 6 * k;
      if (i > 0) {
        const double* Ls = &Lsub[i * 36];
        const double* xp = X + (i - 1) * 6 * k;
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < k; ++c) {
            double t = 0;
            for (int j = 0; j < 6; ++j) t += Ls[6 * r + j] * xp[j * k + c];
            xi[r * k + c] -= t;
          }
      }
      const double* L = &Lii[i * 36];
      for (int c = 0; c < k; ++c)
        for (int r = 0; r < 6; ++r) {
          double t = xi[r * k + c];
          for (int j = 0; j < r; ++j) t -= L[6 * r + j] * xi[j * k + c];
          xi[r * k + c] = t / L[6 * r + r];
        }
    }
    for (size_t ii = N; ii-- > 0;) {
      double* xi = X + ii * 6 * k;
      if (ii + 1 < N) {
        const double* Ls = &Lsub[(ii + 1) * 36];   // L(ii+1, ii): x_ii -= Ls^T x_{ii+1}
        const double* xn = X + (ii + 1) * 6 * k;
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < k; ++c) {
            double t = 0;
            for (int j = 0; j < 6; ++j) t += Ls[6 * j + r] * xn[j * k + c];
            xi[r * k + c] -= t;
          }
      }
      const double* L = &Lii[ii * 36];
      for (int c = 0; c < k; ++c)
        for (int r = 5; r >= 0; --r) {
          double t = xi[r * k + c];
          for (int j = r + 1; j < 6; ++j) t -= L[6 * j + r] * xi[j * k + c];
          xi[r * k + c] = t / L[6 * r + r];
        }
    }
  }
};

// S with Omega = S S^T: S = Q diag(sqrt(max(lambda, 0))) from cyclic Jacobi
void sqrt_psd(const double W[36], double S[36]) {
  double A[36], V[36];
  std::memcpy(A, W, sizeof(A));
  for (int i = 0; i < 36; ++i) V[i] = (i % 7 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) off += A[6 * p + q] * A[6 * p + q];
    if (off == 0) break;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) {
        const double apq = A[6 * p + q];
        if (apq == 0) continue;
        const double theta = (A[6 * q + q] - A[6 * p + p]) / (2 * apq);
        double t = 1 / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        if (theta < 0) t = -t;
        const double c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 6; ++k) {
          const double akp = A[6 * k + p], akq = A[6 * k + q];
          A[6 * k + p] = c * akp - s * akq; A[6 * k + q] = s * akp + c * akq;
          const double vkp = V[6 * k + p], vkq = V[6 * k + q];
          V[6 * k + p] = c * vkp - s * vkq; V[6 * k + q] = s * vkp + c * vkq;
        }
        for (int k = 0; k < 6; ++k) {
          const double apk = A[6 * p + k], aqk = A[6 * q + k];
          A[6 * p + k] = c * apk - s * aqk; A[6 * q + k] = s * apk + c * aqk;
        }
      }
  }
  for (int j = 0; j < 6; ++j) {
    const double l = A[7 * j] > 0 ? std::sqrt(A[7 * j]) : 0.0;
    for (int i = 0; i < 6; ++i) S[6 * i + j] = V[6 * i + j] * l;
  }
}

bool finite_pos(double v) { return std::isfinite(v) && v > 0; }

struct Graph {
  uint64_t n;
  std::vector<Edge> odo, loops;
  std::vector<double> Sl;   // per loop: S (6 x 6), Omega = S S^T
  double chi2(const std::vector<Pose>& x, double* c_odo, double* c_loop, double* per_loop) const {
    double so = 0, sl = 0;
    std::vector<double> T(16 * n);
    for (uint64_t k = 0; k < n; ++k) to_T(x[k], &T[16 * k]);
    for (const Edge& e : odo) { double r[6]; residual(e, &T[16 * e.a], &T[16 * e.b], r, nullptr); so += quad(r, e.W); }
    for (size_t i = 0; i < loops.size(); ++i) {
      const Edge& e = loops[i];
      double r[6];
      residual(e, &T[16 * e.a], &T[16 * e.b], r, nullptr);
      const double c = quad(r, e.W);
      if (per_loop) per_loop[i] = c;
      sl += c;
    }
    if (c_odo) *c_odo = so;
    if (c_loop) *c_loop = sl;
    return so + sl;
  }
  // the Gauss-Newton step delta (6 (n - 1)) at x; false when a factor is not positive definite
  bool step(const std::vector<Pose>& x, std::vector<double>& delta) const {
    const size_t N = n - 1;
    std::vector<double> T(16 * n), Dg(N * 36, 0), B(N * 36, 0), g(N * 6, 0);
    for (uint64_t k = 0; k < n; ++k) to_T(x[k], &T[16 * k]);
    // blocks of node k at index k - 1; node 0 is fixed
    auto add_edge = [&](const Edge& e, const double* Ja, const double r[6], bool chain) {
      double Wr[6], JtW[36], t[6];
      for (int i = 0; i < 6; ++i) { double s = 0; for (int j = 0; j < 6; ++j) s += e.W[6 * i + j] * r[j]; Wr[i] = s; }
      if (e.b > 0) for (int i = 0; i < 6; ++i) g[(e.b - 1) * 6 + i] += Wr[i];
      if (e.a > 0) { mtv(Ja, Wr, t); for (int i = 0; i < 6; ++i) g[(e.a - 1) * 6 + i] += t[i]; }
      if (!chain) return;
      if (e.b > 0) for (int i = 0; i < 36; ++i) Dg[(e.b - 1) * 36 + i] += e.W[i];
      if (e.a > 0) {
        mtm(Ja, e.W, JtW);
        double JtWJ[36];
        mm(JtW, Ja, JtWJ);
        for (int i = 0; i < 36; ++i) Dg[(e.a - 1) * 36 + i] += JtWJ[i];
        for (int i = 0; i < 36; ++i) B[(e.a - 1) * 36 + i] += JtW[i];   // H(a, b) = J_a^T Omega J_b, J_b = I
      }
    };
    for (const Edge& e : odo) {
      double r[6], Ja[36];
      residual(e, &T[16 * e.a], &T[16 * e.b], r, Ja);
      add_edge(e, Ja, r, true);
    }
    // V's nonzero blocks: per loop J_a^T S at node a and S at node b (none at node 0)
    const size_t m = loops.size(), k6 = 6 * m;
    std::vector<double> Va(36 * m, 0), Vb(36 * m, 0);
    for (size_t i = 0; i < m; ++i) {
      const Edge& e = loops[i];
      double r[6], Ja[36];
      residual(e, &T[16 * e.a], &T[16 * e.b], r, Ja);
      add_edge(e, Ja, r, false);
      mtm(Ja, &Sl[36 * i], &Va[36 * i]);
      std::memcpy(&Vb[36 * i], &Sl[36 * i], 36 * sizeof(double));
    }
    // the blocks of loop i as (node, block) pairs
    auto blocks = [&](size_t i, uint64_t node[2], const double* blk[2]) {
      node[0] = loops[i].a; blk[0] = &Va[36 * i];
      node[1] = loops[i].b; blk[1] = &Vb[36 * i];
    };
    Chain ch{N, {}, {}};
    if (!ch.factor(Dg, B)) return false;
    // rhs = -g; y = T^-1 rhs
    std::vector<double> y(N * 6);
    for (size_t i = 0; i < N * 6; ++i) y[i] = -g[i];
    ch.solve(y.data(), 1);
    delta = y;
    if (m == 0) return true;
    // C = I + V^T T^-1 V, one loop's 6 columns at a time
    std::vector<double> Cm(k6 * k6, 0);
#pragma omp parallel for schedule(dynamic) if (m >= 64)   // threads pay for themselves only with many loops
    for (long long j = 0; j < (long long)m; ++j) {
      std::vector<double> X(N * 36, 0);
      uint64_t nd[2];
      const double* bk[2];
      blocks((size_t)j, nd, bk);
      for (int h = 0; h < 2; ++h)
        if (nd[h] > 0)
          for (int q = 0; q < 36; ++q) X[(nd[h] - 1) * 36 + q] += bk[h][q];
      ch.solve(X.data(), 6);
      for (size_t i = 0; i < m; ++i) {
        uint64_t ni[2];
        const double* bi[2];
        blocks(i, ni, bi);
        for (int h = 0; h < 2; ++h) {
          if (ni[h] == 0) continue;
          const double* Xb = &X[(ni[h] - 1) * 36];
          for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
              double s = 0;
              for (int t = 0; t < 6; ++t) s += bi[h][6 * t + r] * Xb[6 * t + c];
              Cm[(6 * i + r) * k6 + 6 * j + c] += s;
            }
        }
      }
    }
    for (size_t i = 0; i < k6; ++i) Cm[i * k6 + i] += 1.0;
    // z = C^-1 V^T y; delta = T^-1 (rhs - V z) = y - T^-1 V z
    std::vector<double> z(k6, 0), w(N * 6, 0);
    for (size_t i = 0; i < m; ++i) {
      uint64_t ni[2];
      const double* bi[2];
      blocks(i, ni, bi);
      for (int h = 0; h < 2; ++h)
        if (ni[h] > 0)
          for (int c = 0; c < 6; ++c)
            for (int t = 0; t < 6; ++t) z[6 * i + c] += bi[h][6 * t + c] * y[(ni[h] - 1) * 6 + t];
    }
    if (!chol(Cm.data(), (int)k6)) return false;
    chol_solve(Cm.data(), (int)k6, z.data(), 1);
    for (size_t i = 0; i < m; ++i) {
      uint64_t ni[2];
      const double* bi[2];
      blocks(i, ni, bi);
      for (int h = 0; h < 2; ++h)
        if (ni[h] > 0)
          for (int t = 0; t < 6; ++t)
            for (int c = 0; c < 6; ++c) w[(ni[h] - 1) * 6 + t] += bi[h][6 * t + c] * z[6 * i + c];
    }
    ch.solve(w.data(), 1);
    for (size_t i = 0; i < N * 6; ++i) delta[i] = y[i] - w[i];
    return true;
  }
};

Edge make_edge(uint64_t a, uint64_t b, const double q[4], const double p[3], const double W[36]) {
  Edge e{};
  e.a = a; e.b = b;
  double Z[16];
  Pose zp;
  std::memcpy(zp.q, q, sizeof(zp.q));
  std::memcpy(zp.p, p, sizeof(zp.p));
  to_T(zp, Z);
  malio_se3::inv_se3(Z, e.Zi);
  std::memcpy(e.W, W, sizeof(e.W));
  return e;
}

}  // namespace

extern "C" int malio_pose_graph_optimize(const malio_pass_state* odo, uint64_t n, const malio_pose_edge* loops, uint32_t n_loops,
                                         const malio_pose_graph_args* a, malio_pass_state* out, double* loop_chi2,
                                         malio_pose_graph_report* rep) {
  if (!odo || !a || !out || !rep || n == 0 || (n_loops && !loops) || n_loops > MALIO_POSE_GRAPH_MAX_LOOPS) return MALIO_ERR_INVALID_ARG;
  if (!finite_pos(a->sigma_rot) || !finite_pos(a->sigma_pos) || !finite_pos(a->eps_rot) || !finite_pos(a->eps_pos) || a->max_iter == 0)
    return MALIO_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n_loops; ++i) {
    const malio_pose_edge& e = loops[i];
    if (e.a >= n || e.b >= n || e.a == e.b) return MALIO_ERR_INVALID_ARG;
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c)
        if (!std::isfinite(e.info[6 * r + c]) || e.info[6 * r + c] != e.info[6 * c + r]) return MALIO_ERR_INVALID_ARG;
    for (double v : {e.rot[0], e.rot[1], e.rot[2], e.rot[3], e.pos[0], e.pos[1], e.pos[2]})
      if (!std::isfinite(v)) return MALIO_ERR_INVALID_ARG;
  }
  const auto t0 = std::chrono::steady_clock::now();
  Graph G;
  G.n = n;
  std::vector<Pose> x(n);
  for (uint64_t k = 0; k < n; ++k) {
    std::memcpy(x[k].q, odo[k].rot, sizeof(x[k].q));
    std::memcpy(x[k].p, odo[k].pos, sizeof(x[k].p));
  }
  const double wr = 1.0 / (a->sigma_rot * a->sigma_rot), wp = 1.0 / (a->sigma_pos * a->sigma_pos);
  double Wodo[36] = {0};
  for (int i = 0; i < 3; ++i) { Wodo[7 * i] = wr; Wodo[7 * (i + 3)] = wp; }
  std::vector<double> T(16 * n);
  for (uint64_t k = 0; k < n; ++k) to_T(x[k], &T[16 * k]);
  for (uint64_t k = 0; k + 1 < n; ++k) {
    Edge e{};
    e.a = k; e.b = k + 1;
    double Ti[16];
    malio_se3::inv_se3(&T[16 * k], Ti);
    double Z[16];
    malio_se3::mul4(Ti, &T[16 * (k + 1)], Z);
    malio_se3::inv_se3(Z, e.Zi);
    std::memcpy(e.W, Wodo, sizeof(e.W));
    G.odo.push_back(e);
  }
  G.Sl.resize(36 * (size_t)n_loops);
  for (uint32_t i = 0; i < n_loops; ++i) {
    G.loops.push_back(make_edge(loops[i].a, loops[i].b, loops[i].rot, loops[i].pos, loops[i].info));
    sqrt_psd(loops[i].info, &G.Sl[36 * i]);
  }
  malio_pose_graph_report R{};
  std::vector<double> per(n_loops ? n_loops : 1);
  double c_odo = 0, c_loop = 0;
  double chi = G.chi2(x, &c_odo, &c_loop, per.data());
  R.chi2_loop_before = c_loop;
  R.converged = 1;
  if (n_loops > 0 && n > 1) {
    R.converged = 0;
    std::vector<double> delta;
    for (uint32_t it = 0; it < a->max_iter; ++it) {
      if (!G.step(x, delta)) break;
      bool small = true;
      for (size_t i = 0; i < delta.size(); ++i)
        if (!(std::fabs(delta[i]) < ((i % 6) < 3 ? a->eps_rot : a->eps_pos))) { small = false; break; }
      std::vector<Pose> xn;
      double cn = 0;
      bool lowered = false;
      for (int half = 0; half <= 20; ++half) {
        xn = x;
        for (uint64_t k = 1; k < n; ++k) right_update(xn[k], &delta[(k - 1) * 6]);
        cn = G.chi2(xn, nullptr, nullptr, nullptr);
        if (cn <= chi) { lowered = true; break; }
        for (double& d : delta) d *= 0.5;
      }
      // no halving lowers chi^2: after accepted steps, the minimum along the first-order step; on the first, a stall
      if (!lowered) { R.converged = it > 0 ? 1 : 0; break; }
      x = xn;
      chi = cn;
      R.iterations = it + 1;
      if (small) { R.converged = 1; break; }
    }
    chi = G.chi2(x, &c_odo, &c_loop, per.data());
  }
  for (uint64_t k = 0; k < n; ++k) {
    out[k] = odo[k];
    if (n_loops > 0) {
      std::memcpy(out[k].rot, x[k].q, sizeof(x[k].q));
      std::memcpy(out[k].pos, x[k].p, sizeof(x[k].p));
    }
  }
  if (loop_chi2) for (uint32_t i = 0; i < n_loops; ++i) loop_chi2[i] = per[i];
  R.chi2_odo = c_odo;
  R.chi2_loop = c_loop;
  R.ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *rep = R;
  return MALIO_OK;
}
