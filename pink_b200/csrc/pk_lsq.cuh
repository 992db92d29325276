// Per-instance QP of the IK step, solved in square-root (least-squares) form.
//
// pink.solve_ik hands qpsolvers the strictly convex QP (pink/solve_ik.py:202,270)
//
//     minimise 1/2 x^T H x + c^T x   subject to  G x <= h
//
// with H = sum_t (W_t J_t)^T (W_t J_t) + (damping + sum_t mu_t) I and
// c = sum_t alpha_t (W_t J_t)^T W_t e_t (pink/tasks/task.py:145-166,
// pink/solve_ik.py:55-60).  When the rows of G come from ConfigurationLimit and
// VelocityLimit they are all +-e_i (pink/limits/configuration_limit.py:119,
// pink/limits/velocity_limit.py:119): the feasible set is a box lo <= x <= hi.
//
// H is a Gram matrix.  With A the stacked weighted task Jacobians (K x n), b the
// stacked weighted errors, and the diagonal terms (posture task, damping, LM)
// folded into d_i x_i + beta_i, the same problem reads
//
//     minimise 1/2 |A x + b|^2 + 1/2 sum_i (d_i x_i + beta_i)^2,  lo <= x <= hi
//
// (H = A^T A + diag(d^2), c = A^T b + d*beta).  Working on [diag(d); A] instead of
// H halves the exponent of the condition number, which is what makes fp32 viable:
// cond(H) reaches 1e6..1e7 on the reference's own humanoid examples (CoM cost 200
// next to posture cost 0.1) while cond([D; A]) stays ~1e3.
//
// Method: primal active set on the box.  Every equality-constrained subproblem is
// a linear least-squares problem on the free coordinates, solved from scratch by
// Householder QR of [diag(d); A] with the diagonal block ON TOP: the reflection of
// column k only involves row k and the K dense rows, so a factorisation costs
// ~2 (K+1) n^2 flops (about what forming H and its Cholesky would) and needs no
// up/down-dating.  Fixed coordinates are masked (unit diagonal, zero column), so
// indices stay static and, for compile-time sizes, everything lives in registers.
// Multipliers come from the factored gradient A^T (A x + b) + d (d x + beta), whose
// rounding error scales with the residual, not with |H| |x|.
//
// The minimiser of a strictly convex QP is unique, so the result equals what
// quadprog's Goldfarb-Idnani iteration returns (the parity target).
#pragma once

#include "pk_math.cuh"

#include "../../include/pink_b200.h"

namespace pk {

// Packed lower triangle (used for the exported Hessian).
PK_HD constexpr int tri(int i, int j) { return i >= j ? i * (i + 1) / 2 + j : j * (j + 1) / 2 + i; }

// General-path solver: run-time sizes K <= KMAX rows, n <= N coordinates, arrays
// addressed dynamically (thread-local memory).  Every subproblem is solved on the
// COMPACTED free set: with tight velocity limits most coordinates sit on a bound
// (24 of 33 on the Draco3-class workload), so a factorisation costs
// ~2 (K+1) |F|^2 instead of ~2 (K+1) n^2.
template <int KMAX, int N>
struct BoxLSQ {
  static constexpr int KA = KMAX > 0 ? KMAX : 1;
  static constexpr int NU = N * (N - 1) / 2 > 0 ? N * (N - 1) / 2 : 1;

  PK_HD static constexpr int ut(int k, int j) { return k * N - k * (k + 1) / 2 + (j - k - 1); }  // j > k

  // Least squares on the free coordinates with x fixed on `act`.  y receives the
  // full solution (fixed entries copied from x).  Returns false if singular.
  static PK_HD bool eqp(const float (&A)[KA][N], const float (&b)[KA], const float (&d)[N], const float (&beta)[N],
                        int K, int n, uint64_t act, const float (&x)[N], float (&y)[N]) {
    float Aw[KA][N];  // free columns, compacted
    float zb[KA];
    float Rd[N], Ru[NU], zt[N];
    int idx[N];
    bool ok = true;
    int nf = 0;
    for (int j = 0; j < n; ++j) {
      y[j] = x[j];
      if (!((act >> j) & 1ull)) idx[nf++] = j;
    }
    // right-hand side = b + A_act x_act; compacted copy of the free columns
    for (int r = 0; r < K; ++r) {
      float s = b[r];
      for (int j = 0; j < n; ++j)
        if ((act >> j) & 1ull) s = fmaf(A[r][j], x[j], s);
      zb[r] = s;
      for (int c = 0; c < nf; ++c) Aw[r][c] = A[r][idx[c]];
    }
    for (int k = 0; k < nf; ++k) {
      float sigma = 0.f;
      for (int r = 0; r < K; ++r) sigma = fmaf(Aw[r][k], Aw[r][k], sigma);
      const float alpha = d[idx[k]];
      zt[k] = beta[idx[k]];
      const float norm = sqrtf(fmaf(alpha, alpha, sigma));
      ok = ok && (norm > 0.f);
      const float v0 = alpha + norm;                               // alpha >= 0: no cancellation
      const float tau = (sigma > 0.f) ? 1.f / (norm * v0) : 0.f;   // 2 / |v|^2
      Rd[k] = (sigma > 0.f) ? -norm : alpha;
      for (int j = k + 1; j < nf; ++j) {
        float s = 0.f;
        for (int r = 0; r < K; ++r) s = fmaf(Aw[r][k], Aw[r][j], s);
        s *= tau;
        Ru[ut(k, j)] = -s * v0;
        for (int r = 0; r < K; ++r) Aw[r][j] = fmaf(-s, Aw[r][k], Aw[r][j]);
      }
      float s = v0 * zt[k];
      for (int r = 0; r < K; ++r) s = fmaf(Aw[r][k], zb[r], s);
      s *= tau;
      zt[k] = fmaf(-s, v0, zt[k]);
      for (int r = 0; r < K; ++r) zb[r] = fmaf(-s, Aw[r][k], zb[r]);
    }
    // R y_F = -zt
    for (int kk = 0; kk < nf; ++kk) {
      const int k = nf - 1 - kk;
      float s = -zt[k];
      for (int j = k + 1; j < nf; ++j) s = fmaf(-Ru[ut(k, j)], zt[j], s);
      zt[k] = (Rd[k] != 0.f) ? s / Rd[k] : 0.f;  // zt now holds the solution
      y[idx[k]] = zt[k];
    }
    return ok;
  }

  // Returns status bits (0, NOT_POSDEF, NO_SOLUTION, ITER_LIMIT).  `active` (unless null): the
  // coordinates the solution holds on a bound (x_i is then exactly lo_i or hi_i).
  static PK_HD int run(const float (&A)[KA][N], const float (&b)[KA], const float (&d)[N], const float (&beta)[N],
                       const float (&lo)[N], const float (&hi)[N], int K, int n, float (&x)[N],
                       uint64_t* active = nullptr) {
    if (active) *active = 0ull;
    int status = 0;
    // infeasible box <=> quadprog reports no solution
    for (int i = 0; i < n; ++i) {
      x[i] = 0.f;
      if (lo[i] > hi[i]) status |= PK_STATUS_NO_SOLUTION;
    }
    if (status) return status;
    float y[N];
    if (!eqp(A, b, d, beta, K, n, 0ull, x, y)) status |= PK_STATUS_NOT_POSDEF;
    uint64_t at_hi = 0ull, at_lo = 0ull;
    for (int i = 0; i < n; ++i) {
      if (y[i] > hi[i]) { at_hi |= (1ull << i); x[i] = hi[i]; }
      else if (y[i] < lo[i]) { at_lo |= (1ull << i); x[i] = lo[i]; }
      else x[i] = y[i];
    }
    if ((at_hi | at_lo) == 0ull) return status;

    const uint64_t all = (n >= 64) ? ~0ull : ((1ull << n) - 1ull);
    const int max_iter = 4 * n + 16;
    // anti-cycling at degenerate vertices (multiplier ~ 0 in fp32): a bound that was
    // released and blocks again at once, with a zero-length step, is not released again
    uint64_t released = 0ull, tabu = 0ull;
    for (int it = 0;; ++it) {
      if (it >= max_iter) { status |= PK_STATUS_ITER_LIMIT; break; }
      const uint64_t act = at_hi | at_lo;
      if (act == all) {
        // every coordinate sits on a bound: nothing to solve
        for (int i = 0; i < n; ++i) y[i] = x[i];
      } else {
#ifdef PK_COUNT_ITERS
        status += 256;
#endif
        eqp(A, b, d, beta, K, n, act, x, y);
      }
      // longest feasible step from x towards y
      float step = 1.f;
      int blk = -1;
      bool blk_hi = false;
      for (int i = 0; i < n; ++i) {
        if (!((act >> i) & 1ull)) {
          const float dlt = y[i] - x[i];
          if (y[i] > hi[i]) {
            const float a = (hi[i] - x[i]) / dlt;
            if (a < step) { step = a; blk = i; blk_hi = true; }
          } else if (y[i] < lo[i]) {
            const float a = (lo[i] - x[i]) / dlt;
            if (a < step) { step = a; blk = i; blk_hi = false; }
          }
        }
      }
      if (blk >= 0) {
        step = fmaxf(step, 0.f);
        for (int i = 0; i < n; ++i) {
          if (!((act >> i) & 1ull)) {
            x[i] = fmaf(step, y[i] - x[i], x[i]);
            if (i == blk) x[i] = blk_hi ? hi[i] : lo[i];
          }
        }
        if (blk_hi) at_hi |= (1ull << blk); else at_lo |= (1ull << blk);
        if (((released >> blk) & 1ull) && step <= 1e-6f) tabu |= (1ull << blk);
        continue;
      }
      for (int i = 0; i < n; ++i) x[i] = y[i];
      // multipliers from the factored gradient g = A^T (A x + b) + d (d x + beta)
      float rho[KA];
      for (int r = 0; r < K; ++r) {
        float s = b[r];
        for (int j = 0; j < n; ++j) s = fmaf(A[r][j], x[j], s);
        rho[r] = s;
      }
      float worst = 0.f;
      int rel = -1;
      uint64_t neg = 0ull;
      for (int i = 0; i < n; ++i) {
        if (((act & ~tabu) >> i) & 1ull) {
          const float rt = fmaf(d[i], x[i], beta[i]);
          float g = d[i] * rt;
          float gabs = fabsf(g);
          for (int r = 0; r < K; ++r) {
            g = fmaf(A[r][i], rho[r], g);
            gabs = fmaf(fabsf(A[r][i]), fabsf(rho[r]), gabs);
          }
          const float lam = ((at_hi >> i) & 1ull) ? -g : g;
          // release only multipliers that are negative beyond the rounding of g
          if (lam < -4e-6f * gabs) {
            neg |= (1ull << i);
            if (lam < worst) { worst = lam; rel = i; }
          }
        }
      }
      if (rel < 0) break;
      // first pass: release every wrong-signed bound; afterwards one at a time
      const uint64_t drop = (it == 0) ? neg : (1ull << rel);
      if (it > 0) released |= drop;
      at_hi &= ~drop;
      at_lo &= ~drop;
    }
    if (active) *active = at_hi | at_lo;
    return status;
  }

  // y_F = (A_F^T A_F + diag(d_F)^2)^-1 g_F on the free coordinates F (bit i of `held` clear), y_i = 0
  // on the held ones.  Householder QR of [diag(d); A] on the compacted free columns as in eqp, so the
  // normal matrix is never formed in fp32; then R^T z = g_F and R y_F = z.  Returns false (y = 0) when
  // a pivot of R is at most 1e-5 of its column's norm: the matrix is not positive definite to fp32
  // accuracy.
  static PK_HD bool normal_solve(const float (&A)[KA][N], const float (&d)[N], int K, int n, uint64_t held,
                                 const float (&g)[N], float (&y)[N]) {
    float Aw[KA][N];
    float Rd[N], Ru[NU], z[N];
    int idx[N];
    int nf = 0;
    for (int j = 0; j < n; ++j) {
      y[j] = 0.f;
      if (!((held >> j) & 1ull)) idx[nf++] = j;
    }
    for (int r = 0; r < K; ++r)
      for (int c = 0; c < nf; ++c) Aw[r][c] = A[r][idx[c]];
    bool ok = true;
    for (int k = 0; k < nf; ++k) {
      float sigma = 0.f;
      for (int r = 0; r < K; ++r) sigma = fmaf(Aw[r][k], Aw[r][k], sigma);
      const float alpha = d[idx[k]];
      const float norm = sqrtf(fmaf(alpha, alpha, sigma));
      const float v0 = alpha + norm;
      const float tau = (sigma > 0.f) ? 1.f / (norm * v0) : 0.f;
      Rd[k] = (sigma > 0.f) ? -norm : alpha;
      for (int j = k + 1; j < nf; ++j) {
        float s = 0.f;
        for (int r = 0; r < K; ++r) s = fmaf(Aw[r][k], Aw[r][j], s);
        s *= tau;
        Ru[ut(k, j)] = -s * v0;
        for (int r = 0; r < K; ++r) Aw[r][j] = fmaf(-s, Aw[r][k], Aw[r][j]);
      }
      // norm of the original column k
      float c2 = alpha * alpha;
      for (int r = 0; r < K; ++r) c2 = fmaf(A[r][idx[k]], A[r][idx[k]], c2);
      ok = ok && fabsf(Rd[k]) > 1e-5f * sqrtf(c2);
    }
    if (!ok) return false;
    for (int k = 0; k < nf; ++k) {
      float s = g[idx[k]];
      for (int j = 0; j < k; ++j) s = fmaf(-Ru[ut(j, k)], z[j], s);
      z[k] = s / Rd[k];
    }
    for (int kk = 0; kk < nf; ++kk) {
      const int k = nf - 1 - kk;
      float s = z[k];
      for (int j = k + 1; j < nf; ++j) s = fmaf(-Ru[ut(k, j)], z[j], s);
      z[k] = s / Rd[k];
      y[idx[k]] = z[k];
    }
    return true;
  }
};

// ---------------------------------------------------------------------------------
// Register-resident variant for small compile-time sizes (the chain kernel).
//
// Same problem and same primal active-set logic as BoxLSQ, different linear
// algebra, chosen from the first ncu captures (profiles/r01*): the Householder
// sweep cost ~1800 instructions per subproblem and the QP was 77 % of the kernel.
//  * Subproblems are Newton steps on the free coordinates with a Cholesky
//    factorisation of the masked Gram matrix H = A^T A + diag(d^2) (~300
//    instructions for n = 6), started from the current gradient H x + c.
//  * The conditioning lost by squaring is bought back only where it matters: the
//    final multipliers always come from the FACTORED gradient
//    A^T (A x + b) + d (d x + beta) (rounding error ~ |A x + b|, not |H| |x|), and
//    when the pivot ratio of the free block says it is ill-conditioned the free
//    coordinates get two steps of iterative refinement with that gradient
//    (corrected semi-normal equations).
//  * No solve at all while every coordinate sits on a bound, and the first
//    multiplier pass releases every wrong-signed bound at once.
// The solver is split into corner_start / gram / round / polish (run() chains them).
// ---------------------------------------------------------------------------------
#ifdef PK_COUNT_ITERS
extern "C" void pk_count_nfree(int nfree, int round);
#endif

template <int N>
struct BoxState {
  static constexpr int NT = N * (N + 1) / 2;
  float H[NT], c[N], lo[N], hi[N], x[N];
  uint32_t at_hi, at_lo;
  float gtol;  // absolute tolerance on multipliers inside the rounds
  float cond;  // pivot ratio of the last factorisation of the free block
  int status;
  int rounds;
};

template <int K, int N>
struct BoxLSQChol {
  static constexpr int KA = K > 0 ? K : 1;
  static constexpr int NT = N * (N + 1) / 2;
  static constexpr uint32_t ALL = (1u << N) - 1u;
  static constexpr int kMaxRounds = 3 * N + 8;
  using State = BoxState<N>;

  // Cholesky of the masked H (act bit => identity row/column); returns the pivot
  // ratio max/min over the free coordinates (0 if a pivot is not positive).
  static PK_HD float factor(const float (&H)[NT], uint32_t act, float (&L)[NT], float (&inv)[N]) {
    float pmax = 0.f, pmin = 3.0e38f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const bool fj = !((act >> j) & 1u);
      float dj = fj ? H[tri(j, j)] : 1.f;
#pragma unroll
      for (int k = 0; k < j; ++k) dj = fmaf(-L[tri(j, k)], L[tri(j, k)], dj);
      if (fj) { pmax = fmaxf(pmax, dj); pmin = fminf(pmin, dj); }
      const float r = rsqrtf(fmaxf(dj, 1e-30f));
      inv[j] = r;
      L[tri(j, j)] = dj * r;
#pragma unroll
      for (int i = j + 1; i < N; ++i) {
        const bool fi = !((act >> i) & 1u);
        float s = (fi && fj) ? H[tri(i, j)] : 0.f;
#pragma unroll
        for (int k = 0; k < j; ++k) s = fmaf(-L[tri(i, k)], L[tri(j, k)], s);
        L[tri(i, j)] = s * r;
      }
    }
    return (pmin > 0.f) ? pmax / pmin : 0.f;
  }

  static PK_HD void solve(const float (&L)[NT], const float (&inv)[N], float (&y)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      float s = y[i];
#pragma unroll
      for (int k = 0; k < i; ++k) s = fmaf(-L[tri(i, k)], y[k], s);
      y[i] = s * inv[i];
    }
#pragma unroll
    for (int ii = 0; ii < N; ++ii) {
      const int i = N - 1 - ii;
      float s = y[i];
#pragma unroll
      for (int k = i + 1; k < N; ++k) s = fmaf(-L[tri(k, i)], y[k], s);
      y[i] = s * inv[i];
    }
  }

  // g = H x + c
  static PK_HD void gradient_h(const State& S, float (&g)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      float s = S.c[i];
#pragma unroll
      for (int j = 0; j < N; ++j) s = fmaf(S.H[tri(i, j)], S.x[j], s);
      g[i] = s;
    }
  }

  // Objective held in registers / thread-local arrays.
  struct ArrayObjective {
    const float (&A)[KA][N];
    const float (&b)[KA];
    const float (&d)[N];
    const float (&beta)[N];
    PK_HD void row(int r, float (&a)[N], float& br) const {
#pragma unroll
      for (int j = 0; j < N; ++j) a[j] = A[r][j];
      br = b[r];
    }
    PK_HD float diag(int i) const { return d[i]; }
    PK_HD float lin(int i) const { return beta[i]; }
  };

  // g = A^T (A x + b) + d (d x + beta), gabs = rounding scale of each entry.  The
  // objective is streamed row by row (Obj::row) so that a caller holding it in
  // shared memory never needs all of A in registers.
  template <class Obj>
  static PK_HD void gradient_factored(const Obj& O, const float (&x)[N], float (&g)[N], float (&gabs)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const float di = O.diag(i);
      const float rt = fmaf(di, x[i], O.lin(i));
      g[i] = di * rt;
      gabs[i] = fabsf(g[i]);
    }
#pragma unroll
    for (int r = 0; r < K; ++r) {
      float a[N], br;
      O.row(r, a, br);
      float rho = br;
#pragma unroll
      for (int j = 0; j < N; ++j) rho = fmaf(a[j], x[j], rho);
      const float ra = fabsf(rho);
#pragma unroll
      for (int i = 0; i < N; ++i) {
        g[i] = fmaf(a[i], rho, g[i]);
        gabs[i] = fmaf(fabsf(a[i]), ra, gabs[i]);
      }
    }
  }

  // Cheap start.  Every coordinate is put on the bound the gradient at the origin
  // points to (c_i < 0 -> upper, c_i > 0 -> lower) and the KKT conditions are tested
  // there with the factored gradient.  On the UR5 benchmark 78 % of the instances are
  // optimal at that corner (the velocity box is tight), which the clamp of the
  // unconstrained minimiser only guessed for 42 % - and this start needs neither the
  // Gram matrix nor a factorisation.  Returns false if x is optimal (or the box is
  // empty); true if rounds are needed (wrong-signed bounds are already released).
  template <class Obj>
  static PK_HD bool corner_start(const Obj& O, const float (&lo)[N], const float (&hi)[N], State& S,
                               bool closed_form = true) {
    S.status = 0;
    S.rounds = 0;
    S.at_hi = S.at_lo = 0u;
    S.cond = 1.f;
    S.gtol = 0.f;
    bool infeasible = false;
    float c[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      S.lo[i] = lo[i];
      S.hi[i] = hi[i];
      S.x[i] = 0.f;
      infeasible = infeasible || (lo[i] > hi[i]);
      c[i] = O.diag(i) * O.lin(i);
    }
    if (infeasible) {  // empty box <=> quadprog reports no solution
      S.status = PK_STATUS_NO_SOLUTION;
      return false;
    }
#pragma unroll
    for (int r = 0; r < K; ++r) {
      float a[N], br;
      O.row(r, a, br);
#pragma unroll
      for (int i = 0; i < N; ++i) c[i] = fmaf(a[i], br, c[i]);
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if (c[i] < 0.f && hi[i] < 3.0e38f) { S.at_hi |= (1u << i); S.x[i] = hi[i]; }
      else if (c[i] > 0.f && lo[i] > -3.0e38f) { S.at_lo |= (1u << i); S.x[i] = lo[i]; }
      else S.x[i] = fminf(fmaxf(0.f, lo[i]), hi[i]);
    }
    const uint32_t act = S.at_hi | S.at_lo;
    float g[N], gabs[N];
    gradient_factored(O, S.x, g, gabs);
    uint32_t neg = 0u;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if ((act >> i) & 1u) {
        const float lam = ((S.at_hi >> i) & 1u) ? -g[i] : g[i];
        if (lam < -4e-6f * gabs[i]) neg |= (1u << i);
      }
    }
    PK_PHASE(kPhaseCorner);
#ifdef PK_COUNT_ITERS
    if (act == ALL && neg == 0u) pk_count_nfree(0, -1);
#endif
    if (act == ALL && neg == 0u) return false;
    const uint32_t at_hi0 = S.at_hi, at_lo0 = S.at_lo;
    S.at_hi &= ~neg;
    S.at_lo &= ~neg;
    // Closed-form active-set steps from the corner.  On the benchmark 78 % of the
    // instances are optimal at the corner, 18 % have ONE free coordinate at the optimum
    // and 3 % two, so the first one or two releases are done here without the Gram
    // matrix: release the coordinate with the most negative multiplier, minimise over
    // the released set F (|F| <= 2) exactly, delta_F = -H_FF^-1 g_F with the columns
    // H_jF = A[:, j] . A[:, F] (+ d^2 on the diagonal) accumulated row by row, and test
    // the KKT signs of the others with g_j + H_jF delta_F.  Anything else (a released
    // coordinate that reaches its other bound, a third release) goes to the rounds.
    if (closed_form && act == ALL && neg != 0u) {
      PK_PHASE_FLAG(kFlagRelease1);
      // most negative multiplier
      float worst = 0.f;
      uint32_t n1 = 0u;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float lam = ((at_hi0 >> j) & 1u) ? -g[j] : g[j];
        if (((neg >> j) & 1u) && lam < worst) { worst = lam; n1 = 1u << j; }
      }
      float m1[N], h1[N];
#pragma unroll
      for (int j = 0; j < N; ++j) {
        m1[j] = ((n1 >> j) & 1u) ? 1.f : 0.f;
        const float dj = O.diag(j);
        h1[j] = m1[j] * dj * dj;
      }
#pragma unroll
      for (int r = 0; r < K; ++r) {
        float a[N], br;
        O.row(r, a, br);
        float a1 = 0.f;
#pragma unroll
        for (int j = 0; j < N; ++j) a1 = fmaf(a[j], m1[j], a1);
#pragma unroll
        for (int j = 0; j < N; ++j) h1[j] = fmaf(a[j], a1, h1[j]);
      }
      float h11 = 0.f, g1 = 0.f, x1 = 0.f, lo1 = 0.f, hi1 = 0.f;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        h11 = fmaf(m1[j], h1[j], h11);
        g1 = fmaf(m1[j], g[j], g1);
        x1 = fmaf(m1[j], S.x[j], x1);
        lo1 = fmaf(m1[j], fmaxf(lo[j], -3.0e38f), lo1);
        hi1 = fmaf(m1[j], fminf(hi[j], 3.0e38f), hi1);
      }
      float d1 = -g1 / h11;
      bool ok = h11 > 0.f;
      // the box is narrow: the released coordinate may run into its opposite bound, where
      // it stays (the corner had picked the wrong side for it)
      const bool flip_hi = (x1 + d1) > hi1, flip_lo = (x1 + d1) < lo1;
      if (flip_hi) d1 = hi1 - x1;
      if (flip_lo) d1 = lo1 - x1;
      const bool flipped = flip_hi || flip_lo;
      // multipliers of the others after the step
      float worst2 = 0.f;
      uint32_t n2 = 0u;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        if (!((n1 >> j) & 1u)) {
          const float gj = fmaf(h1[j], d1, g[j]);
          const float lam = ((at_hi0 >> j) & 1u) ? -gj : gj;
          if (lam < -4e-6f * gabs[j] && lam < worst2) { worst2 = lam; n2 = 1u << j; }
        }
      }
      // side of every bound after stage 1 (the flipped coordinate changed sides)
      const uint32_t hi1m = (at_hi0 & ~n1) | (flip_hi ? n1 : 0u);
      const uint32_t lo1m = (at_lo0 & ~n1) | (flip_lo ? n1 : 0u);
      if (flipped) {
        // multiplier of the flipped coordinate at its new bound
        const float gn = fmaf(h11, d1, g1);
        ok = ok && !((flip_hi ? -gn : gn) < 0.f);
      }
      if (ok && n2 == 0u) {
#ifdef PK_COUNT_ITERS
        pk_count_nfree(flipped ? 3 : 1, -1);
#endif
#pragma unroll
        for (int j = 0; j < N; ++j) {
          S.x[j] = fmaf(m1[j], d1, S.x[j]);
          if (flipped && ((n1 >> j) & 1u)) S.x[j] = flip_hi ? hi[j] : lo[j];
        }
        S.at_hi = hi1m;  // the other wrong-signed bounds turned out to be active
        S.at_lo = lo1m;
        return false;
      }
      if (ok) {
        // second release i2: exact minimiser over {i1, i2} from the corner, or over {i2}
        // alone when i1 sits on its opposite bound
        PK_PHASE_FLAG(kFlagRelease2);
        float m2[N], h2[N];
#pragma unroll
        for (int j = 0; j < N; ++j) {
          m2[j] = ((n2 >> j) & 1u) ? 1.f : 0.f;
          const float dj = O.diag(j);
          h2[j] = m2[j] * dj * dj;
        }
#pragma unroll
        for (int r = 0; r < K; ++r) {
          float a[N], br;
          O.row(r, a, br);
          float a2 = 0.f;
#pragma unroll
          for (int j = 0; j < N; ++j) a2 = fmaf(a[j], m2[j], a2);
#pragma unroll
          for (int j = 0; j < N; ++j) h2[j] = fmaf(a[j], a2, h2[j]);
        }
        float h22 = 0.f, h12 = 0.f, g2 = 0.f, x2 = 0.f, lo2 = 0.f, hi2 = 0.f;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          h22 = fmaf(m2[j], h2[j], h22);
          h12 = fmaf(m2[j], h1[j], h12);
          g2 = fmaf(m2[j], g[j], g2);
          x2 = fmaf(m2[j], S.x[j], x2);
          lo2 = fmaf(m2[j], fmaxf(lo[j], -3.0e38f), lo2);
          hi2 = fmaf(m2[j], fminf(hi[j], 3.0e38f), hi2);
        }
        float d2;
        bool solved;  // the released block was well-conditioned
        if (flipped) {
          d2 = -fmaf(h12, d1, g2) / h22;
          solved = h22 > 0.f;
        } else {
          const float det = fmaf(h11, h22, -h12 * h12);
          const float inv = 1.f / det;
          d1 = (h12 * g2 - h22 * g1) * inv;
          d2 = (h12 * g1 - h11 * g2) * inv;
          solved = det > 1e-6f * h11 * h22;  // otherwise the rounds decide
        }
        // longest feasible step towards the minimiser of the released block
        float alpha = 1.f;
        uint32_t blk = 0u;
        bool blk_hi = false;
        if (!flipped) {
          if (x1 + d1 > hi1) { const float a = (hi1 - x1) / d1; if (a < alpha) { alpha = a; blk = n1; blk_hi = true; } }
          else if (x1 + d1 < lo1) { const float a = (lo1 - x1) / d1; if (a < alpha) { alpha = a; blk = n1; blk_hi = false; } }
        }
        if (x2 + d2 > hi2) { const float a = (hi2 - x2) / d2; if (a < alpha) { alpha = a; blk = n2; blk_hi = true; } }
        else if (x2 + d2 < lo2) { const float a = (lo2 - x2) / d2; if (a < alpha) { alpha = a; blk = n2; blk_hi = false; } }
        alpha = fmaxf(alpha, 0.f);
        const uint32_t freed = flipped ? n2 : (n1 | n2);
        // multipliers of the others at the block minimiser
        float worst3 = 0.f;
        uint32_t n3 = 0u;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          if (!((freed >> j) & 1u)) {
            const float gj = fmaf(h1[j], d1, fmaf(h2[j], d2, g[j]));
            const float lam = ((hi1m >> j) & 1u) ? -gj : gj;
            if (lam < -4e-6f * gabs[j] && lam < worst3) { worst3 = lam; n3 = 1u << j; }
          }
        }
        ok = solved && blk == 0u && n3 == 0u;
#ifdef PK_COUNT_ITERS
        pk_count_nfree(ok ? (flipped ? 4 : 2) : (flipped ? 14 : 12), -1);
#endif
        if (ok) {
#pragma unroll
          for (int j = 0; j < N; ++j) {
            S.x[j] = fmaf(m1[j], d1, fmaf(m2[j], d2, S.x[j]));
            if (flipped && ((n1 >> j) & 1u)) S.x[j] = flip_hi ? hi[j] : lo[j];
          }
          S.at_hi = hi1m & ~n2;
          S.at_lo = lo1m & ~n2;
          return false;
        }
        // Not settled: hand the rounds the furthest state reached here rather than the corner
        // with every wrong-signed bound released.  The kernel ends when the slowest instance
        // does, and this cuts the longest chain on the benchmark from 9 rounds to 5 (state
        // after the first closed-form step) and further (state after the second one).
        if (solved) {
          // (a) a released coordinate reaches a bound on the way: stop there, it becomes active;
          // (b) the block minimiser is feasible but another multiplier is negative: release it
          const float e1 = flipped ? d1 : alpha * d1;  // the flipped coordinate is already placed
          const float e2 = alpha * d2;
#pragma unroll
          for (int j = 0; j < N; ++j) {
            S.x[j] = fmaf(m1[j], e1, fmaf(m2[j], e2, S.x[j]));
            if (flipped && ((n1 >> j) & 1u)) S.x[j] = flip_hi ? hi[j] : lo[j];
            if ((blk >> j) & 1u) S.x[j] = blk_hi ? hi[j] : lo[j];
          }
          S.at_hi = (hi1m & ~n2) | (blk_hi ? blk : 0u);
          S.at_lo = (lo1m & ~n2) | (blk_hi ? 0u : blk);
          if (blk == 0u) { S.at_hi &= ~n3; S.at_lo &= ~n3; }
          return true;
        }
        {
          const float d1s = flipped ? d1 : -g1 / h11;
#pragma unroll
          for (int j = 0; j < N; ++j) {
            S.x[j] = fmaf(m1[j], d1s, S.x[j]);
            if (flipped && ((n1 >> j) & 1u)) S.x[j] = flip_hi ? hi[j] : lo[j];
          }
          S.at_hi = hi1m & ~n2;
          S.at_lo = lo1m & ~n2;
          return true;
        }
      }
#ifdef PK_COUNT_ITERS
      else pk_count_nfree(11, -1);
#endif
    }
    return true;
  }

  // Gram matrix H = A^T A + diag(d^2), c = A^T b + d beta and the tolerance of the
  // rounds, for the instances that need them.
  template <class Obj>
  static PK_HD void gram(const Obj& O, State& S) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const float di = O.diag(i);
#pragma unroll
      for (int j = 0; j <= i; ++j) S.H[tri(i, j)] = (i == j) ? di * di : 0.f;
      S.c[i] = di * O.lin(i);
    }
#pragma unroll
    for (int r = 0; r < K; ++r) {
      float a[N], br;
      O.row(r, a, br);
#pragma unroll
      for (int i = 0; i < N; ++i) {
#pragma unroll
        for (int j = 0; j <= i; ++j) S.H[tri(i, j)] = fmaf(a[i], a[j], S.H[tri(i, j)]);
        S.c[i] = fmaf(a[i], br, S.c[i]);
      }
    }
    // rounding scale of H x + c over the box
    float gs = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      float s = fabsf(S.c[i]);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float xm = fmaxf(fabsf(S.x[j]), fminf(fmaxf(fabsf(S.lo[j]), fabsf(S.hi[j])), 1e3f));
        s = fmaf(fabsf(S.H[tri(i, j)]), xm, s);
      }
      gs = fmaxf(gs, s);
    }
    S.gtol = 4e-6f * gs;
  }

  // One active-set round: Newton step on the free set (with blocking), then release
  // of wrong-signed bounds.  Returns true if another round is needed.
  static PK_HD bool round(State& S) {
    const bool first = S.rounds == 0;
    if (++S.rounds > kMaxRounds) {
      S.status |= PK_STATUS_ITER_LIMIT;
      return false;
    }
    const uint32_t act = S.at_hi | S.at_lo;
    float g[N];
    if (act != ALL) {
#ifdef PK_COUNT_ITERS
      S.status += 256;
      pk_count_nfree(N - __builtin_popcount(act), S.rounds);
#endif
      gradient_h(S, g);
      float L[NT], inv[N], y[N];
      S.cond = factor(S.H, act, L, inv);
#pragma unroll
      for (int i = 0; i < N; ++i) y[i] = ((act >> i) & 1u) ? 0.f : -g[i];
      solve(L, inv, y);
      float step = 1.f;
      int blk = -1;
      bool blk_hi = false;
#pragma unroll
      for (int i = 0; i < N; ++i) {
        if (!((act >> i) & 1u)) {
          const float xn = S.x[i] + y[i];
          if (xn > S.hi[i]) {
            const float a = (S.hi[i] - S.x[i]) / y[i];
            if (a < step) { step = a; blk = i; blk_hi = true; }
          } else if (xn < S.lo[i]) {
            const float a = (S.lo[i] - S.x[i]) / y[i];
            if (a < step) { step = a; blk = i; blk_hi = false; }
          }
        }
      }
      step = fmaxf(step, 0.f);
#pragma unroll
      for (int i = 0; i < N; ++i) {
        if (!((act >> i) & 1u)) {
          S.x[i] = fmaf(step, y[i], S.x[i]);
          if (i == blk) S.x[i] = blk_hi ? S.hi[i] : S.lo[i];
        }
      }
      if (blk >= 0) {
        if (blk_hi) S.at_hi |= (1u << blk); else S.at_lo |= (1u << blk);
        return true;
      }
    }
    // multipliers of the active bounds
    gradient_h(S, g);
    float worst = 0.f;
    int rel = -1;
    uint32_t neg = 0u;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if ((act >> i) & 1u) {
        const float lam = ((S.at_hi >> i) & 1u) ? -g[i] : g[i];
        if (lam < -S.gtol) {
          neg |= (1u << i);
          if (lam < worst) { worst = lam; rel = i; }
        }
      }
    }
    if (rel < 0) return false;
    // first pass: release every wrong-signed bound; afterwards one at a time
    const uint32_t drop = first ? neg : (1u << rel);
    S.at_hi &= ~drop;
    S.at_lo &= ~drop;
    return true;
  }

  // Accurate acceptance test and refinement.  Returns true if more rounds are needed.
  // A refinement step that pushes a free coordinate out of its box is clamped; if a coordinate
  // still sits on a bound when the refinement ends, that bound becomes active and more rounds
  // follow (an ill-conditioned free block otherwise keeps clamping the same coordinates and
  // stalls away from the minimiser: 1 instance in 40000 without a Levenberg-Marquardt term at
  // dt = 0.1, relative stationarity up to 4e-2; profiles/r02i_hostsim_soak.txt).
  template <class Obj>
  static PK_HD bool polish(const Obj& O, State& S) {
    if (S.status & (PK_STATUS_NO_SOLUTION | PK_STATUS_ITER_LIMIT)) return false;
    const uint32_t act = S.at_hi | S.at_lo;
    if (act == 0u && S.cond <= 1e3f) return false;  // interior, well-conditioned: x is the plain solve
    float g[N], gabs[N];
    gradient_factored(O, S.x, g, gabs);
    float worst = 0.f;
    int rel = -1;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if ((act >> i) & 1u) {
        const float lam = ((S.at_hi >> i) & 1u) ? -g[i] : g[i];
        if (lam < -4e-6f * gabs[i] && lam < worst) { worst = lam; rel = i; }
      }
    }
    if (rel >= 0 && S.rounds < kMaxRounds) {
      S.at_hi &= ~(1u << rel);
      S.at_lo &= ~(1u << rel);
      return true;
    }
    if (act != ALL && S.cond > 1e3f) {
      // ill-conditioned free block: iterative refinement with the factored gradient
      // (corrected semi-normal equations) until the correction stalls, 4 steps at most
      float L[NT], inv[N], y[N];
      factor(S.H, act, L, inv);
#pragma unroll 1
      for (int pass = 0; pass < 4; ++pass) {
        float dmax = 0.f, xmax = 0.f;
#pragma unroll
        for (int i = 0; i < N; ++i) y[i] = ((act >> i) & 1u) ? 0.f : -g[i];
        solve(L, inv, y);
#pragma unroll
        for (int i = 0; i < N; ++i) {
          if (!((act >> i) & 1u)) {
            const float xn = fminf(fmaxf(S.x[i] + y[i], S.lo[i]), S.hi[i]);
            dmax = fmaxf(dmax, fabsf(xn - S.x[i]));
            xmax = fmaxf(xmax, fabsf(xn));
            S.x[i] = xn;
          }
        }
#ifdef PK_COUNT_ITERS
        pk_count_nfree(100 + pass, -1);
#endif
        if (dmax <= 2e-7f * xmax) break;
        gradient_factored(O, S.x, g, gabs);
      }
      if (S.rounds < kMaxRounds) {
        uint32_t hit_hi = 0u, hit_lo = 0u;
#pragma unroll
        for (int i = 0; i < N; ++i) {
          if (!((act >> i) & 1u)) {
            if (S.x[i] >= S.hi[i]) hit_hi |= (1u << i);
            else if (S.x[i] <= S.lo[i]) hit_lo |= (1u << i);
          }
        }
        if ((hit_hi | hit_lo) != 0u) {
#ifdef PK_COUNT_ITERS
          pk_count_nfree(200, __builtin_popcount(hit_hi | hit_lo));
#endif
          S.at_hi |= hit_hi;
          S.at_lo |= hit_lo;
          return true;
        }
      }
    }
    return false;
  }

  static PK_HD bool polish(const float (&A)[KA][N], const float (&b)[KA], const float (&d)[N],
                           const float (&beta)[N], State& S) {
    const ArrayObjective O{A, b, d, beta};
    return polish(O, S);
  }

  // Whole solve in one thread.
  static PK_HD int run(const float (&A)[KA][N], const float (&b)[KA], const float (&d)[N], const float (&beta)[N],
                       const float (&lo)[N], const float (&hi)[N], float (&x)[N], int flags = 0) {
    State S;
    const ArrayObjective O{A, b, d, beta};
    // flags: bit 0 = closed-form first releases off (A/B), bit 1 = stop after the corner
    // stage (timing probe only: wrong results for the instances that need rounds)
    const bool rounds = corner_start(O, lo, hi, S, !(flags & 1));
    PK_PHASE(kPhaseClosedForm);
    if (rounds && !(flags & 2)) {
      PK_PHASE_FLAG(kFlagRounds);
      gram(O, S);
      bool more = true;
      for (;;) {
        while (more) more = round(S);
        more = polish(O, S);
        if (!more) break;
      }
    }
    PK_PHASE(kPhaseRounds);
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = S.x[i];
    return S.status;
  }
};

}  // namespace pk
