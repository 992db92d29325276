// Warp-cooperative IK step for joint trees (humanoids): one instance per warp,
// lanes = joints / tangent columns / task rows, all per-instance state in the warp's
// slice of shared memory.  Same arithmetic as the general path (pk_generic.cuh):
// FK over the tree, FrameTask / RelativeFrameTask / PostureTask / ComTask rows in
// square-root form, box limits, active-set QP with a Householder QR of the
// compacted free columns of [diag(d); A].  Reference path: see pk_chain.cuh and
// pk_generic.cuh headers.
//
// Written in the lane-block style of pk_warp.cuh so that tests/hostsim can run it
// on the CPU.
#pragma once

#include "pk_generic.cuh"
#include "pk_warp.cuh"

namespace pk {

constexpr int kTreeMaxJoints = 32;   // lanes = joints
constexpr int kTreeTaskWords = 60;   // per task: Tf 12, A 9, B 9, e 6, Tr 12, Trf 12

// Sizes and workspace offsets (in floats) of one instance; computed on the host.
struct TreePlan {
  int nj, nq, nv, rq, rv, K, ntasks, stride, lda, ldw, maxdepth;
  int row_base[PK_MAX_TASKS];  // first row of A of each task (-1: none)
  int o_q, o_t, o_tw, o_root, o_tf, o_A, o_b, o_d, o_beta, o_lo, o_hi, o_x, o_y, o_g, o_aw, o_ru, o_rd, o_zt, o_zb,
      o_rho, o_ys, o_idx, o_cw, o_xa, words;
  // dense inequality rows (barriers) and the state of the dual method (pk_treedual.cuh); p = 0: none
  // meq: equality rows of solve_ik(..., constraints=...); nct: number of constraint tasks
  int p, ldj, npairs, meq, nct;
  int o_G, o_hg, o_gn, o_J, o_RA, o_dv, o_z, o_r, o_u, o_act, o_xd, o_wd, o_gd, o_rhod, o_ud, o_dist, o_E, o_fe, o_en,
      o_asg;
};

// defined in pk_treedual.cuh
PK_HD int tree_dual_solve(float* W, const TreePlan& L);

constexpr int kTwStride = 13;     // 12 floats per joint transform, padded against bank conflicts
#ifdef PK_COUNT_ITERS
static int g_tree_seq = 0;
static uint64_t g_tree_prev = 0;
#endif
constexpr int kMultiChange = 12;  // iterations with multi-add / multi-release before single steps

struct TreeStep {
  // ---- small accessors -------------------------------------------------------------
  static PK_HD SE3f load_tw(const float* W, const TreePlan& L, int body) {
    if (body == -2) return identity_se3();
    if (body == -1) return load_se3(W + L.o_root);
    return load_se3(W + L.o_tw + kTwStride * body);
  }

  // Column i of the LOCAL Jacobian of a frame at Tf on `body` (as Generic::frame_jac_col).
  static PK_HD void jac_col(const DevModel& M, const float* W, const TreePlan& L, int body, const SE3f& Tf, int i,
                            V3& lin, V3& ang) {
    lin = v3(0.f, 0.f, 0.f);
    ang = v3(0.f, 0.f, 0.f);
    if (i < L.rv) {
      if (body == -2) return;
      const SE3f Trf = act_inv(load_se3(W + L.o_root), Tf);
      const V3 ek = v3(i % 3 == 0 ? 1.f : 0.f, i % 3 == 1 ? 1.f : 0.f, i % 3 == 2 ? 1.f : 0.f);
      if (i < 3) {
        lin = mulT(Trf.R, ek);
      } else {
        lin = mulT(Trf.R, cross(ek, Trf.p));
        ang = mulT(Trf.R, ek);
      }
      return;
    }
    const int j = i - L.rv;
    if (body < 0 || !((M.anc[body + 2] >> j) & 1ull)) return;
    const SE3f Tj = load_se3(W + L.o_tw + kTwStride * j);
    const V3 axis = v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]);
    const V3 aw = mul(Tj.R, axis);
    if (M.jtype[j] == PK_JOINT_REVOLUTE) {
      lin = mulT(Tf.R, cross(aw, Tf.p - Tj.p));
      ang = mulT(Tf.R, aw);
    } else {
      lin = mulT(Tf.R, aw);
    }
  }

  // strict upper triangle of R, packed by rows: entry (k, j), j > k
  static PK_HD int ru(const TreePlan& L, int k, int j) { return k * L.nv - k * (k + 1) / 2 + (j - k - 1); }

  // ---- least squares on the free set (cooperative Householder QR) -------------------
  // Rows of Aw are owned by lanes (r = l, l + 32, ...).  y receives the full solution.
  // TWO: the task set has more than 32 rows, so a lane owns two of them (l and l + 32); with
  // K <= 32 (the Draco3 / G1 example task sets: 24 rows) the second slot is compiled out, which
  // removes a third of the sweep's loads, FMAs and stores (results are bit-identical: the
  // empty slot only ever contributed zeros).
  template <bool TWO>
  static PK_HD bool eqp_impl(float* W, const TreePlan& L, uint64_t act) {
    const int n = L.nv, K = L.K;
    float* A = W + L.o_A;
    float* Aw = W + L.o_aw;
    float* Ru = W + L.o_ru;
    float* Rd = W + L.o_rd;
    float* zt = W + L.o_zt;
    float* zb = W + L.o_zb;
    int* idx = reinterpret_cast<int*>(W + L.o_idx);
    const float* x = W + L.o_x;
    float* y = W + L.o_y;
    const float* bv = W + L.o_b;
    const float* dv = W + L.o_d;
    const float* beta = W + L.o_beta;
    // free index list
#if defined(__CUDA_ARCH__)
    const int nf = n - __popcll(act);
#else
    const int nf = n - __builtin_popcountll(act);
#endif
    float* xa = W + L.o_xa;  // x with the free entries zeroed
#ifdef PK_COUNT_ITERS
    pk_count_nfree(nf, 1000);
    if (g_tree_seq > 0) pk_count_nfree(__builtin_popcountll(act ^ g_tree_prev), 2000 + (g_tree_seq < 9 ? g_tree_seq : 9));
    g_tree_prev = act;
    ++g_tree_seq;
#endif
    PK_LANES(l) {
      #pragma unroll 1
      for (int i = l; i < n; i += 32) {
        y[i] = x[i];
        xa[i] = ((act >> i) & 1ull) ? x[i] : 0.f;
        if (!((act >> i) & 1ull)) {
          const uint64_t below = (i == 0) ? 0ull : (~act & ((1ull << i) - 1ull));
#if defined(__CUDA_ARCH__)
          const int pos = __popcll(below);
#else
          const int pos = __builtin_popcountll(below);
#endif
          idx[pos] = i;
          zt[pos] = beta[i];
        }
      }
    }
    PK_WSYNC();
    // right-hand side and compacted copy, row-parallel (two row slots per lane)
    PK_LANES(l) {
#pragma unroll
      for (int h = 0; h < (TWO ? 2 : 1); ++h) {
        const int r = l + 32 * h;
        if (r < K) {
          const float* Ar = A + r * L.lda;
          float* Awr = Aw + r * L.ldw;
          float s = bv[r];
#pragma unroll 4
          for (int j = 0; j < n; ++j) s = fmaf(Ar[j], xa[j], s);
          zb[r] = s;
#pragma unroll 4
          for (int c = 0; c < nf; ++c) Awr[c] = Ar[idx[c]];
        }
      }
    }
    PK_WSYNC();
    bool ok = true;
    // Householder sweep.  K <= 64: every lane owns at most two rows (l and l + 32),
    // kept in registers for column k; four columns j are reflected per pass so that
    // the four shuffle reductions overlap.
    #pragma unroll 1
    for (int k = 0; k < nf; ++k) {
      LaneVar<float> ak0, ak1, part;
      PK_LANES(l) {
        const float a0 = (l < K) ? Aw[l * L.ldw + k] : 0.f;
        const float a1 = (TWO && l + 32 < K) ? Aw[(l + 32) * L.ldw + k] : 0.f;
        ak0[l] = a0;
        ak1[l] = a1;
        part[l] = fmaf(a0, a0, a1 * a1);
      }
      const float sigma = lane_sum(part);
      const float alpha = dv[idx[k]];
      const float norm = sqrtf(fmaf(alpha, alpha, sigma));
      ok = ok && (norm > 0.f);
      const float v0 = alpha + norm;
      const float tau = (sigma > 0.f) ? 1.f / (norm * v0) : 0.f;
      const float rdk = (sigma > 0.f) ? -norm : alpha;
      #pragma unroll 1
      for (int j = k + 1; j < nf; j += 4) {
        LaneVar<float> c0[4], c1[4], p[4];
        PK_LANES(l) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const bool on = j + c < nf;
            const float a0 = (on && l < K) ? Aw[l * L.ldw + j + c] : 0.f;
            const float a1 = (TWO && on && l + 32 < K) ? Aw[(l + 32) * L.ldw + j + c] : 0.f;
            c0[c][l] = a0;
            c1[c][l] = a1;
            p[c][l] = fmaf(ak0[l], a0, ak1[l] * a1);
          }
        }
        float sc[4];
        lane_sum4(p, sc);
#pragma unroll
        for (int c = 0; c < 4; ++c) sc[c] *= tau;
        PK_LANES(l) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (j + c < nf) {
              if (l < K) Aw[l * L.ldw + j + c] = fmaf(-sc[c], ak0[l], c0[c][l]);
              if (TWO && l + 32 < K) Aw[(l + 32) * L.ldw + j + c] = fmaf(-sc[c], ak1[l], c1[c][l]);
              if (l == 0) Ru[ru(L, k, j + c)] = -sc[c] * v0;
            }
          }
        }
      }
      PK_LANES(l) {
        const float z0 = (l < K) ? zb[l] : 0.f;
        const float z1 = (TWO && l + 32 < K) ? zb[l + 32] : 0.f;
        part[l] = fmaf(ak0[l], z0, ak1[l] * z1);
      }
      const float ztk = zt[k];
      const float s = fmaf(v0, ztk, lane_sum(part)) * tau;
      PK_WSYNC();
      PK_LANES(l) {
        if (l < K) zb[l] = fmaf(-s, ak0[l], zb[l]);
        if (TWO && l + 32 < K) zb[l + 32] = fmaf(-s, ak1[l], zb[l + 32]);
        if (l == 0) {
          zt[k] = fmaf(-s, v0, ztk);
          Rd[k] = rdk;
        }
      }
    }
    PK_WSYNC();
    // R ys = -zt by columns: lane j owns the running sum of row j (two slots); each
    // solved component is broadcast from its owner and folded into the rows above it.
    {
      LaneVar<float> acc0, acc1, sol0, sol1;
      PK_LANES(l) {
        acc0[l] = (l < nf) ? -zt[l] : 0.f;
        acc1[l] = (l + 32 < nf) ? -zt[l + 32] : 0.f;
        sol0[l] = 0.f;
        sol1[l] = 0.f;
      }
      #pragma unroll 1
      for (int kk = 0; kk < nf; ++kk) {
        const int k = nf - 1 - kk;
        const float rd = Rd[k];
        const float num = (k < 32) ? lane_bcast(acc0, k) : lane_bcast(acc1, k - 32);
        const float yk = (rd != 0.f) ? num / rd : 0.f;
        PK_LANES(l) {
          if (l < k) acc0[l] = fmaf(-Ru[ru(L, l, k)], yk, acc0[l]);
          if (l + 32 < k) acc1[l] = fmaf(-Ru[ru(L, l + 32, k)], yk, acc1[l]);
          if (l == (k & 31)) {
            if (k < 32) sol0[l] = yk; else sol1[l] = yk;
          }
        }
      }
      PK_LANES(l) {
        if (l < nf) y[idx[l]] = sol0[l];
        if (l + 32 < nf) y[idx[l + 32]] = sol1[l];
      }
      PK_WSYNC();
    }
    return ok;
  }

  // ---- the same least-squares solve, COLUMN-parallel (round 2) --------------------------
  // For task sets of at most KR <= 32 rows and at most 31 free columns, lane c holds free
  // column c of [diag(d_F); A_F] in registers (KR dense entries; its only non-zero "top" entry
  // is its own diagonal d_c until its turn), lane nf holds the right-hand side.  Step k: the
  // owner's column is the Householder vector; it is broadcast (KR shuffles), every later lane
  // forms its dot product with it locally and reflects its own column - no cross-lane
  // reductions, no shared-memory traffic inside the sweep.  The row-parallel sweep above
  // costs a 5-stage shuffle reduction per dot product and reloads every column from shared
  // memory in every pass; for nf = 9 / 20 free columns it issues about 1.4x / 2x the
  // instructions of this one.  Same mathematics, different summation order.
  template <int KR>
  struct ColRegs {
    float a[KR];
  };

  template <int KR>
  static PK_HD bool eqp_cols(float* W, const TreePlan& L, uint64_t act) {
    const int n = L.nv, K = L.K;
    float* A = W + L.o_A;
    float* Ru = W + L.o_ru;
    float* Rd = W + L.o_rd;
    float* zt = W + L.o_zt;
    float* zb = W + L.o_zb;
    int* idx = reinterpret_cast<int*>(W + L.o_idx);
    const float* x = W + L.o_x;
    float* y = W + L.o_y;
    const float* bv = W + L.o_b;
    const float* dv = W + L.o_d;
    const float* beta = W + L.o_beta;
#if defined(__CUDA_ARCH__)
    const int nf = n - __popcll(act);
#else
    const int nf = n - __builtin_popcountll(act);
#endif
    float* xa = W + L.o_xa;  // x with the free entries zeroed
#ifdef PK_COUNT_ITERS
    pk_count_nfree(nf, 1000);
    if (g_tree_seq > 0) pk_count_nfree(__builtin_popcountll(act ^ g_tree_prev), 2000 + (g_tree_seq < 9 ? g_tree_seq : 9));
    g_tree_prev = act;
    ++g_tree_seq;
#endif
    PK_LANES(l) {
      #pragma unroll 1
      for (int i = l; i < n; i += 32) {
        y[i] = x[i];
        xa[i] = ((act >> i) & 1ull) ? x[i] : 0.f;
        if (!((act >> i) & 1ull)) {
          const uint64_t below = (i == 0) ? 0ull : (~act & ((1ull << i) - 1ull));
#if defined(__CUDA_ARCH__)
          const int pos = __popcll(below);
#else
          const int pos = __builtin_popcountll(below);
#endif
          idx[pos] = i;
          zt[pos] = beta[i];
        }
      }
    }
    PK_WSYNC();
    // right-hand side of the dense rows, row-parallel: zb = b + A x_active
    PK_LANES(l) {
      if (l < K) {
        const float* Ar = A + l * L.lda;
        float s = bv[l];
#pragma unroll 4
        for (int j = 0; j < n; ++j) s = fmaf(Ar[j], xa[j], s);
        zb[l] = s;
      }
    }
    PK_WSYNC();
    // columns into registers: lane c < nf its free column, lane nf the right-hand side
    LaneVar<ColRegs<KR>> C;
    PK_LANES(l) {
      // one strided read per row: a free column of A (stride lda) or the right-hand side (stride 1)
      const bool live = l <= nf;
      const float* src = (l < nf) ? A + idx[l] : zb;
      const int stride = (l < nf) ? L.lda : 1;
#pragma unroll
      for (int r = 0; r < KR; ++r) C[l].a[r] = (live && r < K) ? src[r * stride] : 0.f;
    }
    bool ok = true;
    #pragma unroll 1
    for (int k = 0; k < nf; ++k) {
      // Householder vector = column k (broadcast from its owner)
      float v[KR];
#pragma unroll
      for (int r = 0; r < KR; ++r) {
        LaneVar<float> t;
        PK_LANES(l) { t[l] = C[l].a[r]; }
        v[r] = lane_bcast(t, k);
      }
      float sigma = 0.f;
#pragma unroll
      for (int r = 0; r < KR; ++r) sigma = fmaf(v[r], v[r], sigma);
      const float alpha = dv[idx[k]];
      const float norm = sqrtf(fmaf(alpha, alpha, sigma));
      ok = ok && (norm > 0.f);
      const float v0 = alpha + norm;                              // alpha >= 0: no cancellation
      const float tau = (sigma > 0.f) ? rcp_f(norm * v0) : 0.f;  // 2 / |v|^2
      const float ztk = zt[k];
      PK_WSYNC();
      PK_LANES(l) {
        if (l > k && l <= nf) {
          // top row k of this column: zero for a free column, the diagonal row's right-hand side for lane nf
          const float top = (l == nf) ? ztk : 0.f;
          float sdot = v0 * top;
#pragma unroll
          for (int r = 0; r < KR; ++r) sdot = fmaf(v[r], C[l].a[r], sdot);
          sdot *= tau;
#pragma unroll
          for (int r = 0; r < KR; ++r) C[l].a[r] = fmaf(-sdot, v[r], C[l].a[r]);
          const float tnew = fmaf(-sdot, v0, top);
          if (l == nf) zt[k] = tnew;
          else Ru[ru(L, k, l)] = tnew;
        }
        if (l == 0) Rd[k] = (sigma > 0.f) ? -norm : alpha;
      }
    }
    PK_WSYNC();
    // R ys = -zt by columns (as in the row-parallel variant)
    {
      LaneVar<float> acc0, sol0;
      PK_LANES(l) {
        acc0[l] = (l < nf) ? -zt[l] : 0.f;
        sol0[l] = 0.f;
      }
      #pragma unroll 1
      for (int kk = 0; kk < nf; ++kk) {
        const int k = nf - 1 - kk;
        const float rd = Rd[k];
        const float num = lane_bcast(acc0, k);
        const float yk = (rd != 0.f) ? num * rcp_f(rd) : 0.f;
        PK_LANES(l) {
          if (l < k) acc0[l] = fmaf(-Ru[ru(L, l, k)], yk, acc0[l]);
          if (l == k) sol0[l] = yk;
        }
      }
      PK_LANES(l) {
        if (l < nf) y[idx[l]] = sol0[l];
      }
      PK_WSYNC();
    }
    return ok;
  }

  static PK_HD bool eqp(float* W, const TreePlan& L, uint64_t act) {
#if defined(__CUDA_ARCH__)
    const int nf = L.nv - __popcll(act);
#else
    const int nf = L.nv - __builtin_popcountll(act);
#endif
    if (L.K <= 32 && nf <= 31) {
      if (L.K <= 8) return eqp_cols<8>(W, L, act);
      if (L.K <= 16) return eqp_cols<16>(W, L, act);
      if (L.K <= 24) return eqp_cols<24>(W, L, act);
      return eqp_cols<32>(W, L, act);
    }
    return (L.K > 32) ? eqp_impl<true>(W, L, act) : eqp_impl<false>(W, L, act);
  }

  // ---- box-constrained least squares (as BoxLSQ::run, cooperative) ------------------
  static PK_HD int solve_qp(float* W, const TreePlan& L) {
#ifdef PK_COUNT_ITERS
    g_tree_seq = 0;
#endif
    const int n = L.nv, K = L.K;
    const float* A = W + L.o_A;
    const float* bv = W + L.o_b;
    const float* dv = W + L.o_d;
    const float* beta = W + L.o_beta;
    const float* lo = W + L.o_lo;
    const float* hi = W + L.o_hi;
    float* x = W + L.o_x;
    float* y = W + L.o_y;
    float* rho = W + L.o_rho;
    int status = 0;
    {
      LaneVar<int> bad;
      PK_LANES(l) {
        int f = 0;
        #pragma unroll 1
        for (int i = l; i < n; i += 32) {
          x[i] = 0.f;
          if (lo[i] > hi[i]) f = 1;
        }
        bad[l] = f;
      }
      PK_WSYNC();
      if (lane_or(bad)) return PK_STATUS_NO_SOLUTION;
    }
    // Start: a diagonally scaled gradient step x_i = -c_i / H_ii, clamped, guesses the
    // active set.  With tight velocity limits most coordinates end on a bound, so this
    // replaces the most expensive factorisation (all n columns free) by small ones; the
    // loop below only stops at a point that passes the KKT test, whatever the start.
    uint64_t at_hi, at_lo;
    {
      LaneVar<uint64_t> mh, ml;
      PK_LANES(l) {
        uint64_t h = 0ull, m = 0ull;
        #pragma unroll 1
        for (int i = l; i < n; i += 32) {
          float ci = dv[i] * beta[i];
          float hii = dv[i] * dv[i];
          #pragma unroll 1
          for (int r = 0; r < K; ++r) {
            const float a = A[r * L.lda + i];
            ci = fmaf(a, bv[r], ci);
            hii = fmaf(a, a, hii);
          }
          const float yi = (hii > 0.f) ? -ci / hii : 0.f;
          if (yi > hi[i]) { h |= (1ull << i); x[i] = hi[i]; }
          else if (yi < lo[i]) { m |= (1ull << i); x[i] = lo[i]; }
          else x[i] = yi;
        }
        mh[l] = h;
        ml[l] = m;
      }
      at_hi = lane_or64(mh);
      at_lo = lane_or64(ml);
      PK_WSYNC();
    }
    const uint64_t all = (n >= 64) ? ~0ull : ((1ull << n) - 1ull);
    const int max_iter = 4 * n + 16;
    // anti-cycling at degenerate vertices (multiplier ~ 0 in fp32): a bound that was
    // released and blocks again at once, with a zero-length step, is not released again
    uint64_t released = 0ull, tabu = 0ull;
    for (int it = 0;; ++it) {
      if (it >= max_iter) { status |= PK_STATUS_ITER_LIMIT; break; }
      const uint64_t act = at_hi | at_lo;
      if (act == all) {
        PK_LANES(l) {
          #pragma unroll 1
          for (int i = l; i < n; i += 32) y[i] = x[i];
        }
        PK_WSYNC();
      } else if (!eqp(W, L, act)) {
        status |= PK_STATUS_NOT_POSDEF;
      }
      // longest feasible step from x towards y
      float step;
      int blk;
      {
        LaneVar<float> sv;
        LaneVar<int> si;
        PK_LANES(l) {
          float best = 1.f;
          int bi = 0x7fffffff;
          #pragma unroll 1
          for (int i = l; i < n; i += 32) {
            if (!((act >> i) & 1ull)) {
              const float yi = y[i], xi = x[i];
              float a = 2.f;
              if (yi > hi[i]) a = (hi[i] - xi) / (yi - xi);
              else if (yi < lo[i]) a = (lo[i] - xi) / (yi - xi);
              if (a < best) { best = a; bi = i; }
            }
          }
          sv[l] = best;
          si[l] = bi;
        }
        lane_argmin(sv, si, step, blk);
      }
      if (blk != 0x7fffffff) {
        if (it < kMultiChange) {
          // early iterations: clamp EVERY free coordinate that the Newton point pushes
          // past a bound (primal-dual style; halves the number of factorisations on
          // the humanoid workloads).  Later iterations take the classical single
          // blocking step, which guarantees termination.
          LaneVar<uint64_t> mh, ml;
          PK_LANES(l) {
            uint64_t h = 0ull, m = 0ull;
            #pragma unroll 1
            for (int i = l; i < n; i += 32) {
              if (!((act >> i) & 1ull)) {
                const float yi = y[i];
                if (yi > hi[i]) { h |= (1ull << i); x[i] = hi[i]; }
                else if (yi < lo[i]) { m |= (1ull << i); x[i] = lo[i]; }
                else x[i] = yi;
              }
            }
            mh[l] = h;
            ml[l] = m;
          }
          at_hi |= lane_or64(mh);
          at_lo |= lane_or64(ml);
          PK_WSYNC();
          continue;
        }
        step = fmaxf(step, 0.f);
        const bool blk_hi = y[blk] > hi[blk];
        PK_WSYNC();
        PK_LANES(l) {
          #pragma unroll 1
          for (int i = l; i < n; i += 32) {
            if (!((act >> i) & 1ull)) {
              float xi = fmaf(step, y[i] - x[i], x[i]);
              if (i == blk) xi = blk_hi ? hi[i] : lo[i];
              x[i] = xi;
            }
          }
        }
        PK_WSYNC();
        if (blk_hi) at_hi |= (1ull << blk); else at_lo |= (1ull << blk);
        if (((released >> blk) & 1ull) && step <= 1e-6f) tabu |= (1ull << blk);
        continue;
      }
      PK_LANES(l) {
        #pragma unroll 1
        for (int i = l; i < n; i += 32) x[i] = y[i];
      }
      PK_WSYNC();
      // multipliers from the factored gradient: rho = A x + b (row-parallel) ...
      PK_LANES(l) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = l + 32 * h;
          if (r < K) {
            const float* Ar = A + r * L.lda;
            float s = bv[r];
#pragma unroll 4
            for (int j = 0; j < n; ++j) s = fmaf(Ar[j], x[j], s);
            rho[r] = s;
          }
        }
      }
      PK_WSYNC();
      // ... g_i = A[:, i] . rho + d_i (d_i x_i + beta_i) (column-parallel)
      float worst;
      int rel;
      uint64_t neg;
      {
        LaneVar<float> wv;
        LaneVar<int> wi;
        LaneVar<uint64_t> nm;
        PK_LANES(l) {
          float best = 0.f;
          int bi = 0x7fffffff;
          uint64_t m = 0ull;
          #pragma unroll 1
          for (int i = l; i < n; i += 32) {
            if (((act & ~tabu) >> i) & 1ull) {
              const float rt = fmaf(dv[i], x[i], beta[i]);
              float g = dv[i] * rt;
              float gabs = fabsf(g);
#pragma unroll 4
              for (int r = 0; r < K; ++r) {
                const float a = A[r * L.lda + i];
                g = fmaf(a, rho[r], g);
                gabs = fmaf(fabsf(a), fabsf(rho[r]), gabs);
              }
              const float lam = ((at_hi >> i) & 1ull) ? -g : g;
              if (lam < -4e-6f * gabs) {
                m |= (1ull << i);
                if (lam < best) { best = lam; bi = i; }
              }
            }
          }
          wv[l] = best;
          wi[l] = bi;
          nm[l] = m;
        }
        lane_argmin(wv, wi, worst, rel);
        neg = lane_or64(nm);
      }
      if (neg == 0ull) break;
      const uint64_t drop = (it < kMultiChange) ? neg : (1ull << rel);
      if (it >= kMultiChange) released |= drop;
      at_hi &= ~drop;
      at_lo &= ~drop;
    }
    return status;
  }

  // ---- the whole step ----------------------------------------------------------------
  // ERR (converge): also the stop test `ct` on the task errors, reduced across the warp and made
  // before the rows of A; a step that stops there, or whose instance is outside its limits with
  // safety_break, returns with v = 0.  ct->status is the step's status on every lane.  Test: the
  // stop rule, ct->decide(err), called by the whole warp (ConvergeTest: this instance's own; the
  // multi-start kernel's decides for the CTA's group of seeds, with a barrier).
  template <bool ERR = false, class Test = ConvergeTest>
  static PK_HD void run(const DevModel& M, const DevProblem& P, const TreePlan& L, const float* __restrict__ qg,
                        const float* __restrict__ tg, float* W, float* __restrict__ vg, int32_t* status_out,
                        Test* ct = nullptr) {
    const int nj = L.nj, nv = L.nv, rq = L.rq, rv = L.rv;
    float* qs = W + L.o_q;
    float* ts = W + L.o_t;
    float* A = W + L.o_A;
    // ---- load q and targets (coalesced), limit check --------------------------------
    int status = 0;
    {
      LaneVar<int> bad;
      PK_LANES(l) {
        #pragma unroll 1
        for (int i = l; i < L.nq; i += 32) qs[i] = qg[i];
        #pragma unroll 1
        for (int i = l; i < L.stride; i += 32) ts[i] = tg[i];
        int f = 0;
        #pragma unroll 1
        for (int i = rv + l; i < nv; i += 32) {
          const float qi = qg[i + rq - rv];
          if (qi < P.chk_lo[i] || qi > P.chk_hi[i]) f = 1;
        }
        bad[l] = f;
      }
      PK_WSYNC();
      if (lane_or(bad)) status |= PK_STATUS_OUT_OF_LIMITS;
    }
    if (!ERR && status && P.safety_break) {
      PK_LANES(l) {
        #pragma unroll 1
        for (int i = l; i < nv; i += 32) vg[i] = 0.f;
        if (l == 0 && status_out) *status_out = status;
      }
      return;
    }
    // ---- forward kinematics: local transforms in registers, tree sweep by depth ------
    {
      LaneVar<SE3f> Tl;
      PK_LANES(l) {
        if (l == 0) {
          SE3f root = identity_se3();
          if (M.free_flyer) {
            root.p = v3(qs[0], qs[1], qs[2]);
            root.R = quat_to_matrix(qs[3], qs[4], qs[5], qs[6]);
          }
          store_se3(root, W + L.o_root);
        }
        if (l < nj) {
          const SE3f X = load_se3(M.jX + 12 * l);
          const V3 axis = v3(M.axis[3 * l], M.axis[3 * l + 1], M.axis[3 * l + 2]);
          SE3f T;
          if (M.jtype[l] == PK_JOINT_REVOLUTE) {
            float s, c;
            sincos_f(qs[rq + l], &s, &c);
            T.R = mul(X.R, rot_axis(axis, s, c));
            T.p = X.p;
          } else {
            T.R = X.R;
            T.p = X.p + mul(X.R, qs[rq + l] * axis);
          }
          Tl[l] = T;
        }
      }
      PK_WSYNC();
      for (int dep = 0; dep <= L.maxdepth; ++dep) {
        PK_LANES(l) {
          if (l < nj && M.depth[l] == dep) {
            const int par = M.parent[l];
            const SE3f Tp = load_tw(W, L, par < 0 ? -1 : par);
            store_se3(compose(Tp, Tl[l]), W + L.o_tw + kTwStride * l);
          }
        }
        PK_WSYNC();
      }
    }
    // world CoM of every body (only if a CoM task exists)
    bool has_com = false;
    const int nt = P.ntasks + L.nct;  // objective tasks, then the tasks used as equality constraints
    auto task_at = [&](int t) -> const DevTask& { return t < P.ntasks ? P.tasks[t] : P.ext->constraints[t - P.ntasks]; };
    #pragma unroll 1
    for (int t = 0; t < nt; ++t) has_com = has_com || (task_at(t).type == PK_TASK_COM);
    if (has_com) {
      PK_LANES(l) {
        for (int b = l; b <= nj; b += 32) {  // index b: body b - 1
          const SE3f T = load_tw(W, L, b - 1);
          const V3 cl = v3(M.com[3 * b], M.com[3 * b + 1], M.com[3 * b + 2]);
          const V3 c = mul(T.R, cl) + T.p;
          W[L.o_cw + 3 * b] = c.x; W[L.o_cw + 3 * b + 1] = c.y; W[L.o_cw + 3 * b + 2] = c.z;
        }
      }
      PK_WSYNC();
    }
    // ---- per-task quantities, one task per lane ------------------------------------------
    PK_LANES(l) {
      if (l < nt) {
        const DevTask& Kt = task_at(l);
        float* F = W + L.o_tf + kTreeTaskWords * l;
        const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (ts + Kt.tgt_off);
        if (Kt.type == PK_TASK_FRAME || Kt.type == PK_TASK_RELATIVE_FRAME) {
          const SE3f Tf = compose(load_tw(W, L, Kt.body), load_se3(M.fX + 12 * Kt.frame));
          const SE3f Tt = load_se3(tgt);
          M3 Am, Bm;
          float e[6];
          SE3f Tr = identity_se3(), Trf = identity_se3();
          if (Kt.type == PK_TASK_FRAME) {
            const SE3f Tbt = act_inv(Tf, Tt);
            Log3 Lg = log3(Tbt.R);
            log6(Tbt, Lg, e);
            SE3f Ttb;
            for (int a = 0; a < 3; ++a)
              for (int c = 0; c < 3; ++c) Ttb.R.m[3 * a + c] = Tbt.R.m[3 * c + a];
            Ttb.p = -1.f * mul(Ttb.R, Tbt.p);
            Lg.w = -1.f * Lg.w;
            jlog6(Ttb, Lg, Am, Bm);
          } else {
            Tr = compose(load_tw(W, L, Kt.root_body), load_se3(M.fX + 12 * Kt.root));
            Trf = act_inv(Tr, Tf);
            const SE3f Ttf = act_inv(Tt, Trf);
            const Log3 Lg = log3(Ttf.R);
            log6(Ttf, Lg, e);
            jlog6(Ttf, Lg, Am, Bm);
          }
          store_se3(Tf, F);
          for (int k = 0; k < 9; ++k) { F[12 + k] = Am.m[k]; F[21 + k] = Bm.m[k]; }
          for (int k = 0; k < 6; ++k) F[30 + k] = e[k];
          store_se3(Tr, F + 36);
          store_se3(Trf, F + 48);
        } else if (Kt.type == PK_TASK_LINEAR) {
          // e = A (q - q_0) - b on the joint coordinates (pink/tasks/linear_holonomic_task.py:148-166)
          const float* Al = P.ext->extra + Kt.data_off;
          const float* bl = Al + Kt.rows * nv;
          const float* q0 = bl + Kt.rows;
          #pragma unroll 1
          for (int r = 0; r < 6; ++r) {
            float sacc = 0.f;
            if (r < Kt.rows) {
              sacc = -bl[r];
              #pragma unroll 1
              for (int i = rv; i < nv; ++i) sacc = fmaf(Al[r * nv + i], qs[i + rq - rv] - q0[i + rq - rv], sacc);
            }
            F[30 + r] = sacc;
          }
        } else if (Kt.type == PK_TASK_COM) {
          V3 acc = v3(0.f, 0.f, 0.f);
          for (int b = 0; b <= nj; ++b) {
            const float m = M.mass[b];
            acc = acc + m * v3(W[L.o_cw + 3 * b], W[L.o_cw + 3 * b + 1], W[L.o_cw + 3 * b + 2]);
          }
          const V3 cm = (1.f / M.total_mass) * acc;
          F[0] = cm.x; F[1] = cm.y; F[2] = cm.z;
          F[30] = cm.x - tgt[0]; F[31] = cm.y - tgt[1]; F[32] = cm.z - tgt[2];
          F[33] = F[34] = F[35] = 0.f;
        }
      }
    }
    PK_WSYNC();
    if constexpr (ERR) {
      // the stop test: |e_t|_2 of the selected tasks, the diagonal ones summed across the lanes
      float emax = 0.f;
      #pragma unroll 1
      for (int t = 0; t < P.ntasks; ++t) {
        if (!((ct->mask >> t) & 1u)) continue;
        const DevTask& Kt = P.tasks[t];
        float n2 = 0.f;
        if (is_diag_task(Kt.type)) {
          const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (ts + Kt.tgt_off);
          LaneVar<float> part;
          PK_LANES(l) {
            float s = 0.f;
            #pragma unroll 1
            for (int i = rv + l; i < nv; i += 32) {
              const float e = diag_task_error(Kt.type, qs, tgt, i, rq, rv);
              s = fmaf(e, e, s);
            }
            part[l] = s;
          }
          n2 = lane_sum(part);
        } else {
          const float* F = W + L.o_tf + kTreeTaskWords * t;
          const int k = (Kt.type == PK_TASK_COM) ? 3 : (Kt.type == PK_TASK_LINEAR ? Kt.rows : 6);
          #pragma unroll 1
          for (int r = 0; r < k; ++r) n2 = fmaf(F[30 + r], F[30 + r], n2);
        }
        emax = err_max(emax, sqrtf(n2));
      }
      ct->decide(emax);
      ct->status = status;
      if (ct->stop || (status && P.safety_break)) {
        PK_LANES(l) {
          #pragma unroll 1
          for (int i = l; i < nv; i += 32) vg[i] = 0.f;
        }
        return;
      }
    }
    // ---- rows of A (column-parallel), b, diagonal terms -----------------------------------
    float diag = P.damping;
    int erow = 0;  // next equality row
    #pragma unroll 1
    for (int t = 0; t < nt; ++t) {
      const DevTask& Kt = task_at(t);
      const float* F = W + L.o_tf + kTreeTaskWords * t;
      const bool as_constraint = t >= P.ntasks;  // J dq = -gain e (pink/solve_ik.py:143-148)
      if (is_diag_task(Kt.type)) {
        const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (ts + Kt.tgt_off);
        const float w2 = Kt.cost[0] * Kt.cost[0];
        LaneVar<float> part;
        PK_LANES(l) {
          float s = 0.f;
          #pragma unroll 1
          for (int i = rv + l; i < nv; i += 32) {
            const float e = diag_task_error(Kt.type, qs, tgt, i, rq, rv);
            s = fmaf(e, e, s);
          }
          part[l] = s;
        }
        diag = fmaf(Kt.lm * Kt.gain * Kt.gain * w2, lane_sum(part), diag);
        continue;
      }
      const int k = (Kt.type == PK_TASK_COM) ? 3 : (Kt.type == PK_TASK_LINEAR ? Kt.rows : 6);
      int base;
      if (as_constraint) {
        base = erow;
        erow += k;
      } else {
        float mu = 0.f;
        #pragma unroll 1
        for (int r = 0; r < k; ++r) {
          const float ew = Kt.cost[r] * Kt.gain * F[30 + r];
          mu = fmaf(ew, ew, mu);
        }
        diag = fmaf(Kt.lm, mu, diag);
        base = L.row_base[t];
        if (base < 0) continue;
      }
      PK_LANES(l) {
        // b entries of this task (rows with non-zero cost are packed in order)
        if (l == 0) {
          int row = base;
          #pragma unroll 1
          for (int r = 0; r < k; ++r) {
            if (as_constraint) W[L.o_fe + row++] = -Kt.gain * F[30 + r];
            else if (Kt.cost[r] != 0.f) W[L.o_b + row++] = Kt.cost[r] * Kt.gain * F[30 + r];
          }
        }
        #pragma unroll 1
        for (int i = l; i < nv; i += 32) {
          float col[6];
          if (Kt.type == PK_TASK_LINEAR) {
            const float* Al = P.ext->extra + Kt.data_off;
            #pragma unroll 1
            for (int r = 0; r < 6; ++r) col[r] = (r < Kt.rows) ? Al[r * nv + i] : 0.f;
          } else if (Kt.type == PK_TASK_COM) {
            const V3 cm = v3(F[0], F[1], F[2]);
            V3 c = v3(0.f, 0.f, 0.f);
            if (i < rv) {
              const SE3f root = load_se3(W + L.o_root);
              const V3 ek = v3(i % 3 == 0 ? 1.f : 0.f, i % 3 == 1 ? 1.f : 0.f, i % 3 == 2 ? 1.f : 0.f);
              if (i < 3) c = mul(root.R, ek);
              else c = mul(root.R, cross(ek, mulT(root.R, cm - root.p)));
            } else {
              const int j = i - rv;
              float sm = 0.f;
              V3 smc = v3(0.f, 0.f, 0.f);
              for (int b = 1; b <= nj; ++b) {
                if ((M.anc[b + 1] >> j) & 1ull) {
                  const float m = M.mass[b];
                  sm += m;
                  smc = smc + m * v3(W[L.o_cw + 3 * b], W[L.o_cw + 3 * b + 1], W[L.o_cw + 3 * b + 2]);
                }
              }
              if (sm > 0.f) {
                const SE3f Tj = load_se3(W + L.o_tw + kTwStride * j);
                const V3 axis = v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]);
                const V3 aw = mul(Tj.R, axis);
                const float invM = 1.f / M.total_mass;
                if (M.jtype[j] == PK_JOINT_REVOLUTE) c = (sm * invM) * cross(aw, (1.f / sm) * smc - Tj.p);
                else c = (sm * invM) * aw;
              }
            }
            col[0] = c.x; col[1] = c.y; col[2] = c.z; col[3] = col[4] = col[5] = 0.f;
          } else {
            const SE3f Tf = load_se3(F);
            M3 Am, Bm;
            for (int q9 = 0; q9 < 9; ++q9) { Am.m[q9] = F[12 + q9]; Bm.m[q9] = F[21 + q9]; }
            V3 lin, ang;
            jac_col(M, W, L, Kt.body, Tf, i, lin, ang);
            float sign = -1.f;
            if (Kt.type == PK_TASK_RELATIVE_FRAME) {
              const SE3f Tr = load_se3(F + 36);
              const SE3f Trf = load_se3(F + 48);
              V3 rl, ra;
              jac_col(M, W, L, Kt.root_body, Tr, i, rl, ra);
              lin = lin - mulT(Trf.R, rl - cross(Trf.p, ra));
              ang = ang - mulT(Trf.R, ra);
              sign = 1.f;
            }
            const V3 tl = sign * (mul(Am, lin) + mul(Bm, ang));
            const V3 ta = sign * mul(Am, ang);
            col[0] = tl.x; col[1] = tl.y; col[2] = tl.z; col[3] = ta.x; col[4] = ta.y; col[5] = ta.z;
          }
          int row = base;
          #pragma unroll 1
          for (int r = 0; r < k; ++r) {
            if (as_constraint) W[L.o_E + (row++) * L.lda + i] = col[r];
            else if (Kt.cost[r] != 0.f) A[(row++) * L.lda + i] = Kt.cost[r] * col[r];
          }
        }
      }
    }
    // ---- dense inequality rows of the barriers (pink/barriers/*.py), column-parallel ------
    // G = -J_h / dt, h = gain * alpha(h(q)) (barrier.py:246-252); the safe-displacement
    // term adds safe_gain / |J_h|_F^2 to the diagonal (barrier.py:193-203).  Same
    // arithmetic as Generic::barrier_rows.
    if (L.p > 0) {
      const DevExtras& X = *P.ext;
      int prow = 0;
      if (X.fb_enabled) {
        // FloatingBaseVelocityLimit (pink/limits/floating_base_velocity_limit.py:118-148):
        // +-J_frame[:, root] dq <= dt * twist_max, rows with an infinite bound dropped
        const SE3f Tf = compose(load_tw(W, L, X.fb_body), load_se3(M.fX + 12 * X.fb_frame));
        int nfin = 0;
        #pragma unroll 1
        for (int r = 0; r < 6; ++r) nfin += (X.fb_max[r] < 3.0e38f) ? 1 : 0;
        float* Gb = W + L.o_G;
        float* hb = W + L.o_hg;
        PK_LANES(l) {
          #pragma unroll 1
          for (int i = l; i < nv; i += 32) {
            V3 lin = v3(0.f, 0.f, 0.f), ang = v3(0.f, 0.f, 0.f);
            if (i < rv) jac_col(M, W, L, X.fb_body, Tf, i, lin, ang);
            const float col[6] = {lin.x, lin.y, lin.z, ang.x, ang.y, ang.z};
            int rr = 0;
            #pragma unroll 1
            for (int r = 0; r < 6; ++r)
              if (X.fb_max[r] < 3.0e38f) {
                Gb[rr * L.lda + i] = col[r];
                Gb[(nfin + rr) * L.lda + i] = -col[r];
                ++rr;
              }
          }
          if (l == 0) {
            int rr = 0;
            for (int r = 0; r < 6; ++r)
              if (X.fb_max[r] < 3.0e38f) {
                hb[rr] = hb[nfin + rr] = P.dt * X.fb_max[r];
                ++rr;
              }
          }
        }
        prow += 2 * nfin;
        PK_WSYNC();
      }
      #pragma unroll 1
      for (int bi = 0; bi < X.nbarriers; ++bi) {
        const DevBarrier& Bd = X.barriers[bi];
        float* Gb = W + L.o_G + prow * L.lda;
        float* hb = W + L.o_hg + prow;
        LaneVar<float> fro;
        PK_LANES(l) { fro[l] = 0.f; }
        if (Bd.type == PK_BARRIER_POSITION) {
          const SE3f Tf = compose(load_tw(W, L, Bd.body), load_se3(M.fX + 12 * Bd.frame));
          PK_LANES(l) {
            const float pw[3] = {Tf.p.x, Tf.p.y, Tf.p.z};
            if (l == 0) {
              int r = 0;
              if (Bd.has_min)
                for (int k = 0; k < Bd.nidx; ++k, ++r)
                  hb[r] = Bd.gain[r] * Generic<1, 1>::barrier_gain_fn(Bd.gain_fn, pw[Bd.idx[k]] - Bd.p_min[k]);
              if (Bd.has_max)
                for (int k = 0; k < Bd.nidx; ++k, ++r)
                  hb[r] = Bd.gain[r] * Generic<1, 1>::barrier_gain_fn(Bd.gain_fn, Bd.p_max[k] - pw[Bd.idx[k]]);
            }
            float f = 0.f;
            #pragma unroll 1
            for (int i = l; i < nv; i += 32) {
              V3 lin, ang;
              jac_col(M, W, L, Bd.body, Tf, i, lin, ang);
              const V3 c = mul(Tf.R, lin);
              const float cw[3] = {c.x, c.y, c.z};
              int r = 0;
              if (Bd.has_min)
                for (int k = 0; k < Bd.nidx; ++k, ++r) { Gb[r * L.lda + i] = -cw[Bd.idx[k]] * P.inv_dt; f = fmaf(cw[Bd.idx[k]], cw[Bd.idx[k]], f); }
              if (Bd.has_max)
                for (int k = 0; k < Bd.nidx; ++k, ++r) { Gb[r * L.lda + i] = cw[Bd.idx[k]] * P.inv_dt; f = fmaf(cw[Bd.idx[k]], cw[Bd.idx[k]], f); }
            }
            fro[l] = f;
          }
        } else if (Bd.type == PK_BARRIER_BODY_SPHERICAL) {
          const SE3f T1 = compose(load_tw(W, L, Bd.body), load_se3(M.fX + 12 * Bd.frame));
          const SE3f T2 = compose(load_tw(W, L, Bd.body2), load_se3(M.fX + 12 * Bd.frame2));
          const V3 dp = T1.p - T2.p;
          PK_LANES(l) {
            if (l == 0) hb[0] = Bd.gain[0] * Generic<1, 1>::barrier_gain_fn(Bd.gain_fn, dot(dp, dp) - Bd.d_min * Bd.d_min);
            float f = 0.f;
            #pragma unroll 1
            for (int i = l; i < nv; i += 32) {
              V3 l1, a1, l2, a2;
              jac_col(M, W, L, Bd.body, T1, i, l1, a1);
              jac_col(M, W, L, Bd.body2, T2, i, l2, a2);
              const float jh = Generic<1, 1>::rigid_for_both(M, Bd.body, Bd.body2, i)
                                   ? 0.f
                                   : 2.f * dot(dp, mul(T1.R, l1) - mul(T2.R, l2));
              Gb[i] = -jh * P.inv_dt;
              f = fmaf(jh, jh, f);
            }
            fro[l] = f;
          }
        } else {
          // SELF_COLLISION on sphere pairs: the `dim` smallest distances
          float* dist = W + L.o_dist;
          const int* pr = X.pairs + 2 * Bd.pair_off;
          const float* rad = X.extra + Bd.data_off;
          PK_LANES(l) {
            #pragma unroll 1
            for (int k = l; k < Bd.npairs; k += 32) {
              const int fa = pr[2 * k], fb = pr[2 * k + 1];
              const SE3f Ta = load_tw(W, L, M.frame_body[fa]);
              const SE3f Tb = load_tw(W, L, M.frame_body[fb]);
              const V3 ca = mul(Ta.R, v3(M.fX[12 * fa + 3], M.fX[12 * fa + 7], M.fX[12 * fa + 11])) + Ta.p;
              const V3 cb = mul(Tb.R, v3(M.fX[12 * fb + 3], M.fX[12 * fb + 7], M.fX[12 * fb + 11])) + Tb.p;
              const V3 dp = ca - cb;
              dist[k] = sqrtf(dot(dp, dp)) - rad[2 * k] - rad[2 * k + 1];
            }
          }
          PK_WSYNC();
          #pragma unroll 1
          for (int r = 0; r < Bd.dim; ++r) {
            float bd;
            int best;
            {
              LaneVar<float> dvl;
              LaneVar<int> dil;
              PK_LANES(l) {
                float b0 = 3.0e38f;
                int bi0 = 0x7fffffff;
                #pragma unroll 1
                for (int k = l; k < Bd.npairs; k += 32)
                  if (dist[k] < b0) { b0 = dist[k]; bi0 = k; }
                dvl[l] = b0;
                dil[l] = bi0;
              }
              lane_argmin(dvl, dil, bd, best);
            }
            const bool have = best != 0x7fffffff;
            SE3f Ta = identity_se3(), Tb = identity_se3();
            int ba = -2, bb = -2;
            if (have) {
              const int fa = pr[2 * best], fb = pr[2 * best + 1];
              ba = M.frame_body[fa];
              bb = M.frame_body[fb];
              Ta = compose(load_tw(W, L, ba), load_se3(M.fX + 12 * fa));
              Tb = compose(load_tw(W, L, bb), load_se3(M.fX + 12 * fb));
            }
            const V3 dp = Ta.p - Tb.p;
            const float gap = sqrtf(dot(dp, dp));
            const bool zero = !have || !(gap > 0.f) || fabsf(bd) <= 1e-8f;
            const V3 nrm = zero ? v3(0.f, 0.f, 0.f) : ((bd < 0.f ? -1.f : 1.f) / gap) * dp;
            PK_WSYNC();
            PK_LANES(l) {
              if (l == 0) {
                hb[r] = Bd.gain[0] * Generic<1, 1>::barrier_gain_fn(Bd.gain_fn, bd - Bd.d_min);
                if (have) dist[best] = 3.0e38f;  // taken
              }
              float f = fro[l];
              #pragma unroll 1
              for (int i = l; i < nv; i += 32) {
                float jh = 0.f;
                if (!zero && !Generic<1, 1>::rigid_for_both(M, ba, bb, i)) {
                  V3 l1, a1, l2, a2;
                  jac_col(M, W, L, ba, Ta, i, l1, a1);
                  jac_col(M, W, L, bb, Tb, i, l2, a2);
                  jh = dot(nrm, mul(Ta.R, l1) - mul(Tb.R, l2));
                }
                Gb[r * L.lda + i] = -jh * P.inv_dt;
                f = fmaf(jh, jh, f);
              }
              fro[l] = f;
            }
            PK_WSYNC();
          }
        }
        const float fr = lane_sum(fro);
        if (Bd.safe_gain > 1e-6f) diag += Bd.safe_gain / fr;
        prow += Bd.dim;
        PK_WSYNC();
      }
    }
    // diagonal terms (posture tasks), box
    PK_LANES(l) {
      #pragma unroll 1
      for (int i = l; i < nv; i += 32) {
        float pw2 = 0.f, pc = 0.f;
        const float qi = (i >= rv) ? qs[i + rq - rv] : 0.f;
        #pragma unroll 1
        for (int t = 0; t < P.ntasks; ++t) {
          const DevTask& Kt = P.tasks[t];
          if (is_diag_task(Kt.type) && i >= rv) {
            const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (ts + Kt.tgt_off);
            const float w2 = Kt.cost[0] * Kt.cost[0];
            pw2 += w2;
            pc = fmaf(Kt.gain * w2, diag_task_error(Kt.type, qs, tgt, i, rq, rv), pc);
          }
        }
        const float dd = sqrtf(pw2 + diag);
        W[L.o_d + i] = dd;
        W[L.o_beta + i] = dd > 0.f ? pc / dd : 0.f;
        const float vb = P.dt * P.vel[i];
        float hb = fminf(P.cfg_gain * (P.cfg_hi[i] - qi), vb);
        float lb = fmaxf(P.cfg_gain * (P.cfg_lo[i] - qi), -vb);
        if (P.ext && P.ext->acc_enabled) {
          // AccelerationLimit (pink/limits/acceleration_limit.py:119-200): a box as well
          const DevExtras& X = *P.ext;
          const float a = X.acc_max[i];
          if (a < 3.0e38f) {
            const float pv = X.acc_prev_off >= 0 ? ts[X.acc_prev_off + i] : 0.f;
            const float up = X.acc_qhi[i] - qi, dn = qi - X.acc_qlo[i];
            if (up < 0.f || dn < 0.f) hb = -INFINITY;  // NaN rows in the reference: empty box -> no solution
            const float dt2 = P.dt * P.dt;
            hb = fminf(hb, fminf(fmaf(a, dt2, pv), (up < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(up, 0.f)) : INFINITY));
            lb = fmaxf(lb, -fminf(fmaf(a, dt2, -pv), (dn < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(dn, 0.f)) : INFINITY));
          }
        }
        W[L.o_hi + i] = hb;
        W[L.o_lo + i] = lb;
      }
    }
    PK_WSYNC();
    // ---- QP -------------------------------------------------------------------------------
    status |= (L.p > 0 || L.meq > 0) ? tree_dual_solve(W, L) : solve_qp(W, L);
    PK_LANES(l) {
      #pragma unroll 1
      for (int i = l; i < nv; i += 32) vg[i] = W[L.o_x + i] * P.inv_dt;
      if (l == 0 && status_out) *status_out = status;
    }
    if constexpr (ERR) ct->status = status;
  }

  // Solve to a tolerance (pk_converge_prepared), one instance per warp; the loop of
  // converge_chain (pk_chain.cuh) with run<true>.  qg [nq]: in q_0, out where the instance stopped
  // (updated in place by lane 0); vg [nv]: scratch.  err, steps and status are the same on every
  // lane, so the warp leaves the loop together.
  static PK_HD void converge(const DevModel& M, const DevProblem& P, const TreePlan& L, float* qg, const float* tg,
                             float* W, float* vg, unsigned mask, float tol, int max_steps, float& err, int& steps,
                             int& status_out) {
    int st_all = 0;
    int s = 0;
    #pragma unroll 1
    for (;; ++s) {
      ConvergeTest ct{mask, tol, s == max_steps, 0.f, false, 0};
      run<true>(M, P, L, qg, tg, W, vg, nullptr, &ct);
      PK_WSYNC();
      err = ct.err;
      if (ct.stop) break;
      st_all |= ct.status;
      if (step_failed(st_all, P.safety_break)) {
        ++s;
        break;
      }
      PK_LANES(l) {
        if (l == 0) integrate_configuration(L.nq, M.free_flyer, qg, vg, P.dt, qg);
      }
      PK_WSYNC();
    }
    steps = s;
    status_out = st_all;
  }

  // Closed-loop rollout of instance i, one instance per warp (ik_tree_rollout_kernel): n_steps
  // iterations of run and q (+) v dt on qg [nq] in place (by lane 0), the targets row of step s at
  // targets + s T.target_step + i L.stride, the records of T after every step.  A step that fails
  // the freeze rule is recorded without moving q and ends the loop; the remaining steps are
  // recorded with q unchanged and v = 0.  vg [nv]: the last step's velocity.  Returns the OR of
  // the statuses of the steps that ran, the same on every lane.
  static PK_HD int rollout(const DevModel& M, const DevProblem& P, const TreePlan& L, float* qg, const float* targets,
                           float* W, float* vg, int n_steps, const Trajectory& T, int64_t B, int64_t i) {
    int st_all = 0;
    int s = 0;
    while (s < n_steps) {
      int32_t st = 0;
      run(M, P, L, qg, targets ? targets + s * T.target_step + i * (int64_t)L.stride : nullptr, W, vg, &st);
      PK_WSYNC();
      st = lane0_int(st);  // run() reports through lane 0
      st_all |= st;
      const bool failed = step_failed(st, P.safety_break);
      PK_LANES(l) {
        if (!failed && l == 0) integrate_configuration(L.nq, M.free_flyer, qg, vg, P.dt, qg);
      }
      PK_WSYNC();
      const int recorded = s++;  // advanced before the stores: 4 B fewer spill loads than after them
      PK_LANES(l) record_rows(T, recorded, B, i, L.nq, L.nv, qg, vg, st_all, false, l, 32);
      if (failed) break;
    }
    for (; s < n_steps; ++s)
      PK_LANES(l) record_rows(T, s, B, i, L.nq, L.nv, qg, vg, st_all, true, l, 32);
    return st_all;
  }

  // Instance i of the one-instance-per-warp kernels, W its warp's workspace.  ik_tree_kernel: run on
  // q row i into v row i and status[i] (unless null).
  static PK_HD void solve_instance(const DevModel& M, const DevProblem& P, const TreePlan& L, const float* __restrict__ q,
                                   const float* __restrict__ targets, float* W, float* __restrict__ v,
                                   int32_t* __restrict__ status, int64_t i) {
    run(M, P, L, q + i * L.nq, targets ? targets + i * (int64_t)L.stride : nullptr, W, v + i * L.nv,
        status ? status + i : nullptr);
  }

  // ik_tree_rollout_kernel: q row i into q_out row i, rollout there in place with v row i, then the
  // status (unless null).
  static PK_HD void rollout_instance(const DevModel& M, const DevProblem& P, const TreePlan& L,
                                     const float* __restrict__ q, const float* __restrict__ targets, int n_steps,
                                     float* __restrict__ q_out, float* W, float* __restrict__ v,
                                     int32_t* __restrict__ status, const Trajectory& T, int64_t B, int64_t i) {
    float* qrow = q_out + i * L.nq;
    PK_LANES(l) for (int k = l; k < L.nq; k += 32) qrow[k] = q[i * L.nq + k];
    PK_WSYNC();
    const int st_all = rollout(M, P, L, qrow, targets, W, v + i * L.nv, n_steps, T, B, i);
    PK_LANES(l) if (status && l == 0) status[i] = st_all;
  }

  // ik_tree_converge_kernel: q row i into q_out row i (q_out may alias q), converge there in place
  // with the step's v at word o_v of W (converge_tree_layout), then err, steps and status (each
  // unless null).
  static PK_HD void converge_instance(const DevModel& M, const DevProblem& P, const TreePlan& L, int o_v,
                                      const float* q, const float* __restrict__ targets, unsigned mask, float tol,
                                      int max_steps, float* q_out, float* W, float* __restrict__ err,
                                      int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t i) {
    float* qrow = q_out + i * L.nq;
    PK_LANES(l) for (int k = l; k < L.nq; k += 32) qrow[k] = q[i * L.nq + k];
    PK_WSYNC();
    float e;
    int n, st;
    converge(M, P, L, qrow, targets ? targets + i * (int64_t)L.stride : nullptr, W, W + o_v, mask, tol, max_steps, e,
             n, st);
    PK_LANES(l) {
      if (l == 0) {
        if (err) err[i] = e;
        if (steps) steps[i] = n;
        if (status) status[i] = st;
      }
    }
  }
};

}  // namespace pk
