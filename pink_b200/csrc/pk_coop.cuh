// One IK step of a fixed-base serial chain with L lanes per robot instance
// (L = 1: one instance per thread; L = 2, 4, 8: a sub-warp group per instance).
//
// Path (reference file:line), same as pk_chain.cuh:
//   Configuration.check_limits            pink/configuration.py:181-201
//   FK + LOCAL frame Jacobian             pink/configuration.py:163-164, 233-235
//   FrameTask error / Jacobian            pink/tasks/frame_task.py:176-227
//   PostureTask error / Jacobian          pink/tasks/posture_task.py:100-129
//   Task.compute_qp_objective             pink/tasks/task.py:145-166
//   H = damping I + sum H_t, c = sum c_t  pink/solve_ik.py:55-60
//   ConfigurationLimit / VelocityLimit    pink/limits/configuration_limit.py:108-121,
//                                         pink/limits/velocity_limit.py:115-121
//   QP solve, v = dq / dt                 pink/solve_ik.py:270-275
//
// What is different from the round-1 kernel (pk_chain.cuh), and why (DESIGN.md section 3.1):
//  * Joint frames are re-oriented on the host so that every joint axis is the local z axis
//    (T~_j = oMi[j] A_j with A_j e_z = a_j; origins and world axes are unchanged).  A joint then
//    costs one constant compose and a 2x2 rotation of two columns; the world axis is a column
//    of the running transform.
//  * The chain is cut into L contiguous SEGMENTS of NC = ceil(NJ / L) joints, one per lane.
//    A lane runs forward kinematics of its segment in the segment's own base frame; LOCAL
//    frame Jacobian columns are invariant under the choice of base frame, so a lane needs
//    only (a) its own prefix transforms and (b) the pose of the task frame relative to its
//    segment base, which is a suffix product over the lanes (log2 L shuffle + compose steps).
//    Only the frame pose in the world (lane 0's suffix product) is broadcast, for the error.
//  * The task rows A = W J are stored by COLUMN on the lane that owns the joint, so that
//    c = A^T b, g = A^T rho, and the Gram entries the QP needs are lane-local dot products;
//    rho = A x + b is the only group reduction, done once (afterwards it is updated with the
//    replicated free columns).
//  * QP: primal active set from the box corner, as BoxLSQChol, but as ONE loop over
//    release / solve / ratio-test iterations on up to two free coordinates whose columns are
//    replicated in the group; anything that needs a third free coordinate gathers the problem
//    and runs the Cholesky rounds of pk_lsq.cuh (replicated on the group's lanes).
#pragma once

#include "pk_group.cuh"
#include "pk_lsq.cuh"

namespace pk {

constexpr int kCoopMaxFrameTasks = 2;

// Per-joint constants, 6 x float4 so that a lane can fetch them with 128-bit loads from
// shared memory (lane-varying joint index when L > 1).
struct alignas(16) CoopJoint {
  float Xr[9];  // rotation of the z-aligned placement X~_j = A_{j-1}^T X_j A_j (row-major)
  float Xp[3];  // its translation A_{j-1}^T X_j.p
  float prismatic;  // 1.0 prismatic, 0.0 revolute
  float cfg_lo, cfg_hi, vel;  // q_min, q_max, dt * v_max (box: lo = max(gain (q_min - q), -vel), hi = min(gain (q_max - q), vel))
  float chk_lo, chk_hi;
  float acc_max, acc_qlo, acc_qhi;
  float valid;  // 0 for padding joints beyond NJ
  float pad[2];
};
static_assert(sizeof(CoopJoint) == 96, "CoopJoint must be 6 float4");

struct CoopFrameTask {
  int body;       // joint index the frame is fixed to (-1: world)
  float X[12];    // frame placement in the z-aligned frame of that joint, row-major [R | p]
  float cost[6];  // [pos(3), ori(3)]
  float gain, lm;
  int tgt_off;
  int tgt_shared;
};

// NJP = L * NC joints (padded with identity joints)
template <int NJP>
struct CoopParams {
  CoopJoint joint[NJP];
  int n_frame_tasks;
  CoopFrameTask ft[kCoopMaxFrameTasks];
  int has_posture;
  float posture_w2, posture_gain, posture_lm;
  int posture_off, posture_shared;
  float dt, inv_dt, damping;
  float cfg_gain;
  int target_stride;
  int target_vec4;  // every per-instance frame target is 16-byte aligned (stride and offsets multiples of 4 floats)
  int safety_break;
  float shared[12 * kCoopMaxFrameTasks + NJP];
  int acc_enabled, acc_prev_off;
  int any_prismatic;    // 0: every joint is revolute (the common case skips the per-joint selects)
  int frames_on_last;   // 1: every frame task sits on the last joint (no mid-chain / world frames)
};

template <int NJ, int NFT, int L>
struct CoopStep {
  static_assert(NFT >= 0 && NFT <= kCoopMaxFrameTasks, "unsupported number of frame tasks");
  static_assert(L == 1 || L == 2 || L == 4 || L == 8, "lanes per instance: 1, 2, 4 or 8");
  static constexpr int NC = (NJ + L - 1) / L;  // joints (columns) per lane
  static constexpr int NJP = NC * L;
  static constexpr int K = 6 * NFT;
  static constexpr int KA = K > 0 ? K : 1;
  static constexpr int NT = NFT > 0 ? NFT : 1;
  static constexpr int kMaxFastIters = 2 * NJ + 6;
  using Params = CoopParams<NJP>;
  using Solver = BoxLSQChol<K, NJ>;

  struct Lane {
    float q[NC];
    V3 pj[NC], zj[NC];  // joint origin / axis in the segment's base frame
    SE3f S[NT];         // suffix product: pose of task frame t relative to this lane's segment base
    float A[NC][KA];    // columns of W J of the lane's joints
    float nrm[NC];      // |A[:, j]|
    float x[NC], lo[NC], hi[NC], beta[NC];
    int side[NC];       // +1 on the upper bound, -1 on the lower bound, 0 free
    int flags;          // status bits raised by this lane
    float cand_val;     // scratch of the release search
    int cand_idx;
  };

  // ---- everything up to the QP data --------------------------------------------------
  // jc(j) returns the constants of joint j (constant bank for L = 1, shared memory otherwise).
  // Outputs that are identical on all lanes of the group: b, d, status, skip.
  template <class JC>
  static PK_HD void assemble(const Group<L>& G, const Params& P, JC jc, const float* __restrict__ trow,
                             GVar<Lane, L>& S, float (&b)[KA], float& d, int& status, bool& skip) {
    status = 0;
    // limit check (pink/configuration.py:181-201)
    PK_GLANES(G, h) {
      Lane& s = S[h];
      s.flags = 0;
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const CoopJoint& J = jc(h * NC + k);
        if (s.q[k] < J.chk_lo || s.q[k] > J.chk_hi) s.flags |= PK_STATUS_OUT_OF_LIMITS;
      }
    }
    if (g_any(G, S, [](const Lane& s) { return s.flags != 0; })) status |= PK_STATUS_OUT_OF_LIMITS;
    skip = status && P.safety_break;
    if (skip) return;

    // ---- forward kinematics of the lane's segment, in the segment's base frame ----------
    PK_GLANES(G, h) {
      Lane& s = S[h];
      SE3f T = identity_se3();
      SE3f Tb[NT];
#pragma unroll
      for (int t = 0; t < NT; ++t) Tb[t] = identity_se3();
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        const CoopJoint& J = jc(j);
        SE3f Y;
        if (k == 0) {  // the segment starts at its own base frame: Y = X~
#pragma unroll
          for (int i = 0; i < 9; ++i) Y.R.m[i] = J.Xr[i];
          Y.p = v3(J.Xp[0], J.Xp[1], J.Xp[2]);
        } else {
          M3 Xr;
#pragma unroll
          for (int i = 0; i < 9; ++i) Xr.m[i] = J.Xr[i];
          Y.R = mul(T.R, Xr);
          Y.p = mul(T.R, v3(J.Xp[0], J.Xp[1], J.Xp[2])) + T.p;
        }
        // motion about / along the local z axis
        float sn, cs;
        sincos_f(s.q[k], &sn, &cs);
        float dz = 0.f;
        if (P.any_prismatic) {  // uniform: chains without prismatic joints skip the selects
          const bool pris = J.prismatic != 0.f;
          sn = pris ? 0.f : sn;
          cs = pris ? 1.f : cs;
          dz = pris ? s.q[k] : 0.f;
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float y0 = Y.R.m[3 * r], y1 = Y.R.m[3 * r + 1];
          T.R.m[3 * r] = fmaf(cs, y0, sn * y1);
          T.R.m[3 * r + 1] = fmaf(cs, y1, -sn * y0);
          T.R.m[3 * r + 2] = Y.R.m[3 * r + 2];
        }
        const V3 z = v3(T.R.m[2], T.R.m[5], T.R.m[8]);
        T.p = P.any_prismatic ? Y.p + dz * z : Y.p;
        s.pj[k] = T.p;
        s.zj[k] = z;
        if (!P.frames_on_last) {  // uniform: remember the joint that carries each task frame
#pragma unroll
          for (int t = 0; t < NFT; ++t) {
            const bool here = P.ft[t].body == j;
#pragma unroll
            for (int i = 0; i < 9; ++i) Tb[t].R.m[i] = here ? T.R.m[i] : Tb[t].R.m[i];
            Tb[t].p.x = here ? T.p.x : Tb[t].p.x;
            Tb[t].p.y = here ? T.p.y : Tb[t].p.y;
            Tb[t].p.z = here ? T.p.z : Tb[t].p.z;
          }
        }
      }
      if (P.frames_on_last) {
        // the frame's joint is the last one of the chain: it lives in the last lane's segment
#pragma unroll
        for (int t = 0; t < NFT; ++t) Tb[t] = T;
      }
      // segment factor of the suffix product: the whole segment before the frame's joint, the
      // prefix up to that joint times the frame offset in its segment, identity after it
      // (a frame fixed to the world, body = -1, lives on lane 0)
#pragma unroll
      for (int t = 0; t < NFT; ++t) {
        const int body = P.ft[t].body;
        const int j0 = h * NC;
        const bool inside = (body >= j0 && body < j0 + NC) || (body < 0 && h == 0);
        const bool before = body >= j0 + NC;
        const SE3f withX = compose(Tb[t], load_se3(P.ft[t].X));
        const SE3f I = identity_se3();
#pragma unroll
        for (int i = 0; i < 9; ++i) s.S[t].R.m[i] = inside ? withX.R.m[i] : (before ? T.R.m[i] : I.R.m[i]);
        s.S[t].p.x = inside ? withX.p.x : (before ? T.p.x : 0.f);
        s.S[t].p.y = inside ? withX.p.y : (before ? T.p.y : 0.f);
        s.S[t].p.z = inside ? withX.p.z : (before ? T.p.z : 0.f);
      }
    }
    // suffix product over the lanes: S_h <- S_h S_{h+1} ... S_{L-1}
#pragma unroll
    for (int t = 0; t < NFT; ++t) {
#pragma unroll
      for (int dist = 1; dist < L; dist <<= 1) {
        GVar<SE3f, L> Nx;
        PK_GLANES(G, h) {
          const bool has = h + dist < L;
          const int src = has ? h + dist : h;
          SE3f Gt;
#pragma unroll
          for (int i = 0; i < 9; ++i) {
            const float val = g_get(G, S, src, [&](const Lane& o) { return o.S[t].R.m[i]; });
            Gt.R.m[i] = has ? val : ((i % 4 == 0) ? 1.f : 0.f);
          }
          const float px = g_get(G, S, src, [&](const Lane& o) { return o.S[t].p.x; });
          const float py = g_get(G, S, src, [&](const Lane& o) { return o.S[t].p.y; });
          const float pz = g_get(G, S, src, [&](const Lane& o) { return o.S[t].p.z; });
          Gt.p = has ? v3(px, py, pz) : v3(0.f, 0.f, 0.f);
          Nx[h] = compose(S[h].S[t], Gt);
        }
        PK_GLANES(G, h) { S[h].S[t] = Nx[h]; }
      }
    }

    // ---- task error, Jlog6 (replicated), columns of W J (lane-local) ---------------------
    float diag = P.damping;  // damping + sum of Levenberg-Marquardt terms
#pragma unroll
    for (int t = 0; t < NFT; ++t) {
      const CoopFrameTask& Kt = P.ft[t];
      // frame pose in the world = lane 0's suffix product
      SE3f Tf;
#pragma unroll
      for (int i = 0; i < 9; ++i) Tf.R.m[i] = g_get(G, S, 0, [&](const Lane& o) { return o.S[t].R.m[i]; });
      Tf.p.x = g_get(G, S, 0, [&](const Lane& o) { return o.S[t].p.x; });
      Tf.p.y = g_get(G, S, 0, [&](const Lane& o) { return o.S[t].p.y; });
      Tf.p.z = g_get(G, S, 0, [&](const Lane& o) { return o.S[t].p.z; });
      const SE3f Tt = Kt.tgt_shared ? load_se3(P.shared + Kt.tgt_off) : load_se3_vec4(trow + Kt.tgt_off, P.target_vec4 != 0);
      // e = log6(T_b^-1 T_t)
      const SE3f Tbt = act_inv(Tf, Tt);
      Log3 Lg = log3(Tbt.R);
      float e[6];
      log6(Tbt, Lg, e);
      // J = -Jlog6(T_t^-1 T_b) bJ_b ;  log3(R^T) = -log3(R), same angle and coefficients
      SE3f Ttb;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) Ttb.R.m[3 * i + k] = Tbt.R.m[3 * k + i];
      Ttb.p = -1.f * mul(Ttb.R, Tbt.p);
      Lg.w = -1.f * Lg.w;
      M3 Am, Bm;
      jlog6(Ttb, Lg, Am, Bm);
      float mu = 0.f;
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const float ew = Kt.cost[k] * Kt.gain * e[k];
        b[6 * t + k] = ew;
        mu = fmaf(ew, ew, mu);
      }
      diag = fmaf(Kt.lm, mu, diag);
      // rows of -W Jlog6 (weights and sign folded in once)
      M3 WA, WB, WC;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          WA.m[3 * r + c] = -Kt.cost[r] * Am.m[3 * r + c];
          WB.m[3 * r + c] = -Kt.cost[r] * Bm.m[3 * r + c];
          WC.m[3 * r + c] = -Kt.cost[3 + r] * Am.m[3 * r + c];
        }
      PK_GLANES(G, h) {
        Lane& s = S[h];
        const SE3f& F = s.S[t];
#pragma unroll
        for (int k = 0; k < NC; ++k) {
          const int j = h * NC + k;
          const CoopJoint& J = jc(j);
          const V3 z = s.zj[k];
          const V3 cr = cross(z, F.p - s.pj[k]);
          V3 lin = cr, ang = z;
          if (P.any_prismatic) {
            const bool pris = J.prismatic != 0.f;
            lin = pris ? z : cr;
            ang = pris ? v3(0.f, 0.f, 0.f) : z;
          }
          const V3 jl = mulT(F.R, lin);
          const V3 ja = mulT(F.R, ang);
          const V3 tl = mul(WA, jl) + mul(WB, ja);
          const V3 ta = mul(WC, ja);
          // joints past the frame do not move it; padding joints never do
          const bool on = (P.frames_on_last || j <= Kt.body) && (NJP == NJ || J.valid != 0.f);
          s.A[k][6 * t + 0] = on ? tl.x : 0.f;
          s.A[k][6 * t + 1] = on ? tl.y : 0.f;
          s.A[k][6 * t + 2] = on ? tl.z : 0.f;
          s.A[k][6 * t + 3] = on ? ta.x : 0.f;
          s.A[k][6 * t + 4] = on ? ta.y : 0.f;
          s.A[k][6 * t + 5] = on ? ta.z : 0.f;
        }
      }
    }

    // ---- diagonal part: posture rows w (x_j + alpha e_j) and sqrt(diag) x_j merged into d x_j + beta_j
    float se = 0.f;
    PK_GLANES(G, h) {
      Lane& s = S[h];
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        float pe = 0.f;
        if (P.has_posture) {
          const float* qref = P.posture_shared ? (P.shared + P.posture_off) : (trow + P.posture_off);
          pe = (j < NJ) ? s.q[k] - qref[j < NJ ? j : NJ - 1] : 0.f;
        }
        s.beta[k] = pe;  // scaled below
      }
    }
    const float w2 = P.has_posture ? P.posture_w2 : 0.f;
    if (P.has_posture && P.posture_lm != 0.f) {
      se = g_sum(G, S, [](const Lane& s) {
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < NC; ++k) a = fmaf(s.beta[k], s.beta[k], a);
        return a;
      });
      diag = fmaf(P.posture_lm * P.posture_gain * P.posture_gain * w2, se, diag);
    }
    d = sqrtf(w2 + diag);
    const float kf = (d > 0.f) ? P.posture_gain * w2 / d : 0.f;

    // ---- box rows, column norms ---------------------------------------------------------
    PK_GLANES(G, h) {
      Lane& s = S[h];
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        const CoopJoint& J = jc(j);
        s.beta[k] *= kf;
        s.hi[k] = fminf(P.cfg_gain * (J.cfg_hi - s.q[k]), J.vel);  // the difference first: exact near a limit
        s.lo[k] = fmaxf(P.cfg_gain * (J.cfg_lo - s.q[k]), -J.vel);
        if (P.acc_enabled) {
          // AccelerationLimit (pink/limits/acceleration_limit.py:119-200): a box as well
          const float a = J.acc_max;
          if (a < 3.0e38f) {
            const float dt2 = P.dt * P.dt;
            const float pv = (P.acc_prev_off >= 0 && j < NJ) ? trow[P.acc_prev_off + (j < NJ ? j : 0)] : 0.f;
            const float up = J.acc_qhi - s.q[k], dn = s.q[k] - J.acc_qlo;
            if (up < 0.f || dn < 0.f) s.flags |= PK_STATUS_NO_SOLUTION;  // sqrt of a negative margin: NaN rows
            const float hu = fminf(fmaf(a, dt2, pv), (up < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(up, 0.f)) : INFINITY);
            const float hl = fminf(fmaf(a, dt2, -pv), (dn < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(dn, 0.f)) : INFINITY);
            s.hi[k] = fminf(s.hi[k], hu);
            s.lo[k] = fmaxf(s.lo[k], -hl);
          }
        }
        if (NJP != NJ && J.valid == 0.f) {  // padding joint: pinned at zero, never part of the problem
          s.lo[k] = 0.f;
          s.hi[k] = 0.f;
        }
        // |A[:, k]| for the rounding scale of the multipliers (a tolerance: the rsqrt
        // approximation is plenty)
        float n2 = 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) n2 = fmaf(s.A[k][r], s.A[k][r], n2);
        s.nrm[k] = n2 * rsqrtf(fmaxf(n2, 1e-30f));
      }
    }
    if (P.acc_enabled && g_any(G, S, [](const Lane& s) { return (s.flags & PK_STATUS_NO_SOLUTION) != 0; }))
      status |= PK_STATUS_NO_SOLUTION;
  }

  // ---- QP: primal active set from the box corner -----------------------------------------
  // Returns status bits.  On return S[.].x holds the solution.
  static PK_HD int solve_qp(const Group<L>& G, GVar<Lane, L>& S, const float (&b)[KA], float d) {
    // empty box <=> quadprog reports no solution
    if (g_any(G, S, [](const Lane& s) {
          bool bad = false;
#pragma unroll
          for (int k = 0; k < NC; ++k) bad = bad || (s.lo[k] > s.hi[k]);
          return bad;
        }))
      return PK_STATUS_NO_SOLUTION;

    // corner: every coordinate on the bound the gradient at the origin points to
    PK_GLANES(G, h) {
      Lane& s = S[h];
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        float c = d * s.beta[k];
#pragma unroll
        for (int r = 0; r < K; ++r) c = fmaf(s.A[k][r], b[r], c);
        if (c < 0.f && s.hi[k] < 3.0e38f) { s.side[k] = 1; s.x[k] = s.hi[k]; }
        else if (c > 0.f && s.lo[k] > -3.0e38f) { s.side[k] = -1; s.x[k] = s.lo[k]; }
        else { s.side[k] = 0; s.x[k] = fminf(fmaxf(0.f, s.lo[k]), s.hi[k]); }
      }
    }
    // rho = A x + b (the one group reduction of the solve)
    float rho[KA];
#pragma unroll
    for (int r = 0; r < K; ++r) {
      rho[r] = b[r] + g_sum(G, S, [&](const Lane& s) {
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < NC; ++k) a = fmaf(s.A[k][r], s.x[k], a);
        return a;
      });
    }
    // a coordinate that starts strictly inside its box (c = 0 or infinite bounds) is not
    // covered by the two-slot loop: hand such problems to the rounds
    bool to_rounds = g_any(G, S, [](const Lane& s) {
      bool f = false;
#pragma unroll
      for (int k = 0; k < NC; ++k) f = f || (s.side[k] == 0 && s.lo[k] < s.hi[k]);
      return f;
    });

    // free slots (replicated): coordinate index, its column, Gram entries, box, value
    int nF = 0;
    int fidx[2] = {-1, -1};
    float fcol[2][KA] = {}, fH[2] = {1.f, 1.f}, fx[2] = {0.f, 0.f}, flo[2] = {0.f, 0.f}, fhi[2] = {0.f, 0.f}, fbeta[2] = {0.f, 0.f};
    float H01 = 0.f;
    bool full_step = true;
    int status = 0;
    int it = 0;
#pragma unroll 1
    for (; !to_rounds; ++it) {
      if (it >= kMaxFastIters) { to_rounds = true; break; }
      if (full_step || nF == 0) {
        float r2 = 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) r2 = fmaf(rho[r], rho[r], r2);
        const float rnorm = sqrtf(r2);
        // most negative multiplier among the active bounds: g_k = A[:, k] . rho + d (d x_k + beta_k)
        // against its rounding scale (|A[:, k]| |rho| bounds sum_r |A_rk| |rho_r|, Cauchy-Schwarz)
        PK_GLANES(G, h) {
          Lane& s = S[h];
          s.cand_val = 0.f;
          s.cand_idx = -1;
#pragma unroll
          for (int k = 0; k < NC; ++k) {
            const float rt = fmaf(d, s.x[k], s.beta[k]);
            float g = d * rt;
#pragma unroll
            for (int r = 0; r < K; ++r) g = fmaf(s.A[k][r], rho[r], g);
            const float tol = 4e-6f * fmaf(s.nrm[k], rnorm, fabsf(d * rt));
            const float lam = (s.side[k] > 0) ? -g : g;
            if (s.side[k] != 0 && lam < -tol && lam < s.cand_val) { s.cand_val = lam; s.cand_idx = h * NC + k; }
          }
        }
        float worst;
        int rel;
        g_argmin(G, S, [](const Lane& s) { return s.cand_val; },
                 [](const Lane& s) { return s.cand_idx < 0 ? 0x7fffffff : s.cand_idx; }, worst, rel);
        if (!(worst < 0.f)) break;  // KKT point
        if (nF == 2) {
          // a third free coordinate: release it and let the rounds continue from here
          PK_GLANES(G, h) {
            Lane& s = S[h];
#pragma unroll
            for (int k = 0; k < NC; ++k)
              if (h * NC + k == rel) s.side[k] = 0;
          }
          to_rounds = true;
          break;
        }
        // new slot: the owner publishes the column and the scalars of coordinate `rel`
        // (slot arrays are only ever indexed statically: they must stay in registers)
        const int own = rel / NC, slot = rel % NC;
        const int sN = nF;
        auto pick = [&](const Lane& o, auto member) {
          float val = member(o, 0);
#pragma unroll
          for (int k = 1; k < NC; ++k) val = (slot == k) ? member(o, k) : val;
          return val;
        };
        float ncol[KA];
#pragma unroll
        for (int r = 0; r < K; ++r)
          ncol[r] = g_get(G, S, own, [&](const Lane& o) { return pick(o, [&](const Lane& p, int k) { return p.A[k][r]; }); });
        const float nx = g_get(G, S, own, [&](const Lane& o) { return pick(o, [](const Lane& p, int k) { return p.x[k]; }); });
        const float nlo = g_get(G, S, own, [&](const Lane& o) { return pick(o, [](const Lane& p, int k) { return p.lo[k]; }); });
        const float nhi = g_get(G, S, own, [&](const Lane& o) { return pick(o, [](const Lane& p, int k) { return p.hi[k]; }); });
        const float nbeta = g_get(G, S, own, [&](const Lane& o) { return pick(o, [](const Lane& p, int k) { return p.beta[k]; }); });
        float hh = d * d, h01 = 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) {
          hh = fmaf(ncol[r], ncol[r], hh);
          h01 = fmaf(fcol[0][r], ncol[r], h01);
        }
        if (sN == 0) {
          fidx[0] = rel; fx[0] = nx; flo[0] = nlo; fhi[0] = nhi; fH[0] = hh; fbeta[0] = nbeta;
#pragma unroll
          for (int r = 0; r < K; ++r) fcol[0][r] = ncol[r];
        } else {
          fidx[1] = rel; fx[1] = nx; flo[1] = nlo; fhi[1] = nhi; fH[1] = hh; fbeta[1] = nbeta;
          H01 = h01;
#pragma unroll
          for (int r = 0; r < K; ++r) fcol[1][r] = ncol[r];
        }
        nF = sN + 1;
        PK_GLANES(G, h) {
          Lane& s = S[h];
#pragma unroll
          for (int k = 0; k < NC; ++k)
            if (h * NC + k == rel) s.side[k] = 0;
        }
      }
      // gradient entries of the free coordinates, from their replicated columns
      float gF[2] = {0.f, 0.f};
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        float g = d * fmaf(d, fx[sl], fbeta[sl]);
#pragma unroll
        for (int r = 0; r < K; ++r) g = fmaf(fcol[sl][r], rho[r], g);
        gF[sl] = g;
      }
      // Newton step on the free block
      float p[2] = {0.f, 0.f};
      if (nF == 1) {
        p[0] = -gF[0] / fH[0];
        if (!(fH[0] > 0.f)) { to_rounds = true; break; }
      } else {
        const float det = fmaf(fH[0], fH[1], -H01 * H01);
        if (!(det > 1e-6f * fH[0] * fH[1])) { to_rounds = true; break; }  // nearly dependent columns: the rounds decide
        const float inv = 1.f / det;
        p[0] = (H01 * gF[1] - fH[1] * gF[0]) * inv;
        p[1] = (H01 * gF[0] - fH[0] * gF[1]) * inv;
      }
      // longest feasible step
      float alpha = 1.f;
      int blk = -1;
      bool blk_hi = false;
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        if (sl < nF) {
          const float xn = fx[sl] + p[sl];
          if (xn > fhi[sl]) {
            const float a = (fhi[sl] - fx[sl]) / p[sl];
            if (a < alpha) { alpha = a; blk = sl; blk_hi = true; }
          } else if (xn < flo[sl]) {
            const float a = (flo[sl] - fx[sl]) / p[sl];
            if (a < alpha) { alpha = a; blk = sl; blk_hi = false; }
          }
        }
      }
      alpha = fmaxf(alpha, 0.f);
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        if (sl < nF) {
          const float stp = alpha * p[sl];
          fx[sl] += stp;
          if (sl == blk) fx[sl] = blk_hi ? fhi[sl] : flo[sl];
#pragma unroll
          for (int r = 0; r < K; ++r) rho[r] = fmaf(fcol[sl][r], stp, rho[r]);
        }
      }
      // owners take the new values; a blocking coordinate becomes active
      const int i0 = fidx[0], i1 = fidx[1];
      const float x0 = fx[0], x1 = fx[1];
      const int nF_now = nF;
      const int blk_idx = blk < 0 ? -1 : (blk == 0 ? fidx[0] : fidx[1]);
      PK_GLANES(G, h) {
        Lane& s = S[h];
#pragma unroll
        for (int k = 0; k < NC; ++k) {
          const int j = h * NC + k;
          if (j == i0) s.x[k] = x0;
          if (nF_now == 2 && j == i1) s.x[k] = x1;
          if (j == blk_idx) s.side[k] = blk_hi ? 1 : -1;
        }
      }
      if (blk >= 0) {
        if (blk == 0 && nF == 2) {  // slot 1 moves down
          fidx[0] = fidx[1];
          fH[0] = fH[1];
          fx[0] = fx[1];
          flo[0] = flo[1];
          fhi[0] = fhi[1];
          fbeta[0] = fbeta[1];
#pragma unroll
          for (int r = 0; r < K; ++r) fcol[0][r] = fcol[1][r];
        }
        --nF;
        full_step = false;
      } else {
        full_step = true;
      }
    }
#ifdef PK_COUNT_ITERS
    pk_count_nfree(to_rounds ? 20 + nF : nF, -(it + 2));
#endif
    if (to_rounds) status |= rounds(G, S, b, d);
    return status;
  }

  // Cholesky rounds of pk_lsq.cuh on the gathered problem (every lane of the group runs the
  // same replicated computation), started from the state the fast loop reached.
  static PK_HD int rounds(const Group<L>& G, GVar<Lane, L>& S, const float (&b)[KA], float d) {
    float Af[KA][NJ], dv[NJ], betaf[NJ];
    typename Solver::State St;
    St.status = 0;
    St.rounds = 0;
    St.cond = 1.f;
    St.gtol = 0.f;
    St.at_hi = St.at_lo = 0u;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int own = j / NC, slot = j % NC;
#pragma unroll
      for (int r = 0; r < K; ++r) Af[r][j] = g_get(G, S, own, [&](const Lane& o) { return o.A[slot][r]; });
      St.x[j] = g_get(G, S, own, [&](const Lane& o) { return o.x[slot]; });
      St.lo[j] = g_get(G, S, own, [&](const Lane& o) { return o.lo[slot]; });
      St.hi[j] = g_get(G, S, own, [&](const Lane& o) { return o.hi[slot]; });
      betaf[j] = g_get(G, S, own, [&](const Lane& o) { return o.beta[slot]; });
      const int side = g_get_int(G, S, own, [&](const Lane& o) { return o.side[slot]; });
      if (side > 0) St.at_hi |= (1u << j);
      if (side < 0) St.at_lo |= (1u << j);
      dv[j] = d;
    }
    const typename Solver::ArrayObjective O{Af, b, dv, betaf};
    Solver::gram(O, St);
    bool more = true;
    for (;;) {
      while (more) more = Solver::round(St);
      more = Solver::polish(O, St);
      if (!more) break;
    }
    PK_GLANES(G, h) {
      Lane& s = S[h];
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj)
          if (jj == j) s.x[k] = St.x[jj];
      }
    }
    return St.status;
  }
};

// One step of one instance.  q / v: the lane's NC joints (S[h].q in, vout[h][k] out).
template <int NJ, int NFT, int L, class JC>
PK_HD void ik_step_coop(const Group<L>& G, const CoopParams<CoopStep<NJ, NFT, L>::NJP>& P, JC jc,
                        const float* __restrict__ trow, GVar<typename CoopStep<NJ, NFT, L>::Lane, L>& S,
                        int& status_out) {
  using Step = CoopStep<NJ, NFT, L>;
  float b[Step::KA];
#pragma unroll
  for (int r = 0; r < Step::KA; ++r) b[r] = 0.f;
  float d = 0.f;
  int status = 0;
  bool skip = false;
  Step::assemble(G, P, jc, trow, S, b, d, status, skip);
  const bool solve = !skip && !(status & PK_STATUS_NO_SOLUTION);
  if (solve) status |= Step::solve_qp(G, S, b, d);
  // a NaN / Inf in q or in a target passes every comparison above and ends up in x: report it
  // (the reference's QP back-end fails on such a problem) instead of returning it
  float sum = 0.f;
  if (solve && !(status & PK_STATUS_NO_SOLUTION)) {
    sum = g_sum(G, S, [](const typename Step::Lane& s) {
      float a = 0.f;
#pragma unroll
      for (int k = 0; k < Step::NC; ++k) a += s.x[k];
      return a;
    });
  }
  const bool finite = fabsf(sum) < 3.0e38f;
  if (!finite) status |= PK_STATUS_NO_SOLUTION;
  const bool zero = !solve || !finite || (status & PK_STATUS_NO_SOLUTION);
  PK_GLANES(G, h) {
    typename Step::Lane& s = S[h];
#pragma unroll
    for (int k = 0; k < Step::NC; ++k) s.x[k] = zero ? 0.f : s.x[k] * P.inv_dt;  // v = dq / dt
  }
  status_out = status;
}

// Closed-loop rollout of instance `inst` (ik_coop_kernel), the loop of rollout_chain (pk_chain.cuh)
// with ik_step_coop: S[h].q in, where the instance ended out; S[h].x the last step's velocity.
// Each lane stores the joints it owns into the records of T, lane 0 of the group the status.
template <int NJ, int NFT, int L, class JC>
PK_HD int rollout_coop(const Group<L>& G, const CoopParams<CoopStep<NJ, NFT, L>::NJP>& P, JC jc, const float* trow,
                       GVar<typename CoopStep<NJ, NFT, L>::Lane, L>& S, int n_steps, bool integrate,
                       const Trajectory& T, int64_t B, int64_t inst) {
  constexpr int NC = CoopStep<NJ, NFT, L>::NC;
  // records of step s: the lane's joints of q and v, the status from lane 0 of the group
  auto record = [&](int s, int st_all, bool frozen) {
    const int64_t r = (int64_t)s * B + inst;
    PK_GLANES(G, h) {
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        if (j < NJ) {
          if (T.q) T.q[r * NJ + j] = S[h].q[k];
          if (T.v) T.v[r * NJ + j] = frozen ? 0.f : S[h].x[k];
        }
      }
      if (T.status && h == 0) T.status[r] = st_all;
    }
  };
  int st_all = 0;
  PK_GLANES(G, h) {
#pragma unroll
    for (int k = 0; k < NC; ++k) S[h].x[k] = 0.f;
  }
#pragma unroll 1
  for (int step_no = 0; step_no < n_steps; ++step_no) {
    if (step_failed(st_all, P.safety_break)) {
#pragma unroll 1
      for (int s = step_no; s < n_steps; ++s) record(s, st_all, true);
      break;
    }
    int st;
    ik_step_coop<NJ, NFT, L>(G, P, jc, trow, S, st);
    st_all |= st & 0xff;
    if (n_steps > 1 || integrate) {
      PK_GLANES(G, h) {
#pragma unroll
        for (int k = 0; k < NC; ++k) S[h].q[k] = fmaf(S[h].x[k], P.dt, S[h].q[k]);  // 1-dof joints: q + v dt
      }
    }
    trow += T.target_step;
    record(step_no, st_all, false);
  }
  return st_all;
}

// Instance `inst` of ik_coop_kernel: its q row into the lanes (padding joints at zero), rollout_coop,
// then each lane stores the joints it owns of v and of q_out (unless null), lane 0 of the group the
// status (unless null).
template <int NJ, int NFT, int L, class JC>
PK_HD void coop_instance(const Group<L>& G, const CoopParams<CoopStep<NJ, NFT, L>::NJP>& P, JC jc,
                         const float* __restrict__ q, const float* __restrict__ targets, float* __restrict__ v,
                         int32_t* __restrict__ status, int64_t B, int n_steps, float* __restrict__ q_out,
                         const Trajectory& T, int64_t inst) {
  using Step = CoopStep<NJ, NFT, L>;
  constexpr int NC = Step::NC;
  GVar<typename Step::Lane, L> S;
  const float* qrow = q + inst * NJ;
  PK_GLANES(G, h) {
    if constexpr (L == 1 && NJ % 2 == 0) {
#pragma unroll
      for (int k = 0; k < NJ / 2; ++k) {
        const float2 t = load_ro(reinterpret_cast<const float2*>(qrow) + k);
        S[h].q[2 * k] = t.x;
        S[h].q[2 * k + 1] = t.y;
      }
    } else {
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        S[h].q[k] = (j < NJ) ? load_ro(qrow + (j < NJ ? j : 0)) : 0.f;
      }
    }
  }
  const int st_all = rollout_coop<NJ, NFT, L>(G, P, jc, targets + inst * (int64_t)P.target_stride, S, n_steps,
                                              q_out != nullptr, T, B, inst);
  float* vrow = v + inst * NJ;
  PK_GLANES(G, h) {
    if constexpr (L == 1 && NJ % 2 == 0) {
#pragma unroll
      for (int k = 0; k < NJ / 2; ++k) reinterpret_cast<float2*>(vrow)[k] = make_float2(S[h].x[2 * k], S[h].x[2 * k + 1]);
    } else {
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        if (j < NJ) vrow[j] = S[h].x[k];
      }
    }
    if (q_out) {
      float* orow = q_out + inst * NJ;
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int j = h * NC + k;
        if (j < NJ) orow[j] = S[h].q[k];
      }
    }
    if (status && h == 0) status[inst] = st_all;
  }
}

}  // namespace pk
