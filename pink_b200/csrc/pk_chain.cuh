// One IK step of a fixed-base serial chain, one instance per thread, all state in
// registers (UR5-class arms: nq = nv = NJ <= 8).
//
// Path (reference file:line):
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
// The parameter block is passed by value as a kernel argument, i.e. it lives in
// the constant bank: every thread reads the same address at the same time, so
// model constants cost no registers and no memory traffic.
#pragma once

#include "pk_math.cuh"
#include "pk_lsq.cuh"

namespace pk {

constexpr int kChainMaxFrameTasks = 2;
// longest targets row the PDL instantiation of ik_chain_kernel copies: frame targets, posture and dq_prev
PK_HD constexpr int chain_row_words(int nj, int nft) { return 12 * nft + 2 * nj; }

struct ChainJoint {
  float X[12];  // placement in the parent joint frame, row-major [R | p]
  float ax, ay, az;
  int type;  // PK_JOINT_*
  // X.R Rot(a, q) = X.R + sin q (X.R [a]x) + (1 - cos q) (X.R (a a^T - I)): the two
  // constant matrices, and X.R a for prismatic joints, are folded on the host
  float M1[9], M2[9];
  float Xa[3];
};

struct ChainFrameTask {
  int body;       // joint index the frame is fixed to (-1: world)
  float X[12];    // frame placement in that body
  float cost[6];  // [pos(3), ori(3)]
  float gain, lm;
  int tgt_off;
  int tgt_shared;
};

template <int NJ>
struct ChainParams {
  ChainJoint joint[NJ];
  int n_frame_tasks;
  ChainFrameTask ft[kChainMaxFrameTasks];
  int has_posture;
  float posture_w2, posture_gain, posture_lm;
  int posture_off, posture_shared;
  float dt, inv_dt, damping;
  float cfg_gain;
  float cfg_lo[NJ], cfg_hi[NJ], vel[NJ], chk_lo[NJ], chk_hi[NJ];
  int target_stride;
  int target_vec4;  // per-instance frame targets are 16-byte aligned: three 128-bit loads per target
  int safety_break;
  float shared[12 * kChainMaxFrameTasks + NJ];
  // AccelerationLimit (pink/limits/acceleration_limit.py:119-200): a box as well
  int acc_enabled, acc_prev_off;  // dq_prev per instance at acc_prev_off of the targets row (< 0: zeros)
  float acc_max[NJ], acc_qlo[NJ], acc_qhi[NJ];
};

// NFT = number of FrameTasks (compile time, so that the stacked Jacobian has a
// static shape and stays in registers).
//
// ChainStep::assemble runs everything up to the QP data (limit check, FK, task
// rows, box); the QP itself is BoxLSQChol (pk_lsq.cuh), either run to completion
// in the same thread (ik_step_chain).
template <int NJ, int NFT>
struct ChainStep {
  static_assert(NFT >= 0 && NFT <= kChainMaxFrameTasks, "unsupported number of frame tasks");
  static constexpr int K = 6 * NFT;
  static constexpr int KA = K > 0 ? K : 1;
  float A[KA][NJ];
  float b[KA];
  float d[NJ], beta[NJ], lo[NJ], hi[NJ];

  // Returns status bits; `skip` is set when the instance must not be solved
  // (outside limits with safety_break).
  // ERR (converge_chain): also store in *err the largest unweighted, gain-free |e_t|_2 of the
  // tasks of `emask` in chain slots (bit k < NFT: ft[k], bit NFT: the posture task).  An
  // instance outside its limits still runs the forward kinematics then, because its error is
  // wanted too; it returns right after the task errors.
  template <bool ERR = false>
  PK_HD int assemble(const ChainParams<NJ>& P, const float (&q)[NJ], const float* __restrict__ trow, bool& skip,
                     unsigned emask = 0u, float* err = nullptr) {
  int status = 0;
  float emax = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j)
    if (q[j] < P.chk_lo[j] || q[j] > P.chk_hi[j]) status |= PK_STATUS_OUT_OF_LIMITS;
  skip = status && P.safety_break;
  if (skip && !ERR) return status;

  // ---- forward kinematics: oMi[j] = oMi[j-1] X_j exp(S_j q_j) -----------------
  SE3f T = identity_se3();
  V3 pj[NJ], wj[NJ];  // world origin and world axis of every joint
  SE3f Tf[NFT > 0 ? NFT : 1], Tb[NFT > 0 ? NFT : 1];
#pragma unroll
  for (int t = 0; t < NFT; ++t) Tb[t] = identity_se3();  // frames fixed to the world body
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const ChainJoint& Jn = P.joint[j];
    const V3 axis = v3(Jn.ax, Jn.ay, Jn.az);
    SE3f X = load_se3(Jn.X);
    SE3f Tl;
    if (Jn.type == PK_JOINT_REVOLUTE) {
      float s, c;
      sincos_f(q[j], &s, &c);
      const float t = 1.f - c;
#pragma unroll
      for (int k = 0; k < 9; ++k) Tl.R.m[k] = fmaf(s, Jn.M1[k], fmaf(t, Jn.M2[k], X.R.m[k]));
      Tl.p = X.p;
    } else {
      Tl.R = X.R;
      Tl.p = X.p + q[j] * v3(Jn.Xa[0], Jn.Xa[1], Jn.Xa[2]);
    }
    T = compose(T, Tl);
    pj[j] = T.p;
    wj[j] = mul(T.R, axis);
    // remember the placement of the joint that carries each task frame (selects only;
    // the frame offset is composed once, after the sweep)
#pragma unroll
    for (int t = 0; t < NFT; ++t) {
      const bool here = P.ft[t].body == j;
#pragma unroll
      for (int k = 0; k < 9; ++k) Tb[t].R.m[k] = here ? T.R.m[k] : Tb[t].R.m[k];
      Tb[t].p.x = here ? T.p.x : Tb[t].p.x;
      Tb[t].p.y = here ? T.p.y : Tb[t].p.y;
      Tb[t].p.z = here ? T.p.z : Tb[t].p.z;
    }
  }
#pragma unroll
  for (int t = 0; t < NFT; ++t) Tf[t] = compose(Tb[t], load_se3(P.ft[t].X));

  // ---- objective in square-root form: rows of A / b are W J and W alpha e ----------
  float diag = P.damping;  // damping + sum of Levenberg-Marquardt terms

#pragma unroll
  for (int t = 0; t < NFT; ++t) {
    const ChainFrameTask& Kt = P.ft[t];
    const SE3f Tt = Kt.tgt_shared ? load_se3(P.shared + Kt.tgt_off) : load_se3_vec4(trow + Kt.tgt_off, P.target_vec4 != 0);
    // e = log6(T_b^-1 T_t)
    const SE3f Tbt = act_inv(Tf[t], Tt);
    Log3 L = log3(Tbt.R);
    float e[6];
    log6(Tbt, L, e);
    if constexpr (ERR) {
      if ((emask >> t) & 1u) {
        float n2 = 0.f;
#pragma unroll
        for (int k = 0; k < 6; ++k) n2 = fmaf(e[k], e[k], n2);
        emax = err_max(emax, sqrtf(n2));
      }
    }
    // J = -Jlog6(T_t^-1 T_b) bJ_b ;  log3(R^T) = -log3(R), same angle and coefficients
    SE3f Ttb;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) Ttb.R.m[3 * i + k] = Tbt.R.m[3 * k + i];
    Ttb.p = -1.f * mul(Ttb.R, Tbt.p);
    L.w = -1.f * L.w;
    M3 Am, Bm;
    jlog6(Ttb, L, Am, Bm);

    float mu = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float ew = Kt.cost[k] * Kt.gain * e[k];
      b[6 * t + k] = ew;
      mu = fmaf(ew, ew, mu);
    }
    diag = fmaf(Kt.lm, mu, diag);

#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      V3 lin, ang;
      if (P.joint[j].type == PK_JOINT_REVOLUTE) {
        ang = wj[j];
        lin = cross(wj[j], Tf[t].p - pj[j]);
      } else {
        ang = v3(0.f, 0.f, 0.f);
        lin = wj[j];
      }
      const V3 jl = mulT(Tf[t].R, lin);
      const V3 ja = mulT(Tf[t].R, ang);
      const V3 tl = mul(Am, jl) + mul(Bm, ja);
      const V3 ta = mul(Am, ja);
      const float on = (j <= Kt.body) ? -1.f : 0.f;  // joints past the frame do not move it
      A[6 * t + 0][j] = on * Kt.cost[0] * tl.x;
      A[6 * t + 1][j] = on * Kt.cost[1] * tl.y;
      A[6 * t + 2][j] = on * Kt.cost[2] * tl.z;
      A[6 * t + 3][j] = on * Kt.cost[3] * ta.x;
      A[6 * t + 4][j] = on * Kt.cost[4] * ta.y;
      A[6 * t + 5][j] = on * Kt.cost[5] * ta.z;
    }
  }

  // diagonal part: posture rows w (x_j + alpha e_j) and sqrt(diag) x_j merged into d_j x_j + beta_j
  {
    float se = 0.f;
    float pe[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      pe[j] = 0.f;
      if (P.has_posture) {
        const float* qref = P.posture_shared ? (P.shared + P.posture_off) : (trow + P.posture_off);
        pe[j] = q[j] - qref[j];
        se = fmaf(pe[j], pe[j], se);
      }
    }
    const float w2 = P.has_posture ? P.posture_w2 : 0.f;
    diag = fmaf(P.posture_lm * P.posture_gain * P.posture_gain * w2, se, diag);
    const float dd = sqrtf(w2 + diag);
    const float k = (dd > 0.f) ? P.posture_gain * w2 / dd : 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      d[j] = dd;
      beta[j] = k * pe[j];
    }
    if constexpr (ERR) {
      if ((emask >> NFT) & 1u) emax = err_max(emax, sqrtf(se));
      *err = emax;
      if (skip) return status;
    }
  }

  // ---- box rows ------------------------------------------------------------------
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const float vb = P.dt * P.vel[j];
    hi[j] = fminf(P.cfg_gain * (P.cfg_hi[j] - q[j]), vb);
    lo[j] = fmaxf(P.cfg_gain * (P.cfg_lo[j] - q[j]), -vb);
  }
  if (P.acc_enabled) {
    const float dt2 = P.dt * P.dt;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const float a = P.acc_max[j];
      if (a < 3.0e38f) {
        const float pv = P.acc_prev_off >= 0 ? trow[P.acc_prev_off + j] : 0.f;
        const float up = P.acc_qhi[j] - q[j], dn = q[j] - P.acc_qlo[j];
        if (up < 0.f || dn < 0.f) status |= PK_STATUS_NO_SOLUTION;  // sqrt of a negative margin: NaN rows
        const float hu = fminf(fmaf(a, dt2, pv), (up < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(up, 0.f)) : INFINITY);
        const float hl = fminf(fmaf(a, dt2, -pv), (dn < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(dn, 0.f)) : INFINITY);
        hi[j] = fminf(hi[j], hu);
        lo[j] = fmaxf(lo[j], -hl);
      }
    }
  }

  return status;
  }
};

template <int NJ, int NFT>
PK_HD void ik_step_chain(const ChainParams<NJ>& P, const float (&q)[NJ], const float* __restrict__ trow,
                         float (&v)[NJ], int& status_out, int flags = 0) {
  ChainStep<NJ, NFT> C;
  bool skip;
  int status = C.assemble(P, q, trow, skip);
  float x[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) x[j] = 0.f;
  if (!skip && !(status & PK_STATUS_NO_SOLUTION))
    status |= BoxLSQChol<6 * NFT, NJ>::run(C.A, C.b, C.d, C.beta, C.lo, C.hi, x, flags);
  // a NaN / Inf in q or in a target passes every comparison above and ends up in x:
  // report it (the reference's QP back-end fails on such a problem) instead of returning it
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) sum += x[j];
  const bool finite = fabsf(sum) < 3.0e38f;
  if (!finite) status |= PK_STATUS_NO_SOLUTION;
#pragma unroll
  for (int j = 0; j < NJ; ++j) v[j] = finite ? x[j] * P.inv_dt : 0.f;
  status_out = status;
}

// The rest of a converge step after C.assemble<true> returned `status` and `skip`: the QP of
// ik_step_chain, its status ORed into st_all.  Returns false, with q unchanged, when the freeze
// rule of the rollouts fires; otherwise moves q to q (+) v dt.
template <int NJ, int NFT>
PK_HD bool converge_chain_advance(const ChainParams<NJ>& P, ChainStep<NJ, NFT>& C, int status, bool skip,
                                  float (&q)[NJ], int& st_all, int flags) {
  int st = status;
  float x[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) x[j] = 0.f;
  if (!skip && !(st & PK_STATUS_NO_SOLUTION))
    st |= BoxLSQChol<6 * NFT, NJ>::run(C.A, C.b, C.d, C.beta, C.lo, C.hi, x, flags);
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) sum += x[j];
  const bool finite = fabsf(sum) < 3.0e38f;
  if (!finite) st |= PK_STATUS_NO_SOLUTION;
  st_all |= st & 0xff;
  if (step_failed(st_all, P.safety_break)) return false;
#pragma unroll
  for (int k = 0; k < NJ; ++k) q[k] = fmaf(finite ? x[k] * P.inv_dt : 0.f, P.dt, q[k]);  // q (+) v dt = q + v dt
  return true;
}

// Solve to a tolerance (pk_converge_prepared), one instance, q in registers.  For s = 0, 1, ...:
// err(q_s) = the largest |e_t|_2 of the tasks of `emask` (chain slots, see assemble); stop at
// q_s when err <= tol or s == max_steps; otherwise take the step ik_step_chain takes (its status
// ORed into status_out), stop at q_s if the freeze rule of the rollouts fires, and move to
// q_s (+) v dt.  On return q is where the instance stopped, err its error, steps the solves.
template <int NJ, int NFT>
PK_HD void converge_chain(const ChainParams<NJ>& P, float (&q)[NJ], const float* __restrict__ trow, unsigned emask,
                          float tol, int max_steps, float& err, int& steps, int& status_out, int flags = 0) {
  int st_all = 0;
  int s = 0;
#pragma unroll 1
  for (;; ++s) {
    ChainStep<NJ, NFT> C;
    bool skip;
    float e;
    const int status = C.template assemble<true>(P, q, trow, skip, emask, &e);
    err = e;
    if (e <= tol || s == max_steps) break;
    if (!converge_chain_advance(P, C, status, skip, q, st_all, flags)) {
      ++s;
      break;
    }
  }
  steps = s;
  status_out = st_all;
}

}  // namespace pk
