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
  // X~_j: placement in the parent joint frame with every joint axis re-oriented to the local
  // z axis (z_axis_joint_frames, pk_marshal.hpp), row-major [R | p]
  float X[12];
  int type;  // PK_JOINT_*
};

struct ChainFrameTask {
  int body;       // joint index the frame is fixed to (-1: world)
  float X[12];    // frame placement in that body's z-axis frame (z_axis_frame), or in the world
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
  // the arm shape (make_chain_params): at least one frame task, every joint revolute, every frame
  // task on the last joint, no AccelerationLimit; ik_chain_kernel then runs ChainStep::assemble<.., ARM>
  int arm;
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
  // ARM: the problem has the arm shape (ChainParams::arm), so the joint types, the bodies of the
  // frame tasks and acc_enabled are known at compile time; the results are bitwise those of ARM = false.
  // ERR (converge_chain): also store in *err the largest unweighted, gain-free |e_t|_2 of the
  // tasks of `emask` in chain slots (bit k < NFT: ft[k], bit NFT: the posture task).  An
  // instance outside its limits still runs the forward kinematics then, because its error is
  // wanted too; it returns right after the task errors.
  // POSE: a frame task's error is pose_err over the axes of `amask` (bit 6 k + r: row r of ft[k];
  // chain_axis_mask) with rscale = tol / orientation_tol, the separate-tolerance test.
  template <bool ERR = false, bool POSE = false, bool ARM = false>
  PK_HD int assemble(const ChainParams<NJ>& P, const float (&q)[NJ], const float* __restrict__ trow, bool& skip,
                     unsigned emask = 0u, float* err = nullptr, unsigned amask = 0u, float rscale = 0.f) {
  int status = 0;
  float emax = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j)
    if (q[j] < P.chk_lo[j] || q[j] > P.chk_hi[j]) status |= PK_STATUS_OUT_OF_LIMITS;
  skip = status && P.safety_break;
  if (skip && !ERR) return status;

  // ---- forward kinematics in z-axis joint frames: T~_j = T~_{j-1} X~_j M_z(q_j) ---------
  // T~_j has the origin of oMi[j] and the world axis of joint j as its third column
  SE3f T = identity_se3();
  V3 pj[NJ], wj[NJ];  // world origin and world axis of every joint
  SE3f Tf[NFT > 0 ? NFT : 1], Tb[NFT > 0 ? NFT : 1];
#pragma unroll
  for (int t = 0; t < NFT; ++t) Tb[t] = identity_se3();  // frames fixed to the world body
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const ChainJoint& Jn = P.joint[j];
    const SE3f X = load_se3(Jn.X);
    T = (j == 0) ? X : compose(T, X);  // T~_{-1} = I
    if (ARM || Jn.type == PK_JOINT_REVOLUTE) {
      float s, c;
      sincos_f(q[j], &s, &c);
#pragma unroll
      for (int r = 0; r < 3; ++r) {  // R Rz(q): rotate the first two columns
        const float x = T.R.m[3 * r], y = T.R.m[3 * r + 1];
        T.R.m[3 * r] = fmaf(c, x, s * y);
        T.R.m[3 * r + 1] = fmaf(c, y, -s * x);
      }
    } else {
      T.p = T.p + q[j] * v3(T.R.m[2], T.R.m[5], T.R.m[8]);
    }
    pj[j] = T.p;
    wj[j] = v3(T.R.m[2], T.R.m[5], T.R.m[8]);
    // remember the placement of the joint that carries each task frame (selects only;
    // the frame offset is composed once, after the sweep)
#pragma unroll
    for (int t = 0; t < (ARM ? 0 : NFT); ++t) {
      const bool here = P.ft[t].body == j;
#pragma unroll
      for (int k = 0; k < 9; ++k) Tb[t].R.m[k] = here ? T.R.m[k] : Tb[t].R.m[k];
      Tb[t].p.x = here ? T.p.x : Tb[t].p.x;
      Tb[t].p.y = here ? T.p.y : Tb[t].p.y;
      Tb[t].p.z = here ? T.p.z : Tb[t].p.z;
    }
  }
#pragma unroll
  for (int t = 0; t < NFT; ++t) Tf[t] = compose(ARM ? T : Tb[t], load_se3(P.ft[t].X));

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
    if constexpr (ERR && POSE) {
      if ((emask >> t) & 1u) {
        float l2 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if ((amask >> (6 * t + k)) & 1u) l2 = fmaf(e[k], e[k], l2);
          if ((amask >> (6 * t + 3 + k)) & 1u) a2 = fmaf(e[3 + k], e[3 + k], a2);
        }
        emax = err_max(emax, pose_err(l2, a2, rscale));
      }
    } else if constexpr (ERR) {
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
    M3 Am, Cm;
    jlog6_ac(Ttb, L, Am, Cm);
    // A column of the task is -diag(cost) [Am Tf^T lin + Cm Am Tf^T ang; Am Tf^T ang]: the
    // three 3x3 factors are formed once per task, so that a column costs 27 FMAs
    const M3 G = mulNT(Am, Tf[t].R);
    const M3 CG = mul(Cm, G);
    M3 Pl, Ql, Pa;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        Pl.m[3 * i + k] = -Kt.cost[i] * G.m[3 * i + k];
        Ql.m[3 * i + k] = -Kt.cost[i] * CG.m[3 * i + k];
        Pa.m[3 * i + k] = -Kt.cost[3 + i] * G.m[3 * i + k];
      }

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
      V3 tl, ta;
      if (ARM || P.joint[j].type == PK_JOINT_REVOLUTE) {
        const V3 lin = cross(wj[j], Tf[t].p - pj[j]);
        tl = mul(Pl, lin) + mul(Ql, wj[j]);
        ta = mul(Pa, wj[j]);
      } else {
        tl = mul(Pl, wj[j]);
        ta = v3(0.f, 0.f, 0.f);
      }
      // joints past the frame do not move it; ARM: a constant 1, whose products fold away
      const float on = (ARM || j <= Kt.body) ? 1.f : 0.f;
      A[6 * t + 0][j] = on * tl.x;
      A[6 * t + 1][j] = on * tl.y;
      A[6 * t + 2][j] = on * tl.z;
      A[6 * t + 3][j] = on * ta.x;
      A[6 * t + 4][j] = on * ta.y;
      A[6 * t + 5][j] = on * ta.z;
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
  if (!ARM && P.acc_enabled) {
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

template <int NJ, int NFT, bool ARM = false>
PK_HD void ik_step_chain(const ChainParams<NJ>& P, const float (&q)[NJ], const float* __restrict__ trow,
                         float (&v)[NJ], int& status_out, int flags = 0) {
  ChainStep<NJ, NFT> C;
  bool skip;
  int status = C.template assemble<false, false, ARM>(P, q, trow, skip);
  PK_PHASE(kPhaseAssembled);
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
// POSE, amask, rscale: the separate-tolerance test (ChainStep::assemble).
template <int NJ, int NFT, bool POSE = false>
PK_HD void converge_chain(const ChainParams<NJ>& P, float (&q)[NJ], const float* __restrict__ trow, unsigned emask,
                          float tol, int max_steps, float& err, int& steps, int& status_out, int flags = 0,
                          unsigned amask = 0u, float rscale = 0.f) {
  int st_all = 0;
  int s = 0;
#pragma unroll 1
  for (;; ++s) {
    ChainStep<NJ, NFT> C;
    bool skip;
    float e;
    const int status = C.template assemble<true, POSE>(P, q, trow, skip, emask, &e, amask, rscale);
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

// Instance i of ik_chain_converge_kernel: converge_chain from q row i, where it stopped into q_out
// row i, then err, steps and status (each unless null).  q_out may alias q (the row is read before
// it is written).  POSE, amask, rscale: as converge_chain.
template <int NJ, int NFT, bool POSE = false>
PK_HD void converge_chain_instance(const ChainParams<NJ>& P, const float* q, const float* __restrict__ targets,
                                   unsigned emask, float tol, int max_steps, float* q_out, float* __restrict__ err,
                                   int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t i,
                                   unsigned amask = 0u, float rscale = 0.f) {
  float qi[NJ];
#pragma unroll
  for (int k = 0; k < NJ; ++k) qi[k] = q[i * NJ + k];
  float e;
  int n, st;
  converge_chain<NJ, NFT, POSE>(P, qi, targets + i * (int64_t)P.target_stride, emask, tol, max_steps, e, n, st, 0,
                                amask, rscale);
#pragma unroll
  for (int k = 0; k < NJ; ++k) q_out[i * NJ + k] = qi[k];
  if (err) err[i] = e;
  if (steps) steps[i] = n;
  if (status) status[i] = st;
}

// Records of step s of a trajectory (thread-per-instance chain kernel); `frozen`: v row of zeros.
template <int NJ>
PK_HD void chain_record(const Trajectory& T, int s, int64_t B, int64_t i, const float (&qi)[NJ],
                        const float (&vi)[NJ], int st_all, bool frozen) {
  const int64_t r = (int64_t)s * B + i;
  if (T.q) {
#pragma unroll
    for (int k = 0; k < NJ; ++k) T.q[r * NJ + k] = qi[k];
  }
  if (T.v) {
#pragma unroll
    for (int k = 0; k < NJ; ++k) T.v[r * NJ + k] = frozen ? 0.f : vi[k];
  }
  if (T.status) T.status[r] = st_all;
}

// Closed-loop rollout of instance i (ik_chain_kernel): n_steps iterations of ik_step_chain, each
// followed by q <- q (+) v dt when n_steps > 1 or `integrate`; an instance whose statuses so far
// fail the freeze rule takes no further step.  Returns the OR of the statuses of the steps that
// ran; v is the last step's.  RECORD: the targets row advances by T.target_step after every step,
// and the records of T are stored (a frozen instance fills its remaining steps with q unchanged
// and v = 0).
template <int NJ, int NFT, bool RECORD, bool ARM = false>
PK_HD int rollout_chain(const ChainParams<NJ>& P, float (&qi)[NJ], const float* trow, float (&vi)[NJ], int n_steps,
                        bool integrate, int flags, const Trajectory& T, int64_t B, int64_t i) {
  int st_all = 0;
#pragma unroll
  for (int k = 0; k < NJ; ++k) vi[k] = 0.f;
#pragma unroll 1
  for (int step_no = 0; step_no < n_steps; ++step_no) {
    if (step_failed(st_all, P.safety_break)) {
      if constexpr (RECORD) {
#pragma unroll 1
        for (int s = step_no; s < n_steps; ++s) chain_record<NJ>(T, s, B, i, qi, vi, st_all, true);
      }
      break;
    }
    int st;
    ik_step_chain<NJ, NFT, ARM>(P, qi, trow, vi, st, flags);
    st_all |= st & 0xff;
    if (n_steps > 1 || integrate) {
#pragma unroll
      for (int k = 0; k < NJ; ++k) qi[k] = fmaf(vi[k], P.dt, qi[k]);  // 1-dof joints: q (+) v dt = q + v dt
    }
    if constexpr (RECORD) {
      trow += T.target_step;
      chain_record<NJ>(T, step_no, B, i, qi, vi, st_all, false);
    }
  }
  return st_all;
}

}  // namespace pk
