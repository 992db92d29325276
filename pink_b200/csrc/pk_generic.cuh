// General IK step: any joint tree (optional free-flyer), any mix of FrameTask /
// RelativeFrameTask / PostureTask / ComTask, box limits.  One instance per thread
// with run-time sized per-thread arrays.  This is the path every model can take;
// it also backs the export entry points (build_ik, task terms, FK, frame Jacobian).
// The register-resident chain kernel (pk_chain.cuh) and the warp-cooperative tree
// kernel (pk_tree.cuh) are specialisations that must agree with it.
//
// Reference path: see the list at the top of pk_chain.cuh, plus
//   RelativeFrameTask   pink/tasks/relative_frame_task.py:173-246
//   ComTask             pink/tasks/com_task.py:120-148
//   free-flyer columns  pink/configuration.py:220-228 (SURVEY.md section 9)
#pragma once

#include "pk_math.cuh"
#include "pk_lsq.cuh"
#include "pk_dualqp.cuh"

namespace pk {

// Device-resident constant tables of a model (pointers into one device buffer).
struct DevModel {
  int njoints, free_flyer, nq, nv, nframes;
  const int* parent;       // [njoints]
  const int* jtype;        // [njoints]
  const float* jX;         // [njoints][12]
  const float* axis;       // [njoints][3]
  const int* frame_body;   // [nframes]
  const float* fX;         // [nframes][12]
  const float* mass;       // [njoints + 1]
  const float* com;        // [njoints + 1][3]
  const uint64_t* anc;     // [njoints + 2] joints on the path to body b (index b + 2)
  const int* depth;        // [njoints] number of 1-dof ancestors
  int maxdepth;
  float total_mass;
};

struct DevTask {
  int type, frame, root, tgt_off, tgt_shared, body, root_body;
  float cost[6];
  float gain, lm;
  int rows, data_off;  // PK_TASK_LINEAR
};

struct DevBarrier {
  int type, frame, frame2, body, body2, dim, nidx, idx[3], has_min, has_max;
  float p_min[3], p_max[3], gain[6], d_min, safe_gain;
  int gain_fn, npairs, pair_off, data_off;
};

// Optional parts of a problem (barriers, equality constraints, opt-in limits, constant
// data of LINEAR tasks); lives in device memory, reached through DevProblem::ext.
struct DevExtras {
  int nbarriers;
  DevBarrier barriers[PK_MAX_BARRIERS];
  int nconstraints;
  DevTask constraints[PK_MAX_CONSTRAINTS];
  int fb_enabled, fb_frame, fb_body;
  float fb_max[6];
  int acc_enabled, acc_prev_off, acc_prev_shared;
  float acc_max[PK_MAX_NV], acc_qlo[PK_MAX_NV], acc_qhi[PK_MAX_NV];
  const float* extra;
  const int* pairs;
  int n_ineq_rows, n_eq_rows;  // totals (validated against PK_MAX_*_ROWS on the host)
};

// Problem description as the kernels read it (filled from PkProblemDesc).
struct DevProblem {
  int ntasks;
  DevTask tasks[PK_MAX_TASKS];
  float dt, inv_dt, damping, cfg_gain;
  int target_stride, safety_break;
  float cfg_lo[PK_MAX_NV], cfg_hi[PK_MAX_NV], vel[PK_MAX_NV], chk_lo[PK_MAX_NV], chk_hi[PK_MAX_NV];
  float shared[PK_MAX_SHARED];
  const DevExtras* ext;  // nullptr: tasks + box limits only
};

// Tasks whose Jacobian is I[root_nv:, :] (they only touch the diagonal terms).
PK_HD bool is_diag_task(int type) { return type == PK_TASK_POSTURE || type == PK_TASK_JOINT_VELOCITY; }
// Error of such a task on tangent coordinate i >= rv: posture q_i - q*_i
// (pink/tasks/posture_task.py:100-107), joint velocity dq_ref,i
// (pink/tasks/joint_velocity_task.py:59-80; zeros for DampingTask).
PK_HD float diag_task_error(int type, const float* q, const float* tgt, int i, int rq, int rv) {
  return type == PK_TASK_POSTURE ? q[i + rq - rv] - tgt[i + rq - rv] : tgt[i - rv];
}

// Optional per-instance outputs of the export entry points (nullptr = skip).
struct GenericOut {
  float* v;        // [nv]
  int32_t* status; // [1]
  float* H;        // [nv][nv]
  float* c;        // [nv]
  float* h;        // [4][nv]
  float* e;        // [k]   of task `task_index`
  float* J;        // [k][nv]
  int task_index;
  float* oMf;      // [nframes][12]
  float* com;      // [3]
  float* Jf;       // [6][nv] LOCAL Jacobian of frame `jac_frame`
  int jac_frame;
  float* G;        // [PK_MAX_INEQ_ROWS][nv] dense inequality rows
  float* hG;       // [PK_MAX_INEQ_ROWS]
  float* E;        // [PK_MAX_EQ_ROWS][nv] equality rows
  float* f;        // [PK_MAX_EQ_ROWS]
  float* lo;       // [nv] box
  float* hi;       // [nv]
};

// The same outputs for a whole batch (rows of instance i at i times the row sizes above), with
// the inputs; task_k = rows of task `task_index`.
struct GenericArgs {
  const float* q;
  const float* targets;
  float* v;
  int32_t* status;
  float* H;
  float* c;
  float* h;
  float* e;
  float* J;
  int task_index;
  int task_k;
  float* oMf;
  float* com;
  float* Jf;
  int jac_frame;
  float* G;
  float* hG;
  float* E;
  float* f;
  float* lo;
  float* hi;
};

// Outputs of instance i.
PK_HD GenericOut generic_out(const DevModel& M, const GenericArgs& A, int64_t i) {
  const int nv = M.nv;
  GenericOut out;
  out.v = A.v ? A.v + i * nv : nullptr;
  out.status = A.status ? A.status + i : nullptr;
  out.H = A.H ? A.H + i * nv * nv : nullptr;
  out.c = A.c ? A.c + i * nv : nullptr;
  out.h = A.h ? A.h + i * 4 * nv : nullptr;
  out.e = A.e ? A.e + i * A.task_k : nullptr;
  out.J = A.J ? A.J + i * A.task_k * nv : nullptr;
  out.task_index = A.task_index;
  out.oMf = A.oMf ? A.oMf + i * M.nframes * 12 : nullptr;
  out.com = A.com ? A.com + i * 3 : nullptr;
  out.Jf = A.Jf ? A.Jf + i * 6 * nv : nullptr;
  out.jac_frame = A.jac_frame;
  out.G = A.G ? A.G + i * PK_MAX_INEQ_ROWS * nv : nullptr;
  out.hG = A.hG ? A.hG + i * PK_MAX_INEQ_ROWS : nullptr;
  out.E = A.E ? A.E + i * PK_MAX_EQ_ROWS * nv : nullptr;
  out.f = A.f ? A.f + i * PK_MAX_EQ_ROWS : nullptr;
  out.lo = A.lo ? A.lo + i * nv : nullptr;
  out.hi = A.hi ? A.hi + i * nv : nullptr;
  return out;
}

// stacked task rows: 6 per frame task, 3 per CoM task; every task set the ABI can describe fits
// (nothing is ever truncated)
constexpr int kGenericMaxRows = 6 * PK_MAX_TASKS;
static_assert(kGenericMaxRows >= 6 * PK_MAX_TASKS, "a describable task set must fit the row buffer");

template <int NJMAX, int NVMAX>
struct Generic {
  SE3f root;
  SE3f Tw[NJMAX];

  PK_HD SE3f body_placement(int body) const {
    if (body == -2) return identity_se3();
    if (body == -1) return root;
    return Tw[body];
  }

  PK_HD void forward_kinematics(const DevModel& M, const float* q) {
    int rq = 0;
    root = identity_se3();
    if (M.free_flyer) {
      root.p = v3(q[0], q[1], q[2]);
      root.R = quat_to_matrix(q[3], q[4], q[5], q[6]);
      rq = 7;
    }
    for (int j = 0; j < M.njoints; ++j) {
      const SE3f X = load_se3(M.jX + 12 * j);
      const V3 axis = v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]);
      SE3f Tl;
      if (M.jtype[j] == PK_JOINT_REVOLUTE) {
        float s, c;
        sincos_f(q[rq + j], &s, &c);
        Tl.R = mul(X.R, rot_axis(axis, s, c));
        Tl.p = X.p;
      } else {
        Tl.R = X.R;
        Tl.p = X.p + mul(X.R, q[rq + j] * axis);
      }
      const int par = M.parent[j];
      Tw[j] = compose(par < 0 ? root : Tw[par], Tl);
    }
  }

  // Column `i` (tangent index) of the LOCAL Jacobian of a frame placed at Tf on `body`.
  PK_HD void frame_jac_col(const DevModel& M, int body, const SE3f& Tf, int i, V3& lin, V3& ang) const {
    lin = v3(0.f, 0.f, 0.f);
    ang = v3(0.f, 0.f, 0.f);
    const int rv = M.free_flyer ? 6 : 0;
    if (i < rv) {
      if (body == -2) return;
      // Ad_{(oM_root^-1 oMf)^-1}: base twist seen from the frame
      const SE3f Trf = act_inv(root, Tf);
      const V3 ek = v3(i % 3 == 0 ? 1.f : 0.f, i % 3 == 1 ? 1.f : 0.f, i % 3 == 2 ? 1.f : 0.f);
      if (i < 3) {
        lin = mulT(Trf.R, ek);
      } else {
        lin = mulT(Trf.R, cross(ek, Trf.p));
        ang = mulT(Trf.R, ek);
      }
      return;
    }
    const int j = i - rv;
    if (body < 0 || !((M.anc[body + 2] >> j) & 1ull)) return;
    const V3 axis = v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]);
    const V3 aw = mul(Tw[j].R, axis);
    if (M.jtype[j] == PK_JOINT_REVOLUTE) {
      lin = mulT(Tf.R, cross(aw, Tf.p - Tw[j].p));
      ang = mulT(Tf.R, aw);
    } else {
      lin = mulT(Tf.R, aw);
    }
  }

  PK_HD V3 center_of_mass(const DevModel& M) const {
    V3 acc = v3(0.f, 0.f, 0.f);
    for (int b = -1; b < M.njoints; ++b) {
      const float m = M.mass[b + 1];
      if (m == 0.f) continue;
      const SE3f T = body_placement(b);
      const V3 cl = v3(M.com[3 * (b + 1)], M.com[3 * (b + 1) + 1], M.com[3 * (b + 1) + 2]);
      acc = acc + m * (mul(T.R, cl) + T.p);
    }
    return (1.f / M.total_mass) * acc;
  }

  // Error e[k] and Jacobian Jw[k][nv] of one (non-diagonal) task; returns k.
  // FrameTask pink/tasks/frame_task.py:178-227, RelativeFrameTask
  // relative_frame_task.py:173-246, ComTask com_task.py:120-148, LinearHolonomicTask
  // linear_holonomic_task.py:148-192.
  PK_HD int task_rows(const DevModel& M, const DevProblem& P, const DevTask& Kt, const float* q, const float* tgt,
                      float (&e)[6], float (&Jw)[6][NVMAX]) const {
    const int nv = M.nv;
    const int rq = M.free_flyer ? 7 : 0;
    const int rv = M.free_flyer ? 6 : 0;
    if (Kt.type == PK_TASK_LINEAR) {
      const float* A = P.ext->extra + Kt.data_off;
      const float* bb = A + Kt.rows * nv;
      const float* q0 = bb + Kt.rows;
      for (int r = 0; r < Kt.rows; ++r) {
        float s = -bb[r];
        for (int i = 0; i < nv; ++i) {
          Jw[r][i] = A[r * nv + i];
          if (i >= rv) s = fmaf(A[r * nv + i], q[i + rq - rv] - q0[i + rq - rv], s);
        }
        e[r] = s;
      }
      for (int r = Kt.rows; r < 6; ++r) e[r] = 0.f;
      return Kt.rows;
    }
    if (Kt.type == PK_TASK_COM) {
      const V3 cm = center_of_mass(M);
      e[0] = cm.x - tgt[0]; e[1] = cm.y - tgt[1]; e[2] = cm.z - tgt[2];
      e[3] = e[4] = e[5] = 0.f;
      // subtree masses and first moments, leaves to root
      float sm[NJMAX];
      V3 smc[NJMAX];
      for (int j = 0; j < M.njoints; ++j) {
        const V3 cl = v3(M.com[3 * (j + 1)], M.com[3 * (j + 1) + 1], M.com[3 * (j + 1) + 2]);
        sm[j] = M.mass[j + 1];
        smc[j] = sm[j] * (mul(Tw[j].R, cl) + Tw[j].p);
      }
      for (int j = M.njoints - 1; j >= 0; --j) {
        const int par = M.parent[j];
        if (par >= 0) { sm[par] += sm[j]; smc[par] = smc[par] + smc[j]; }
      }
      const float invM = 1.f / M.total_mass;
      for (int i = 0; i < nv; ++i) {
        V3 col = v3(0.f, 0.f, 0.f);
        if (i < rv) {
          const V3 ek = v3(i % 3 == 0 ? 1.f : 0.f, i % 3 == 1 ? 1.f : 0.f, i % 3 == 2 ? 1.f : 0.f);
          if (i < 3) col = mul(root.R, ek);
          else col = mul(root.R, cross(ek, mulT(root.R, cm - root.p)));
        } else {
          const int j = i - rv;
          if (sm[j] > 0.f) {
            const V3 axis = v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]);
            const V3 aw = mul(Tw[j].R, axis);
            if (M.jtype[j] == PK_JOINT_REVOLUTE)
              col = (sm[j] * invM) * cross(aw, (1.f / sm[j]) * smc[j] - Tw[j].p);
            else
              col = (sm[j] * invM) * aw;
          }
        }
        Jw[0][i] = col.x; Jw[1][i] = col.y; Jw[2][i] = col.z;
      }
      return 3;
    }
    const SE3f Tf = compose(body_placement(Kt.body), load_se3(M.fX + 12 * Kt.frame));
    const SE3f Tt = load_se3(tgt);
    M3 Am, Bm;
    float sign;
    SE3f Trf;  // relative task: frame in root-frame coordinates
    SE3f Tr;
    if (Kt.type == PK_TASK_FRAME) {
      const SE3f Tbt = act_inv(Tf, Tt);
      Log3 L = log3(Tbt.R);
      log6(Tbt, L, e);
      SE3f Ttb;
      for (int a = 0; a < 3; ++a)
        for (int c2 = 0; c2 < 3; ++c2) Ttb.R.m[3 * a + c2] = Tbt.R.m[3 * c2 + a];
      Ttb.p = -1.f * mul(Ttb.R, Tbt.p);
      L.w = -1.f * L.w;
      jlog6(Ttb, L, Am, Bm);
      sign = -1.f;
      Trf = identity_se3();
      Tr = identity_se3();
    } else {
      Tr = compose(body_placement(Kt.root_body), load_se3(M.fX + 12 * Kt.root));
      Trf = act_inv(Tr, Tf);
      const SE3f Ttf = act_inv(Tt, Trf);
      const Log3 L = log3(Ttf.R);
      log6(Ttf, L, e);
      jlog6(Ttf, L, Am, Bm);
      sign = 1.f;
    }
    for (int i = 0; i < nv; ++i) {
      V3 lin, ang;
      frame_jac_col(M, Kt.body, Tf, i, lin, ang);
      if (Kt.type == PK_TASK_RELATIVE_FRAME) {
        V3 rl, ra;
        frame_jac_col(M, Kt.root_body, Tr, i, rl, ra);
        // Ad_{T_rf^-1} [rl; ra] = [R^T (rl - p x ra); R^T ra]
        lin = lin - mulT(Trf.R, rl - cross(Trf.p, ra));
        ang = ang - mulT(Trf.R, ra);
      }
      const V3 tl = sign * (mul(Am, lin) + mul(Bm, ang));
      const V3 ta = sign * mul(Am, ang);
      Jw[0][i] = tl.x; Jw[1][i] = tl.y; Jw[2][i] = tl.z;
      Jw[3][i] = ta.x; Jw[4][i] = ta.y; Jw[5][i] = ta.z;
    }
    return 6;
  }

  // World-frame velocity of the origin of a frame placed at Tf on `body`, per unit of
  // tangent coordinate i: R_f J_f[:3, i] (pink/barriers/position_barrier.py:139-146).
  PK_HD V3 point_jac_col(const DevModel& M, int body, const SE3f& Tf, int i) const {
    V3 lin, ang;
    frame_jac_col(M, body, Tf, i, lin, ang);
    return mul(Tf.R, lin);
  }

  // Distance-type barriers between two bodies of the same robot do not depend on
  // coordinates that move both bodies rigidly: the floating base and every joint that
  // supports both.  Analytically those Jacobian columns are exactly zero; computed as a
  // difference of two point Jacobians in fp32 they come out as ~1e-7 |J| / dt of
  // cancellation noise, which an active barrier row with a large multiplier turns into
  // visible motion of the unbounded base.  true -> the column is zero by construction.
  PK_HD static bool rigid_for_both(const DevModel& M, int body_a, int body_b, int i) {
    if (body_a == -2 || body_b == -2) return false;
    const int rv = M.free_flyer ? 6 : 0;
    if (i < rv) return true;
    const uint64_t common = M.anc[body_a + 2] & M.anc[body_b + 2];
    return (common >> (i - rv)) & 1ull;
  }

  PK_HD static float barrier_gain_fn(int fn, float h) { return fn == PK_GAINFN_SATURATING ? h / (1.f + fabsf(h)) : h; }

  // Rows of one barrier: Jh[dim][nv] = dh/dq and hv[dim] = h(q).
  PK_HD void barrier_rows(const DevModel& M, const DevExtras& X, const DevBarrier& Bd, float (*Jh)[NVMAX],
                          float* hv) const {
    const int nv = M.nv;
    if (Bd.type == PK_BARRIER_POSITION) {
      const SE3f Tf = compose(body_placement(Bd.body), load_se3(M.fX + 12 * Bd.frame));
      const float pw[3] = {Tf.p.x, Tf.p.y, Tf.p.z};
      int r = 0;
      if (Bd.has_min)
        for (int k = 0; k < Bd.nidx; ++k) hv[r++] = pw[Bd.idx[k]] - Bd.p_min[k];
      if (Bd.has_max)
        for (int k = 0; k < Bd.nidx; ++k) hv[r++] = Bd.p_max[k] - pw[Bd.idx[k]];
      for (int i = 0; i < nv; ++i) {
        const V3 c = point_jac_col(M, Bd.body, Tf, i);
        const float cw[3] = {c.x, c.y, c.z};
        int rr = 0;
        if (Bd.has_min)
          for (int k = 0; k < Bd.nidx; ++k) Jh[rr++][i] = cw[Bd.idx[k]];
        if (Bd.has_max)
          for (int k = 0; k < Bd.nidx; ++k) Jh[rr++][i] = -cw[Bd.idx[k]];
      }
      return;
    }
    if (Bd.type == PK_BARRIER_BODY_SPHERICAL) {
      const SE3f T1 = compose(body_placement(Bd.body), load_se3(M.fX + 12 * Bd.frame));
      const SE3f T2 = compose(body_placement(Bd.body2), load_se3(M.fX + 12 * Bd.frame2));
      const V3 dp = T1.p - T2.p;
      hv[0] = dot(dp, dp) - Bd.d_min * Bd.d_min;
      for (int i = 0; i < nv; ++i)
        Jh[0][i] = rigid_for_both(M, Bd.body, Bd.body2, i)
                       ? 0.f
                       : 2.f * dot(dp, point_jac_col(M, Bd.body, T1, i) - point_jac_col(M, Bd.body2, T2, i));
      return;
    }
    // SELF_COLLISION on sphere pairs: the `dim` smallest distances
    // (pink/barriers/self_collision_barrier.py:108-127, 169-224)
    float dist[PK_MAX_PAIRS];
    const int* pr = X.pairs + 2 * Bd.pair_off;
    const float* rad = X.extra + Bd.data_off;
    for (int k = 0; k < Bd.npairs; ++k) {
      const int fa = pr[2 * k], fb = pr[2 * k + 1];
      const SE3f Ta = body_placement(M.frame_body[fa]);
      const SE3f Tb = body_placement(M.frame_body[fb]);
      const V3 ca = mul(Ta.R, v3(M.fX[12 * fa + 3], M.fX[12 * fa + 7], M.fX[12 * fa + 11])) + Ta.p;
      const V3 cb = mul(Tb.R, v3(M.fX[12 * fb + 3], M.fX[12 * fb + 7], M.fX[12 * fb + 11])) + Tb.p;
      const V3 dp = ca - cb;
      dist[k] = sqrtf(dot(dp, dp)) - rad[2 * k] - rad[2 * k + 1];
    }
    for (int r = 0; r < Bd.dim; ++r) {
      int best = -1;
      float bd = 3.0e38f;
      for (int k = 0; k < Bd.npairs; ++k)
        if (dist[k] < bd) { bd = dist[k]; best = k; }
      hv[r] = bd - Bd.d_min;
      for (int i = 0; i < nv; ++i) Jh[r][i] = 0.f;
      if (best < 0) continue;
      dist[best] = 3.0e38f;  // taken
      const int fa = pr[2 * best], fb = pr[2 * best + 1];
      const SE3f Ta = compose(body_placement(M.frame_body[fa]), load_se3(M.fX + 12 * fa));
      const SE3f Tb = compose(body_placement(M.frame_body[fb]), load_se3(M.fX + 12 * fb));
      const V3 dp = Ta.p - Tb.p;
      const float gap = sqrtf(dot(dp, dp));
      // nearest points w1 - w2 = (gap - ra - rb) u: coincident -> zero row (:198-199)
      if (!(gap > 0.f) || fabsf(bd) <= 1e-8f) continue;
      const V3 n = ((bd < 0.f ? -1.f : 1.f) / gap) * dp;
      for (int i = 0; i < nv; ++i)
        Jh[r][i] = rigid_for_both(M, M.frame_body[fa], M.frame_body[fb], i)
                       ? 0.f
                       : dot(n, point_jac_col(M, M.frame_body[fa], Ta, i) - point_jac_col(M, M.frame_body[fb], Tb, i));
    }
  }

  // One step. `q` [nq], `trow` per-instance targets.
  // ERR (converge_generic): also the stop test `ct` on the task errors, made before the QP; a
  // step that stops there writes only *out.status (and ct).  Test: the stop rule, ct->decide(err)
  // (ConvergeTest: this instance's own; the multi-start kernel's decides for a group of seeds).
  template <bool ERR = false, class Test = ConvergeTest>
  PK_HD void step(const DevModel& M, const DevProblem& P, const float* q, const float* trow, const GenericOut& out,
                  Test* ct = nullptr) {
    const int nv = M.nv;
    const int rq = M.free_flyer ? 7 : 0;
    const int rv = M.free_flyer ? 6 : 0;
    int status = 0;
    for (int i = rv; i < nv; ++i) {
      const float qi = q[i + rq - rv];
      if (qi < P.chk_lo[i] || qi > P.chk_hi[i]) status |= PK_STATUS_OUT_OF_LIMITS;
    }
    const bool skip = status && P.safety_break;

    forward_kinematics(M, q);

    if (out.oMf) {
      for (int f = 0; f < M.nframes; ++f) {
        const SE3f Tf = compose(body_placement(M.frame_body[f]), load_se3(M.fX + 12 * f));
        store_se3(Tf, out.oMf + 12 * f);
      }
    }
    if (out.com) {
      const V3 cm = center_of_mass(M);
      out.com[0] = cm.x; out.com[1] = cm.y; out.com[2] = cm.z;
    }
    if (out.Jf) {
      const int f = out.jac_frame;
      const int body = M.frame_body[f];
      const SE3f Tf = compose(body_placement(body), load_se3(M.fX + 12 * f));
      for (int i = 0; i < nv; ++i) {
        V3 lin, ang;
        frame_jac_col(M, body, Tf, i, lin, ang);
        out.Jf[0 * nv + i] = lin.x; out.Jf[1 * nv + i] = lin.y; out.Jf[2 * nv + i] = lin.z;
        out.Jf[3 * nv + i] = ang.x; out.Jf[4 * nv + i] = ang.y; out.Jf[5 * nv + i] = ang.z;
      }
    }
    if (!P.ntasks && !out.v && !out.H && !out.G && !out.E && !out.lo) {
      if (out.status) *out.status = status;
      return;
    }

    // square-root form of the objective: rows of A / b, diagonal terms d / beta
    float A[kGenericMaxRows][NVMAX];
    float b[kGenericMaxRows];
    float d[NVMAX], beta[NVMAX];
    float pw2[NVMAX], pc[NVMAX];  // posture contributions to H_ii and c_i
    for (int i = 0; i < nv; ++i) { pw2[i] = 0.f; pc[i] = 0.f; }
    int K = 0;
    float diag = P.damping;
    float Jw[6][NVMAX];
    float emax = 0.f;  // ERR: largest |e_t|_2 of the tasks of ct->mask

    for (int t = 0; t < P.ntasks; ++t) {
      const DevTask& Kt = P.tasks[t];
      const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (trow + Kt.tgt_off);
      const bool want = (out.e != nullptr || out.J != nullptr) && out.task_index == t;
      if (is_diag_task(Kt.type)) {
        // J = I[root_nv:, :]; e = (q (-) q*)[root_nv:] or dq_ref
        const float w2 = Kt.cost[0] * Kt.cost[0];
        float se = 0.f;
        for (int i = rv; i < nv; ++i) {
          const float e = diag_task_error(Kt.type, q, tgt, i, rq, rv);
          se = fmaf(e, e, se);
          pw2[i] += w2;
          pc[i] = fmaf(Kt.gain * w2, e, pc[i]);
          if (want && out.e) out.e[i - rv] = e;
        }
        diag = fmaf(Kt.lm * Kt.gain * Kt.gain * w2, se, diag);
        if constexpr (ERR) {
          if ((ct->mask >> t) & 1u) emax = err_max(emax, sqrtf(se));
        }
        if (want && out.J)
          for (int r = 0; r < nv - rv; ++r)
            for (int i = 0; i < nv; ++i) out.J[r * nv + i] = (i == r + rv) ? 1.f : 0.f;
        continue;
      }
      float e[6];
      const int k = task_rows(M, P, Kt, q, tgt, e, Jw);
      if constexpr (ERR) {
        if ((ct->mask >> t) & 1u) {
          float n2 = 0.f;
          for (int r = 0; r < k; ++r) n2 = fmaf(e[r], e[r], n2);
          emax = err_max(emax, sqrtf(n2));
        }
      }
      if (want) {
        if (out.e)
          for (int r = 0; r < k; ++r) out.e[r] = e[r];
        if (out.J)
          for (int r = 0; r < k; ++r)
            for (int i = 0; i < nv; ++i) out.J[r * nv + i] = Jw[r][i];
      }
      float mu = 0.f;
      for (int r = 0; r < k; ++r) {
        const float ew = Kt.cost[r] * Kt.gain * e[r];
        mu = fmaf(ew, ew, mu);
        if (Kt.cost[r] == 0.f) continue;  // zero cost == row deleted (tests/test_frame_task.py:143-181)
        if (K < kGenericMaxRows) {
          b[K] = ew;
          for (int i = 0; i < nv; ++i) A[K][i] = Kt.cost[r] * Jw[r][i];
        }
        ++K;
      }
      diag = fmaf(Kt.lm, mu, diag);
    }
    if (K > kGenericMaxRows) { status |= PK_STATUS_NOT_POSDEF; K = kGenericMaxRows; }
    if constexpr (ERR) {
      ct->decide(emax);
      ct->status = status;
      if (ct->stop) {
        if (out.status) *out.status = status;
        return;
      }
    }

    // box of all +-e_i rows: configuration and velocity limits ...
    float lo[NVMAX], hi[NVMAX];
    for (int i = 0; i < nv; ++i) {
      const float qi = (i >= rv) ? q[i + rq - rv] : 0.f;
      const float vb = P.dt * P.vel[i];
      const float ch = P.cfg_gain * (P.cfg_hi[i] - qi);
      const float cl = P.cfg_gain * (P.cfg_lo[i] - qi);
      hi[i] = fminf(ch, vb);
      lo[i] = fmaxf(cl, -vb);
      if (out.h) {
        out.h[0 * nv + i] = ch;
        out.h[1 * nv + i] = -cl;
        out.h[2 * nv + i] = vb;
        out.h[3 * nv + i] = vb;
      }
    }

    // ---- optional parts: dense inequality rows, equality rows, acceleration box ----
    constexpr int MG = PK_MAX_INEQ_ROWS, ME = PK_MAX_EQ_ROWS;
    int p = 0, meq = 0;
    if (P.ext) {
      const DevExtras& X = *P.ext;
      float Gg[MG][NVMAX], hg[MG], Eq[ME][NVMAX], fe[ME];
      if (X.acc_enabled) {
        // ... and AccelerationLimit (pink/limits/acceleration_limit.py:119-200)
        const float* prev = X.acc_prev_off < 0 ? nullptr
                                                : (X.acc_prev_shared ? P.shared + X.acc_prev_off : trow + X.acc_prev_off);
        const float dt2 = P.dt * P.dt;
        for (int i = 0; i < nv; ++i) {
          const float a = X.acc_max[i];
          if (!(a < 3.0e38f)) continue;
          const float pv = prev ? prev[i] : 0.f;
          const float qi = (i >= rv) ? q[i + rq - rv] : 0.f;
          const float up = X.acc_qhi[i] - qi, dn = qi - X.acc_qlo[i];
          if (up < 0.f || dn < 0.f) status |= PK_STATUS_NO_SOLUTION;  // sqrt of a negative margin: NaN rows
          const float hu = fminf(fmaf(a, dt2, pv), (up < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(up, 0.f)) : INFINITY);
          const float hl = fminf(fmaf(a, dt2, -pv), (dn < 3.0e38f) ? P.dt * sqrtf(2.f * a * fmaxf(dn, 0.f)) : INFINITY);
          hi[i] = fminf(hi[i], hu);
          lo[i] = fmaxf(lo[i], -hl);
        }
      }
      if (X.fb_enabled) {
        // FloatingBaseVelocityLimit (pink/limits/floating_base_velocity_limit.py:118-148)
        const SE3f Tf = compose(body_placement(X.fb_body), load_se3(M.fX + 12 * X.fb_frame));
        const int p0 = p;
        int nfin = 0;
        for (int r = 0; r < 6; ++r) nfin += (X.fb_max[r] < 3.0e38f) ? 1 : 0;
        for (int i = 0; i < nv; ++i) {
          V3 lin = v3(0.f, 0.f, 0.f), ang = v3(0.f, 0.f, 0.f);
          if (i < rv) frame_jac_col(M, X.fb_body, Tf, i, lin, ang);
          const float col[6] = {lin.x, lin.y, lin.z, ang.x, ang.y, ang.z};
          int rr = 0;
          for (int r = 0; r < 6; ++r)
            if (X.fb_max[r] < 3.0e38f) {
              Gg[p0 + rr][i] = col[r];
              Gg[p0 + nfin + rr][i] = -col[r];
              ++rr;
            }
        }
        int rr = 0;
        for (int r = 0; r < 6; ++r)
          if (X.fb_max[r] < 3.0e38f) {
            hg[p0 + rr] = hg[p0 + nfin + rr] = P.dt * X.fb_max[r];
            ++rr;
          }
        p += 2 * nfin;
      }
      for (int bi = 0; bi < X.nbarriers; ++bi) {
        const DevBarrier& Bd = X.barriers[bi];
        barrier_rows(M, X, Bd, &Gg[p], &hg[p]);
        float fro = 0.f;
        for (int r = 0; r < Bd.dim; ++r) {
          const float g = Bd.gain[Bd.type == PK_BARRIER_POSITION ? r : 0];
          hg[p + r] = g * barrier_gain_fn(Bd.gain_fn, hg[p + r]);
          for (int i = 0; i < nv; ++i) {
            fro = fmaf(Gg[p + r][i], Gg[p + r][i], fro);
            Gg[p + r][i] *= -P.inv_dt;  // G = -J_h / dt (pink/barriers/barrier.py:246)
          }
        }
        if (Bd.safe_gain > 1e-6f) diag += Bd.safe_gain / fro;  // barrier.py:193-203
        p += Bd.dim;
      }
      for (int ci = 0; ci < X.nconstraints; ++ci) {
        // J dq = -gain e (pink/solve_ik.py:143-148)
        const DevTask& Kt = X.constraints[ci];
        const float* tgt = Kt.tgt_shared ? (P.shared + Kt.tgt_off) : (trow + Kt.tgt_off);
        float e[6];
        const int k = task_rows(M, P, Kt, q, tgt, e, Jw);
        for (int r = 0; r < k; ++r) {
          fe[meq] = -Kt.gain * e[r];
          for (int i = 0; i < nv; ++i) Eq[meq][i] = Jw[r][i];
          ++meq;
        }
      }
      if (out.G)
        for (int r = 0; r < MG; ++r) {
          out.hG[r] = r < p ? hg[r] : INFINITY;
          for (int i = 0; i < nv; ++i) out.G[r * nv + i] = r < p ? Gg[r][i] : 0.f;
        }
      if (out.E)
        for (int r = 0; r < ME; ++r) {
          out.f[r] = r < meq ? fe[r] : 0.f;
          for (int i = 0; i < nv; ++i) out.E[r * nv + i] = r < meq ? Eq[r][i] : 0.f;
        }
      finish(M, P, out, A, b, d, beta, pw2, pc, diag, lo, hi, K, status, skip, Gg, hg, p, Eq, fe, meq);
      return;
    }
    if (out.G)
      for (int r = 0; r < MG; ++r) {
        out.hG[r] = INFINITY;
        for (int i = 0; i < nv; ++i) out.G[r * nv + i] = 0.f;
      }
    if (out.E)
      for (int r = 0; r < ME; ++r) {
        out.f[r] = 0.f;
        for (int i = 0; i < nv; ++i) out.E[r * nv + i] = 0.f;
      }
    finish(M, P, out, A, b, d, beta, pw2, pc, diag, lo, hi, K, status, skip, nullptr, nullptr, 0, nullptr, nullptr, 0);
  }

  // Diagonal terms, exports and the QP solve.
  PK_HD void finish(const DevModel& M, const DevProblem& P, const GenericOut& out, const float (&A)[kGenericMaxRows][NVMAX],
                    const float (&b)[kGenericMaxRows], float (&d)[NVMAX], float (&beta)[NVMAX], const float (&pw2)[NVMAX],
                    const float (&pc)[NVMAX], float diag, const float (&lo)[NVMAX], const float (&hi)[NVMAX], int K,
                    int status, bool skip, const float (*Gg)[NVMAX], const float* hg, int p, const float (*Eq)[NVMAX],
                    const float* fe, int meq) {
    const int nv = M.nv;
    for (int i = 0; i < nv; ++i) {
      const float dd = sqrtf(pw2[i] + diag);
      d[i] = dd;
      beta[i] = dd > 0.f ? pc[i] / dd : 0.f;
    }
    if (out.lo)
      for (int i = 0; i < nv; ++i) { out.lo[i] = lo[i]; out.hi[i] = hi[i]; }
    if (out.H)
      for (int i = 0; i < nv; ++i)
        for (int j = 0; j < nv; ++j) {
          float s = (i == j) ? d[i] * d[i] : 0.f;
          for (int r = 0; r < K; ++r) s = fmaf(A[r][i], A[r][j], s);
          out.H[i * nv + j] = s;
        }
    if (out.c)
      for (int i = 0; i < nv; ++i) {
        float s = d[i] * beta[i];
        for (int r = 0; r < K; ++r) s = fmaf(A[r][i], b[r], s);
        out.c[i] = s;
      }

    if (out.v) {
      float x[NVMAX];
      if (skip || (status & PK_STATUS_NO_SOLUTION)) {
        for (int i = 0; i < nv; ++i) out.v[i] = 0.f;
      } else {
        if (p + meq == 0) {
          status |= BoxLSQ<kGenericMaxRows, NVMAX>::run(A, b, d, beta, lo, hi, K, nv, x);
        } else {
          using QP = DualQP<kGenericMaxRows, NVMAX, PK_MAX_INEQ_ROWS, PK_MAX_EQ_ROWS>;
          typename QP::Problem Q{A, b, d, beta, lo, hi, Gg, hg, Eq, fe, K, nv, p, meq};
          status |= QP::run(Q, x);
        }
        if (status & PK_STATUS_NO_SOLUTION)
          for (int i = 0; i < nv; ++i) x[i] = 0.f;
        for (int i = 0; i < nv; ++i) out.v[i] = x[i] * P.inv_dt;
      }
    }
    if (out.status) *out.status = status;
  }
};

// Solve to a tolerance (pk_converge_prepared), one instance on the general path; the loop of
// converge_chain (pk_chain.cuh) with Generic::step.  q [nq]: in q_0, out where the instance
// stopped (updated in place); v [nv]: scratch.
template <int NJMAX, int NVMAX>
PK_HD void converge_generic(Generic<NJMAX, NVMAX>& G, const DevModel& M, const DevProblem& P, float* q,
                            const float* trow, float* v, unsigned mask, float tol, int max_steps, float& err,
                            int& steps, int& status_out) {
  int32_t st = 0;
  GenericOut out{};
  out.v = v;
  out.status = &st;
  out.task_index = -1;
  int st_all = 0;
  int s = 0;
  for (;; ++s) {
    ConvergeTest ct{mask, tol, s == max_steps, 0.f, false, 0};
    G.template step<true>(M, P, q, trow, out, &ct);
    err = ct.err;
    if (ct.stop) break;
    st_all |= st;
    if (step_failed(st_all, P.safety_break)) {
      ++s;
      break;
    }
    integrate_configuration(M.nq, M.free_flyer, q, v, P.dt, q);
  }
  steps = s;
  status_out = st_all;
}

}  // namespace pk
