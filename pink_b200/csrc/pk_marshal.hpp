// Host-side marshalling shared by the CUDA library (pk_cabi.cu) and the CPU
// test harness (tests/hostsim): PkModelDesc -> flat fp32 tables, PkProblemDesc ->
// DevProblem / ChainParams, kernel eligibility.  Plain C++, no CUDA calls.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/pink_b200.h"
#include "pk_chain.cuh"
#include "pk_coop.cuh"
#include "pk_generic.cuh"
#include "pk_tree.cuh"
#include "pk_treedual.cuh"

namespace pk {

struct HostModel {
  int njoints = 0, free_flyer = 0, nq = 0, nv = 0, nframes = 0;
  std::vector<int> parent, jtype, frame_body, depth;
  int maxdepth = 0;
  std::vector<float> jX, axis, fX, mass, com;
  std::vector<uint64_t> anc;
  float total_mass = 0.f;
  bool serial_chain = false;

  // DevModel whose pointers alias the host vectors (CPU harness only).
  DevModel host_view() const {
    DevModel d{};
    d.njoints = njoints; d.free_flyer = free_flyer; d.nq = nq; d.nv = nv; d.nframes = nframes;
    d.parent = parent.data(); d.jtype = jtype.data(); d.jX = jX.data(); d.axis = axis.data();
    d.frame_body = frame_body.data(); d.fX = fX.data(); d.mass = mass.data(); d.com = com.data();
    d.anc = anc.data(); d.total_mass = total_mass;
    d.depth = depth.data(); d.maxdepth = maxdepth;
    return d;
  }
};

// Returns an empty string on success, else the error message.
inline std::string build_host_model(const PkModelDesc* d, HostModel* m) {
  if (!d || !m) return "null model description";
  if (d->njoints < 0 || d->njoints > PK_MAX_JOINTS) return "njoints out of range";
  if (d->nframes < 0 || d->nframes > PK_MAX_FRAMES) return "nframes out of range";
  const int nj = d->njoints;
  const int ff = d->free_flyer ? 1 : 0;
  if (d->nq != nj + 7 * ff || d->nv != nj + 6 * ff) return "nq/nv inconsistent with njoints/free_flyer";
  m->njoints = nj;
  m->free_flyer = ff;
  m->nq = d->nq;
  m->nv = d->nv;
  m->nframes = d->nframes;
  m->parent.assign(d->parent, d->parent + nj);
  m->jtype.assign(d->jtype, d->jtype + nj);
  m->jX.resize(12 * nj);
  m->axis.resize(3 * nj);
  for (int i = 0; i < 12 * nj; ++i) m->jX[i] = (float)d->joint_placement[i];
  for (int j = 0; j < nj; ++j) {
    const double* a = d->axis + 3 * j;
    const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    if (!(n > 0.0)) return "zero joint axis";
    for (int k = 0; k < 3; ++k) m->axis[3 * j + k] = (float)(a[k] / n);
    if (m->parent[j] >= j || m->parent[j] < -1) return "joints must be ordered parents-first";
    if (m->jtype[j] != PK_JOINT_REVOLUTE && m->jtype[j] != PK_JOINT_PRISMATIC) return "unknown joint type";
  }
  m->frame_body.assign(d->frame_body, d->frame_body + d->nframes);
  for (int f = 0; f < d->nframes; ++f)
    if (m->frame_body[f] < -2 || m->frame_body[f] >= nj) return "frame body out of range";
  m->fX.resize(12 * d->nframes);
  for (int i = 0; i < 12 * d->nframes; ++i) m->fX[i] = (float)d->frame_placement[i];
  m->mass.resize(nj + 1);
  m->com.resize(3 * (nj + 1));
  double total = 0.0;
  for (int b = 0; b <= nj; ++b) {
    m->mass[b] = d->mass ? (float)d->mass[b] : 0.f;
    total += d->mass ? d->mass[b] : 0.0;
    for (int k = 0; k < 3; ++k) m->com[3 * b + k] = d->com ? (float)d->com[3 * b + k] : 0.f;
  }
  m->total_mass = (float)total;
  m->anc.assign(nj + 2, 0ull);
  for (int j = 0; j < nj; ++j) {
    const uint64_t up = m->parent[j] >= 0 ? m->anc[m->parent[j] + 2] : 0ull;
    m->anc[j + 2] = up | (1ull << j);
  }
  m->depth.assign(nj > 0 ? nj : 1, 0);
  m->maxdepth = 0;
  for (int j = 0; j < nj; ++j) {
    m->depth[j] = m->parent[j] >= 0 ? m->depth[m->parent[j]] + 1 : 0;
    m->maxdepth = std::max(m->maxdepth, m->depth[j]);
  }
  m->serial_chain = !ff && nj >= 1;
  for (int j = 0; j < nj; ++j)
    if (m->parent[j] != j - 1) m->serial_chain = false;
  return "";
}

inline int target_size(const HostModel& m, const PkTaskDesc& t) {
  switch (t.type) {
    case PK_TASK_FRAME:
    case PK_TASK_RELATIVE_FRAME: return 12;
    case PK_TASK_POSTURE: return m.nq;
    case PK_TASK_JOINT_VELOCITY: return m.nv - (m.free_flyer ? 6 : 0);
    case PK_TASK_COM: return 3;
    case PK_TASK_LINEAR: return 0;
    default: return -1;
  }
}

// Host image of the optional problem parts; `X.extra` / `X.pairs` point into the
// vectors here until the C-ABI layer re-points them at device copies.
struct HostExtras {
  DevExtras X;
  std::vector<float> extra;
  std::vector<int> pairs;
  bool present = false;
  // no dense inequality rows and no equalities (only constant data of LINEAR tasks and / or an
  // AccelerationLimit, which is a box): the chain and tree kernels handle these problems.  A
  // shared (not per-instance) non-zero dq_prev stays on the general path.
  bool box_only() const {
    return present && X.nbarriers == 0 && X.nconstraints == 0 && !X.fb_enabled &&
           !(X.acc_enabled && X.acc_prev_shared && X.acc_prev_off >= 0);
  }
};

inline std::string fill_dev_task(const HostModel& m, const PkProblemDesc* p, const PkTaskDesc& s, DevTask& d,
                                 bool as_constraint) {
  const int ts = target_size(m, s);
  if (ts < 0) return "unknown task type";
  const int limit = s.target_shared ? PK_MAX_SHARED : p->target_stride;
  if (ts > 0 && (s.target_offset < 0 || s.target_offset + ts > limit)) return "task target does not fit its buffer";
  d.type = s.type;
  d.frame = s.frame;
  d.root = s.root;
  d.tgt_off = s.target_offset;
  d.tgt_shared = s.target_shared ? 1 : 0;
  d.body = d.root_body = -2;
  d.rows = 0;
  d.data_off = 0;
  if (s.type == PK_TASK_FRAME || s.type == PK_TASK_RELATIVE_FRAME) {
    if (s.frame < 0 || s.frame >= m.nframes) return "task frame index out of range";
    d.body = m.frame_body[s.frame];
  }
  if (s.type == PK_TASK_RELATIVE_FRAME) {
    if (s.root < 0 || s.root >= m.nframes) return "task root frame index out of range";
    d.root_body = m.frame_body[s.root];
  }
  if (s.type == PK_TASK_LINEAR) {
    if (s.rows < 1 || s.rows > 6) return "linear task: rows must be in 1..6";
    const int need = s.rows * m.nv + s.rows + m.nq;
    if (s.data_offset < 0 || !p->extra || s.data_offset + need > p->n_extra) return "linear task data does not fit `extra`";
    const int rv = m.free_flyer ? 6 : 0;
    for (int r = 0; r < s.rows; ++r)
      for (int i = 0; i < rv; ++i)
        if (p->extra[s.data_offset + r * m.nv + i] != 0.f) return "linear task: root columns of A must be zero";
    d.rows = s.rows;
    d.data_off = s.data_offset;
  }
  if (as_constraint && is_diag_task(s.type)) return "posture / joint-velocity tasks cannot be equality constraints";
  for (int k = 0; k < 6; ++k) {
    if (s.cost[k] < 0.f) return "negative task cost";
    d.cost[k] = s.cost[k];
  }
  d.gain = s.gain;
  d.lm = s.lm_damping;
  return "";
}

inline int task_row_count(const HostModel& m, const DevTask& d) {
  if (d.type == PK_TASK_COM) return 3;
  if (d.type == PK_TASK_LINEAR) return d.rows;
  return 6;
}

// Rows of e and J that the task-terms export writes for task `d`.
inline int task_terms_rows(const HostModel& m, const DevTask& d) {
  return is_diag_task(d.type) ? m.nv - (m.free_flyer ? 6 : 0) : task_row_count(m, d);
}

// Arguments of pk_converge_prepared; "" when valid.  Joint-velocity-type tasks cannot be in the
// mask: their error does not depend on q.
inline std::string check_converge_args(const DevProblem& P, uint32_t mask, float tol, int max_steps) {
  if (mask == 0u) return "empty task mask";
  if (P.ntasks < 32 && (mask >> P.ntasks) != 0u) return "task mask has bits at or above the number of tasks";
  for (int t = 0; t < P.ntasks; ++t)
    if (((mask >> t) & 1u) && P.tasks[t].type == PK_TASK_JOINT_VELOCITY)
      return "a joint-velocity task (JointVelocityTask, DampingTask, LowAccelerationTask) cannot be in the task mask";
  if (!(tol >= 0.f) || !std::isfinite(tol)) return "tol must be finite and >= 0";
  if (max_steps < 0) return "max_steps must be >= 0";
  return "";
}

// Seeds per target of pk_converge_multistart_prepared: a power of two that fits one warp, so that
// a group of seeds is S adjacent lanes.
constexpr int kMaxSeeds = 32;
inline bool valid_num_seeds(int S) { return S >= 1 && S <= kMaxSeeds && (S & (S - 1)) == 0; }

// Problem of the forward-kinematics and frame-Jacobian exports: no tasks, no limits.
inline DevProblem kinematics_problem() {
  DevProblem P;
  memset(&P, 0, sizeof(P));
  for (int i = 0; i < PK_MAX_NV; ++i) {
    P.chk_lo[i] = -INFINITY;
    P.chk_hi[i] = INFINITY;
  }
  return P;
}

inline std::string make_dev_problem(const HostModel& m, const PkProblemDesc* p, DevProblem* out,
                                    HostExtras* hx = nullptr) {
  if (!p) return "null problem";
  if (p->ntasks < 0 || p->ntasks > PK_MAX_TASKS) return "ntasks out of range";
  if (!(p->dt > 0.f)) return "dt must be positive";
  if (p->target_stride < 0) return "negative target_stride";
  DevProblem& P = *out;
  memset(&P, 0, sizeof(P));
  P.ntasks = p->ntasks;
  bool any_linear = false;
  for (int t = 0; t < p->ntasks; ++t) {
    const std::string e = fill_dev_task(m, p, p->tasks[t], P.tasks[t], false);
    if (!e.empty()) return e;
    any_linear = any_linear || p->tasks[t].type == PK_TASK_LINEAR;
  }
  P.dt = p->dt;
  P.inv_dt = 1.f / p->dt;
  P.damping = p->damping;
  P.cfg_gain = p->cfg_gain;
  P.target_stride = p->target_stride;
  P.safety_break = p->safety_break ? 1 : 0;
  for (int i = 0; i < PK_MAX_NV; ++i) {
    const bool in = i < m.nv;
    P.cfg_lo[i] = in ? p->cfg_lo[i] : -INFINITY;
    P.cfg_hi[i] = in ? p->cfg_hi[i] : INFINITY;
    P.vel[i] = in ? p->vel[i] : INFINITY;
    P.chk_lo[i] = in ? p->chk_lo[i] : -INFINITY;
    P.chk_hi[i] = in ? p->chk_hi[i] : INFINITY;
  }
  memcpy(P.shared, p->shared, sizeof(P.shared));
  P.ext = nullptr;

  // ---- optional parts (ABI 2) ----
  const bool present = any_linear || p->nbarriers > 0 || p->nconstraints > 0 || p->fb_enabled || p->acc_enabled;
  if (!present) {
    if (hx) hx->present = false;
    return "";
  }
  if (!hx) return "this entry point does not support barriers / constraints / opt-in limits";
  hx->present = true;
  DevExtras& X = hx->X;
  memset(&X, 0, sizeof(X));
  if (p->nbarriers < 0 || p->nbarriers > PK_MAX_BARRIERS) return "nbarriers out of range";
  if (p->nconstraints < 0 || p->nconstraints > PK_MAX_CONSTRAINTS) return "nconstraints out of range";
  if (p->n_extra < 0 || p->n_pairs < 0 || (p->n_extra > 0 && !p->extra) || (p->n_pairs > 0 && !p->pairs))
    return "extra / pairs buffers inconsistent";
  hx->extra.assign(p->extra, p->extra + p->n_extra);
  hx->pairs.assign(p->pairs, p->pairs + 2 * (size_t)p->n_pairs);
  int rows = 0;
  if (p->fb_enabled) {
    if (!m.free_flyer) return "FloatingBaseVelocityLimit requires a floating-base root joint";
    if (p->fb_frame < 0 || p->fb_frame >= m.nframes) return "floating-base frame index out of range";
    if (m.frame_body[p->fb_frame] != -1) return "floating-base frame is not attached to the root joint";
    X.fb_enabled = 1;
    X.fb_frame = p->fb_frame;
    X.fb_body = -1;
    int nfin = 0;
    for (int r = 0; r < 6; ++r) {
      if (!(p->fb_max[r] >= 0.f)) return "floating-base velocity bounds must be non-negative";
      X.fb_max[r] = p->fb_max[r];
      nfin += std::isfinite(p->fb_max[r]) ? 1 : 0;
    }
    if (nfin == 0) X.fb_enabled = 0;  // no finite bound: the limit contributes no row
    rows += 2 * nfin;
  }
  X.nbarriers = p->nbarriers;
  for (int b = 0; b < p->nbarriers; ++b) {
    const PkBarrierDesc& s = p->barriers[b];
    DevBarrier& d = X.barriers[b];
    d.type = s.type;
    d.frame = s.frame;
    d.frame2 = s.frame2;
    d.body = d.body2 = -2;
    d.d_min = s.d_min;
    d.safe_gain = s.safe_displacement_gain;
    d.gain_fn = s.gain_function;
    if (s.gain_function != PK_GAINFN_IDENTITY && s.gain_function != PK_GAINFN_SATURATING) return "unknown barrier gain function";
    for (int k = 0; k < 6; ++k) d.gain[k] = s.gain[k];
    if (s.type == PK_BARRIER_POSITION) {
      if (s.frame < 0 || s.frame >= m.nframes) return "barrier frame index out of range";
      if (s.nidx < 1 || s.nidx > 3) return "position barrier: 1..3 indices";
      if (!s.has_min && !s.has_max) return "position barrier needs p_min or p_max";
      d.body = m.frame_body[s.frame];
      d.nidx = s.nidx;
      d.has_min = s.has_min ? 1 : 0;
      d.has_max = s.has_max ? 1 : 0;
      for (int k = 0; k < s.nidx; ++k) {
        if (s.indices[k] < 0 || s.indices[k] > 2) return "position barrier index out of range";
        d.idx[k] = s.indices[k];
        d.p_min[k] = s.p_min[k];
        d.p_max[k] = s.p_max[k];
      }
      d.dim = s.nidx * (d.has_min + d.has_max);
    } else if (s.type == PK_BARRIER_BODY_SPHERICAL) {
      if (s.frame < 0 || s.frame >= m.nframes || s.frame2 < 0 || s.frame2 >= m.nframes) return "barrier frame index out of range";
      if (s.d_min < 0.f) return "negative minimum distance";
      d.body = m.frame_body[s.frame];
      d.body2 = m.frame_body[s.frame2];
      d.dim = 1;
    } else if (s.type == PK_BARRIER_SELF_COLLISION) {
      if (s.d_min < 0.f) return "negative minimum distance";
      if (s.npairs < 0 || s.npairs > PK_MAX_PAIRS) return "self-collision barrier: too many pairs";
      if (s.dim < 0 || s.dim > s.npairs) return "self-collision barrier: dim exceeds the number of collision pairs";
      if (s.pair_offset < 0 || s.pair_offset + s.npairs > p->n_pairs) return "self-collision pairs out of range";
      if (s.data_offset < 0 || s.data_offset + 2 * s.npairs > p->n_extra) return "self-collision radii out of range";
      for (int k = 0; k < 2 * s.npairs; ++k) {
        const int f = p->pairs[2 * s.pair_offset + k];
        if (f < 0 || f >= m.nframes) return "self-collision frame index out of range";
      }
      d.dim = s.dim;
      d.npairs = s.npairs;
      d.pair_off = s.pair_offset;
      d.data_off = s.data_offset;
    } else {
      return "unknown barrier type";
    }
    if (d.dim != s.dim) return "barrier dim does not match its definition";
    rows += d.dim;
  }
  if (rows > PK_MAX_INEQ_ROWS) return "too many dense inequality rows (PK_MAX_INEQ_ROWS)";
  X.n_ineq_rows = rows;
  X.nconstraints = p->nconstraints;
  int erows = 0;
  for (int c = 0; c < p->nconstraints; ++c) {
    const std::string e = fill_dev_task(m, p, p->constraints[c], X.constraints[c], true);
    if (!e.empty()) return e;
    erows += task_row_count(m, X.constraints[c]);
  }
  if (erows > PK_MAX_EQ_ROWS) return "too many equality rows (PK_MAX_EQ_ROWS)";
  X.n_eq_rows = erows;
  if (p->acc_enabled) {
    X.acc_enabled = 1;
    X.acc_prev_off = p->acc_prev_offset;
    X.acc_prev_shared = p->acc_prev_shared ? 1 : 0;
    if (p->acc_prev_offset >= 0) {
      const int limit = p->acc_prev_shared ? PK_MAX_SHARED : p->target_stride;
      if (p->acc_prev_offset + m.nv > limit) return "acceleration-limit dq_prev does not fit its buffer";
    }
    for (int i = 0; i < PK_MAX_NV; ++i) {
      const bool in = i < m.nv;
      X.acc_max[i] = in ? p->acc_max[i] : INFINITY;
      X.acc_qlo[i] = in ? p->acc_qlo[i] : -INFINITY;
      X.acc_qhi[i] = in ? p->acc_qhi[i] : INFINITY;
    }
  }
  X.extra = hx->extra.data();
  X.pairs = hx->pairs.data();
  return "";
}

// Does the register-resident chain kernel cover this (model, problem)?
inline bool chain_eligible(const HostModel& m, const DevProblem& P, bool has_extras = false) {
  if (has_extras) return false;
  if (!m.serial_chain || m.njoints > 7 || m.njoints < 2) return false;
  int nf = 0, np = 0;
  for (int t = 0; t < P.ntasks; ++t) {
    const DevTask& d = P.tasks[t];
    if (d.type == PK_TASK_FRAME) {
      if (d.body == -2) return false;
      ++nf;
    } else if (d.type == PK_TASK_POSTURE) {
      ++np;
    } else {
      return false;
    }
  }
  if (nf > kChainMaxFrameTasks || np > 1) return false;
  int shared_need = 0;
  for (int t = 0; t < P.ntasks; ++t)
    if (P.tasks[t].tgt_shared)
      shared_need = std::max(shared_need, P.tasks[t].tgt_off + (P.tasks[t].type == PK_TASK_FRAME ? 12 : m.nq));
  return shared_need <= 12 * kChainMaxFrameTasks + m.njoints;
}

// Workspace layout of the warp-cooperative tree kernel; `ok` false if the problem
// does not fit it (then the general path is used).
// Workspace layout of one instance (offsets in floats) from L.nj / nq / nv / K / p / npairs.
inline void tree_layout(TreePlan& L, int ntasks, int stride) {
  int off = 0;
  auto take = [&](int& cursor, int words) { const int at = cursor; cursor += (words + 3) / 4 * 4; return at; };
  const int K = L.K;
  const int Kp = K > 0 ? K : 1;
  L.lda = L.nv | 1;
  L.ldw = L.nv | 1;
  L.ldj = L.nv | 1;
  L.o_A = take(off, Kp * L.lda);
  L.o_b = take(off, K);
  L.o_d = take(off, L.nv);
  L.o_beta = take(off, L.nv);
  L.o_lo = take(off, L.nv);
  L.o_hi = take(off, L.nv);
  L.o_x = take(off, L.nv);
  L.o_y = take(off, L.nv);
  L.o_g = off;  // unused
  if (L.p > 0 || L.meq > 0) {
    // dense rows and dual-method state: persistent (not overlaid with the assembly scratch)
    L.o_G = take(off, (L.p > 0 ? L.p : 1) * L.lda);
    L.o_hg = take(off, L.p > 0 ? L.p : 1);
    L.o_gn = take(off, L.p > 0 ? L.p : 1);
    L.o_E = take(off, (L.meq > 0 ? L.meq : 1) * L.lda);
    L.o_fe = take(off, L.meq > 0 ? L.meq : 1);
    L.o_en = take(off, L.meq > 0 ? L.meq : 1);
    L.o_asg = take(off, L.nv + 1);
    L.o_J = take(off, L.nv * L.ldj);
    L.o_dv = take(off, L.nv);
    L.o_z = take(off, L.nv);
    L.o_r = take(off, L.nv + 1);
    L.o_u = take(off, L.nv + 1);
    L.o_act = take(off, L.nv + 1);
    L.o_xd = take(off, 2 * L.nv);
    L.o_wd = take(off, 2 * (L.nv + 1));
    L.o_gd = take(off, 2 * L.nv);
    L.o_rhod = take(off, 2 * Kp);
    L.o_ud = take(off, 2 * (L.nv + 1));
    L.o_dist = take(off, L.npairs > 0 ? L.npairs : 1);
  }
  // Then one region that is used twice - by the assembly phase (q, targets, joint
  // transforms, per-task blocks, body CoMs) and, once A / b / box are built, by the QR
  // scratch (compacted columns, R, right-hand sides).  Overlaying the two and packing R
  // roughly halves the footprint, which is what bounds the number of resident warps per SM.
  const int shared_base = off;
  int a = shared_base;  // assembly view
  L.o_q = take(a, L.nq);
  L.o_t = take(a, stride);
  L.o_tw = take(a, kTwStride * (L.nj > 0 ? L.nj : 1));
  L.o_root = take(a, 12);
  L.o_tf = take(a, kTreeTaskWords * (ntasks + L.nct > 0 ? ntasks + L.nct : 1));
  L.o_cw = take(a, 3 * (L.nj + 1));
  int b2 = shared_base;  // QP view
  L.o_aw = take(b2, Kp * L.ldw);
  L.o_ru = take(b2, L.nv * (L.nv - 1) / 2 + 1);
  L.o_rd = take(b2, L.nv);
  L.o_zt = take(b2, L.nv);
  L.o_zb = take(b2, K);
  L.o_rho = take(b2, K);
  L.o_ys = b2;  // unused
  L.o_idx = take(b2, L.nv);
  L.o_xa = take(b2, L.nv);
  L.words = a > b2 ? a : b2;
  if (L.p > 0 || L.meq > 0) {
    // third use of the region: once J = R^-1 is built the QR scratch is dead, and the
    // triangular factor of the active normals (written from the first entering constraint
    // on) takes its place
    int c3 = shared_base;
    L.o_RA = take(c3, L.nv * L.ldj);
    L.words = c3 > L.words ? c3 : L.words;
  }
}

// `X` (host image of the extras): barriers become the dense rows of the warp-cooperative
// dual method, like the rows of the floating-base limit and the equality rows of constraint tasks.
inline TreePlan make_tree_plan(const HostModel& m, const DevProblem& P, bool* ok, const DevExtras* X = nullptr) {
  TreePlan L;
  memset(&L, 0, sizeof(L));
  if (X) {
    if (X->fb_enabled)
      for (int r = 0; r < 6; ++r) L.p += std::isfinite(X->fb_max[r]) ? 2 : 0;
    L.meq = X->n_eq_rows;
    L.nct = X->nconstraints;
    for (int b = 0; b < X->nbarriers; ++b) {
      L.p += X->barriers[b].dim;
      if (X->barriers[b].type == PK_BARRIER_SELF_COLLISION) L.npairs = std::max(L.npairs, X->barriers[b].npairs);
    }
  }
  L.nj = m.njoints;
  L.nq = m.nq;
  L.nv = m.nv;
  L.rq = m.free_flyer ? 7 : 0;
  L.rv = m.free_flyer ? 6 : 0;
  L.ntasks = P.ntasks;
  L.stride = P.target_stride;
  L.maxdepth = m.maxdepth;
  int K = 0;
  for (int t = 0; t < PK_MAX_TASKS; ++t) L.row_base[t] = -1;
  for (int t = 0; t < P.ntasks; ++t) {
    const DevTask& d = P.tasks[t];
    if (is_diag_task(d.type)) continue;
    const int k = d.type == PK_TASK_COM ? 3 : (d.type == PK_TASK_LINEAR ? d.rows : 6);
    int rows = 0;
    for (int r = 0; r < k; ++r) rows += d.cost[r] != 0.f ? 1 : 0;
    if (rows) {
      L.row_base[t] = K;
      K += rows;
    }
  }
  L.K = K;
  L.lda = L.nv | 1;
  L.ldw = L.nv | 1;
  // Layout: persistent QP data first; then one region that is used twice - by the
  // assembly phase (q, targets, joint transforms, per-task blocks, body CoMs) and,
  // once A / b / box are built, by the QR scratch (compacted columns, R, right-hand
  // sides).  Overlaying the two and packing R roughly halves the footprint, which is
  // what bounds the number of resident warps per SM.
  tree_layout(L, P.ntasks, L.stride);
  const bool dense_ok = !X || (L.p <= 32 && L.meq <= 32 && L.p + L.meq <= 60 && P.ntasks + L.nct <= 32 &&
                               !(X->acc_enabled && X->acc_prev_shared && X->acc_prev_off >= 0));
  *ok = dense_ok && m.njoints >= 1 && m.njoints <= kTreeMaxJoints && m.nv <= 64 && P.ntasks <= 32 && K <= 64 &&
        (size_t)L.words * 4 <= 48 * 1024;
  return L;
}

template <int NJ>
void make_chain_params(const HostModel& m, const DevProblem& P, ChainParams<NJ>* out, const DevExtras* X = nullptr) {
  ChainParams<NJ>& C = *out;
  memset(&C, 0, sizeof(C));
  C.acc_prev_off = -1;
  if (X && X->acc_enabled) {  // host image of the extras (P.ext may be a device pointer)
    C.acc_enabled = 1;
    C.acc_prev_off = X->acc_prev_shared ? -1 : X->acc_prev_off;
    for (int j = 0; j < NJ; ++j) {
      C.acc_max[j] = X->acc_max[j];
      C.acc_qlo[j] = X->acc_qlo[j];
      C.acc_qhi[j] = X->acc_qhi[j];
    }
  }
  for (int j = 0; j < NJ; ++j) {
    memcpy(C.joint[j].X, &m.jX[12 * j], sizeof(float) * 12);
    C.joint[j].ax = m.axis[3 * j];
    C.joint[j].ay = m.axis[3 * j + 1];
    C.joint[j].az = m.axis[3 * j + 2];
    C.joint[j].type = m.jtype[j];
    {
      // fold the constant factors of X.R Rot(a, q) in double precision
      const float* X = &m.jX[12 * j];
      const double a[3] = {m.axis[3 * j], m.axis[3 * j + 1], m.axis[3 * j + 2]};
      const double Kx[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
      double R[9];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[3 * r + c] = X[4 * r + c];
      for (int r = 0; r < 3; ++r) {
        double xa = 0.0;
        for (int c = 0; c < 3; ++c) {
          double m1 = 0.0, m2 = 0.0;
          for (int k = 0; k < 3; ++k) {
            m1 += R[3 * r + k] * Kx[3 * k + c];
            m2 += R[3 * r + k] * (a[k] * a[c] - (k == c ? 1.0 : 0.0));
          }
          C.joint[j].M1[3 * r + c] = (float)m1;
          C.joint[j].M2[3 * r + c] = (float)m2;
          xa += R[3 * r + c] * a[c];
        }
        C.joint[j].Xa[r] = (float)xa;
      }
    }
    C.cfg_lo[j] = P.cfg_lo[j];
    C.cfg_hi[j] = P.cfg_hi[j];
    C.vel[j] = P.vel[j];
    C.chk_lo[j] = P.chk_lo[j];
    C.chk_hi[j] = P.chk_hi[j];
  }
  for (int t = 0; t < kChainMaxFrameTasks; ++t) {
    // inert defaults so that unused slots are well defined
    const float I[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    memcpy(C.ft[t].X, I, sizeof(I));
    C.ft[t].body = -1;
  }
  for (int t = 0; t < P.ntasks; ++t) {
    const DevTask& d = P.tasks[t];
    if (d.type == PK_TASK_FRAME) {
      ChainFrameTask& f = C.ft[C.n_frame_tasks++];
      f.body = d.body;
      memcpy(f.X, &m.fX[12 * d.frame], sizeof(float) * 12);
      memcpy(f.cost, d.cost, sizeof(float) * 6);
      f.gain = d.gain;
      f.lm = d.lm;
      f.tgt_off = d.tgt_off;
      f.tgt_shared = d.tgt_shared;
    } else {
      C.has_posture = 1;
      C.posture_w2 = d.cost[0] * d.cost[0];
      C.posture_gain = d.gain;
      C.posture_lm = d.lm;
      C.posture_off = d.tgt_off;
      C.posture_shared = d.tgt_shared;
    }
  }
  C.dt = P.dt;
  C.inv_dt = P.inv_dt;
  C.damping = P.damping;
  C.cfg_gain = P.cfg_gain;
  C.target_stride = P.target_stride;
  C.target_vec4 = (P.target_stride % 4) == 0;
  for (int t = 0; t < C.n_frame_tasks; ++t)
    if (!C.ft[t].tgt_shared && (C.ft[t].tgt_off % 4) != 0) C.target_vec4 = 0;
  C.safety_break = P.safety_break;
  memcpy(C.shared, P.shared, sizeof(C.shared));
}

// Parameter block of the sub-warp chain kernel (pk_coop.cuh): joint frames re-oriented so
// that every joint axis is the local z axis.  With A_j the rotation that takes e_z to the
// axis a_j, T~_j = oMi[j] A_j satisfies T~_j = T~_{j-1} X~_j M_z(q_j), X~_j = A_{j-1}^T X_j A_j
// (A_{-1} = I), and a frame fixed to joint b sits at A_b^T X_f in T~_b.  All folding in double.
template <int NJ, int L>
void make_coop_params(const HostModel& m, const DevProblem& P, CoopParams<((NJ + L - 1) / L) * L>* out,
                      const DevExtras* X = nullptr) {
  constexpr int NJP = ((NJ + L - 1) / L) * L;
  CoopParams<NJP>& C = *out;
  memset(&C, 0, sizeof(C));
  C.acc_prev_off = -1;
  if (X && X->acc_enabled) {
    C.acc_enabled = 1;
    C.acc_prev_off = X->acc_prev_shared ? -1 : X->acc_prev_off;
  }
  double Aprev[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  std::vector<double> Aall(9 * NJ);
  for (int j = 0; j < NJ; ++j) {
    const double a[3] = {m.axis[3 * j], m.axis[3 * j + 1], m.axis[3 * j + 2]};
    double A[9];
    const double c = a[2];  // e_z . a
    if (c > 1.0 - 1e-12) {
      const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
      memcpy(A, I, sizeof(A));
    } else if (c < -1.0 + 1e-12) {
      const double Rx[9] = {1, 0, 0, 0, -1, 0, 0, 0, -1};  // half turn about x
      memcpy(A, Rx, sizeof(A));
    } else {
      // Rodrigues about v = e_z x a = (-a_y, a_x, 0): A = I + [v]x + [v]x^2 / (1 + c)
      const double vx = -a[1], vy = a[0];
      const double k = 1.0 / (1.0 + c);
      const double Kx[9] = {0, 0, vy, 0, 0, -vx, -vy, vx, 0};
      for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 3; ++cc) {
          double k2 = 0.0;
          for (int t = 0; t < 3; ++t) k2 += Kx[3 * r + t] * Kx[3 * t + cc];
          A[3 * r + cc] = (r == cc ? 1.0 : 0.0) + Kx[3 * r + cc] + k * k2;
        }
    }
    memcpy(&Aall[9 * j], A, sizeof(A));
    const float* Xj = &m.jX[12 * j];
    CoopJoint& J = C.joint[j];
    // X~.R = Aprev^T X.R A, X~.p = Aprev^T X.p
    double XA[9];
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc) {
        double s = 0.0;
        for (int t = 0; t < 3; ++t) s += (double)Xj[4 * r + t] * A[3 * t + cc];
        XA[3 * r + cc] = s;
      }
    for (int r = 0; r < 3; ++r) {
      for (int cc = 0; cc < 3; ++cc) {
        double s = 0.0;
        for (int t = 0; t < 3; ++t) s += Aprev[3 * t + r] * XA[3 * t + cc];
        J.Xr[3 * r + cc] = (float)s;
      }
      double sp = 0.0;
      for (int t = 0; t < 3; ++t) sp += Aprev[3 * t + r] * (double)Xj[4 * t + 3];
      J.Xp[r] = (float)sp;
    }
    memcpy(Aprev, A, sizeof(A));
    J.prismatic = (m.jtype[j] == PK_JOINT_REVOLUTE) ? 0.f : 1.f;
    if (m.jtype[j] != PK_JOINT_REVOLUTE) C.any_prismatic = 1;
    J.cfg_lo = P.cfg_lo[j];
    J.cfg_hi = P.cfg_hi[j];
    J.vel = P.dt * P.vel[j];  // the same fp32 product the kernel used to form
    J.chk_lo = P.chk_lo[j];
    J.chk_hi = P.chk_hi[j];
    J.acc_max = (X && X->acc_enabled) ? X->acc_max[j] : INFINITY;
    J.acc_qlo = (X && X->acc_enabled) ? X->acc_qlo[j] : -INFINITY;
    J.acc_qhi = (X && X->acc_enabled) ? X->acc_qhi[j] : INFINITY;
    J.valid = 1.f;
  }
  for (int j = NJ; j < NJP; ++j) {  // padding: identity joints that never move
    CoopJoint& J = C.joint[j];
    J.Xr[0] = J.Xr[4] = J.Xr[8] = 1.f;
    J.cfg_lo = J.chk_lo = J.acc_qlo = -INFINITY;
    J.cfg_hi = J.chk_hi = J.acc_qhi = J.vel = J.acc_max = INFINITY;
    J.valid = 0.f;
  }
  for (int t = 0; t < kCoopMaxFrameTasks; ++t) {
    const float I[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    memcpy(C.ft[t].X, I, sizeof(I));
    C.ft[t].body = -1;
  }
  bool vec4 = (P.target_stride % 4) == 0;
  for (int t = 0; t < P.ntasks; ++t) {
    const DevTask& d = P.tasks[t];
    if (d.type == PK_TASK_FRAME) {
      CoopFrameTask& f = C.ft[C.n_frame_tasks++];
      f.body = d.body;
      const float* Xf = &m.fX[12 * d.frame];
      if (d.body >= 0) {
        const double* A = &Aall[9 * d.body];
        for (int r = 0; r < 3; ++r)
          for (int cc = 0; cc < 4; ++cc) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += A[3 * k + r] * (double)Xf[4 * k + cc];
            f.X[4 * r + cc] = (float)s;
          }
      } else {
        memcpy(f.X, Xf, sizeof(float) * 12);
      }
      memcpy(f.cost, d.cost, sizeof(float) * 6);
      f.gain = d.gain;
      f.lm = d.lm;
      f.tgt_off = d.tgt_off;
      f.tgt_shared = d.tgt_shared;
      if (!d.tgt_shared && (d.tgt_off % 4) != 0) vec4 = false;
    } else {
      C.has_posture = 1;
      C.posture_w2 = d.cost[0] * d.cost[0];
      C.posture_gain = d.gain;
      C.posture_lm = d.lm;
      C.posture_off = d.tgt_off;
      C.posture_shared = d.tgt_shared;
    }
  }
  C.frames_on_last = 1;
  for (int t = 0; t < C.n_frame_tasks; ++t)
    if (C.ft[t].body != NJ - 1) C.frames_on_last = 0;
  C.dt = P.dt;
  C.inv_dt = P.inv_dt;
  C.damping = P.damping;
  C.cfg_gain = P.cfg_gain;
  C.target_stride = P.target_stride;
  C.target_vec4 = vec4 ? 1 : 0;
  C.safety_break = P.safety_break;
  static_assert(sizeof(C.shared) >= sizeof(float) * (12 * kChainMaxFrameTasks + NJ), "shared target block too small");
  memcpy(C.shared, P.shared, sizeof(float) * (12 * kChainMaxFrameTasks + NJ));
}

}  // namespace pk
