/*
 * pink_b200 -- C ABI of the batched differential-IK engine (sm_90a).
 *
 * The reference (stephane-caron/pink) is pure Python and has
 * no FFI: its boundary for this path is the Python API
 *   pink.solve_ik(configuration, tasks, dt, solver, damping, limits, ...)
 *     -> pink/solve_ik.py:206-275
 *   pink.build_ik(...) -> qpsolvers.Problem(P, q, G, h, A, b)
 *     -> pink/solve_ik.py:152-203
 *   pink.Configuration.update / get_frame_jacobian / get_transform_frame_to_world
 *     -> pink/configuration.py:131-164, 203-254
 *   Task.compute_error / compute_jacobian -> pink/tasks/task.py:66-113
 * Each entry point below names the reference interface it evaluates for a
 * whole batch of independent instances.  The Python classes in pink_b200/
 * (same names and arguments as the reference's) marshal into these calls
 * through ctypes; see INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it
 *    asynchronously, no host synchronisation, no allocation on the hot path;
 *  - the caller owns every buffer; device entry points take DEVICE pointers,
 *    *_host entry points take HOST pointers (pinned for best throughput) and
 *    perform the H2D / D2H copies themselves on `stream`;
 *  - return value: 0 on success, non-zero for API misuse / CUDA errors
 *    (message via pk_last_error()).  Per-instance numerical outcomes never
 *    fail the call; they are reported in status[].
 *  - SE(3) values are 12 floats, row-major [R | p] (3 rows of 4);
 *    twists and Jacobian rows are [linear(3); angular(3)];
 *    free-flyer q = [x y z qx qy qz qw | joints], v = [v(3) w(3) | rates].
 */
#ifndef PINK_B200_H
#define PINK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PK_ABI_VERSION 3

#define PK_MAX_JOINTS 58  /* 1-dof joints (free-flyer excluded)            */
#define PK_MAX_NV 64      /* PK_MAX_JOINTS + 6 (active sets are 64-bit masks) */
#define PK_MAX_FRAMES 256
#define PK_MAX_TASKS 12
#define PK_MAX_SHARED 192 /* floats of targets shared by all instances     */
#define PK_MAX_INEQ_ROWS 24 /* dense inequality rows per instance (barriers, floating-base velocity limit) */
#define PK_MAX_EQ_ROWS 12   /* equality rows per instance (solve_ik(..., constraints=...)) */

/* per-instance status bits written by the solve entry points */
#define PK_STATUS_OK 0
#define PK_STATUS_NO_SOLUTION 1   /* pink.exceptions.NoSolutionFound (solve_ik.py:271-273): infeasible rows, or a
                                     NaN / Inf in q or a target (bit 1 or 4 is set then); v = 0 for the instance */
#define PK_STATUS_OUT_OF_LIMITS 2 /* NotWithinConfigurationLimits (configuration.py:186-194) */
#define PK_STATUS_NOT_POSDEF 4    /* Hessian not positive definite in fp32 */
#define PK_STATUS_ITER_LIMIT 8    /* active-set iteration cap hit; v is feasible, maybe sub-optimal */

/* joint types */
#define PK_JOINT_REVOLUTE 0
#define PK_JOINT_PRISMATIC 1

/* task types (pink/tasks/{frame,relative_frame,posture,com}_task.py) */
#define PK_TASK_FRAME 0
#define PK_TASK_RELATIVE_FRAME 1
#define PK_TASK_POSTURE 2
#define PK_TASK_COM 3
#define PK_TASK_JOINT_VELOCITY 4 /* pink/tasks/joint_velocity_task.py, damping_task.py: e = target (nv - root_nv floats), J = I[root_nv:] */
#define PK_TASK_LINEAR 5         /* pink/tasks/linear_holonomic_task.py:148-192 (JointCouplingTask: joint_coupling_task.py:82-100):
                                    e = A (q (-) q_0) - b, J = A, with A zero on the root columns; `rows` <= 6;
                                    extra[data_offset ...] = A[rows][nv], b[rows], q_0[nq]                      */

/* barriers (pink/barriers/*.py) */
#define PK_MAX_BARRIERS 8
#define PK_MAX_CONSTRAINTS 4
#define PK_MAX_PAIRS 256
#define PK_BARRIER_POSITION 0       /* position_barrier.py:95-153        */
#define PK_BARRIER_BODY_SPHERICAL 1 /* body_spherical_barrier.py:73-143  */
#define PK_BARRIER_SELF_COLLISION 2 /* self_collision_barrier.py:85-224, sphere-sphere pairs */
#define PK_GAINFN_IDENTITY 0        /* barrier.py:75-77                  */
#define PK_GAINFN_SATURATING 1      /* h / (1 + |h|), body_spherical_barrier.py:65 */

/* bodies: -2 universe, -1 root body (floating base if free_flyer, else the
 * universe), j >= 0 the body moved by 1-dof joint j                        */

typedef struct PkModelDesc {
  int32_t njoints;      /* number of 1-dof joints, parents-first order   */
  int32_t free_flyer;   /* 1: root is a free-flyer ("root_joint")        */
  int32_t nq;           /* njoints (+7)                                   */
  int32_t nv;           /* njoints (+6)                                   */
  const int32_t* parent;        /* [njoints] parent body (-1 or joint index) */
  const int32_t* jtype;         /* [njoints] PK_JOINT_*                   */
  const double* joint_placement;/* [njoints][12] placement in parent body */
  const double* axis;           /* [njoints][3] unit axis in joint frame  */
  int32_t nframes;
  const int32_t* frame_body;    /* [nframes] body the frame is fixed to   */
  const double* frame_placement;/* [nframes][12]                          */
  const double* mass;           /* [njoints+1] by body+1 (root body first)*/
  const double* com;            /* [njoints+1][3] CoM in body frame       */
} PkModelDesc;

typedef struct PkTaskDesc {
  int32_t type;          /* PK_TASK_*                                     */
  int32_t frame;         /* frame index (FRAME / RELATIVE_FRAME)          */
  int32_t root;          /* root frame index (RELATIVE_FRAME)             */
  int32_t target_offset; /* float offset of the target: inside one row of
                            `targets` (per instance) or inside
                            PkProblemDesc.shared (target_shared = 1).
                            frame: 12 floats [R|p]; posture: nq; com: 3;
                            joint velocity: nv - root_nv (dq_ref)       */
  int32_t target_shared;
  float cost[6];         /* frame: [pos(3), ori(3)]; com: [3]; posture / joint velocity: cost[0] */
  float gain;            /* Task.gain   (pink/tasks/task.py:146)          */
  float lm_damping;      /* Task.lm_damping (pink/tasks/task.py:160)      */
  int32_t rows;          /* LINEAR: number of rows p (cost[0..p))         */
  int32_t data_offset;   /* LINEAR: float offset into PkProblemDesc.extra */
} PkTaskDesc;

/* One barrier h(q) >= 0 (pink/barriers/barrier.py): rows  -J_h / dt dq <= gain_i alpha(h_i)
 * (barrier.py:246-252) and, if safe_displacement_gain > 1e-6, the objective term
 * safe_displacement_gain / |J_h|_F^2 * I (barrier.py:193-203, zero safe displacement). */
typedef struct PkBarrierDesc {
  int32_t type;            /* PK_BARRIER_*                                 */
  int32_t frame;           /* POSITION: monitored frame; BODY_SPHERICAL: first frame */
  int32_t frame2;          /* BODY_SPHERICAL: second frame                 */
  int32_t dim;             /* rows: POSITION nidx * (has_min + has_max); BODY_SPHERICAL 1;
                              SELF_COLLISION the n closest pairs           */
  int32_t nidx;            /* POSITION: number of monitored coordinates    */
  int32_t indices[3];      /* POSITION: 0..2 = x..z                         */
  int32_t has_min, has_max;
  float p_min[3], p_max[3];/* POSITION: bounds, by position in `indices`   */
  float gain[6];           /* POSITION: per row; otherwise gain[0]         */
  float d_min;             /* BODY_SPHERICAL / SELF_COLLISION              */
  float safe_displacement_gain;
  int32_t gain_function;   /* PK_GAINFN_*                                  */
  int32_t npairs;          /* SELF_COLLISION: collision pairs ...          */
  int32_t pair_offset;     /* ... pairs[2 (pair_offset + k)] = the frames of the two sphere centres */
  int32_t data_offset;     /* ... extra[data_offset + 2 k] = their radii   */
} PkBarrierDesc;

typedef struct PkProblemDesc {
  int32_t ntasks;
  PkTaskDesc tasks[PK_MAX_TASKS];
  float dt;              /* solve_ik(..., dt)                             */
  float damping;         /* solve_ik(..., damping)                        */
  int32_t target_stride; /* floats per instance in `targets`              */
  int32_t safety_break;  /* 1: out-of-limit instances are not solved and
                            get PK_STATUS_OUT_OF_LIMITS; 0: flagged but solved */
  /* Box inequality rows, per tangent index i (q index = i + nq - nv):
   *   ConfigurationLimit (pink/limits/configuration_limit.py:108-121):
   *      +dq_i <= cfg_gain (cfg_hi[i] - q_i),  -dq_i <= -cfg_gain (cfg_lo[i] - q_i)
   *   VelocityLimit (pink/limits/velocity_limit.py:115-121):
   *      +-dq_i <= dt * vel[i]
   * +-INFINITY disables a row.                                            */
  float cfg_gain;
  float cfg_lo[PK_MAX_NV];
  float cfg_hi[PK_MAX_NV];
  float vel[PK_MAX_NV];
  /* Configuration.check_limits (pink/configuration.py:181-201), tolerance
   * already applied by the caller: flagged if q_i < chk_lo[i] or > chk_hi[i] */
  float chk_lo[PK_MAX_NV];
  float chk_hi[PK_MAX_NV];
  float shared[PK_MAX_SHARED];
  /* ---- ABI 2: barriers, equality constraints, opt-in limits (all optional, zero = absent) ---- */
  int32_t nbarriers;
  PkBarrierDesc barriers[PK_MAX_BARRIERS];
  /* solve_ik(..., constraints=[tasks]) (pink/solve_ik.py:125-149): J dq = -gain e;
   * FRAME, RELATIVE_FRAME, COM and LINEAR tasks                             */
  int32_t nconstraints;
  PkTaskDesc constraints[PK_MAX_CONSTRAINTS];
  /* FloatingBaseVelocityLimit (pink/limits/floating_base_velocity_limit.py:118-148):
   * +-J_frame[:, root] dq <= dt fb_max, rows with infinite fb_max dropped   */
  int32_t fb_enabled;
  int32_t fb_frame;
  float fb_max[6];        /* [linear(3); angular(3)]                        */
  /* AccelerationLimit (pink/limits/acceleration_limit.py:119-200), per tangent index:
   *   +dq_i <= min(a dt^2 + dq_prev_i, dt sqrt(2 a (acc_qhi_i - q_i)))
   *   -dq_i <= min(a dt^2 - dq_prev_i, dt sqrt(2 a (q_i - acc_qlo_i)))
   * acc_max = INFINITY: no row; acc_qlo/acc_qhi = -+INFINITY: no braking term.
   * dq_prev = v_prev * dt: nv floats at acc_prev_offset of the targets row
   * (of `shared` if acc_prev_shared); acc_prev_offset < 0: zeros            */
  int32_t acc_enabled;
  int32_t acc_prev_offset;
  int32_t acc_prev_shared;
  float acc_max[PK_MAX_NV];
  float acc_qlo[PK_MAX_NV];
  float acc_qhi[PK_MAX_NV];
  /* constant data referenced by LINEAR tasks and SELF_COLLISION barriers (host
   * pointers, copied at pk_problem_create / at every pk_solve_ik_batched call) */
  const float* extra;
  int32_t n_extra;
  const int32_t* pairs;   /* [n_pairs][2] frame indices                     */
  int32_t n_pairs;
} PkProblemDesc;

typedef struct PkModel PkModel; /* opaque; immutable after creation */

int pk_abi_version(void);
/* sizeof of the descriptor structs as compiled (0 PkModelDesc, 1 PkTaskDesc,
 * 2 PkBarrierDesc, 3 PkProblemDesc): lets a binding verify its own layout.   */
int pk_struct_size(int which);
const char* pk_last_error(void); /* thread-local */

/* Build device-resident constant tables of a model on CUDA device `device`. */
int pk_model_create(const PkModelDesc* desc, int device, PkModel** out);
void pk_model_destroy(PkModel* model);

/* pink.solve_ik for B instances (pink/solve_ik.py:206-275).
 *   q[B][nq], targets[B][target_stride] -> v[B][nv], status[B] (may be NULL). */
int pk_solve_ik_batched(const PkModel* model, const PkProblemDesc* prob,
                        const float* q, const float* targets, float* v,
                        int32_t* status, int64_t B, void* stream);

/* Prepared form for hot loops: validate and marshal the problem once, then every
 * call costs one kernel launch.  A PkProblem is immutable and tied to the model
 * it was created for.                                                      */
typedef struct PkProblem PkProblem;
int pk_problem_create(const PkModel* model, const PkProblemDesc* prob, PkProblem** out);
void pk_problem_destroy(PkProblem* problem);
int pk_solve_ik_prepared(const PkModel* model, const PkProblem* problem,
                         const float* q, const float* targets, float* v,
                         int32_t* status, int64_t B, void* stream);
int pk_solve_ik_prepared_host(PkModel* model, const PkProblem* problem,
                              const float* q_host, const float* targets_host,
                              float* v_host, int32_t* status_host, int64_t B,
                              void* stream);

/* Closed loop of n_steps iterations of  v = solve_ik(q); q <- q (+) v dt
 * (the loop of examples/arm_ur5.py:65-86 with fixed targets): q_out[B][nq] final
 * configurations, v[B][nv] last velocities, status = OR over steps; an instance
 * that fails a step keeps its configuration.  Serial chains run all steps in one
 * launch with q resident in registers, joint trees (warp kernel) in one launch with
 * the instance's rows re-read by the warp that wrote them; models beyond the warp
 * kernel alternate solve / integrate launches (status then reports the last step).   */
int pk_rollout_prepared(const PkModel* model, const PkProblem* problem,
                        const float* q, const float* targets, int32_t n_steps,
                        float* q_out, float* v, int32_t* status, int64_t B,
                        void* stream);

/* Trajectory rollout: n_steps iterations of  v = solve_ik(q, targets_s); q <- q (+) v dt,
 * where the targets row of instance i at step s is
 *   targets + s * target_step + i * target_stride
 * (target_step in floats, >= 0; 0 = the same row every step, as pk_rollout_prepared).
 * q_out[B][nq] final q (may alias q), v[B][nv] velocity of the last step that ran,
 * status[B] = OR over the steps that ran (may be NULL).
 * Optional records (NULL = not written), step-major:
 *   q_traj[n_steps][B][nq]  q after step s,
 *   v_traj[n_steps][B][nv]  velocity of step s,
 *   status_traj[n_steps][B] OR of the statuses of steps 0..s.
 * Every path freezes an instance that fails a step (NO_SOLUTION / NOT_POSDEF, or
 * OUT_OF_LIMITS with safety_break): from then on q stays, v_traj rows are 0 and
 * status_traj repeats.  One launch on every path (chains, joint trees and the general
 * path); no host synchronisation and no allocation, so the call can be captured in a
 * CUDA graph.  The dq_prev words of AccelerationLimit / LowAccelerationTask are read
 * from each step's targets row as given: the rollout does not feed its own previous
 * velocity back into them.                                                            */
int pk_rollout_trajectory_prepared(const PkModel* model, const PkProblem* problem,
                                   const float* q, const float* targets, int64_t target_step,
                                   int32_t n_steps, float* q_out, float* v, int32_t* status,
                                   float* q_traj, float* v_traj, int32_t* status_traj,
                                   int64_t B, void* stream);

/* Solve to a tolerance (the loop of the reference's examples/inverse_kinematics_ur10.py:
 * while err > stop_thres), per instance, with fixed targets (one row per instance, as
 * pk_rollout_prepared).  err(q) = max over the tasks t of task_mask (bit t = problem task t)
 * of |e_t(q)|_2, the unweighted, gain-free error of pk_task_terms_batched.  For s = 0, 1, ...:
 * stop at q_s if err(q_s) <= tol or s == max_steps; else solve step s (the step
 * pk_rollout_prepared takes), stop at q_s if it fails (NO_SOLUTION / NOT_POSDEF, or
 * OUT_OF_LIMITS with safety_break), else q_{s+1} = q_s (+) v dt.
 *   q_out[B][nq]  where the instance stopped (required; may alias q),
 *   err[B]        err(q_out); an instance has converged iff err <= tol (a NaN never has),
 *   steps[B]      solves that ran,
 *   status[B]     OR of their statuses (0 if none ran); err, steps, status may be NULL.
 * Joint-velocity-type tasks cannot be in the mask (their error does not depend on q);
 * barriers and constraints act in every step but do not enter err.  In fp32 a pose
 * resolves to about 1e-7, so a tol below about 1e-6 may run to max_steps.  One launch on
 * every path (serial chains always take the thread-per-instance kernel, whatever
 * PK_CHAIN_LANES says); no host synchronisation and no allocation, so the call can be
 * captured in a CUDA graph.                                                              */
int pk_converge_prepared(const PkModel* model, const PkProblem* problem,
                         const float* q, const float* targets, uint32_t task_mask, float tol,
                         int32_t max_steps, float* q_out, float* err, int32_t* steps,
                         int32_t* status, int64_t B, void* stream);

/* Multi-start solve to a tolerance: target b is solved from the num_seeds = S seeds
 * q_seeds[b][j] (row b*S + j of q_seeds[B*S][nq], only read) with the one targets row b
 * (targets[B][target_stride]).  The S seeds advance in lockstep rounds s = 0, 1, ...: each seed
 * that has not failed computes err(q_s) of pk_converge_prepared; the group stops when some seed
 * has err <= tol, s == max_steps, or every seed has failed; otherwise every seed that has not
 * failed takes the pk_converge_prepared step, and a seed whose step fails keeps q_s and its
 * error.  The winner is the seed with the smallest error at the stopping round (a NaN counts as
 * +inf, ties go to the lowest index).  Per target:
 *   q_out[B][nq]  the winner's configuration (required; must not overlap q_seeds),
 *   err[B]        its error, seed[B] its index, steps[B] the rounds the group ran,
 *   status[B]     the OR of the winner's step statuses (0 if none ran); err, seed, steps,
 *                 status may be NULL.
 * S is 1, 2, 4, 8, 16 or 32; on the tree kernel S <= 8 and the S warp workspaces must fit one
 * CTA's shared memory.  With S = 1 the outputs equal pk_converge_prepared's.  One launch, no
 * host synchronisation and no allocation, so the call can be captured in a CUDA graph.      */
int pk_converge_multistart_prepared(const PkModel* model, const PkProblem* problem,
                                    const float* q_seeds, int32_t num_seeds, const float* targets,
                                    uint32_t task_mask, float tol, int32_t max_steps, float* q_out,
                                    float* err, int32_t* seed, int32_t* steps, int32_t* status,
                                    int64_t B, void* stream);

/* Goal-set solve to a tolerance: instance b is solved toward any of num_goals = G targets rows
 * (goals) from num_seeds = S seeds, in one launch.  q_seeds[B*S][nq] as in
 * pk_converge_multistart_prepared (every goal uses the same seeds); targets[B*G][target_stride]
 * holds G complete rows per instance, goal g of instance b at row b*G + g.  The G*S members of
 * an instance, j = g*S + s (goal-major, starting at q_seeds[b*S + s] toward goal g), form one
 * group of pk_converge_multistart_prepared's rule: lockstep rounds, the group stops when one
 * member has err <= tol, at max_steps, or when every member has failed, and the winner is the
 * member with the smallest error at the stopping round (NaN counts as +inf, ties go to the
 * lowest j: the earlier goal, then the earlier seed).  Per instance:
 *   q_out[B][nq]  the winner's configuration (required; must not overlap q_seeds),
 *   err[B]        its error, goal[B] = j / S, seed[B] = j % S, steps[B] the rounds the group
 *                 ran, status[B] the OR of the winner's step statuses; all but q_out may be NULL.
 * G and S are powers of two with G*S in {1, 2, 4, 8, 16, 32}; on the tree kernel G*S <= 8 and
 * the G*S warp workspaces must fit one CTA's shared memory.  A goal count that is not a power
 * of two is padded by repeating a goal: a duplicate never changes the winner.  G = 1 is
 * pk_converge_multistart_prepared.  One launch, no host synchronisation and no allocation, so
 * the call can be captured in a CUDA graph.                                                 */
int pk_converge_goalset_prepared(const PkModel* model, const PkProblem* problem, const float* q_seeds,
                                 int32_t num_seeds, const float* targets, int32_t num_goals,
                                 uint32_t task_mask, float tol, int32_t max_steps, float* q_out,
                                 float* err, int32_t* goal, int32_t* seed, int32_t* steps,
                                 int32_t* status, int64_t B, void* stream);

/* Solve to separate position and orientation tolerances: pk_converge_prepared with another
 * err(q), the largest over the tasks of task_mask of
 *   frame, relative frame   max(|e[0:3]|, (tol / orientation_tol) |e[3:6]|),
 *   CoM, linear (holonomic, joint coupling)   |e|,
 *   posture                 |e|,
 * where e is the task's unweighted, gain-free error (log6's twist for a pose) restricted to the
 * rows whose cost is > 0: an instance stops when every weighed translation part is <= tol, every
 * weighed rotation part (the rotation angle when all three axes are weighed) is <= orientation_tol
 * and every other task is <= tol.  orientation_tol = +inf leaves the rotation rows out of the
 * test.  tol must be finite and > 0, orientation_tol > 0, and every task of task_mask must keep a
 * row to test.  The loop, the step, the outputs and the launch are those of pk_converge_prepared. */
int pk_converge_pose_tol_prepared(const PkModel* model, const PkProblem* problem,
                                  const float* q, const float* targets, uint32_t task_mask, float tol,
                                  float orientation_tol, int32_t max_steps, float* q_out, float* err,
                                  int32_t* steps, int32_t* status, int64_t B, void* stream);

/* Goal-set (and, with num_goals = 1, multi-start) solve to separate position and orientation
 * tolerances: pk_converge_goalset_prepared with the err(q) of pk_converge_pose_tol_prepared; the
 * rounds, the winner's order and the outputs are unchanged.                                  */
int pk_converge_goalset_pose_tol_prepared(const PkModel* model, const PkProblem* problem,
                                          const float* q_seeds, int32_t num_seeds, const float* targets,
                                          int32_t num_goals, uint32_t task_mask, float tol,
                                          float orientation_tol, int32_t max_steps, float* q_out,
                                          float* err, int32_t* goal, int32_t* seed, int32_t* steps,
                                          int32_t* status, int64_t B, void* stream);

/* Gradient of a loss with respect to the targets at solutions of pk_converge_prepared /
 * pk_converge_multistart_prepared: grad_targets[b] = (d q_star / d T)^T grad_q[b] at q_star[b]
 * (targets[B][target_stride] the rows the solutions were converged to, grad_q[B][nq] the loss
 * gradient in q coordinates).  The converge loop stops where the step's linear term vanishes on
 * the coordinates it leaves off the configuration limits; the gradient is that condition's
 * implicit derivative with the Gauss-Newton matrix N = sum_t alpha_t J_t^T W_t^2 J_t (DESIGN.md
 * section 3.2f).  Coordinates held on a configuration limit do not move; a frame target's 12
 * floats [R | p] receive [1/2 R [g_w]x | R g_v] from the gradient (g_v, g_w) of the twist d in
 * T <- T exp(d); shared targets get nothing (their row entries stay 0).
 *   status[B]  0, or PK_STATUS_NOT_POSDEF: N on the free coordinates is not positive definite
 *              in fp32 (the row is 0); may be NULL.
 * The caller zeroes the rows of instances that did not converge.  Problems with barriers,
 * equality constraints or an AccelerationLimit are rejected.  One launch of the general
 * path's kernel on every model; no host synchronisation and no allocation, so the call can
 * be captured in a CUDA graph.                                                             */
int pk_converge_vjp_prepared(const PkModel* model, const PkProblem* problem, const float* q_star,
                             const float* targets, const float* grad_q, float* grad_targets,
                             int32_t* status, int64_t B, void* stream);

/* ---- multi-GPU: all-gather of v through NVLink peer memory (SURVEY.md section 8e) ----
 * One process per GPU; instances are independent, so the only exchange is the one
 * BASELINE north_star names: collecting v.  Instead of a collective after the kernel, the
 * solve kernel itself stores every velocity row into the gather buffer of every peer
 * (posted NVLink writes from the epilogue, overlapped with the remaining instances); a
 * one-warp kernel behind it publishes "gather k complete" in every peer's flag block and
 * waits for the peers' - on a side stream if the next solve should not wait for it.
 *   pk_peer_alloc   zero-filled device buffer that other processes can map + its IPC handle
 *   pk_peer_open    map a peer's buffer from its handle (enables peer access)
 *   pk_solve_ik_prepared_gather   pk_solve_ik_prepared + store v[i] to row (row_offset + i)
 *                   of each of the n_peers buffers (peer_v[k] = base of [rows][nv] floats;
 *                   the caller's own buffer is one of them; v may be NULL for serial chains).
 *                   peer_flags (NULL: no flow control, the caller synchronises by other means)
 *                   = the flag blocks of all ranks, PK_PEER_FLAG_WORDS uint32 each, allocated
 *                   with pk_peer_alloc: in its first instructions the kernel checks that every
 *                   peer has released the gather that used the same buffer slot n_buffers
 *                   calls ago (normally long done: n local words per CTA).
 *   pk_peer_sync    one-warp kernel, queued behind the gather kernel (same stream, or another
 *                   stream that waits for it - then the next solve overlaps it):
 *                   post: publish "my gather k is complete" in every rank's flag block;
 *                   wait: hold the stream until the oldest gather this rank has not waited
 *                   for yet has been published by every rank (its rows are then visible);
 *                   release: tell the peers that this rank is done with that buffer slot.
 * Every rank issues the same sequence of gathers, one post and one wait + release per gather.
 * All counters live in device memory: every launch can be replayed from a CUDA graph.      */
#define PK_MAX_PEERS 16
#define PK_IPC_HANDLE_BYTES 64
#define PK_PEER_FLAG_WORDS 48
int pk_peer_alloc(int device, int64_t bytes, void** ptr, unsigned char* handle /*[64]*/);
int pk_peer_open(int device, const unsigned char* handle /*[64]*/, void** ptr);
int pk_peer_close(int device, void* ptr);
int pk_peer_free(int device, void* ptr);
int pk_solve_ik_prepared_gather(const PkModel* model, const PkProblem* problem,
                                const float* q, const float* targets, float* v,
                                int32_t* status, int64_t B, void* const* peer_v,
                                int32_t n_peers, int64_t row_offset,
                                void* const* peer_flags, int32_t rank, int32_t n_buffers,
                                void* stream);
int pk_peer_sync(int device, void* const* peer_flags, int32_t n_peers, int32_t rank,
                 int32_t post, int32_t wait, int32_t release, void* stream);

/* Schedule of the host-buffer entry points for this model: 0 = uploads and downloads staged
 * by the copy engines, one direction at a time (default); 2 = staged uploads, results
 * written by the kernels straight into the caller's pinned host buffers; 1 = zero-copy both
 * ways; -1 = the PK_HOST_MODE environment default.  Results are identical; which is faster
 * depends on the platform's PCIe root complex, so the caller measures.                  */
int pk_model_set_host_schedule(PkModel* model, int mode);

/* Same through HOST buffers: H2D of q/targets, solve, D2H of v/status, all on
 * `stream`, chunked so copies overlap the kernels.  Returns after enqueueing;
 * the caller synchronises the stream before reading v.                     */
int pk_solve_ik_batched_host(PkModel* model, const PkProblemDesc* prob,
                             const float* q_host, const float* targets_host,
                             float* v_host, int32_t* status_host, int64_t B,
                             void* stream);

/* pink.build_ik for B instances (pink/solve_ik.py:152-203):
 *   H[B][nv][nv], c[B][nv], h[B][4][nv] with rows
 *   [cfg upper, cfg lower, vel upper, vel lower] (the right-hand sides of
 *   G = [P;-P;P;-P], +INFINITY where the row does not exist).             */
int pk_build_ik_batched(const PkModel* model, const PkProblemDesc* prob,
                        const float* q, const float* targets, float* H,
                        float* c, float* h, int64_t B, void* stream);

/* The dense rows of the same QP that pk_build_ik_batched leaves out:
 *   G[B][PK_MAX_INEQ_ROWS][nv], hG[B][PK_MAX_INEQ_ROWS]  (floating-base limit rows, then
 *   barrier rows in list order; unused rows are zero with hG = +INFINITY),
 *   E[B][PK_MAX_EQ_ROWS][nv], f[B][PK_MAX_EQ_ROWS]       (equality constraints; unused: 0),
 *   lo[B][nv], hi[B][nv]  the box  lo <= dq <= hi  of all +-e_i rows (configuration,
 *   velocity and acceleration limits).  Any output may be NULL.              */
int pk_constraint_rows_batched(const PkModel* model, const PkProblemDesc* prob,
                               const float* q, const float* targets, float* G,
                               float* hG, float* E, float* f, float* lo,
                               float* hi, int64_t B, void* stream);

/* Task.compute_error / compute_jacobian of task `task_index`
 * (pink/tasks/task.py:66-113): e[B][k], J[B][k][nv]; k = 6 frame tasks,
 * 3 com, nv - root_nv posture.                                             */
int pk_task_terms_batched(const PkModel* model, const PkProblemDesc* prob,
                          int32_t task_index, const float* q,
                          const float* targets, float* e, float* J, int64_t B,
                          void* stream);

/* Configuration.update (pink/configuration.py:163-164): frame placements
 * oMf[B][nframes][12]; `com` [B][3] optional (pin.centerOfMass).           */
int pk_forward_kinematics_batched(const PkModel* model, const float* q,
                                  float* oMf, float* com, int64_t B,
                                  void* stream);

/* Forward kinematics of selected frames, differentiable (DESIGN.md section 3.2i).
 * frames: HOST array of num_frames frame indices (0 <= f < nframes, repeats allowed), copied into
 * the launch; oMf[B][num_frames][12] (row-major [R | p]); com[B][3] or NULL.  0 <= num_frames <=
 * PK_MAX_FRAMES.  Bitwise the matching rows of pk_forward_kinematics_batched.  A CoM request on a
 * model of total mass 0 is rejected.  No allocation: the call can be captured in a CUDA graph.  */
int pk_frame_placements_batched(const PkModel* model, const int32_t* frames, int32_t num_frames,
                                const float* q, float* oMf, float* com, int64_t B, void* stream);

/* grad_q[B][nq] = (d (oMf, com) / d q)^T (grad_oMf, grad_com), fully written; grad_oMf
 * [B][num_frames][12] or NULL, grad_com [B][3] or NULL (NULL: that term is zero).  On a
 * free-flyer root the quaternion's gradient is that of the normalised map (no radial part).
 * Frames as pk_frame_placements_batched; one launch, no allocation.                           */
int pk_frame_placements_vjp_batched(const PkModel* model, const int32_t* frames, int32_t num_frames,
                                    const float* q, const float* grad_oMf, const float* grad_com,
                                    float* grad_q, int64_t B, void* stream);

/* Configuration.get_frame_jacobian (pink/configuration.py:203-236), LOCAL:
 * J[B][6][nv].                                                             */
int pk_frame_jacobian_batched(const PkModel* model, int32_t frame,
                              const float* q, float* J, int64_t B,
                              void* stream);

/* Configuration.integrate (pink/configuration.py:273-283):
 * q_out = q (+) v * dt, quaternion renormalised.                           */
int pk_integrate_batched(const PkModel* model, const float* q, const float* v,
                         float dt, float* q_out, int64_t B, void* stream);

/* Number of kernels this library has launched in the calling process
 * (instrumentation for bench.py's gpu_launches).                           */
int64_t pk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* PINK_B200_H */
