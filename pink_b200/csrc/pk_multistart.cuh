// Goal-set and multi-start solves to a tolerance (pk_converge_goalset_prepared, and
// pk_converge_multistart_prepared, its G = 1 case): instance b is solved toward G goals (targets
// rows) from S seeds at once, and its group of G S members stops at the first round where one of
// them has converged.  Member j = g S + s (goal-major) starts at seed row b S + s and reads
// targets row b G + g.  Device code only; the host build (hs_converge_goalset in hostsim.cpp)
// runs the same step bodies in two passes per round.
//
// The members of a group advance in lockstep rounds s = 0, 1, ...: every member that has not
// failed computes err(q_s) (the error of converge); the group stops when some member has
// err <= tol, s == max_steps, or every member has failed; otherwise every member that has not
// failed takes the converge step, and a member whose step fails keeps q_s and its error (the
// freeze rule of the rollouts).  The winner is the first member in seed_before's order at the
// stopping round: the earlier goal, then the earlier seed, on ties.
//
// Chains and the general path run one member per thread, the G S members of a group in adjacent
// lanes; joint trees run one instance per CTA, one member per warp.  The bodies whose stop test
// sits in the middle of the step (Generic::step, TreeStep::run) take a test type whose decide()
// makes the group's decision there.
//
// Their siblings under separate position and orientation tolerances are in pk_pose_tol.cu.
#pragma once

#include "pk_chain.cuh"
#include "pk_generic.cuh"
#include "pk_select.hpp"

namespace pk {

// The lanes of this thread's group of S members (S a power of two <= 32, blockDim a multiple of 32).
__device__ __forceinline__ unsigned seed_lanes(int S) {
  const unsigned m = S == 32 ? 0xffffffffu : ((1u << S) - 1u);
  return m << ((threadIdx.x & 31) & ~(S - 1));
}

// The winning member of the group: a butterfly over (error, member index) in seed_before's order.
__device__ __forceinline__ int group_winner(unsigned lanes, int S, float e, int j) {
  int w = j;
#pragma unroll 1
  for (int off = 1; off < S; off <<= 1) {
    const float e2 = __shfl_xor_sync(lanes, e, off);
    const int w2 = __shfl_xor_sync(lanes, w, off);
    if (seed_before(e2, w2, e, w)) {
      e = e2;
      w = w2;
    }
  }
  return w;
}

// Group stop test over the lanes of a group (Generic::step).  A failed member still calls the
// step (its lanes take part in the votes) and keeps the error it had where it failed.
struct LaneGroupTest {
  static constexpr bool kPose = false;
  unsigned mask;
  float tol;
  bool last;
  float err;  // in: the error a failed seed kept
  bool stop;  // out: this seed returns before its QP (the group stops, or it has failed)
  int status;
  unsigned lanes;  // the group's lanes
  bool failed;     // this seed failed an earlier step
  bool group;      // out: the group stops at this round
  __device__ __forceinline__ void decide(float e) {
    if (!failed) err = e;
    group = __any_sync(lanes, err <= tol) || last || __all_sync(lanes, failed);
    stop = group || failed;
  }
};

// Group stop test over the S warps (members) of a CTA (TreeStep::run): each warp publishes its error and
// failed flag in this round's slots, and after the barrier every warp makes the same decision
// from the same slots.  Every warp of the CTA calls the step in every round, so the barrier is
// reached by all of them; the slots alternate between two rounds, so a warp that runs ahead
// cannot overwrite slots another warp has yet to read.
struct CtaGroupTest {
  static constexpr bool kPose = false;
  unsigned mask;
  float tol;
  bool last;
  float err;
  bool stop;
  int status;
  float* slot_err;   // [S] this round's errors (shared memory)
  int* slot_failed;  // [S] this round's failed flags
  int S, seed;
  bool failed;
  bool group;
  __device__ __forceinline__ void decide(float e) {
    if (!failed) err = e;
    if ((threadIdx.x & 31) == 0) {
      slot_err[seed] = err;
      slot_failed[seed] = failed;
    }
    __syncthreads();
    bool hit = false, all_failed = true;
#pragma unroll 1
    for (int k = 0; k < S; ++k) {
      hit = hit || slot_err[k] <= tol;
      all_failed = all_failed && slot_failed[k];
    }
    group = hit || last || all_failed;
    stop = group || failed;
  }
};

// Chains: one member per thread, q in registers; thread i runs member j of instance b, i = b G S + j.
// emask: the task mask in chain slots (chain_task_mask).  q_seeds [B S][NJ] and targets
// [B G][target_stride] are only read; the winner of instance b writes row b of q_out [B][NJ] and
// of err, goal, seed, steps, status (any may be null but q_out).  GOALS = false is the launch
// with G = 1 (multi-start): its indexing reduces to row i and targets row b at compile time, so
// the multi-start loop keeps the registers and spills it had before goal sets.
template <int NJ, int NFT, bool GOALS>
__global__ void __launch_bounds__(128, 4)
    ik_chain_multistart_kernel(const __grid_constant__ ChainParams<NJ> P, const float* __restrict__ q_seeds, int S,
                               const float* __restrict__ targets, int G, unsigned emask, float tol, int max_steps,
                               float* __restrict__ q_out, float* __restrict__ err, int32_t* __restrict__ goal,
                               int32_t* __restrict__ seed, int32_t* __restrict__ steps, int32_t* __restrict__ status,
                               int64_t B) {
  const int GS = GOALS ? G * S : S;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * GS) return;  // whole groups: B G S is a multiple of G S
  const int64_t b = i / GS;
  const int j = (int)(i - b * GS);
  const unsigned lanes = seed_lanes(GS);
  const int64_t row = GOALS ? b * S + j % S : i;
  float qi[NJ];
#pragma unroll
  for (int k = 0; k < NJ; ++k) qi[k] = q_seeds[row * NJ + k];
  const float* trow = targets + (GOALS ? b * G + j / S : b) * (int64_t)P.target_stride;
  float e = 0.f;
  bool failed = false;
  int st_all = 0;
  int s = 0;
#pragma unroll 1
  for (;; ++s) {
    ChainStep<NJ, NFT> C;
    bool skip = false;
    int st = 0;
    if (!failed) st = C.template assemble<true>(P, qi, trow, skip, emask, &e);
    const bool hit = __any_sync(lanes, e <= tol);
    const bool all_failed = __all_sync(lanes, failed);
    if (hit || s == max_steps || all_failed) break;
    if (!failed && !converge_chain_advance(P, C, st, skip, qi, st_all, 0)) failed = true;
  }
  if (group_winner(lanes, GS, e, j) != j) return;
#pragma unroll
  for (int k = 0; k < NJ; ++k) q_out[b * NJ + k] = qi[k];
  if (err) err[b] = e;
  if (goal) goal[b] = GOALS ? j / S : 0;
  if (seed) seed[b] = GOALS ? j % S : j;
  if (steps) steps[b] = s;
  if (status) status[b] = st_all;
}

// General path: one member per thread, the lane grouping of the chain kernel; the member's q in
// local memory, Generic::step with LaneGroupTest.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_multistart_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                 const float* __restrict__ q_seeds, int S, const float* __restrict__ targets, int G,
                                 unsigned mask, float tol, int max_steps, float* __restrict__ q_out,
                                 float* __restrict__ err, int32_t* __restrict__ goal, int32_t* __restrict__ seed,
                                 int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t B) {
  const int GS = G * S;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * GS) return;
  const int64_t b = i / GS;
  const int j = (int)(i - b * GS);
  const unsigned lanes = seed_lanes(GS);
  const int nq = M.nq;
  float q[NVMAX + 1];  // nq <= nv + 1 (the free flyer's quaternion)
  for (int k = 0; k < nq; ++k) q[k] = q_seeds[(b * S + j % S) * nq + k];
  const float* trow = targets ? targets + (b * G + j / S) * (int64_t)P.target_stride : nullptr;
  float v[NVMAX];
  Generic<NJMAX, NVMAX> Gen;
  int32_t st = 0;
  GenericOut out{};
  out.v = v;
  out.status = &st;
  out.task_index = -1;
  float e = 0.f;
  bool failed = false;
  int st_all = 0;
  int s = 0;
  for (;; ++s) {
    LaneGroupTest ct{mask, tol, s == max_steps, e, false, 0, lanes, failed, false};
    Gen.template step<true>(M, P, q, trow, out, &ct);
    e = ct.err;
    if (ct.group) break;
    if (failed) continue;
    st_all |= st;
    if (step_failed(st_all, P.safety_break)) {
      failed = true;
      continue;
    }
    integrate_configuration(nq, M.free_flyer, q, v, P.dt, q);
  }
  if (group_winner(lanes, GS, e, j) != j) return;
  for (int k = 0; k < nq; ++k) q_out[b * nq + k] = q[k];
  if (err) err[b] = e;
  if (goal) goal[b] = j / S;
  if (seed) seed[b] = j % S;
  if (steps) steps[b] = s;
  if (status) status[b] = st_all;
}

#ifndef PK_NO_TREE_MULTISTART_KERNEL  // pk_pose_tol.cu: a translation unit of other kernels
// Joint trees: instance b = blockIdx.x, member j = warp, blockDim = 32 G S.  Warp j's workspace
// (MultistartTreeLayout) holds the plan's words, the step's v at o_v and the member's q at o_q;
// the group's slots follow the G S workspaces.  All warps run the same rounds (CtaGroupTest), and
// the winner is read from the slots of the stopping round.
__global__ void __launch_bounds__(32 * kTreeMaxSeeds)
    ik_tree_multistart_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                              const __grid_constant__ TreePlan L, int o_v, int o_q, const float* __restrict__ q_seeds,
                              int S, const float* __restrict__ targets, int G, unsigned mask, float tol,
                              int max_steps, float* __restrict__ q_out, float* __restrict__ err,
                              int32_t* __restrict__ goal, int32_t* __restrict__ seed, int32_t* __restrict__ steps,
                              int32_t* __restrict__ status, int64_t B) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int GS = G * S;
  const int64_t b = blockIdx.x;
  float* W = tree_smem + (size_t)warp * L.words;
  float* slots = tree_smem + (size_t)GS * L.words;  // round parity p: errors at 2 G S p, flags after them
  float* qw = W + o_q;
  float* vw = W + o_v;
  const int64_t row = b * S + warp % S;
  for (int k = lane; k < L.nq; k += 32) qw[k] = q_seeds[row * L.nq + k];
  __syncwarp();
  const float* tg = targets ? targets + (b * G + warp / S) * (int64_t)L.stride : nullptr;
  float e = 0.f;
  bool failed = false;
  int st_all = 0;
  int s = 0;
#pragma unroll 1
  for (;; ++s) {
    float* se = slots + (s & 1) * 2 * GS;
    CtaGroupTest ct{mask, tol, s == max_steps, e, false, 0, se, reinterpret_cast<int*>(se + GS), GS, warp, failed,
                    false};
    TreeStep::run<true>(M, P, L, qw, tg, W, vw, nullptr, &ct);
    __syncwarp();
    e = ct.err;
    if (ct.group) break;
    if (failed) continue;
    st_all |= ct.status;
    if (step_failed(st_all, P.safety_break)) {
      failed = true;
      continue;
    }
    if (lane == 0) integrate_configuration(L.nq, M.free_flyer, qw, vw, P.dt, qw);
    __syncwarp();
  }
  const float* fe = slots + (s & 1) * 2 * GS;
  int w = 0;
#pragma unroll 1
  for (int k = 1; k < GS; ++k)
    if (seed_before(fe[k], k, fe[w], w)) w = k;
  if (warp != w) return;
  for (int k = lane; k < L.nq; k += 32) q_out[b * L.nq + k] = qw[k];
  if (lane == 0) {
    if (err) err[b] = e;
    if (goal) goal[b] = w / S;
    if (seed) seed[b] = w % S;
    if (steps) steps[b] = s;
    if (status) status[b] = st_all;
  }
}
#endif

}  // namespace pk
