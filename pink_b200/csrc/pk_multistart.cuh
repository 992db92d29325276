// Multi-start solve to a tolerance (pk_converge_multistart_prepared): each target is solved
// from S seeds at once, and the group of S seeds stops at the first round where one of them
// has converged.  Device code only; the host build (tests/hostsim/multistart.cpp) runs the
// same step bodies in two passes per round.
//
// The S seeds of a target advance in lockstep rounds s = 0, 1, ...: every seed that has not
// failed computes err(q_s) (the error of converge); the group stops when some seed has
// err <= tol, s == max_steps, or every seed has failed; otherwise every seed that has not
// failed takes the converge step, and a seed whose step fails keeps q_s and its error (the
// freeze rule of the rollouts).  The winner is the first seed in seed_before's order at the
// stopping round.
//
// Chains and the general path run one seed per thread, the S seeds of a target in S adjacent
// lanes; joint trees run one target per CTA, one seed per warp.  The bodies whose stop test sits
// in the middle of the step (Generic::step, TreeStep::run) take a test type whose decide() makes
// the group's decision there.
#pragma once

#include "pk_chain.cuh"
#include "pk_generic.cuh"
#include "pk_select.hpp"

namespace pk {

// The lanes of this thread's group of S seeds (S a power of two <= 32, blockDim a multiple of 32).
__device__ __forceinline__ unsigned seed_lanes(int S) {
  const unsigned m = S == 32 ? 0xffffffffu : ((1u << S) - 1u);
  return m << ((threadIdx.x & 31) & ~(S - 1));
}

// The winning seed of the group: a butterfly over (error, seed index) in seed_before's order.
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

// Group stop test over the S lanes of a group (Generic::step).  A failed seed still calls the
// step (its lanes take part in the votes) and keeps the error it had where it failed.
struct LaneGroupTest {
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

// Group stop test over the S warps of a CTA (TreeStep::run): each warp publishes its error and
// failed flag in this round's slots, and after the barrier every warp makes the same decision
// from the same slots.  Every warp of the CTA calls the step in every round, so the barrier is
// reached by all of them; the slots alternate between two rounds, so a warp that runs ahead
// cannot overwrite slots another warp has yet to read.
struct CtaGroupTest {
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

// Chains: one seed per thread, q in registers; thread i runs seed row i = b S + j.  emask: the
// task mask in chain slots (chain_task_mask).  q_seeds [B S][NJ] is only read; the winner of
// target b writes row b of q_out [B][NJ] and of err, seed, steps, status (any may be null but
// q_out).
template <int NJ, int NFT>
__global__ void __launch_bounds__(128, 4)
    ik_chain_multistart_kernel(const __grid_constant__ ChainParams<NJ> P, const float* __restrict__ q_seeds, int S,
                               const float* __restrict__ targets, unsigned emask, float tol, int max_steps,
                               float* __restrict__ q_out, float* __restrict__ err, int32_t* __restrict__ seed,
                               int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * S) return;  // whole groups: B S is a multiple of S
  const int64_t b = i / S;
  const int j = (int)(i - b * S);
  const unsigned lanes = seed_lanes(S);
  float qi[NJ];
#pragma unroll
  for (int k = 0; k < NJ; ++k) qi[k] = q_seeds[i * NJ + k];
  const float* trow = targets + b * (int64_t)P.target_stride;
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
  if (group_winner(lanes, S, e, j) != j) return;
#pragma unroll
  for (int k = 0; k < NJ; ++k) q_out[b * NJ + k] = qi[k];
  if (err) err[b] = e;
  if (seed) seed[b] = j;
  if (steps) steps[b] = s;
  if (status) status[b] = st_all;
}

// General path: one seed per thread, the lane grouping of the chain kernel; the seed's q in local
// memory, Generic::step with LaneGroupTest.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_multistart_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                 const float* __restrict__ q_seeds, int S, const float* __restrict__ targets,
                                 unsigned mask, float tol, int max_steps, float* __restrict__ q_out,
                                 float* __restrict__ err, int32_t* __restrict__ seed, int32_t* __restrict__ steps,
                                 int32_t* __restrict__ status, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * S) return;
  const int64_t b = i / S;
  const int j = (int)(i - b * S);
  const unsigned lanes = seed_lanes(S);
  const int nq = M.nq;
  float q[NVMAX + 1];  // nq <= nv + 1 (the free flyer's quaternion)
  for (int k = 0; k < nq; ++k) q[k] = q_seeds[i * nq + k];
  const float* trow = targets ? targets + b * (int64_t)P.target_stride : nullptr;
  float v[NVMAX];
  Generic<NJMAX, NVMAX> G;
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
    G.template step<true>(M, P, q, trow, out, &ct);
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
  if (group_winner(lanes, S, e, j) != j) return;
  for (int k = 0; k < nq; ++k) q_out[b * nq + k] = q[k];
  if (err) err[b] = e;
  if (seed) seed[b] = j;
  if (steps) steps[b] = s;
  if (status) status[b] = st_all;
}

// Joint trees: target b = blockIdx.x, seed j = warp, blockDim = 32 S.  Warp j's workspace
// (MultistartTreeLayout) holds the plan's words, the step's v at o_v and the seed's q at o_q; the
// group's slots follow the S workspaces.  All warps run the same rounds (CtaGroupTest), and the
// winner is read from the slots of the stopping round.
__global__ void __launch_bounds__(32 * kTreeMaxSeeds)
    ik_tree_multistart_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                              const __grid_constant__ TreePlan L, int o_v, int o_q, const float* __restrict__ q_seeds,
                              int S, const float* __restrict__ targets, unsigned mask, float tol, int max_steps,
                              float* __restrict__ q_out, float* __restrict__ err, int32_t* __restrict__ seed,
                              int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t B) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t b = blockIdx.x;
  float* W = tree_smem + (size_t)warp * L.words;
  float* slots = tree_smem + (size_t)S * L.words;  // round parity p: errors at 2 S p, flags after them
  float* qw = W + o_q;
  float* vw = W + o_v;
  const int64_t row = b * S + warp;
  for (int k = lane; k < L.nq; k += 32) qw[k] = q_seeds[row * L.nq + k];
  __syncwarp();
  const float* tg = targets ? targets + b * (int64_t)L.stride : nullptr;
  float e = 0.f;
  bool failed = false;
  int st_all = 0;
  int s = 0;
#pragma unroll 1
  for (;; ++s) {
    float* se = slots + (s & 1) * 2 * S;
    CtaGroupTest ct{mask, tol, s == max_steps, e, false, 0, se, reinterpret_cast<int*>(se + S), S, warp, failed, false};
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
  const float* fe = slots + (s & 1) * 2 * S;
  int w = 0;
#pragma unroll 1
  for (int k = 1; k < S; ++k)
    if (seed_before(fe[k], k, fe[w], w)) w = k;
  if (warp != w) return;
  for (int k = lane; k < L.nq; k += 32) q_out[b * L.nq + k] = qw[k];
  if (lane == 0) {
    if (err) err[b] = e;
    if (seed) seed[b] = w;
    if (steps) steps[b] = s;
    if (status) status[b] = st_all;
  }
}

}  // namespace pk
