// Device wrapper of pk_coop.cuh: L lanes per instance, 128 threads per CTA.
// n_steps > 1: closed-loop rollout (rollout_coop), q <- q (+) v dt after every step with q kept
// in registers (pink/configuration.py:285-293 after pink/solve_ik.py:274); an instance that
// fails a step (no solution / outside limits with safety_break) is frozen.  T: per-step targets
// rows and records of a trajectory call (pk_rollout_trajectory_prepared).
#pragma once

#include "pk_coop.cuh"

namespace pk {

constexpr int kCoopThreads = 128;

// resident CTAs per SM the register allocation aims at: one wave of B = 65536 instances
// on the 132 SMs of an H100 needs 65536 L / (132 * 128) = 3.9 L CTAs per SM (L = 2 at 7 CTAs
// per SM runs in a little more than one wave)
template <int L>
struct CoopOccupancy {
  static constexpr int min_blocks = (L == 1) ? 4 : (L == 2) ? 7 : 8;
};

template <int NJ, int NFT, int L>
__global__ void __launch_bounds__(kCoopThreads, CoopOccupancy<L>::min_blocks)
    ik_coop_kernel(const __grid_constant__ CoopParams<CoopStep<NJ, NFT, L>::NJP> P, const float* __restrict__ q,
                   const float* __restrict__ targets, float* __restrict__ v, int32_t* __restrict__ status,
                   int64_t B, int n_steps, float* __restrict__ q_out, const __grid_constant__ Trajectory T) {
  using Step = CoopStep<NJ, NFT, L>;
  // lane-varying joint index (L > 1): the per-joint constants come from shared memory
  __shared__ CoopJoint sj[L > 1 ? Step::NJP : 1];
  if constexpr (L > 1) {
    constexpr int words = (int)(sizeof(CoopJoint) / 4) * Step::NJP;
    const float* src = reinterpret_cast<const float*>(P.joint);
    float* dst = reinterpret_cast<float*>(sj);
    for (int w = threadIdx.x; w < words; w += kCoopThreads) dst[w] = src[w];
    __syncthreads();
  }
  const Group<L> G;
  const int64_t inst = ((int64_t)blockIdx.x * kCoopThreads + threadIdx.x) / L;
  if (inst >= B) return;
  auto jc = [&](int j) -> const CoopJoint& {
    if constexpr (L > 1) return sj[j];
    else return P.joint[j];
  };
  coop_instance<NJ, NFT, L>(G, P, jc, q, targets, v, status, B, n_steps, q_out, T, inst);
}

}  // namespace pk
