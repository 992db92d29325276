// Device wrapper of pk_coop.cuh: L lanes per instance, 128 threads per CTA.
// n_steps > 1: closed-loop rollout, q <- q (+) v dt after every step with q kept in
// registers (pink/configuration.py:285-293 after pink/solve_ik.py:274); an instance that
// fails a step (no solution / outside limits with safety_break) is frozen.  T: per-step targets
// rows and records of a trajectory call (pk_rollout_trajectory_prepared); each lane stores the
// joints it owns, and a frozen instance fills its remaining steps (q unchanged, v = 0).
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
  constexpr int NC = Step::NC;
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
  GVar<typename Step::Lane, L> S;
  // records of step s: the lane's joints of q and v, the status from lane 0 of the group
  auto record = [&](int s, int st_all, bool frozen) {
    const int64_t r = (int64_t)s * B + inst;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int j = G.h * NC + k;
      if (j < NJ) {
        if (T.q) T.q[r * NJ + j] = S.v.q[k];
        if (T.v) T.v[r * NJ + j] = frozen ? 0.f : S.v.x[k];
      }
    }
    if (T.status && G.h == 0) T.status[r] = st_all;
  };
  const float* qrow = q + inst * NJ;
  if constexpr (L == 1 && NJ % 2 == 0) {
#pragma unroll
    for (int k = 0; k < NJ / 2; ++k) {
      const float2 t = __ldg(reinterpret_cast<const float2*>(qrow) + k);
      S.v.q[2 * k] = t.x;
      S.v.q[2 * k + 1] = t.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int j = G.h * NC + k;
      S.v.q[k] = (j < NJ) ? __ldg(qrow + (j < NJ ? j : 0)) : 0.f;
    }
  }
  const float* trow = targets + inst * (int64_t)P.target_stride;
  int st_all = 0;
#pragma unroll
  for (int k = 0; k < NC; ++k) S.v.x[k] = 0.f;
#pragma unroll 1
  for (int step_no = 0; step_no < n_steps; ++step_no) {
    const bool frozen =
        (st_all & (PK_STATUS_NO_SOLUTION | PK_STATUS_NOT_POSDEF)) || ((st_all & PK_STATUS_OUT_OF_LIMITS) && P.safety_break);
    if (frozen) {
#pragma unroll 1
      for (int s = step_no; s < n_steps; ++s) record(s, st_all, true);
      break;
    }
    int st;
    ik_step_coop<NJ, NFT, L>(G, P, jc, trow, S, st);
    st_all |= st & 0xff;
    if (n_steps > 1 || q_out) {
#pragma unroll
      for (int k = 0; k < NC; ++k) S.v.q[k] = fmaf(S.v.x[k], P.dt, S.v.q[k]);  // 1-dof joints: q (+) v dt = q + v dt
    }
    trow += T.target_step;
    record(step_no, st_all, false);
  }
  float* vrow = v + inst * NJ;
  if constexpr (L == 1 && NJ % 2 == 0) {
#pragma unroll
    for (int k = 0; k < NJ / 2; ++k) reinterpret_cast<float2*>(vrow)[k] = make_float2(S.v.x[2 * k], S.v.x[2 * k + 1]);
  } else {
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int j = G.h * NC + k;
      if (j < NJ) vrow[j] = S.v.x[k];
    }
  }
  if (q_out) {
    float* orow = q_out + inst * NJ;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int j = G.h * NC + k;
      if (j < NJ) orow[j] = S.v.q[k];
    }
  }
  if (status && G.h == 0) status[inst] = st_all;
}

}  // namespace pk
