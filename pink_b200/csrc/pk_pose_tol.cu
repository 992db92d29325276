// Kernels of the solves to separate position and orientation tolerances
// (pk_converge_pose_tol_prepared, pk_converge_goalset_pose_tol_prepared, DESIGN.md section 3.2h)
// and their launches (pk_pose_tol.hpp).  Each is the default kernel of pk_cabi.cu or
// pk_multistart.cuh with the pose-tolerance step bodies (ChainStep::assemble<true, true>,
// PoseTolTest).  A translation unit of its own, so that nvcc compiles it in parallel with
// pk_cabi.cu; the multi-start loops are written out rather than shared with the default
// kernels, whose machine code an inlined common body would change.
#define PK_NO_TREE_MULTISTART_KERNEL
#include "pk_pose_tol.hpp"

#include <mutex>

#include "../../include/pink_b200.h"
#include "pk_chain.cuh"
#include "pk_generic.cuh"
#include "pk_multistart.cuh"

namespace pk {

// Separate position and orientation tolerances (pk_converge_pose_tol_prepared): ik_chain_converge_kernel
// with the test of ChainStep::assemble<true, true>; amask: chain_axis_mask, rscale = tol /
// orientation_tol.
template <int NJ, int NFT>
__global__ void __launch_bounds__(128, 4)
    ik_chain_converge_pose_tol_kernel(const __grid_constant__ ChainParams<NJ> P, const float* q,
                                      const float* __restrict__ targets, unsigned emask, float tol, int max_steps,
                                      float* q_out, float* __restrict__ err, int32_t* __restrict__ steps,
                                      int32_t* __restrict__ status, int64_t B, unsigned amask, float rscale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  converge_chain_instance<NJ, NFT, true>(P, q, targets, emask, tol, max_steps, q_out, err, steps, status, i, amask,
                                         rscale);
}

// ik_generic_converge_kernel with the separate-tolerance test, rot_scale = tol / orientation_tol.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_converge_pose_tol_kernel(const DevModel M, const __grid_constant__ DevProblem P, const float* q,
                                        const float* __restrict__ targets, unsigned mask, float tol, int max_steps,
                                        float* q_out, float* __restrict__ err, int32_t* __restrict__ steps,
                                        int32_t* __restrict__ status, int64_t B, float rot_scale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  Generic<NJMAX, NVMAX> G;
  converge_generic_instance<NJMAX, NVMAX, true>(G, M, P, q, targets, mask, tol, max_steps, q_out, err, steps, status, i,
                                                rot_scale);
}

// ik_tree_converge_kernel with the separate-tolerance test, rot_scale = tol / orientation_tol.
__global__ void __launch_bounds__(32 * kTreeWarpsPerBlock)
    ik_tree_converge_pose_tol_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                     const __grid_constant__ TreePlan L, int o_v, const float* q,
                                     const float* __restrict__ targets, unsigned mask, float tol, int max_steps,
                                     float* q_out, float* __restrict__ err, int32_t* __restrict__ steps,
                                     int32_t* __restrict__ status, int64_t B, float rot_scale) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * kTreeWarpsPerBlock + warp;
  if (i >= B) return;
  TreeStep::converge_instance<true>(M, P, L, o_v, q, targets, mask, tol, max_steps, q_out,
                                    tree_smem + (size_t)warp * L.words, err, steps, status, i, rot_scale);
}

// ik_chain_multistart_kernel with ChainStep::assemble<true, true>: amask (chain_axis_mask) and
// rscale = tol / orientation_tol.
template <int NJ, int NFT, bool GOALS>
__global__ void __launch_bounds__(128, 4)
    ik_chain_multistart_pose_tol_kernel(const __grid_constant__ ChainParams<NJ> P, const float* __restrict__ q_seeds,
                                        int S, const float* __restrict__ targets, int G, unsigned emask, float tol,
                                        int max_steps, float* __restrict__ q_out, float* __restrict__ err,
                                        int32_t* __restrict__ goal, int32_t* __restrict__ seed,
                                        int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t B,
                                        unsigned amask, float rscale) {
  const int GS = GOALS ? G * S : S;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * GS) return;
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
    if (!failed) st = C.template assemble<true, true>(P, qi, trow, skip, emask, &e, amask, rscale);
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

// ik_generic_multistart_kernel with PoseTolTest<LaneGroupTest>, rot_scale = tol / orientation_tol.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_multistart_pose_tol_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                          const float* __restrict__ q_seeds, int S, const float* __restrict__ targets,
                                          int G, unsigned mask, float tol, int max_steps, float* __restrict__ q_out,
                                          float* __restrict__ err, int32_t* __restrict__ goal,
                                          int32_t* __restrict__ seed, int32_t* __restrict__ steps,
                                          int32_t* __restrict__ status, int64_t B, float rot_scale) {
  const int GS = G * S;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * GS) return;
  const int64_t b = i / GS;
  const int j = (int)(i - b * GS);
  const unsigned lanes = seed_lanes(GS);
  const int nq = M.nq;
  float q[NVMAX + 1];
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
    PoseTolTest<LaneGroupTest> ct{{mask, tol, s == max_steps, e, false, 0, lanes, failed, false}, rot_scale};
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

// ik_tree_multistart_kernel with PoseTolTest<CtaGroupTest>, rot_scale = tol / orientation_tol.
__global__ void __launch_bounds__(32 * kTreeMaxSeeds)
    ik_tree_multistart_pose_tol_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                       const __grid_constant__ TreePlan L, int o_v, int o_q,
                                       const float* __restrict__ q_seeds, int S, const float* __restrict__ targets,
                                       int G, unsigned mask, float tol, int max_steps, float* __restrict__ q_out,
                                       float* __restrict__ err, int32_t* __restrict__ goal, int32_t* __restrict__ seed,
                                       int32_t* __restrict__ steps, int32_t* __restrict__ status, int64_t B,
                                       float rot_scale) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int GS = G * S;
  const int64_t b = blockIdx.x;
  float* W = tree_smem + (size_t)warp * L.words;
  float* slots = tree_smem + (size_t)GS * L.words;
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
    PoseTolTest<CtaGroupTest> ct{
        {mask, tol, s == max_steps, e, false, 0, se, reinterpret_cast<int*>(se + GS), GS, warp, failed, false},
        rot_scale};
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


namespace {

template <class... Params, class... Args>
cudaError_t launch_rows(void (*kernel)(Params...), int64_t rows, int block, cudaStream_t stream, const Args&... args) {
  kernel<<<(unsigned)((rows + block - 1) / block), block, 0, stream>>>(args...);
  return cudaSuccess;
}

// Dynamic shared memory a tree kernel has been granted, per device ordinal (as in pk_cabi.cu).
struct SmemGrant {
  std::mutex mu;
  size_t bytes[64] = {};
};
SmemGrant g_converge_smem, g_multistart_smem;

template <class... Params, class... Args>
cudaError_t launch_tree(void (*kernel)(Params...), SmemGrant& grant, int device, int64_t grid, int block, size_t smem,
                        cudaStream_t stream, const Args&... args) {
  {
    std::lock_guard<std::mutex> lock(grant.mu);
    const int dev = (device >= 0 && device < 64) ? device : 0;
    if (smem > grant.bytes[dev] || device >= 64) {
      const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      grant.bytes[dev] = smem;
    }
  }
  kernel<<<(unsigned)grid, block, smem, stream>>>(args...);
  return cudaSuccess;
}

float rot_scale(const PoseTolLaunch& a) { return a.orientation_tol < INFINITY ? a.tol / a.orientation_tol : 0.f; }

}  // namespace

cudaError_t launch_converge_pose_tol(const PoseTolLaunch& a) {
  const Selection& sel = *a.sel;
  const DevProblem& P = *a.P;
  const float rs = rot_scale(a);
  if (sel.path == kPathChain) {
    const unsigned emask = chain_task_mask(P, a.mask, sel.nft);
    const unsigned amask = chain_axis_mask(P, a.mask, a.orientation_tol);
    return with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
      return launch_rows(ik_chain_converge_pose_tol_kernel<NJ, NFT>, a.B, 128, a.stream,
                         *static_cast<const ChainParams<NJ>*>(a.chain_params), a.q, a.targets, emask, a.tol,
                         a.max_steps, a.q_out, a.err, a.steps, a.status, a.B, amask, rs);
    });
  }
  if (sel.path == kPathTree) {
    const ConvergeTreeLayout T = converge_tree_layout(sel.plan);
    return launch_tree(ik_tree_converge_pose_tol_kernel, g_converge_smem, a.device,
                       (a.B + kTreeWarpsPerBlock - 1) / kTreeWarpsPerBlock, 32 * kTreeWarpsPerBlock,
                       (size_t)T.plan.words * 4 * kTreeWarpsPerBlock, a.stream, a.dev, P, T.plan, T.o_v, a.q, a.targets,
                       a.mask, a.tol, a.max_steps, a.q_out, a.err, a.steps, a.status, a.B, rs);
  }
  return with_generic(sel.generic_class, [&](auto nj, auto nv) {
    return launch_rows(ik_generic_converge_pose_tol_kernel<decltype(nj)::value, decltype(nv)::value>, a.B, 64,
                       a.stream, a.dev, P, a.q, a.targets, a.mask, a.tol, a.max_steps, a.q_out, a.err, a.steps,
                       a.status, a.B, rs);
  });
}

cudaError_t launch_goalset_pose_tol(const PoseTolLaunch& a) {
  const Selection& sel = *a.sel;
  const DevProblem& P = *a.P;
  const float rs = rot_scale(a);
  const int S = a.S, G = a.G;
  if (sel.path == kPathTree) {
    const MultistartTreeLayout T = multistart_tree_layout(sel.plan);
    return launch_tree(ik_tree_multistart_pose_tol_kernel, g_multistart_smem, a.device, a.B, 32 * G * S,
                       T.smem_bytes(G * S), a.stream, a.dev, P, T.plan, T.o_v, T.o_q, a.q, S, a.targets, G, a.mask,
                       a.tol, a.max_steps, a.q_out, a.err, a.goal, a.seed, a.steps, a.status, a.B, rs);
  }
  if (sel.path == kPathChain) {
    const unsigned emask = chain_task_mask(P, a.mask, sel.nft);
    const unsigned amask = chain_axis_mask(P, a.mask, a.orientation_tol);
    return with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
      auto launch = [&](auto kernel) {
        return launch_rows(kernel, a.B * G * S, 128, a.stream, *static_cast<const ChainParams<NJ>*>(a.chain_params),
                           a.q, S, a.targets, G, emask, a.tol, a.max_steps, a.q_out, a.err, a.goal, a.seed, a.steps,
                           a.status, a.B, amask, rs);
      };
      return G == 1 ? launch(ik_chain_multistart_pose_tol_kernel<NJ, NFT, false>)
                    : launch(ik_chain_multistart_pose_tol_kernel<NJ, NFT, true>);
    });
  }
  return with_generic(sel.generic_class, [&](auto nj, auto nv) {
    return launch_rows(ik_generic_multistart_pose_tol_kernel<decltype(nj)::value, decltype(nv)::value>, a.B * G * S,
                       64, a.stream, a.dev, P, a.q, S, a.targets, G, a.mask, a.tol, a.max_steps, a.q_out, a.err,
                       a.goal, a.seed, a.steps, a.status, a.B, rs);
  });
}

}  // namespace pk
