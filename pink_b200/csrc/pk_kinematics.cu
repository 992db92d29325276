// Kernels of the differentiable forward kinematics (pk_frame_placements_batched,
// pk_frame_placements_vjp_batched, DESIGN.md section 3.2i) and their launches (pk_kinematics.hpp):
// one thread per instance at the size classes of the general path, running the bodies of
// pk_kinematics.cuh.
#include "pk_kinematics.hpp"

#include "pk_select.hpp"

namespace pk {

template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    frame_placements_kernel(const DevModel M, const __grid_constant__ FrameList L, const float* __restrict__ q,
                            float* __restrict__ oMf, float* __restrict__ com, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  Generic<NJMAX, NVMAX> G;
  frame_placements_instance(G, M, L, q, oMf, com, i);
}

template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    frame_placements_vjp_kernel(const DevModel M, const __grid_constant__ FrameList L, const float* __restrict__ q,
                                const float* __restrict__ grad_oMf, const float* __restrict__ grad_com,
                                float* __restrict__ grad_q, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  FramePlacementsVjp<NJMAX, NVMAX> K;
  frame_placements_vjp_instance(K, M, L, q, grad_oMf, grad_com, grad_q, i);
}

namespace {
constexpr int kBlock = 64;
unsigned grid_of(int64_t B) { return (unsigned)((B + kBlock - 1) / kBlock); }
}  // namespace

cudaError_t launch_frame_placements(int size_class, const DevModel& M, const FrameList& L, const float* q, float* oMf,
                                    float* com, int64_t B, cudaStream_t stream) {
  return with_generic(size_class, [&](auto nj, auto nv) {
    frame_placements_kernel<decltype(nj)::value, decltype(nv)::value><<<grid_of(B), kBlock, 0, stream>>>(M, L, q, oMf,
                                                                                                       com, B);
    return cudaGetLastError();
  });
}

cudaError_t launch_frame_placements_vjp(int size_class, const DevModel& M, const FrameList& L, const float* q,
                                        const float* grad_oMf, const float* grad_com, float* grad_q, int64_t B,
                                        cudaStream_t stream) {
  return with_generic(size_class, [&](auto nj, auto nv) {
    frame_placements_vjp_kernel<decltype(nj)::value, decltype(nv)::value><<<grid_of(B), kBlock, 0, stream>>>(
        M, L, q, grad_oMf, grad_com, grad_q, B);
    return cudaGetLastError();
  });
}

}  // namespace pk
