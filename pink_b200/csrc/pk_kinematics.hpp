// Launches of the differentiable forward kinematics (pk_frame_placements_batched,
// pk_frame_placements_vjp_batched).  Their kernels live in pk_kinematics.cu, a translation unit of
// their own: it compiles in parallel with pk_cabi.cu, and the kernels there keep their machine
// code.  Host C++ only.
#pragma once

#include <cuda_runtime.h>

#include "pk_kinematics.cuh"

namespace pk {

// Enqueue the kernel of the general path's size class `size_class` (generic_size_class); the
// launch error, if any.
cudaError_t launch_frame_placements(int size_class, const DevModel& M, const FrameList& L, const float* q, float* oMf,
                                    float* com, int64_t B, cudaStream_t stream);
cudaError_t launch_frame_placements_vjp(int size_class, const DevModel& M, const FrameList& L, const float* q,
                                        const float* grad_oMf, const float* grad_com, float* grad_q, int64_t B,
                                        cudaStream_t stream);

}  // namespace pk
