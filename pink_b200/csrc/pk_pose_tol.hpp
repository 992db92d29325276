// Launches of the solves to separate position and orientation tolerances
// (pk_converge_pose_tol_prepared, pk_converge_goalset_pose_tol_prepared).  Their kernels live in
// pk_pose_tol.cu, a translation unit of their own: it compiles in parallel with pk_cabi.cu, and
// the default kernels in pk_cabi.cu keep their machine code.  Host C++ only.
#pragma once

#include <cuda_runtime.h>

#include "pk_select.hpp"

namespace pk {

// One launch: the problem (its selection, device model and problem, and the chain kernels'
// parameter block), the arguments of the C entry, and the stream.  S = G = 1 for converge.
struct PoseTolLaunch {
  const Selection* sel;
  DevModel dev;
  const DevProblem* P;
  const void* chain_params;  // ChainParams<sel->nj>
  int device;                // ordinal of the opt-in to dynamic shared memory
  const float* q;            // converge: q [B][nq]; goal sets: q_seeds [B S][nq]
  int S;
  const float* targets;      // [B G][target_stride]
  int G;
  unsigned mask;
  float tol, orientation_tol;
  int max_steps;
  float* q_out;
  float* err;
  int32_t *goal, *seed, *steps, *status;
  int64_t B;
  cudaStream_t stream;
};

// Enqueue the kernel; the launch error, if any (the caller checks cudaGetLastError).
cudaError_t launch_converge_pose_tol(const PoseTolLaunch& a);
cudaError_t launch_goalset_pose_tol(const PoseTolLaunch& a);

}  // namespace pk
