// Warp-cooperative programming layer for the tree kernel (pk_tree.cuh).
//
// One robot instance is handled by one warp.  The algorithm is written as a
// sequence of lane-parallel blocks that communicate only through the instance's
// workspace (shared memory on the device) and through the reductions below.
// The same source compiles for the host, where a "warp" is a plain loop over 32
// lanes; this is how tests/hostsim runs the cooperative kernel on the CPU
// (test harness only).
//
// Rules that keep both builds equivalent:
//  * inside PK_LANES(l) a lane may read workspace words written before the
//    previous PK_WSYNC(), and may write words no other lane touches in the block;
//  * values that are identical on every lane (read from the workspace, results of
//    reductions) live in ordinary variables outside PK_LANES blocks;
//  * per-lane values that must survive from one PK_LANES block to the next live in
//    a LaneVar<T> (a register on the device, an array of 32 on the host).
#pragma once

#include "pk_math.cuh"

namespace pk {

#if defined(__CUDA_ARCH__)

#define PK_LANES(l) for (int l = (int)(threadIdx.x & 31u), pk_once_##l = 1; pk_once_##l; pk_once_##l = 0)
#define PK_WSYNC() __syncwarp()

template <class T>
struct LaneVar {
  T v;
  __device__ __forceinline__ T& operator[](int) { return v; }
  __device__ __forceinline__ const T& operator[](int) const { return v; }
};

__device__ __forceinline__ float lane_sum(const LaneVar<float>& a) {
  float s = a.v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}
// Four sums at once with 10 shuffles instead of 20: after each of the first two
// butterfly stages a lane keeps only half of the values (the other half travels to
// its partner), the last three stages run on a single value, and the four results
// are broadcast from the lane groups that own them.  Same pairing as lane_sum.
__device__ __forceinline__ void lane_sum4(const LaneVar<float> (&p)[4], float (&out)[4]) {
  const unsigned lane = threadIdx.x & 31u;
  const bool h16 = lane & 16u;
  float k0 = h16 ? p[2].v : p[0].v;
  float k1 = h16 ? p[3].v : p[1].v;
  const float s0 = h16 ? p[0].v : p[2].v;
  const float s1 = h16 ? p[1].v : p[3].v;
  k0 += __shfl_xor_sync(0xffffffffu, s0, 16);
  k1 += __shfl_xor_sync(0xffffffffu, s1, 16);
  const bool h8 = lane & 8u;
  float k = h8 ? k1 : k0;
  const float s = h8 ? k0 : k1;
  k += __shfl_xor_sync(0xffffffffu, s, 8);
  k += __shfl_xor_sync(0xffffffffu, k, 4);
  k += __shfl_xor_sync(0xffffffffu, k, 2);
  k += __shfl_xor_sync(0xffffffffu, k, 1);
  out[0] = __shfl_sync(0xffffffffu, k, 0);
  out[1] = __shfl_sync(0xffffffffu, k, 8);
  out[2] = __shfl_sync(0xffffffffu, k, 16);
  out[3] = __shfl_sync(0xffffffffu, k, 24);
}
// smallest value and the index that carries it (ties: smallest index)
__device__ __forceinline__ void lane_argmin(const LaneVar<float>& val, const LaneVar<int>& idx, float& best,
                                            int& best_idx) {
  float s = val.v;
  int i = idx.v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float so = __shfl_xor_sync(0xffffffffu, s, o);
    const int io = __shfl_xor_sync(0xffffffffu, i, o);
    if (so < s || (so == s && io < i)) { s = so; i = io; }
  }
  best = s;
  best_idx = i;
}
__device__ __forceinline__ uint64_t lane_or64(const LaneVar<uint64_t>& a) {
  uint64_t s = a.v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s |= __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}
__device__ __forceinline__ int lane_or(const LaneVar<int>& a) {
  return __reduce_or_sync(0xffffffffu, a.v);
}
// value held by lane `src`, on every lane
__device__ __forceinline__ float lane_bcast(const LaneVar<float>& a, int src) {
  return __shfl_sync(0xffffffffu, a.v, src);
}
// lane 0's x, on every lane (on the host x is the one value lane 0 wrote)
__device__ __forceinline__ int lane0_int(int x) { return __shfl_sync(0xffffffffu, x, 0); }
__device__ __forceinline__ double lane_sum_d(const LaneVar<double>& a) {
  double s = a.v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

#else  // host emulation: one "warp" = a loop over 32 lanes

#define PK_LANES(l) for (int l = 0; l < 32; ++l)
#define PK_WSYNC() ((void)0)

template <class T>
struct LaneVar {
  T v[32];
  T& operator[](int l) { return v[l]; }
  const T& operator[](int l) const { return v[l]; }
};

inline float lane_sum(const LaneVar<float>& a) {
  // same pairing as the xor-butterfly on the device, so that rounding matches
  float t[32];
  for (int l = 0; l < 32; ++l) t[l] = a.v[l];
  for (int o = 16; o > 0; o >>= 1) {
    float n[32];
    for (int l = 0; l < 32; ++l) n[l] = t[l] + t[l ^ o];
    for (int l = 0; l < 32; ++l) t[l] = n[l];
  }
  return t[0];
}
inline void lane_sum4(const LaneVar<float> (&p)[4], float (&out)[4]) {
  for (int c = 0; c < 4; ++c) out[c] = lane_sum(p[c]);
}
inline void lane_argmin(const LaneVar<float>& val, const LaneVar<int>& idx, float& best, int& best_idx) {
  best = val.v[0];
  best_idx = idx.v[0];
  for (int l = 1; l < 32; ++l)
    if (val.v[l] < best || (val.v[l] == best && idx.v[l] < best_idx)) { best = val.v[l]; best_idx = idx.v[l]; }
}
inline uint64_t lane_or64(const LaneVar<uint64_t>& a) {
  uint64_t s = 0;
  for (int l = 0; l < 32; ++l) s |= a.v[l];
  return s;
}
inline int lane_or(const LaneVar<int>& a) {
  int s = 0;
  for (int l = 0; l < 32; ++l) s |= a.v[l];
  return s;
}
inline float lane_bcast(const LaneVar<float>& a, int src) { return a.v[src]; }
inline int lane0_int(int x) { return x; }
inline double lane_sum_d(const LaneVar<double>& a) {
  double t[32];
  for (int l = 0; l < 32; ++l) t[l] = a.v[l];
  for (int o = 16; o > 0; o >>= 1) {
    double n[32];
    for (int l = 0; l < 32; ++l) n[l] = t[l] + t[l ^ o];
    for (int l = 0; l < 32; ++l) t[l] = n[l];
  }
  return t[0];
}

#endif

}  // namespace pk
