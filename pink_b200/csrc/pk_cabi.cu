// C ABI of pink_b200 (include/pink_b200.h): model tables, problem marshalling,
// kernel selection and launches.  No torch types; built with plain nvcc into
// pink_b200/libpink_b200.so.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/pink_b200.h"
#include "pk_chain.cuh"
#include "pk_coop_kernel.cuh"
#include "pk_generic.cuh"
#include "pk_kinematics.hpp"
#include "pk_multistart.cuh"
#include "pk_pose_tol.hpp"
#include "pk_select.hpp"

namespace {

thread_local std::string g_error;
std::atomic<int64_t> g_launches{0};
std::atomic<bool> g_chain_pdl_rejected{false};  // a PDL launch of the chain kernel failed once

int fail(const std::string& msg) {
  g_error = msg;
  return 1;
}

#define PK_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t err__ = (expr);                                                         \
    if (err__ != cudaSuccess)                                                           \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(err__));              \
  } while (0)

}  // namespace

// --------------------------------------------------------------------------------------
// model
// --------------------------------------------------------------------------------------

struct PkModel {
  int device = 0;
  pk::HostModel hm;
  int njoints = 0, free_flyer = 0, nq = 0, nv = 0, nframes = 0;
  void* dev_buf = nullptr;
  pk::DevModel dev{};
  // staging of the host entry point: two independent sets (device buffers, internal streams,
  // events) used alternately, so that two calls submitted on two caller streams pipeline
  // (the upload of one under the kernel / download of the other); a call on the same caller
  // stream as its predecessor is ordered behind it by the stream itself
  std::mutex mu;
  struct Staging {
    float* st_q = nullptr;
    float* st_t = nullptr;
    float* st_v = nullptr;
    int32_t* st_s = nullptr;
    int64_t st_cap = 0;
    int st_tstride = 0;
    cudaStream_t st_streams[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t st_fork = nullptr;
    cudaEvent_t st_join[3] = {nullptr, nullptr, nullptr};
    bool st_busy = false;
    cudaEvent_t st_in[64] = {};    // H2D of chunk k complete
    cudaEvent_t st_kern[64] = {};  // kernel of chunk k complete
  };
  Staging st[2];
  int st_next = 0;
  // schedule of the host entry point: -1 = PK_HOST_MODE from the environment (default 0),
  // 0 = staged uploads and downloads, 1 = zero-copy, 2 = staged uploads, results written by the
  // kernels straight into the pinned host buffers (pk_model_set_host_schedule)
  int host_mode = -1;
  static constexpr int kMaxChunks = 64;
};

namespace {

template <typename T>
size_t align_up(size_t off) {
  return (off + alignof(T) - 1) / alignof(T) * alignof(T);
}

}  // namespace

extern "C" int pk_abi_version(void) { return PK_ABI_VERSION; }
extern "C" int pk_struct_size(int which) {
  switch (which) {
    case 0: return (int)sizeof(PkModelDesc);
    case 1: return (int)sizeof(PkTaskDesc);
    case 2: return (int)sizeof(PkBarrierDesc);
    case 3: return (int)sizeof(PkProblemDesc);
    default: return -1;
  }
}
extern "C" const char* pk_last_error(void) { return g_error.c_str(); }
extern "C" int64_t pk_launch_count(void) { return g_launches.load(); }
#ifdef PK_CHAIN_PHASE_CLOCKS
// Copies the phase records (pk::ChainPhaseRecord, pk_math.cuh) of the warps that started since
// the last call, at most n, to host memory `dst` and frees every slot; returns the number
// copied, or -1 on a CUDA error.  Instrumented builds only; call with the device idle.
extern "C" int pk_chain_phase_records(void* dst, int n, int warps_per_cta) {
  unsigned ctas = 0u;
  if (cudaMemcpyFromSymbol(&ctas, pk::g_chain_phase_ctas, sizeof(ctas)) != cudaSuccess) return -1;
  n = (int)std::min<int64_t>({(int64_t)std::max(n, 0), (int64_t)pk::kChainPhaseMaxWarps, (int64_t)ctas * warps_per_cta});
  if (n > 0 && cudaMemcpyFromSymbol(dst, pk::g_chain_phase, sizeof(pk::ChainPhaseRecord) * n) != cudaSuccess) return -1;
  ctas = 0u;
  if (cudaMemcpyToSymbol(pk::g_chain_phase_ctas, &ctas, sizeof(ctas)) != cudaSuccess) return -1;
  return n;
}
#endif

extern "C" int pk_model_create(const PkModelDesc* d, int device, PkModel** out) {
  if (!d || !out) return fail("pk_model_create: null argument");
  PkModel* m = new PkModel();
  const std::string err_msg = pk::build_host_model(d, &m->hm);
  if (!err_msg.empty()) {
    delete m;
    return fail("pk_model_create: " + err_msg);
  }
  m->device = device;
  const int nj = m->hm.njoints;
  const int ff = m->hm.free_flyer;
  m->njoints = nj;
  m->free_flyer = ff;
  m->nq = m->hm.nq;
  m->nv = m->hm.nv;
  m->nframes = m->hm.nframes;

  // one device buffer holding every table
  size_t off = 0;
  auto reserve = [&](size_t bytes, size_t align) {
    off = (off + align - 1) / align * align;
    size_t at = off;
    off += bytes;
    return at;
  };
  const size_t o_anc = reserve(sizeof(uint64_t) * (nj + 2), 8);
  const size_t o_parent = reserve(sizeof(int) * std::max(nj, 1), 4);
  const size_t o_jtype = reserve(sizeof(int) * std::max(nj, 1), 4);
  const size_t o_jX = reserve(sizeof(float) * 12 * std::max(nj, 1), 16);
  const size_t o_axis = reserve(sizeof(float) * 3 * std::max(nj, 1), 4);
  const size_t o_fb = reserve(sizeof(int) * std::max(d->nframes, 1), 4);
  const size_t o_fX = reserve(sizeof(float) * 12 * std::max(d->nframes, 1), 16);
  const size_t o_mass = reserve(sizeof(float) * (nj + 1), 4);
  const size_t o_com = reserve(sizeof(float) * 3 * (nj + 1), 4);
  const size_t o_depth = reserve(sizeof(int) * std::max(nj, 1), 4);
  std::vector<char> host(off, 0);
  memcpy(host.data() + o_anc, m->hm.anc.data(), sizeof(uint64_t) * (nj + 2));
  if (nj) {
    memcpy(host.data() + o_parent, m->hm.parent.data(), sizeof(int) * nj);
    memcpy(host.data() + o_jtype, m->hm.jtype.data(), sizeof(int) * nj);
    memcpy(host.data() + o_jX, m->hm.jX.data(), sizeof(float) * 12 * nj);
    memcpy(host.data() + o_axis, m->hm.axis.data(), sizeof(float) * 3 * nj);
  }
  if (d->nframes) {
    memcpy(host.data() + o_fb, m->hm.frame_body.data(), sizeof(int) * d->nframes);
    memcpy(host.data() + o_fX, m->hm.fX.data(), sizeof(float) * 12 * d->nframes);
  }
  memcpy(host.data() + o_mass, m->hm.mass.data(), sizeof(float) * (nj + 1));
  memcpy(host.data() + o_com, m->hm.com.data(), sizeof(float) * 3 * (nj + 1));
  memcpy(host.data() + o_depth, m->hm.depth.data(), sizeof(int) * std::max(nj, 1));

  cudaError_t err = cudaSetDevice(device);
  if (err == cudaSuccess) err = cudaMalloc(&m->dev_buf, off);
  if (err == cudaSuccess) err = cudaMemcpy(m->dev_buf, host.data(), off, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    const std::string msg = std::string("pk_model_create: ") + cudaGetErrorString(err);
    if (m->dev_buf) cudaFree(m->dev_buf);
    delete m;
    return fail(msg);
  }
  char* base = (char*)m->dev_buf;
  m->dev.njoints = nj;
  m->dev.free_flyer = ff;
  m->dev.nq = m->nq;
  m->dev.nv = m->nv;
  m->dev.nframes = d->nframes;
  m->dev.anc = (const uint64_t*)(base + o_anc);
  m->dev.parent = (const int*)(base + o_parent);
  m->dev.jtype = (const int*)(base + o_jtype);
  m->dev.jX = (const float*)(base + o_jX);
  m->dev.axis = (const float*)(base + o_axis);
  m->dev.frame_body = (const int*)(base + o_fb);
  m->dev.fX = (const float*)(base + o_fX);
  m->dev.mass = (const float*)(base + o_mass);
  m->dev.com = (const float*)(base + o_com);
  m->dev.total_mass = m->hm.total_mass;
  m->dev.depth = (const int*)(base + o_depth);
  m->dev.maxdepth = m->hm.maxdepth;
  *out = m;
  return 0;
}

// Which of the host-buffer schedules pk_solve_ik_*_host uses for this model: 0 = uploads and
// downloads staged through device buffers by the copy engines, one direction at a time;
// 2 = staged uploads, the kernels write v / status straight into the caller's pinned host
// buffers (no download phase; falls back to 0 when a result buffer is not pinned);
// 1 = zero-copy both ways; -1 = back to the PK_HOST_MODE environment default.  Which one is
// faster depends on how the platform's PCIe root handles both directions at once, so the
// caller measures: BatchedIK.tune_host_path() times them on its own buffers.
extern "C" int pk_model_set_host_schedule(PkModel* m, int mode) {
  if (!m) return fail("null model");
  if (mode < -1 || mode > 2) return fail("host schedule must be -1, 0, 1 or 2");
  std::lock_guard<std::mutex> lock(m->mu);
  m->host_mode = mode;
  return 0;
}

extern "C" void pk_model_destroy(PkModel* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->dev_buf) cudaFree(m->dev_buf);
  for (PkModel::Staging& S : m->st) {
    if (S.st_q) cudaFree(S.st_q);
    if (S.st_t) cudaFree(S.st_t);
    if (S.st_v) cudaFree(S.st_v);
    if (S.st_s) cudaFree(S.st_s);
    for (int i = 0; i < 3; ++i) {
      if (S.st_streams[i]) cudaStreamDestroy(S.st_streams[i]);
      if (S.st_join[i]) cudaEventDestroy(S.st_join[i]);
    }
    if (S.st_fork) cudaEventDestroy(S.st_fork);
    for (int i = 0; i < PkModel::kMaxChunks; ++i) {
      if (S.st_in[i]) cudaEventDestroy(S.st_in[i]);
      if (S.st_kern[i]) cudaEventDestroy(S.st_kern[i]);
    }
  }
  delete m;
}

// --------------------------------------------------------------------------------------
// kernels
// --------------------------------------------------------------------------------------

namespace pk {

// Chain kernel: one instance per thread, everything in registers - limit check, FK,
// task rows, box, corner start with the closed-form first releases, and (for the few
// instances that still need them) the Cholesky active-set rounds and the polish
// (pk_chain.cuh, pk_lsq.cuh).  n_steps > 1: closed-loop rollout, q <- q (+) v dt after
// every step with q kept in registers (pink/configuration.py:285-293 after
// pink/solve_ik.py:274); an instance that fails a step (no solution / outside limits
// with safety_break) is frozen.
//
// History (profiles/, DESIGN.md section 3.1): an earlier version parked the unfinished QPs
// of a CTA in shared memory and ran their rounds on compacted warps; once the corner
// start and the closed-form releases settle 99.3 % of the benchmark instances in the
// uniform part, that machinery (barriers, slot traffic) cost more than the sparse warps
// it saved (21.6 us vs 18.4 us per 65536-instance launch) and was removed.
// Gather targets of the fused epilogue (pk_solve_ik_prepared_gather): velocity row i goes to
// row (row_offset + i) of each peer buffer.  n == 0: no gather.
struct PeerOut {
  float* ptr[PK_MAX_PEERS];
  int n;
  int64_t row_offset;
  // flow control (optional, flags[0] != nullptr): flags[p] = flag block of rank p (peer-mapped)
  unsigned* flags[PK_MAX_PEERS];
  int rank;
  int n_buffers;  // gather buffers the caller rotates through
};

// Flag block of a rank (uint32 words; written by peers with release stores, zero at start):
//   [p]       produced[p]: gathers rank p has completed (its rows of that gather are visible)
//   [16 + p]  consumed[p]: gathers rank p has released (it no longer reads that buffer slot)
//   [32] gathers this rank has published, [33] waits it has issued, [34] CTA counter, [35] time-outs,
//   [36] gather kernels this rank has run
constexpr int kPeerProduced = 0, kPeerConsumed = PK_MAX_PEERS, kPeerCalls = 2 * PK_MAX_PEERS,
              kPeerWaits = 2 * PK_MAX_PEERS + 1, kPeerCtas = 2 * PK_MAX_PEERS + 2, kPeerTimeouts = 2 * PK_MAX_PEERS + 3,
              kPeerLaunched = 2 * PK_MAX_PEERS + 4;
constexpr long long kPeerSpinLimit = 4000000000ll;  // ~2 s: a peer that never arrives must not hang the GPU

__device__ __forceinline__ unsigned peer_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void peer_st_release(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// First instructions of a kernel that stores gather number k (= kernels run so far + 1) into
// slot k % n_buffers of the peers' buffers: every peer must have released gather k - n_buffers,
// which used the same slot.  Almost always true already: one pass over n local words per CTA.
__device__ __forceinline__ void peer_gate(const PeerOut& peers) {
  if (peers.n > 0 && peers.flags[0] != nullptr) {
    if (threadIdx.x < (unsigned)peers.n) {
      unsigned* mine = peers.flags[peers.rank];
      const unsigned k = mine[kPeerLaunched] + 1u;  // stable: written at the end of the previous kernel
      const long long t0 = clock64();
      while ((int)(peer_ld_acquire(mine + kPeerConsumed + threadIdx.x) + (unsigned)peers.n_buffers - k) < 0) {
        if (clock64() - t0 > kPeerSpinLimit) {
          atomicAdd(mine + kPeerTimeouts, 1u);
          break;
        }
      }
    }
    __syncthreads();
  }
}
// Last instructions of that kernel (thread 0 of every CTA): count the kernel once all CTAs are through.
// No fence: only the next kernel of the stream reads the count.
__device__ __forceinline__ void peer_count_kernel(const PeerOut& peers) {
  if (peers.n > 0 && peers.flags[0] != nullptr && threadIdx.x == 0) {
    unsigned* mine = peers.flags[peers.rank];
    if (atomicAdd(mine + kPeerCtas, 1u) == gridDim.x - 1u) {
      mine[kPeerCtas] = 0u;
      mine[kPeerLaunched] += 1u;
    }
  }
}

// Programmatic dependent launch (PDL).  The chain kernel is one wave whose end waits for
// its slowest warps (the few instances in Cholesky rounds); launched with the
// programmatic-serialization attribute, the next launch on the stream starts its CTAs in
// the slots those tail CTAs leave free.  Protocol of the PDL instantiation:
//   - griddepcontrol.launch_dependents first: the next grid may start at once;
//   - q and the targets row are read and solved before griddepcontrol.wait, which every
//     valid thread executes before its first global store: no grid completes before its
//     predecessor, so stream order holds for whatever runs after it;
//   - the library cannot see what ran before it on the stream (our own previous call
//     writing this call's q, or a foreign kernel that triggers early and then writes q or
//     the targets), so after the wait the q row and the targets row are read again from L2
//     (cp.async.cg / ld.global.cg) and compared bitwise with the values the steps used.  On a
//     difference every step of the instance is recomputed from the re-read values.
// Before the wait, each thread stages its targets row in its slot of the CTA's shared memory
// (ChainPdlSlot) with cp.async, so that every copy of the row is in flight at once and none
// takes a register; the re-read goes to a second row of the same slot, in flight at once too.
// The steps read the row from that slot, never through the read-only path, so "the values the
// steps used" are exactly the slot, and a line the L1 cached before the wait cannot leak into
// the recompute.
// Right after the trigger, CTAs 0 .. l2_ctas - 1 prefetch the whole grid's q and targets rows into
// L2 (pk::chain_l2_prefetch_ctas).  Under PDL those CTAs start early, in the slots the previous
// grid leaves free, while the rest of the grid starts together once the previous one retires;
// the prefetch lets that burst load from L2 instead of HBM.  It fills L2 only, the point of
// coherence: a predecessor's later write replaces the line there and the post-wait re-read (from
// L2) sees it, so a line prefetched before that write cannot reach the results.
// PK_CHAIN_PDL=0 (compile time) launches the plain instantiation only, for A/B runs.
#ifndef PK_CHAIN_PDL
#define PK_CHAIN_PDL 1
#endif
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// flags bit: after the wait, recompute every instance as if its inputs had changed (tests)
constexpr int kChainForceRecompute = 4;

// One thread's slot of the PDL instantiation's staging buffer, in words: [targets row | q row |
// re-read targets row], each part starting on a 16-byte boundary and sized for the longest row
// the instantiation accepts (chain_row_words), so that every offset is a compile-time constant.
// The slot stride is 4 words times an odd number: the eight threads of each phase of a 128-bit
// shared load hit eight distinct 16-byte bank groups.
template <int NJ, int NFT>
struct ChainPdlSlot {
  static constexpr int kRow = (chain_row_words(NJ, NFT) + 3) & ~3;
  static constexpr int kQ = kRow;
  static constexpr int kReread = (kQ + NJ + 3) & ~3;
  static constexpr int kWords = ((kReread + kRow) / 4) % 2 ? kReread + kRow : kReread + kRow + 4;
  // this thread's slot in a CTA of at most 128 threads; %tid.x is read with a volatile move,
  // so the address is formed where it is used instead of being held in a register across
  // the steps
  static __device__ __forceinline__ float* row() {
    __shared__ __align__(16) float rows[128 * kWords];
    unsigned tid;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
    return rows + tid * kWords;
  }
};

__device__ __forceinline__ void cp_async_cg16(float* dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
               "l"(__cvta_generic_to_global(src))
               : "memory");
}
__device__ __forceinline__ void cp_async_ca4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
               "l"(__cvta_generic_to_global(src))
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Issue the copies of the `n`-word targets row `src` into shared `dst`, all of them before any
// completes.  v4: n is a multiple of 4 and src is 16-byte aligned (128-bit copies, L2 only);
// otherwise one 4-byte copy per word.  Nothing past the row is read.
__device__ __forceinline__ void chain_stage_row(float* dst, const float* src, int n, bool v4) {
  if (v4) {
#pragma unroll 1
    for (int k = 0; k < n; k += 4) cp_async_cg16(dst + k, src + k);
  } else {
#pragma unroll 1
    for (int k = 0; k < n; ++k) cp_async_ca4(dst + k, src + k);
  }
}
// The re-read after the wait: from L2 only (a line the L1 cached before the wait may be stale).
// The 4-byte form has no L2-only cp.async, so it loads with ld.global.cg.
__device__ __forceinline__ void chain_reread_row(float* dst, const float* src, int n, bool v4) {
  if (v4) {
#pragma unroll 1
    for (int k = 0; k < n; k += 4) cp_async_cg16(dst + k, src + k);
  } else {
#pragma unroll 4
    for (int k = 0; k < n; ++k) dst[k] = __ldcg(src + k);
  }
}
// Whether the first `n` words of the shared rows a and b (16-byte aligned) are bitwise equal.
__device__ __forceinline__ bool chain_rows_equal(const float* a, const float* b, int n) {
  unsigned diff = 0u;
  int k = 0;
#pragma unroll 1
  for (; k + 4 <= n; k += 4) {
    const uint4 x = *reinterpret_cast<const uint4*>(a + k), y = *reinterpret_cast<const uint4*>(b + k);
    diff |= (x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w);
  }
#pragma unroll 1
  for (; k < n; ++k) diff |= __float_as_uint(a[k]) ^ __float_as_uint(b[k]);
  return diff == 0u;
}

// L2 prefetch of the floats [base, base + n) by the threads of CTAs 0 .. nctas - 1, each its own
// slice of whole 16-byte groups of the range's 16-byte-aligned interior; the ragged ends are left
// to the loads.  A hint: nothing is waited for, and no byte outside the range is addressed.
__device__ __forceinline__ void chain_l2_prefetch(const float* base, int64_t n, int nctas) {
  const uintptr_t a0 = (reinterpret_cast<uintptr_t>(base) + 15u) & ~uintptr_t(15);
  const uintptr_t a1 = reinterpret_cast<uintptr_t>(base + n) & ~uintptr_t(15);
  if (a1 <= a0) return;
  const int64_t groups = (int64_t)((a1 - a0) >> 4), parts = (int64_t)nctas * blockDim.x;
  const int64_t part = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t g0 = groups * part / parts, g1 = groups * (part + 1) / parts;
  // one bulk prefetch per thread: faster on the benchmark than one prefetch.global.L2 per
  // 128-byte line (DESIGN §3.1)
  if (g1 > g0)
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a0 + 16 * (uintptr_t)g0),
                 "r"((unsigned)(16 * (g1 - g0))));
}

// T: per-step targets and records of a trajectory call, read by the plain instantiation only.
// The PDL protocol validates one copied targets row after the wait and stores nothing before
// it, so it cannot cover K rows or per-step stores: trajectory calls with a step stride or
// records always launch <NJ, NFT, false>.  Every step's row is read through load_se3_vec4,
// which checks each address, so a step stride that is not a multiple of 4 floats takes the
// scalar loads.  ARM: the problem has the arm shape (ChainParams::arm, ChainStep::assemble).
template <int NJ, int NFT, bool PDL, bool ARM = false>
__global__ void __launch_bounds__(128, 4)
    ik_chain_kernel(const __grid_constant__ ChainParams<NJ> P, const float* __restrict__ q,
                    const float* __restrict__ targets, float* __restrict__ v, int32_t* __restrict__ status,
                    int64_t B, int flags, int n_steps, float* __restrict__ q_out,
                    const __grid_constant__ PeerOut peers, const __grid_constant__ Trajectory T, int l2_ctas) {
  PK_PHASE(kPhaseEntry);
  if constexpr (PDL) {
    pdl_launch_dependents();
    if (blockIdx.x < (unsigned)l2_ctas) {
      chain_l2_prefetch(q, B * NJ, l2_ctas);
      chain_l2_prefetch(targets, B * (int64_t)P.target_stride, l2_ctas);
    }
  }
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  peer_gate(peers);
  if (i >= B) return;
  float qi[NJ], vi[NJ];
  const float* qrow = q + i * NJ;
  if constexpr (NJ % 2 == 0) {
#pragma unroll
    for (int k = 0; k < NJ / 2; ++k) {
      const float2 t = __ldg(reinterpret_cast<const float2*>(qrow) + k);
      qi[2 * k] = t.x;
      qi[2 * k + 1] = t.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < NJ; ++k) qi[k] = __ldg(qrow + k);
  }
  const float* const grow = targets + i * (int64_t)P.target_stride;
  int st_all;
  if constexpr (!PDL) {
    st_all = rollout_chain<NJ, NFT, true, ARM>(P, qi, grow, vi, n_steps, q_out != nullptr, flags, T, B, i);
  } else {
    using L = ChainPdlSlot<NJ, NFT>;
    const int n = P.target_stride;  // <= chain_row_words(NJ, NFT)
    const bool v4 = (n & 3) == 0 && (reinterpret_cast<uintptr_t>(grow) & 15u) == 0u;
    {
      float* const row = L::row();
      chain_stage_row(row, grow, n, v4);
#pragma unroll
      for (int k = 0; k < NJ; ++k) row[L::kQ + k] = qi[k];
    }
    cp_async_wait_all();  // each thread reads only its own slot: no barrier
    PK_PHASE(kPhaseLoaded);
#pragma unroll 1
    for (int pass = 0;; ++pass) {
      st_all = rollout_chain<NJ, NFT, false, ARM>(P, qi, L::row() + (pass ? L::kReread : 0), vi, n_steps,
                                                  q_out != nullptr, flags, T, B, i);
      if (pass > 0) break;
      pdl_wait();
      // the inputs as the predecessors left them; one recompute at most (nothing writes
      // them once the predecessors are complete)
      float* const row = L::row();
      chain_reread_row(row + L::kReread, grow, n, v4);
      float qn[NJ];
      bool same = !(flags & kChainForceRecompute);
#pragma unroll
      for (int k = 0; k < NJ; ++k) {
        qn[k] = __ldcg(qrow + k);
        same &= __float_as_uint(qn[k]) == __float_as_uint(row[L::kQ + k]);
      }
      cp_async_wait_all();
      if (same && chain_rows_equal(row, row + L::kReread, n)) break;
#pragma unroll
      for (int k = 0; k < NJ; ++k) qi[k] = qn[k];
    }
  }
  PK_PHASE(kPhaseWaited);
  if (v) {
    float* vrow = v + i * NJ;
    if constexpr (NJ % 2 == 0) {
#pragma unroll
      for (int k = 0; k < NJ / 2; ++k) reinterpret_cast<float2*>(vrow)[k] = make_float2(vi[2 * k], vi[2 * k + 1]);
    } else {
#pragma unroll
      for (int k = 0; k < NJ; ++k) vrow[k] = vi[k];
    }
  }
  // fused all-gather: posted stores into every peer's buffer (NVLink).  A warp's 32 rows are
  // 32 NJ contiguous floats: they are transposed through shared memory so that every store
  // instruction writes 512 contiguous bytes per warp (full 128-byte lines on the wire) instead
  // of 8-byte pieces at a 4 NJ-byte stride (measured at N = 8: the strided form ran the link at
  // about a third of its rate).
  if constexpr (!PDL) {  // the PDL instantiation never runs with peers
    if (peers.n > 0) {
      __shared__ __align__(16) float stage[8][32 * NJ];
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      const int64_t row0 = i - lane;  // first row of this warp
      const bool vec = (row0 + 32 <= B) && warp < 8 && ((peers.row_offset * NJ) % 4 == 0);
      if (vec) {
        float* st = stage[warp];
#pragma unroll
        for (int k = 0; k < NJ; ++k) st[lane * NJ + k] = vi[k];
        __syncwarp();
        constexpr int NV4 = 32 * NJ / 4;
        // destinations in a per-rank, per-CTA rotated order: all ranks storing to peer 0 first,
        // then peer 1, ... would converge on one NVSwitch port at a time
        const int first = peers.rank + 1 + (int)(blockIdx.x % (unsigned)peers.n);
#pragma unroll 1
        for (int t = 0; t < peers.n; ++t) {
          const int p = (first + t) % peers.n;
          float4* dst = reinterpret_cast<float4*>(peers.ptr[p] + (peers.row_offset + row0) * NJ);
#pragma unroll
          for (int f = lane; f < NV4; f += 32) dst[f] = reinterpret_cast<const float4*>(st)[f];
        }
      } else {
#pragma unroll 1
        for (int p = 0; p < peers.n; ++p) {
          float* prow = peers.ptr[p] + (peers.row_offset + i) * NJ;
#pragma unroll
          for (int k = 0; k < NJ; ++k) prow[k] = vi[k];
        }
      }
    }
  }
  if (q_out) {
    float* orow = q_out + i * NJ;
#pragma unroll
    for (int k = 0; k < NJ; ++k) orow[k] = qi[k];
  }
  if (status) status[i] = st_all;
  peer_count_kernel(peers);
  PK_PHASE(kPhaseStored);
}

// Solve to a tolerance on chains (pk_converge_prepared): converge_chain_instance per thread, q in
// registers.  A plain launch: no PDL, no peer epilogue, no records.  emask: the task mask in chain
// slots (chain_task_mask).
template <int NJ, int NFT>
__global__ void __launch_bounds__(128, 4)
    ik_chain_converge_kernel(const __grid_constant__ ChainParams<NJ> P, const float* q,
                             const float* __restrict__ targets, unsigned emask, float tol, int max_steps,
                             float* q_out, float* __restrict__ err, int32_t* __restrict__ steps,
                             int32_t* __restrict__ status, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  converge_chain_instance<NJ, NFT>(P, q, targets, emask, tol, max_steps, q_out, err, steps, status, i);
}

// General path: one instance per thread, per-thread arrays in local memory.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64) ik_generic_kernel(const DevModel M, const __grid_constant__ DevProblem P,
                                                        const GenericArgs A, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const GenericOut out = generic_out(M, A, i);
  Generic<NJMAX, NVMAX> G;
  G.step(M, P, A.q + i * M.nq, A.targets ? A.targets + i * (int64_t)P.target_stride : nullptr, out);
}

// Trajectory rollout of the general path in one launch: rollout_generic_instance per thread.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_rollout_kernel(const DevModel M, const __grid_constant__ DevProblem P, const float* q,
                              const float* __restrict__ targets, int n_steps, float* q_out, float* __restrict__ v,
                              int32_t* __restrict__ status, int64_t B, const __grid_constant__ Trajectory T) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  Generic<NJMAX, NVMAX> G;
  rollout_generic_instance(G, M, P, q, targets, n_steps, q_out, v, status, T, B, i);
}

// Solve to a tolerance on the general path (pk_converge_prepared): converge_generic_instance per thread.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_converge_kernel(const DevModel M, const __grid_constant__ DevProblem P, const float* q,
                               const float* __restrict__ targets, unsigned mask, float tol, int max_steps, float* q_out,
                               float* __restrict__ err, int32_t* __restrict__ steps, int32_t* __restrict__ status,
                               int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  Generic<NJMAX, NVMAX> G;
  converge_generic_instance(G, M, P, q, targets, mask, tol, max_steps, q_out, err, steps, status, i);
}

// Gradient with respect to the targets at converged solutions (pk_converge_vjp_prepared), on every
// model: solution_vjp_instance per thread.
template <int NJMAX, int NVMAX>
__global__ void __launch_bounds__(64)
    ik_generic_solution_vjp_kernel(const DevModel M, const __grid_constant__ DevProblem P, const float* q_star,
                                   const float* targets, const float* grad_q, float* grad_targets,
                                   int32_t* __restrict__ status, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  Generic<NJMAX, NVMAX> G;
  solution_vjp_instance(G, M, P, q_star, targets, grad_q, grad_targets, status, i);
}

// Tree kernel: one instance per warp, per-instance state in the warp's slice of
// dynamic shared memory (pk_tree.cuh); kTreeWarpsPerBlock in pk_select.hpp.
// resident CTAs per SM the register allocation aims at: 10 (96 registers, 40 B of spills) ran
// 4 % faster than 8 (128 registers) on configs 3 / 4 (scripts/r2_tree_ab.sh)
#ifndef PK_TREE_MIN_BLOCKS
#define PK_TREE_MIN_BLOCKS 10
#endif
__global__ void __launch_bounds__(32 * kTreeWarpsPerBlock, PK_TREE_MIN_BLOCKS)
    ik_tree_kernel(const DevModel M, const __grid_constant__ DevProblem P, const __grid_constant__ TreePlan L,
                   const float* __restrict__ q, const float* __restrict__ targets, float* __restrict__ v,
                   int32_t* __restrict__ status, int64_t B) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * kTreeWarpsPerBlock + warp;
  if (i >= B) return;
  TreeStep::solve_instance(M, P, L, q, targets, tree_smem + (size_t)warp * L.words, v, status, i);
}

// Closed-loop rollout of the tree kernel in ONE launch: TreeStep::rollout_instance per warp, the q / v
// rows re-read by the warp that wrote them (they stay in L1 / L2; no per-step launch pair and its two
// full passes over HBM).
__global__ void __launch_bounds__(32 * kTreeWarpsPerBlock)
    ik_tree_rollout_kernel(const DevModel M, const __grid_constant__ DevProblem P, const __grid_constant__ TreePlan L,
                           const float* __restrict__ q, const float* __restrict__ targets, int n_steps,
                           float* __restrict__ q_out, float* __restrict__ v, int32_t* __restrict__ status, int64_t B,
                           const __grid_constant__ Trajectory T) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * kTreeWarpsPerBlock + warp;
  if (i >= B) return;
  TreeStep::rollout_instance(M, P, L, q, targets, n_steps, q_out, tree_smem + (size_t)warp * L.words, v, status, T, B,
                             i);
}

// Solve to a tolerance on joint trees (pk_converge_prepared): TreeStep::converge_instance per warp,
// L and o_v from converge_tree_layout.  The warp leaves its loop as soon as its instance stops.
__global__ void __launch_bounds__(32 * kTreeWarpsPerBlock)
    ik_tree_converge_kernel(const DevModel M, const __grid_constant__ DevProblem P, const __grid_constant__ TreePlan L,
                            int o_v, const float* q, const float* __restrict__ targets, unsigned mask, float tol,
                            int max_steps, float* q_out, float* __restrict__ err, int32_t* __restrict__ steps,
                            int32_t* __restrict__ status, int64_t B) {
  extern __shared__ __align__(16) float tree_smem[];
  const int warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * kTreeWarpsPerBlock + warp;
  if (i >= B) return;
  TreeStep::converge_instance(M, P, L, o_v, q, targets, mask, tol, max_steps, q_out, tree_smem + (size_t)warp * L.words,
                              err, steps, status, i);
}

// q (+) v dt
__global__ void integrate_kernel(int nq, int nv, int free_flyer, const float* __restrict__ q,
                                 const float* __restrict__ v, float dt, float* __restrict__ qo, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  integrate_configuration(nq, free_flyer, q + i * nq, v + i * nv, dt, qo + i * nq);
}

// Gather for the kernels without a fused epilogue: rows of the local v to every peer buffer.
__global__ void peer_scatter_kernel(const float* __restrict__ v, int64_t n_floats, const __grid_constant__ PeerOut peers,
                                    int nv) {
  peer_gate(peers);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_floats; k += stride) {
    const float x = v[k];
    for (int p = 0; p < peers.n; ++p) peers.ptr[p][peers.row_offset * nv + k] = x;
  }
  peer_count_kernel(peers);
}

struct PeerFlags {
  unsigned* ptr[PK_MAX_PEERS];
};

// One warp, one thread per peer; queued behind the kernel that stored a gather (whose stores
// are complete at the kernel boundary), on that stream or on any stream that waits for it.
//   post:    publish "gather k complete" (k = this rank's own count) in every peer's block;
//   wait:    hold the stream until the next gather this rank has not waited for yet has been
//            published by every rank;
//   release: then tell all peers that this rank is done with that gather's buffer slot.
__global__ void peer_sync_kernel(const __grid_constant__ PeerFlags F, int n, int rank, int post, int wait, int release) {
  const int t = threadIdx.x;
  unsigned* mine = F.ptr[rank];
  if (post) {
    unsigned k = 0;
    if (t == 0) {
      k = mine[kPeerCalls] + 1u;
      mine[kPeerCalls] = k;
      __threadfence_system();
    }
    k = __shfl_sync(0xffffffffu, k, 0);
    if (t < n) peer_st_release(F.ptr[t] + kPeerProduced + rank, k);
  }
  if (wait) {
    unsigned w = 0;
    if (t == 0) {
      w = mine[kPeerWaits] + 1u;
      mine[kPeerWaits] = w;
    }
    w = __shfl_sync(0xffffffffu, w, 0);
    if (t < n) {
      const long long t0 = clock64();
      while ((int)(peer_ld_acquire(mine + kPeerProduced + t) - w) < 0) {
        if (clock64() - t0 > kPeerSpinLimit) {
          atomicAdd(mine + kPeerTimeouts, 1u);
          break;
        }
      }
    }
    __syncwarp();
    if (release && t < n) peer_st_release(F.ptr[t] + kPeerConsumed + rank, w);
  }
}

}  // namespace pk

namespace {

int env_int(const char* name, int dflt) {
  const char* s = getenv(name);
  return s ? atoi(s) : dflt;
}

// Epilogue of every kernel launch.
int launched() {
  g_launches.fetch_add(1);
  PK_CUDA(cudaGetLastError());
  return 0;
}

const pk::PeerOut kNoPeers{};
const pk::Trajectory kNoTrajectory{};

// A kernel with one thread per row: `rows` threads in blocks of `block`.
template <class... Params, class... Args>
int launch_rows(void (*kernel)(Params...), int64_t rows, int block, cudaStream_t stream, const Args&... args) {
  kernel<<<(unsigned)((rows + block - 1) / block), block, 0, stream>>>(args...);
  return launched();
}

// a call the PDL instantiation of the chain kernel cannot run: per-step targets rows or records
bool per_step(const pk::Trajectory& T) { return T.target_step != 0 || T.q || T.v || T.status; }

// CTAs of the PDL chain kernel `kernel` the device holds at once at `block` threads, and its L2
// size in bytes, queried once per device ordinal.  Zero when a query fails: no prefetch.
struct ChainResidency {
  std::mutex mu;
  int64_t ctas[64] = {}, l2[64] = {};
};
template <class Kernel>
void chain_residency(ChainResidency& r, Kernel kernel, int block, int64_t* ctas, int64_t* l2) {
  int dev = 0;
  *ctas = *l2 = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return;
  std::lock_guard<std::mutex> lock(r.mu);
  if (dev >= 0 && dev < 64 && r.ctas[dev] > 0) {
    *ctas = r.ctas[dev];
    *l2 = r.l2[dev];
    return;
  }
  int per_sm = 0, sms = 0, l2_bytes = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, dev) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  *ctas = (int64_t)per_sm * sms;
  *l2 = l2_bytes;
  if (dev >= 0 && dev < 64) {
    r.ctas[dev] = *ctas;
    r.l2[dev] = *l2;
  }
}

template <int NJ, int NFT, bool ARM>
int launch_chain_shape(const pk::ChainParams<NJ>& C, bool pdl_row_fits, const float* q, const float* targets, float* v,
                       int32_t* status, int64_t B, cudaStream_t stream, int n_steps, float* q_out,
                       const pk::PeerOut& peers, const pk::Trajectory& traj) {
  // A/B and probe switches (timing experiments; see scripts/ab.sh)
  static const int flags = (env_int("PK_CLOSED_FORM", 1) ? 0 : 1) | (env_int("PK_PROBE_SKIP_ROUNDS", 0) ? 2 : 0) |
                           (env_int("PK_CHAIN_FORCE_RECOMPUTE", 0) ? pk::kChainForceRecompute : 0);
  static const int block = env_int("PK_CHAIN_BLOCK", 128);
  static const bool l2_prefetch = env_int("PK_CHAIN_L2_PREFETCH", 1) != 0;
  static ChainResidency residency;
  const int64_t grid = (B + block - 1) / block;
  // PDL unless the fused peer gather is on (peer_gate and its flag protocol assume full stream
  // order), the targets row is longer than the kernel's copy of it, or a trajectory call reads
  // a row per step or stores records
  if (PK_CHAIN_PDL && peers.n == 0 && pdl_row_fits && !per_step(traj) &&
      !g_chain_pdl_rejected.load(std::memory_order_relaxed)) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(block);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int l2_ctas = 0;
    if (l2_prefetch) {
      int64_t resident, l2;
      chain_residency(residency, pk::ik_chain_kernel<NJ, NFT, true, ARM>, block, &resident, &l2);
      l2_ctas = pk::chain_l2_prefetch_ctas(grid, resident, B * 4 * (NJ + (int64_t)C.target_stride), l2);
    }
    if (cudaLaunchKernelEx(&cfg, pk::ik_chain_kernel<NJ, NFT, true, ARM>, C, q, targets, v, status, B, flags, n_steps,
                           q_out, peers, traj, l2_ctas) == cudaSuccess)
      return launched();
    // a driver or capture mode that rejects the attribute: plain launches from now on
    cudaGetLastError();
    g_chain_pdl_rejected.store(true, std::memory_order_relaxed);
  }
  pk::ik_chain_kernel<NJ, NFT, false, ARM><<<(unsigned)grid, block, 0, stream>>>(C, q, targets, v, status, B, flags,
                                                                               n_steps, q_out, peers, traj, 0);
  return launched();
}

// the arm-shape instantiation when the problem has that shape (only with frame tasks: NFT > 0)
template <int NJ, int NFT>
int launch_chain(const pk::ChainParams<NJ>& C, bool pdl_row_fits, const float* q, const float* targets, float* v,
                 int32_t* status, int64_t B, cudaStream_t stream, int n_steps, float* q_out, const pk::PeerOut& peers,
                 const pk::Trajectory& traj) {
  // test switch: the general instantiation for every problem (read once)
  static const bool force_general = env_int("PK_CHAIN_FORCE_GENERAL", 0) != 0;
  if constexpr (NFT > 0) {
    if (C.arm && !force_general)
      return launch_chain_shape<NJ, NFT, true>(C, pdl_row_fits, q, targets, v, status, B, stream, n_steps, q_out, peers,
                                               traj);
  }
  return launch_chain_shape<NJ, NFT, false>(C, pdl_row_fits, q, targets, v, status, B, stream, n_steps, q_out, peers,
                                            traj);
}

// size_class: pk::generic_size_class of the model
int launch_generic(const PkModel* m, int size_class, const pk::DevProblem& P, const pk::GenericArgs& A, int64_t B,
                   cudaStream_t stream) {
  return pk::with_generic(size_class, [&](auto nj, auto nv) {
    return launch_rows(pk::ik_generic_kernel<decltype(nj)::value, decltype(nv)::value>, B, 64, stream, m->dev, P, A, B);
  });
}

// Dynamic shared memory a kernel has been granted, per device ordinal: the opt-in is per device,
// and the entry points may run on several host threads.
struct SmemGrant {
  std::mutex mu;
  size_t bytes[64] = {};
};
SmemGrant g_tree_smem, g_tree_rollout_smem, g_tree_converge_smem, g_tree_multistart_smem;

// A tree kernel with `smem` bytes of dynamic shared memory per CTA, opted into beyond the default.
template <class... Params, class... Args>
int launch_tree(void (*kernel)(Params...), SmemGrant& grant, const PkModel* m, int64_t grid, int block, size_t smem,
                cudaStream_t stream, const Args&... args) {
  {
    std::lock_guard<std::mutex> lock(grant.mu);
    const int dev = (m->device >= 0 && m->device < 64) ? m->device : 0;
    if (smem > grant.bytes[dev] || m->device >= 64) {
      PK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      grant.bytes[dev] = smem;
    }
  }
  kernel<<<(unsigned)grid, block, smem, stream>>>(args...);
  return launched();
}

// A tree kernel with one instance per warp and `plan.words` floats of dynamic shared memory per warp.
template <class... Params, class... Args>
int launch_tree_warps(void (*kernel)(Params...), SmemGrant& grant, const PkModel* m, const pk::TreePlan& plan,
                      int64_t B, cudaStream_t stream, const Args&... args) {
  return launch_tree(kernel, grant, m, (B + pk::kTreeWarpsPerBlock - 1) / pk::kTreeWarpsPerBlock,
                     32 * pk::kTreeWarpsPerBlock, (size_t)plan.words * 4 * pk::kTreeWarpsPerBlock, stream, args...);
}

}  // namespace

// A validated problem with its kernel selection and parameter blocks precomputed, so that the
// per-call host cost is one kernel launch.
struct PkProblem {
  pk::DevProblem P;
  void* dev_ext = nullptr;  // DevExtras + extra floats + pair indices (one allocation)
  // temporary problems of the un-prepared entry points: the image is allocated, filled and
  // released in stream order (no device-wide synchronisation per call)
  bool ext_async = false;
  cudaStream_t ext_stream = nullptr;
  ~PkProblem() {
    if (!dev_ext) return;
    if (ext_async) cudaFreeAsync(dev_ext, ext_stream);
    else cudaFree(dev_ext);
  }
  pk::Selection sel;
  std::string vjp_error;  // pk::check_vjp_problem: why pk_converge_vjp_prepared rejects the problem
  alignas(16) unsigned char chain_params[sizeof(pk::ChainParams<7>)];
  // parameter block of the sub-warp chain kernel's variant sel.lanes (the padding joints depend on it)
  alignas(16) unsigned char coop_params[sizeof(pk::CoopParams<8>)];

  // the parameter blocks, typed: ik_chain_kernel<NJ, *>'s and ik_coop_kernel<NJ, NFT, L>'s
  template <int NJ>
  pk::ChainParams<NJ>& chain() {
    static_assert(sizeof(pk::ChainParams<NJ>) <= sizeof(chain_params), "parameter block too small");
    return *reinterpret_cast<pk::ChainParams<NJ>*>(chain_params);
  }
  template <int NJ, int NFT, int L, class Params = pk::CoopParams<pk::CoopStep<NJ, NFT, L>::NJP>>
  Params& coop() {
    static_assert(sizeof(Params) <= sizeof(coop_params), "parameter block too small");
    return *reinterpret_cast<Params*>(coop_params);
  }
  template <int NJ> const auto& chain() const { return const_cast<PkProblem*>(this)->chain<NJ>(); }
  template <int NJ, int NFT, int L> const auto& coop() const { return const_cast<PkProblem*>(this)->coop<NJ, NFT, L>(); }
};

namespace {

// Device image of the optional problem parts: [DevExtras | extra | pairs] in one buffer.
// With `stream` the allocation and copies are stream-ordered (temporary problems of the
// un-prepared entry points, released with cudaFreeAsync after the launch).
int upload_extras(pk::HostExtras& hx, cudaStream_t stream, bool async, void** out) {
  const size_t o_extra = (sizeof(pk::DevExtras) + 15) & ~size_t(15);
  const size_t o_pairs = (o_extra + sizeof(float) * hx.extra.size() + 15) & ~size_t(15);
  const size_t total = o_pairs + sizeof(int) * hx.pairs.size() + 16;
  unsigned char* dev = nullptr;
  if (async) PK_CUDA(cudaMallocAsync((void**)&dev, total, stream));
  else PK_CUDA(cudaMalloc((void**)&dev, total));
  std::vector<unsigned char> img(total, 0);
  pk::DevExtras X = hx.X;
  X.extra = reinterpret_cast<const float*>(dev + o_extra);
  X.pairs = reinterpret_cast<const int*>(dev + o_pairs);
  memcpy(img.data(), &X, sizeof(X));
  if (!hx.extra.empty()) memcpy(img.data() + o_extra, hx.extra.data(), sizeof(float) * hx.extra.size());
  if (!hx.pairs.empty()) memcpy(img.data() + o_pairs, hx.pairs.data(), sizeof(int) * hx.pairs.size());
  // pageable source: the copy is staged before the call returns
  if (async) PK_CUDA(cudaMemcpyAsync(dev, img.data(), total, cudaMemcpyHostToDevice, stream));
  else PK_CUDA(cudaMemcpy(dev, img.data(), total, cudaMemcpyHostToDevice));
  *out = dev;
  return 0;
}

int prepare_problem(const PkModel* m, const PkProblemDesc* desc, PkProblem* pr, cudaStream_t stream = nullptr,
                    bool async = false) {
  if (!m) return fail("null model");
  pk::HostExtras hx;
  const std::string perr = pk::make_dev_problem(m->hm, desc, &pr->P, &hx);
  if (!perr.empty()) return fail(perr);
  if (hx.present) {
    if (upload_extras(hx, stream, async, &pr->dev_ext)) return 1;
    pr->ext_async = async;
    pr->ext_stream = stream;
    pr->P.ext = reinterpret_cast<const pk::DevExtras*>(pr->dev_ext);
  }
  // PK_CHAIN_LANES: 0 = round-1 kernel (one instance per thread, pk_chain.cuh); 1 / 2 / 4 / 8 =
  // sub-warp kernel (pk_coop.cuh) with that many lanes per instance
  static const pk::SelectOptions opts = [] {
    pk::SelectOptions o;
    o.use_chain = !env_int("PK_FORCE_GENERIC", 0);
    o.use_tree = o.use_chain && env_int("PK_TREE", 1);
    o.chain_lanes = env_int("PK_CHAIN_LANES", 0);
    return o;
  }();
  const pk::Selection& s = pr->sel = pk::select_kernel(m->hm, pr->P, hx, opts);
  pr->vjp_error = pk::check_vjp_problem(hx);
  if (s.path != pk::kPathChain) return 0;
  const pk::DevExtras* X = hx.present ? &hx.X : nullptr;
  pk::with_chain(s, [&](auto nj, auto nft) {
    constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
    pk::make_chain_params<NJ>(m->hm, pr->P, &pr->chain<NJ>(), X);
    if (!s.lanes) return;
    pk::with_lanes<NJ, NFT>(s.lanes, [&](auto lanes) {
      constexpr int L = decltype(lanes)::value;
      pk::make_coop_params<NJ, L>(m->hm, pr->P, &pr->coop<NJ, NFT, L>(), X);
    });
  });
  return 0;
}

// The chain kernels of a prepared chain problem; n_steps > 1 or q_out: closed-loop rollout.
// `peers`: the fused gather epilogue, which lives in the thread-per-instance kernel.  `traj`:
// per-step targets rows and records of a trajectory rollout.
int launch_chain_prepared(const PkProblem& pr, const float* q, const float* targets, float* v, int32_t* status,
                          int64_t B, cudaStream_t stream, int n_steps, float* q_out, const pk::PeerOut* peers,
                          const pk::Trajectory& traj = kNoTrajectory) {
  return pk::with_chain(pr.sel, [&](auto nj, auto nft) {
    constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
    if (pr.sel.lanes && !peers) {
      return pk::with_lanes<NJ, NFT>(pr.sel.lanes, [&](auto lanes) {
        constexpr int L = decltype(lanes)::value;
        return launch_rows(pk::ik_coop_kernel<NJ, NFT, L>, B * L, pk::kCoopThreads, stream, pr.coop<NJ, NFT, L>(), q,
                           targets, v, status, B, n_steps, q_out, traj);
      });
    }
    return launch_chain<NJ, NFT>(pr.chain<NJ>(), pr.sel.pdl_row_fits, q, targets, v, status, B, stream, n_steps, q_out,
                                 peers ? *peers : kNoPeers, traj);
  });
}

int solve_device(const PkModel* m, const PkProblem& pr, const float* q, const float* targets, float* v,
                 int32_t* status, int64_t B, cudaStream_t stream) {
  if (B == 0) return 0;
  if (pr.sel.path == pk::kPathChain) return launch_chain_prepared(pr, q, targets, v, status, B, stream, 1, nullptr, nullptr);
  if (pr.sel.path == pk::kPathTree)
    return launch_tree_warps(pk::ik_tree_kernel, g_tree_smem, m, pr.sel.plan, B, stream, m->dev, pr.P, pr.sel.plan,
                             q, targets, v, status, B);
  pk::GenericArgs A{};
  A.q = q;
  A.targets = targets;
  A.v = v;
  A.status = status;
  A.task_index = -1;
  return launch_generic(m, pr.sel.generic_class, pr.P, A, B, stream);
}

int check_common(const PkModel* m, const void* q, int64_t B) {
  if (!m) return fail("null model");
  if (B < 0) return fail("negative batch size");
  if (B > 0 && !q) return fail("null q");
  if (B > (int64_t)2147483647 * 32) return fail("batch too large");
  return 0;
}

// The argument checks of the *_prepared entries, in this order: check_common, the problem, the
// entry's own checks `more()` (nonzero: failed), the targets.
template <class More>
int check_prepared(const PkModel* m, const PkProblem* pr, const void* q, const void* targets, int64_t B, More more) {
  if (check_common(m, q, B)) return 1;
  if (!pr) return fail("null problem");
  if (more()) return 1;
  if (B > 0 && pr->P.target_stride > 0 && !targets) return fail("null targets");
  return 0;
}
int no_more_checks() { return 0; }

}  // namespace

// --------------------------------------------------------------------------------------
// entry points
// --------------------------------------------------------------------------------------

extern "C" int pk_problem_create(const PkModel* m, const PkProblemDesc* desc, PkProblem** out) {
  if (!out) return fail("null output");
  PkProblem* pr = new PkProblem();
  if (prepare_problem(m, desc, pr)) {
    delete pr;
    return 1;
  }
  *out = pr;
  return 0;
}

extern "C" void pk_problem_destroy(PkProblem* pr) { delete pr; }

static int solve_host_impl(PkModel* m, const PkProblem& pr, const float* q_host, const float* targets_host,
                           float* v_host, int32_t* status_host, int64_t B, cudaStream_t stream);

extern "C" int pk_solve_ik_prepared(const PkModel* m, const PkProblem* pr, const float* q, const float* targets,
                                    float* v, int32_t* status, int64_t B, void* stream) {
  if (check_prepared(m, pr, q, targets, B, [&] { return B > 0 && !v ? fail("null v") : 0; })) return 1;
  return solve_device(m, *pr, q, targets, v, status, B, (cudaStream_t)stream);
}

extern "C" int pk_solve_ik_prepared_host(PkModel* m, const PkProblem* pr, const float* q_host,
                                         const float* targets_host, float* v_host, int32_t* status_host, int64_t B,
                                         void* stream) {
  if (check_prepared(m, pr, q_host, targets_host, B, [&] { return B > 0 && !v_host ? fail("null v") : 0; })) return 1;
  return solve_host_impl(m, *pr, q_host, targets_host, v_host, status_host, B, (cudaStream_t)stream);
}

// ---- multi-GPU gather over peer memory -------------------------------------------------

extern "C" int pk_peer_alloc(int device, int64_t bytes, void** ptr, unsigned char* handle) {
  if (!ptr || !handle || bytes <= 0) return fail("pk_peer_alloc: bad arguments");
  PK_CUDA(cudaSetDevice(device));
  void* p = nullptr;
  PK_CUDA(cudaMalloc(&p, (size_t)bytes));
  PK_CUDA(cudaMemset(p, 0, (size_t)bytes));
  cudaIpcMemHandle_t h;
  static_assert(sizeof(h) == PK_IPC_HANDLE_BYTES, "IPC handle size");
  if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) {
    cudaFree(p);
    return fail(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(cudaGetLastError()));
  }
  memcpy(handle, &h, sizeof(h));
  *ptr = p;
  return 0;
}

extern "C" int pk_peer_open(int device, const unsigned char* handle, void** ptr) {
  if (!ptr || !handle) return fail("pk_peer_open: bad arguments");
  PK_CUDA(cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  PK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

extern "C" int pk_peer_close(int device, void* ptr) {
  if (!ptr) return 0;
  PK_CUDA(cudaSetDevice(device));
  PK_CUDA(cudaIpcCloseMemHandle(ptr));
  return 0;
}

extern "C" int pk_peer_free(int device, void* ptr) {
  if (!ptr) return 0;
  PK_CUDA(cudaSetDevice(device));
  PK_CUDA(cudaFree(ptr));
  return 0;
}

static int fill_peer_out(pk::PeerOut* po, void* const* peer_v, int32_t n_peers, int64_t row_offset,
                         void* const* peer_flags, int32_t rank, int32_t n_buffers) {
  if (n_peers < 0 || n_peers > PK_MAX_PEERS) return fail("n_peers out of range");
  if (n_peers > 0 && !peer_v) return fail("null peer_v");
  if (row_offset < 0) return fail("negative row_offset");
  memset(po, 0, sizeof(*po));
  po->n = n_peers;
  po->row_offset = row_offset;
  for (int k = 0; k < n_peers; ++k) {
    if (!peer_v[k]) return fail("null peer buffer");
    po->ptr[k] = static_cast<float*>(peer_v[k]);
  }
  if (rank >= 0 && rank < n_peers) po->rank = rank;
  if (peer_flags) {
    if (rank < 0 || rank >= n_peers) return fail("rank out of range");
    if (n_buffers < 1) return fail("n_buffers must be >= 1");
    for (int k = 0; k < n_peers; ++k) {
      if (!peer_flags[k]) return fail("null flag block");
      po->flags[k] = static_cast<unsigned*>(peer_flags[k]);
    }
    po->rank = rank;
    po->n_buffers = n_buffers;
  }
  return 0;
}

extern "C" int pk_solve_ik_prepared_gather(const PkModel* m, const PkProblem* pr, const float* q, const float* targets,
                                           float* v, int32_t* status, int64_t B, void* const* peer_v,
                                           int32_t n_peers, int64_t row_offset, void* const* peer_flags,
                                           int32_t rank, int32_t n_buffers, void* stream_) {
  if (check_prepared(m, pr, q, targets, B, no_more_checks)) return 1;
  if (B == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  pk::PeerOut po;
  if (fill_peer_out(&po, peer_v, n_peers, row_offset, peer_flags, rank, n_buffers)) return 1;
  if (pr->sel.path == pk::kPathChain) return launch_chain_prepared(*pr, q, targets, v, status, B, stream, 1, nullptr, &po);
  // kernels without the fused epilogue: solve into v, then one scatter kernel
  if (!v) return fail("this model needs a local v buffer for the gather");
  if (solve_device(m, *pr, q, targets, v, status, B, stream)) return 1;
  if (n_peers == 0) return 0;
  const int64_t n = B * m->nv;
  const int block = 256;
  int sms = 0;
  PK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->device));
  const int64_t grid = std::min<int64_t>((n + block - 1) / block, (int64_t)sms * 8);
  pk::peer_scatter_kernel<<<(unsigned)grid, block, 0, stream>>>(v, n, po, m->nv);
  return launched();
}

extern "C" int pk_peer_sync(int device, void* const* peer_flags, int32_t n_peers, int32_t rank, int32_t post,
                            int32_t wait, int32_t release, void* stream_) {
  if (n_peers < 1 || n_peers > PK_MAX_PEERS || !peer_flags) return fail("pk_peer_sync: bad arguments");
  if (rank < 0 || rank >= n_peers) return fail("pk_peer_sync: rank out of range");
  PK_CUDA(cudaSetDevice(device));
  pk::PeerFlags F{};
  for (int k = 0; k < n_peers; ++k) {
    if (!peer_flags[k]) return fail("null flag block");
    F.ptr[k] = static_cast<unsigned*>(peer_flags[k]);
  }
  pk::peer_sync_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>(F, n_peers, rank, post ? 1 : 0, wait ? 1 : 0, release ? 1 : 0);
  PK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int pk_rollout_prepared(const PkModel* m, const PkProblem* pr, const float* q, const float* targets,
                                   int32_t n_steps, float* q_out, float* v, int32_t* status, int64_t B,
                                   void* stream_) {
  if (check_prepared(m, pr, q, targets, B, [&] {
        if (n_steps < 1) return fail("n_steps must be >= 1");
        return B > 0 && (!v || !q_out) ? fail("null v or q_out") : 0;
      }))
    return 1;
  if (B == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  // chains and joint trees: the whole loop in one launch, the trajectory kernels with fixed rows
  // and no records
  if (pr->sel.path != pk::kPathGeneral)
    return pk_rollout_trajectory_prepared(m, pr, q, targets, 0, n_steps, q_out, v, status, nullptr, nullptr, nullptr, B,
                                          stream_);
  // the general path: the same closed loop as separate launches (solve, then integrate in place)
  if (q_out != q) PK_CUDA(cudaMemcpyAsync(q_out, q, sizeof(float) * B * m->nq, cudaMemcpyDeviceToDevice, stream));
  for (int s = 0; s < n_steps; ++s) {
    if (solve_device(m, *pr, q_out, targets, v, status, B, stream)) return 1;
    if (pk_integrate_batched(m, q_out, v, pr->P.dt, q_out, B, stream)) return 1;
  }
  return 0;
}

extern "C" int pk_rollout_trajectory_prepared(const PkModel* m, const PkProblem* pr, const float* q,
                                              const float* targets, int64_t target_step, int32_t n_steps,
                                              float* q_out, float* v, int32_t* status, float* q_traj, float* v_traj,
                                              int32_t* status_traj, int64_t B, void* stream_) {
  if (check_prepared(m, pr, q, targets, B, [&] {
        if (n_steps < 1) return fail("n_steps must be >= 1");
        if (target_step < 0) return fail("negative target_step");
        return B > 0 && (!v || !q_out) ? fail("null v or q_out") : 0;
      }))
    return 1;
  if (B == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  const pk::Trajectory traj{target_step, q_traj, v_traj, status_traj};
  if (pr->sel.path == pk::kPathChain)
    return launch_chain_prepared(*pr, q, targets, v, status, B, stream, n_steps, q_out, nullptr, traj);
  if (pr->sel.path == pk::kPathTree)
    return launch_tree_warps(pk::ik_tree_rollout_kernel, g_tree_rollout_smem, m, pr->sel.plan, B, stream, m->dev,
                             pr->P, pr->sel.plan, q, targets, n_steps, q_out, v, status, B, traj);
  return pk::with_generic(pr->sel.generic_class, [&](auto nj, auto nv) {
    return launch_rows(pk::ik_generic_rollout_kernel<decltype(nj)::value, decltype(nv)::value>, B, 64, stream, m->dev,
                       pr->P, q, targets, n_steps, q_out, v, status, B, traj);
  });
}

namespace {

// Stopping test of a converge call: the default one (pose = false), or separate position and
// orientation tolerances (pk_converge_pose_tol_prepared), whose kernels pk_pose_tol.cu launches.
struct StopMode {
  bool pose = false;
  float orientation_tol = 0.f;
};

// The launch of pk_converge_prepared and pk_converge_pose_tol_prepared.
int launch_converge(const PkModel* m, const PkProblem* pr, const float* q, const float* targets, uint32_t task_mask,
             float tol, int32_t max_steps, float* q_out, float* err, int32_t* steps, int32_t* status, int64_t B,
             void* stream_, const StopMode& mode) {
  if (check_prepared(m, pr, q, targets, B, [&] {
        std::string aerr = pk::check_converge_args(pr->P, task_mask, tol, max_steps);
        if (aerr.empty() && mode.pose) aerr = pk::check_pose_tol_args(pr->P, task_mask, tol, mode.orientation_tol);
        if (!aerr.empty()) return fail(aerr);
        return B > 0 && !q_out ? fail("null q_out") : 0;
      }))
    return 1;
  if (B == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  const pk::Selection& sel = pr->sel;
  if (mode.pose) {
    const pk::PoseTolLaunch a{&sel, m->dev, &pr->P, pr->chain_params, m->device, q, 1, targets, 1, task_mask, tol,
                              mode.orientation_tol, (int)max_steps, q_out, err, nullptr, nullptr, steps, status, B,
                              stream};
    PK_CUDA(pk::launch_converge_pose_tol(a));
    return launched();
  }
  if (sel.path == pk::kPathChain) {
    // always the thread-per-instance kernel: PK_CHAIN_LANES selects only the solve entries' variant
    const unsigned emask = pk::chain_task_mask(pr->P, task_mask, sel.nft);
    return pk::with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
      return launch_rows(pk::ik_chain_converge_kernel<NJ, NFT>, B, 128, stream, pr->chain<NJ>(), q, targets, emask, tol,
                         (int)max_steps, q_out, err, steps, status, B);
    });
  }
  if (sel.path == pk::kPathTree) {
    const pk::ConvergeTreeLayout T = pk::converge_tree_layout(sel.plan);
    return launch_tree_warps(pk::ik_tree_converge_kernel, g_tree_converge_smem, m, T.plan, B, stream, m->dev, pr->P,
                             T.plan, T.o_v, q, targets, task_mask, tol, (int)max_steps, q_out, err, steps, status, B);
  }
  return pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
    constexpr int NJ = decltype(nj)::value, NV = decltype(nv)::value;
    return launch_rows(pk::ik_generic_converge_kernel<NJ, NV>, B, 64, stream, m->dev, pr->P, q, targets, task_mask, tol,
                       (int)max_steps, q_out, err, steps, status, B);
  });
}

// The launch of pk_converge_goalset_prepared and pk_converge_goalset_pose_tol_prepared.
int launch_converge_goalset(const PkModel* m, const PkProblem* pr, const float* q_seeds, int32_t num_seeds,
                     const float* targets, int32_t num_goals, uint32_t task_mask, float tol, int32_t max_steps,
                     float* q_out, float* err, int32_t* goal, int32_t* seed, int32_t* steps, int32_t* status,
                     int64_t B, void* stream_, const StopMode& mode) {
  if (check_prepared(m, pr, q_seeds, targets, B, [&] {
        std::string aerr = pk::check_converge_args(pr->P, task_mask, tol, max_steps);
        if (aerr.empty() && mode.pose) aerr = pk::check_pose_tol_args(pr->P, task_mask, tol, mode.orientation_tol);
        if (!aerr.empty()) return fail(aerr);
        const std::string serr = pk::check_goalset_members(pr->sel, num_goals, num_seeds);
        if (!serr.empty()) return fail(serr);
        if (B > (int64_t)2147483647 * 32 / (num_goals * num_seeds)) return fail("batch too large");
        return B > 0 && !q_out ? fail("null q_out") : 0;
      }))
    return 1;
  if (B == 0) return 0;
  const pk::Selection& sel = pr->sel;
  const int S = num_seeds, G = num_goals;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (sel.path == pk::kPathTree && B > 2147483647) return fail("batch too large");
  if (mode.pose) {
    const pk::PoseTolLaunch a{&sel, m->dev, &pr->P, pr->chain_params, m->device, q_seeds, S, targets, G, task_mask, tol,
                              mode.orientation_tol, (int)max_steps, q_out, err, goal, seed, steps, status, B, stream};
    PK_CUDA(pk::launch_goalset_pose_tol(a));
    return launched();
  }
  if (sel.path == pk::kPathTree) {
    const pk::MultistartTreeLayout T = pk::multistart_tree_layout(sel.plan);
    return launch_tree(pk::ik_tree_multistart_kernel, g_tree_multistart_smem, m, B, 32 * G * S, T.smem_bytes(G * S),
                       stream, m->dev, pr->P, T.plan, T.o_v, T.o_q, q_seeds, S, targets, G, task_mask, tol,
                       (int)max_steps, q_out, err, goal, seed, steps, status, B);
  }
  if (sel.path == pk::kPathChain) {
    const unsigned emask = pk::chain_task_mask(pr->P, task_mask, sel.nft);
    return pk::with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
      auto launch = [&](auto kernel) {
        return launch_rows(kernel, B * G * S, 128, stream, pr->chain<NJ>(), q_seeds, S, targets, G, emask, tol,
                           (int)max_steps, q_out, err, goal, seed, steps, status, B);
      };
      return G == 1 ? launch(pk::ik_chain_multistart_kernel<NJ, NFT, false>)
                    : launch(pk::ik_chain_multistart_kernel<NJ, NFT, true>);
    });
  }
  return pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
    constexpr int NJ = decltype(nj)::value, NV = decltype(nv)::value;
    return launch_rows(pk::ik_generic_multistart_kernel<NJ, NV>, B * G * S, 64, stream, m->dev, pr->P, q_seeds, S,
                       targets, G, task_mask, tol, (int)max_steps, q_out, err, goal, seed, steps, status, B);
  });
}

}  // namespace

extern "C" int pk_converge_prepared(const PkModel* m, const PkProblem* pr, const float* q, const float* targets,
                                    uint32_t task_mask, float tol, int32_t max_steps, float* q_out, float* err,
                                    int32_t* steps, int32_t* status, int64_t B, void* stream_) {
  return launch_converge(m, pr, q, targets, task_mask, tol, max_steps, q_out, err, steps, status, B, stream_, StopMode{});
}

extern "C" int pk_converge_pose_tol_prepared(const PkModel* m, const PkProblem* pr, const float* q,
                                             const float* targets, uint32_t task_mask, float tol,
                                             float orientation_tol, int32_t max_steps, float* q_out, float* err,
                                             int32_t* steps, int32_t* status, int64_t B, void* stream_) {
  return launch_converge(m, pr, q, targets, task_mask, tol, max_steps, q_out, err, steps, status, B, stream_,
                  StopMode{true, orientation_tol});
}

extern "C" int pk_converge_goalset_prepared(const PkModel* m, const PkProblem* pr, const float* q_seeds,
                                            int32_t num_seeds, const float* targets, int32_t num_goals,
                                            uint32_t task_mask, float tol, int32_t max_steps, float* q_out, float* err,
                                            int32_t* goal, int32_t* seed, int32_t* steps, int32_t* status, int64_t B,
                                            void* stream_) {
  return launch_converge_goalset(m, pr, q_seeds, num_seeds, targets, num_goals, task_mask, tol, max_steps, q_out, err, goal,
                          seed, steps, status, B, stream_, StopMode{});
}

extern "C" int pk_converge_goalset_pose_tol_prepared(const PkModel* m, const PkProblem* pr, const float* q_seeds,
                                                     int32_t num_seeds, const float* targets, int32_t num_goals,
                                                     uint32_t task_mask, float tol, float orientation_tol,
                                                     int32_t max_steps, float* q_out, float* err, int32_t* goal,
                                                     int32_t* seed, int32_t* steps, int32_t* status, int64_t B,
                                                     void* stream_) {
  return launch_converge_goalset(m, pr, q_seeds, num_seeds, targets, num_goals, task_mask, tol, max_steps, q_out, err, goal,
                          seed, steps, status, B, stream_, StopMode{true, orientation_tol});
}

extern "C" int pk_converge_multistart_prepared(const PkModel* m, const PkProblem* pr, const float* q_seeds,
                                               int32_t num_seeds, const float* targets, uint32_t task_mask, float tol,
                                               int32_t max_steps, float* q_out, float* err, int32_t* seed,
                                               int32_t* steps, int32_t* status, int64_t B, void* stream_) {
  return pk_converge_goalset_prepared(m, pr, q_seeds, num_seeds, targets, 1, task_mask, tol, max_steps, q_out, err,
                                      nullptr, seed, steps, status, B, stream_);
}

extern "C" int pk_converge_vjp_prepared(const PkModel* m, const PkProblem* pr, const float* q_star,
                                        const float* targets, const float* grad_q, float* grad_targets,
                                        int32_t* status, int64_t B, void* stream_) {
  if (check_prepared(m, pr, q_star, targets, B, [&] {
        if (!pr->vjp_error.empty()) return fail(pr->vjp_error);
        if (B > 0 && !grad_q) return fail("null grad_q");
        return B > 0 && pr->P.target_stride > 0 && !grad_targets ? fail("null grad_targets") : 0;
      }))
    return 1;
  if (B == 0) return 0;
  return pk::with_generic(pk::generic_size_class(m->hm), [&](auto nj, auto nv) {
    return launch_rows(pk::ik_generic_solution_vjp_kernel<decltype(nj)::value, decltype(nv)::value>, B, 64,
                       (cudaStream_t)stream_, m->dev, pr->P, q_star, targets, grad_q, grad_targets, status, B);
  });
}

extern "C" int pk_solve_ik_batched(const PkModel* m, const PkProblemDesc* prob, const float* q,
                                   const float* targets, float* v, int32_t* status, int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  if (B > 0 && !v) return fail("null v");
  PkProblem pr;
  if (prepare_problem(m, prob, &pr, (cudaStream_t)stream, true)) return 1;
  if (B > 0 && pr.P.target_stride > 0 && !targets) return fail("null targets");
  return solve_device(m, pr, q, targets, v, status, B, (cudaStream_t)stream);
}

extern "C" int pk_solve_ik_batched_host(PkModel* m, const PkProblemDesc* prob, const float* q_host,
                                        const float* targets_host, float* v_host, int32_t* status_host,
                                        int64_t B, void* stream_) {
  if (check_common(m, q_host, B)) return 1;
  if (B > 0 && !v_host) return fail("null v");
  PkProblem pr;
  if (prepare_problem(m, prob, &pr, (cudaStream_t)stream_, true)) return 1;
  if (B > 0 && pr.P.target_stride > 0 && !targets_host) return fail("null targets");
  return solve_host_impl(m, pr, q_host, targets_host, v_host, status_host, B, (cudaStream_t)stream_);
}

static int solve_host_impl(PkModel* m, const PkProblem& pr, const float* q_host, const float* targets_host,
                           float* v_host, int32_t* status_host, int64_t B, cudaStream_t stream) {
  if (B == 0) return 0;
  const pk::DevProblem& P = pr.P;
  // Zero-copy mode: when every buffer is pinned (device-addressable under UVA) the
  // kernel can pull q / targets over PCIe itself and push v / status back: one
  // launch, no staging copies.  PK_HOST_MODE=1 selects it; default is staged DMA.
  static const int host_mode_env = env_int("PK_HOST_MODE", 0);
  const int host_mode = m->host_mode >= 0 ? m->host_mode : host_mode_env;
  if (host_mode == 1) {
    auto pinned = [](const void* ptr) {
      if (!ptr) return true;
      cudaPointerAttributes a{};
      return cudaPointerGetAttributes(&a, ptr) == cudaSuccess && a.type == cudaMemoryTypeHost && a.devicePointer;
    };
    if (pinned(q_host) && pinned(targets_host) && pinned(v_host) && pinned(status_host)) {
      PK_CUDA(cudaSetDevice(m->device));
      return solve_device(m, pr, q_host, targets_host, v_host, status_host, B, stream);
    }
    cudaGetLastError();  // clear the error of a failed attribute query on pageable memory
  }
  std::lock_guard<std::mutex> lock(m->mu);
  PK_CUDA(cudaSetDevice(m->device));
  PkModel::Staging& S = m->st[m->st_next];
  m->st_next ^= 1;
  const int ts = P.target_stride;
  if (B > S.st_cap || ts > S.st_tstride) {
    // (re)size staging; happens on the first call or when the batch grows
    PK_CUDA(cudaStreamSynchronize(stream));
    for (int i = 0; i < 3; ++i)
      if (S.st_streams[i]) PK_CUDA(cudaStreamSynchronize(S.st_streams[i]));
    if (S.st_q) cudaFree(S.st_q);
    if (S.st_t) cudaFree(S.st_t);
    if (S.st_v) cudaFree(S.st_v);
    if (S.st_s) cudaFree(S.st_s);
    S.st_q = S.st_t = S.st_v = nullptr;
    S.st_s = nullptr;
    const int64_t cap = std::max<int64_t>(B, S.st_cap);
    const int tcap = std::max(ts, S.st_tstride);
    PK_CUDA(cudaMalloc(&S.st_q, sizeof(float) * cap * m->nq));
    PK_CUDA(cudaMalloc(&S.st_t, sizeof(float) * cap * std::max(tcap, 1)));
    PK_CUDA(cudaMalloc(&S.st_v, sizeof(float) * cap * m->nv));
    PK_CUDA(cudaMalloc(&S.st_s, sizeof(int32_t) * cap));
    S.st_cap = cap;
    S.st_tstride = tcap;
  }
  if (!S.st_fork) {
    PK_CUDA(cudaEventCreateWithFlags(&S.st_fork, cudaEventDisableTiming));
    for (int i = 0; i < 3; ++i) {
      PK_CUDA(cudaStreamCreateWithFlags(&S.st_streams[i], cudaStreamNonBlocking));
      PK_CUDA(cudaEventCreateWithFlags(&S.st_join[i], cudaEventDisableTiming));
    }
  }
  static const int64_t chunk_env = env_int("PK_HOST_CHUNK", 32768);
  int64_t chunk = std::max<int64_t>(1024, chunk_env);
  if ((B + chunk - 1) / chunk > PkModel::kMaxChunks) chunk = (B + PkModel::kMaxChunks - 1) / PkModel::kMaxChunks;
  const int64_t nchunks = (B + chunk - 1) / chunk;
  // chunk k: rows [k chunk, k chunk + rows(k)) of the call
  auto rows = [&](int64_t k) { return std::min(chunk, B - k * chunk); };
  auto upload = [&](int64_t k, cudaStream_t s) {
    const int64_t b0 = k * chunk;
    PK_CUDA(cudaMemcpyAsync(S.st_q + b0 * m->nq, q_host + b0 * m->nq, sizeof(float) * rows(k) * m->nq,
                            cudaMemcpyHostToDevice, s));
    if (ts > 0)
      PK_CUDA(cudaMemcpyAsync(S.st_t + b0 * ts, targets_host + b0 * ts, sizeof(float) * rows(k) * ts,
                              cudaMemcpyHostToDevice, s));
    return 0;
  };
  // v / status of the chunk into v_out / status_out: the staging buffers or the caller's pinned ones
  auto solve = [&](int64_t k, float* v_out, int32_t* status_out, cudaStream_t s) {
    const int64_t b0 = k * chunk;
    return solve_device(m, pr, S.st_q + b0 * m->nq, S.st_t + b0 * ts, v_out + b0 * m->nv,
                        status_out ? status_out + b0 : nullptr, rows(k), s);
  };
  auto download = [&](int64_t k, cudaStream_t s) {
    const int64_t b0 = k * chunk;
    PK_CUDA(cudaMemcpyAsync(v_host + b0 * m->nv, S.st_v + b0 * m->nv, sizeof(float) * rows(k) * m->nv,
                            cudaMemcpyDeviceToHost, s));
    if (status_host)
      PK_CUDA(cudaMemcpyAsync(status_host + b0, S.st_s + b0, sizeof(int32_t) * rows(k), cudaMemcpyDeviceToHost, s));
    return 0;
  };
  // PK_HOST_DUPLEX=1: chunks round-robin over three internal streams, so that the H2D of
  // chunk k+1, the kernel of chunk k and the D2H of chunk k-1 overlap.  Default (0): the
  // two directions never overlap - all uploads on one stream, each kernel as soon as its
  // chunk has landed (hidden behind the next upload), all downloads after the last upload.
  // On the boxes measured, concurrent H2D + D2H run far below the sum of the one-way rates
  // (4.7 MiB up with 1.8 MiB down: 290 us together, 125 us back to back;
  // scripts/pcie_probe.py), so serialising the directions is the faster schedule.
  static const int duplex = env_int("PK_HOST_DUPLEX", 0);
  PK_CUDA(cudaEventRecord(S.st_fork, stream));
  if (duplex) {
    const int nstreams = (int)std::min<int64_t>(3, nchunks);
    for (int i = 0; i < nstreams; ++i) PK_CUDA(cudaStreamWaitEvent(S.st_streams[i], S.st_fork, 0));
    for (int64_t k = 0; k < nchunks; ++k) {
      cudaStream_t s = S.st_streams[k % nstreams];
      if (upload(k, s) || solve(k, S.st_v, S.st_s, s) || download(k, s)) return 1;
    }
    for (int i = 0; i < nstreams; ++i) {
      PK_CUDA(cudaEventRecord(S.st_join[i], S.st_streams[i]));
      PK_CUDA(cudaStreamWaitEvent(stream, S.st_join[i], 0));
    }
    return 0;
  }
  // PK_HOST_MODE=2 ("direct"): uploads staged, but the kernels write v / status straight into
  // the caller's pinned host buffers (posted PCIe writes, no download phase); staged downloads
  // when a result buffer is not pinned
  float* v_dev = nullptr;
  int32_t* s_dev = nullptr;
  if (host_mode == 2) {
    auto dev_ptr = [](const void* ptr) -> void* {
      if (!ptr) return nullptr;
      cudaPointerAttributes a{};
      if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess || a.type != cudaMemoryTypeHost) return nullptr;
      return a.devicePointer;
    };
    v_dev = static_cast<float*>(dev_ptr(v_host));
    s_dev = static_cast<int32_t*>(dev_ptr(status_host));
    cudaGetLastError();
  }
  const bool direct = v_dev && (s_dev || !status_host);
  cudaStream_t s_in = S.st_streams[0], s_k = S.st_streams[1], s_out = S.st_streams[2];
  for (int i = 0; i < (direct ? 2 : 3); ++i) PK_CUDA(cudaStreamWaitEvent(S.st_streams[i], S.st_fork, 0));
  // calls submitted on different caller streams share the staging buffers: the next upload
  // waits for the previous call's last download (a no-op for calls on one stream)
  if (S.st_busy) PK_CUDA(cudaStreamWaitEvent(s_in, S.st_join[2], 0));
  S.st_busy = true;
  for (int64_t k = 0; k < nchunks; ++k) {
    if (!S.st_in[k]) {
      PK_CUDA(cudaEventCreateWithFlags(&S.st_in[k], cudaEventDisableTiming));
      PK_CUDA(cudaEventCreateWithFlags(&S.st_kern[k], cudaEventDisableTiming));
    }
    if (upload(k, s_in)) return 1;
    PK_CUDA(cudaEventRecord(S.st_in[k], s_in));
    PK_CUDA(cudaStreamWaitEvent(s_k, S.st_in[k], 0));
    if (solve(k, direct ? v_dev : S.st_v, direct ? s_dev : S.st_s, s_k)) return 1;
    if (!direct) PK_CUDA(cudaEventRecord(S.st_kern[k], s_k));
  }
  if (!direct) {
    // downloads start once the last upload is through (st_in[nchunks-1] on the in-order s_in)
    PK_CUDA(cudaStreamWaitEvent(s_out, S.st_in[nchunks - 1], 0));
    for (int64_t k = 0; k < nchunks; ++k) {
      PK_CUDA(cudaStreamWaitEvent(s_out, S.st_kern[k], 0));
      if (download(k, s_out)) return 1;
    }
  }
  // the caller's stream resumes when everything is back; s_in / s_k are ordered before s_out
  PK_CUDA(cudaEventRecord(S.st_join[2], direct ? s_k : s_out));
  PK_CUDA(cudaStreamWaitEvent(stream, S.st_join[2], 0));
  return 0;
}

extern "C" int pk_build_ik_batched(const PkModel* m, const PkProblemDesc* prob, const float* q,
                                   const float* targets, float* H, float* c, float* h, int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  PkProblem pr;
  if (prepare_problem(m, prob, &pr, (cudaStream_t)stream, true)) return 1;
  const pk::DevProblem& P = pr.P;
  if (B == 0) return 0;
  if (!H) return fail("null H");
  pk::GenericArgs A{};
  A.q = q;
  A.targets = targets;
  A.H = H;
  A.c = c;
  A.h = h;
  A.task_index = -1;
  return launch_generic(m, pr.sel.generic_class, P, A, B, (cudaStream_t)stream);
}

extern "C" int pk_constraint_rows_batched(const PkModel* m, const PkProblemDesc* prob, const float* q,
                                          const float* targets, float* G, float* hG, float* E, float* f, float* lo,
                                          float* hi, int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  PkProblem pr;
  if (prepare_problem(m, prob, &pr, (cudaStream_t)stream, true)) return 1;
  if ((G == nullptr) != (hG == nullptr) || (E == nullptr) != (f == nullptr) || (lo == nullptr) != (hi == nullptr))
    return fail("G/hG, E/f and lo/hi come in pairs");
  if (B == 0) return 0;
  if (pr.P.target_stride > 0 && !targets) return fail("null targets");
  pk::GenericArgs A{};
  A.q = q;
  A.targets = targets;
  A.G = G;
  A.hG = hG;
  A.E = E;
  A.f = f;
  A.lo = lo;
  A.hi = hi;
  A.task_index = -1;
  return launch_generic(m, pr.sel.generic_class, pr.P, A, B, (cudaStream_t)stream);
}

extern "C" int pk_task_terms_batched(const PkModel* m, const PkProblemDesc* prob, int32_t task_index,
                                     const float* q, const float* targets, float* e, float* J, int64_t B,
                                     void* stream) {
  if (check_common(m, q, B)) return 1;
  PkProblem pr;
  if (prepare_problem(m, prob, &pr, (cudaStream_t)stream, true)) return 1;
  const pk::DevProblem& P = pr.P;
  if (task_index < 0 || task_index >= P.ntasks) return fail("task_index out of range");
  if (B == 0) return 0;
  pk::GenericArgs A{};
  A.q = q;
  A.targets = targets;
  A.e = e;
  A.J = J;
  A.task_index = task_index;
  A.task_k = pk::task_terms_rows(m->hm, P.tasks[task_index]);
  // H must be accumulated for the task loop to run; give the kernel no v/H outputs
  // but keep ntasks > 0 so the loop executes
  return launch_generic(m, pr.sel.generic_class, P, A, B, (cudaStream_t)stream);
}

extern "C" int pk_forward_kinematics_batched(const PkModel* m, const float* q, float* oMf, float* com,
                                             int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  if (B == 0) return 0;
  pk::GenericArgs A{};
  A.q = q;
  A.oMf = oMf;
  A.com = com;
  A.task_index = -1;
  return launch_generic(m, pk::generic_size_class(m->hm), pk::kinematics_problem(), A, B, (cudaStream_t)stream);
}

extern "C" int pk_frame_placements_batched(const PkModel* m, const int32_t* frames, int32_t num_frames, const float* q,
                                           float* oMf, float* com, int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  pk::FrameList L;
  const std::string e = pk::make_frame_list(m->hm, frames, num_frames, com != nullptr, &L);
  if (!e.empty()) return fail(e);
  if (B > 0 && num_frames > 0 && !oMf) return fail("null oMf");
  if (B == 0 || (num_frames == 0 && !com)) return 0;
  PK_CUDA(pk::launch_frame_placements(pk::generic_size_class(m->hm), m->dev, L, q, oMf, com, B, (cudaStream_t)stream));
  return launched();
}

extern "C" int pk_frame_placements_vjp_batched(const PkModel* m, const int32_t* frames, int32_t num_frames,
                                               const float* q, const float* grad_oMf, const float* grad_com,
                                               float* grad_q, int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  pk::FrameList L;
  const std::string e = pk::make_frame_list(m->hm, frames, num_frames, grad_com != nullptr, &L);
  if (!e.empty()) return fail(e);
  if (B > 0 && !grad_q) return fail("null grad_q");
  if (B == 0) return 0;
  PK_CUDA(pk::launch_frame_placements_vjp(pk::generic_size_class(m->hm), m->dev, L, q, grad_oMf, grad_com, grad_q, B,
                                          (cudaStream_t)stream));
  return launched();
}

extern "C" int pk_frame_jacobian_batched(const PkModel* m, int32_t frame, const float* q, float* J, int64_t B,
                                         void* stream) {
  if (check_common(m, q, B)) return 1;
  if (frame < 0 || frame >= m->nframes) return fail("frame index out of range");
  if (B == 0) return 0;
  pk::GenericArgs A{};
  A.q = q;
  A.Jf = J;
  A.jac_frame = frame;
  A.task_index = -1;
  return launch_generic(m, pk::generic_size_class(m->hm), pk::kinematics_problem(), A, B, (cudaStream_t)stream);
}

extern "C" int pk_integrate_batched(const PkModel* m, const float* q, const float* v, float dt, float* q_out,
                                    int64_t B, void* stream) {
  if (check_common(m, q, B)) return 1;
  if (B == 0) return 0;
  if (!v || !q_out) return fail("null v or q_out");
  return launch_rows(pk::integrate_kernel, B, 128, (cudaStream_t)stream, m->nq, m->nv, m->free_flyer, q, v, dt, q_out, B);
}
