// Kernel selection shared by the CUDA library (pk_cabi.cu) and its host build (tests/hostsim):
// which kernel, instantiation and variant runs a (model, problem), and the dispatch from the
// run-time shape to the compile-time one.  Plain C++, no CUDA calls.
#pragma once

#include <cassert>
#include <type_traits>

#include "pk_marshal.hpp"

namespace pk {

enum KernelPath : int { kPathChain = 0, kPathTree = 1, kPathGeneral = 2 };

struct SelectOptions {
  bool use_chain = true;  // false: the chain kernels are skipped (PK_FORCE_GENERIC)
  bool use_tree = true;   // false: the tree kernel is skipped (PK_FORCE_GENERIC, PK_TREE=0)
  int chain_lanes = 0;    // PK_CHAIN_LANES: lanes per instance of the sub-warp chain kernel, 0 = ik_chain_kernel
};

struct Selection {
  int path = kPathGeneral;
  int nj = 0, nft = 0;  // chains: joints and frame tasks, the <NJ, NFT> of the chain kernels
  TreePlan plan;        // trees: workspace layout of ik_tree_kernel / ik_tree_rollout_kernel
  int generic_class = 2;  // ik_generic_kernel instantiation, see with_generic
  int lanes = 0;          // sub-warp chain kernel's lanes per instance for the solve entries; 0: ik_chain_kernel
  bool pdl_row_fits = false;  // the targets row fits the PDL instantiation's copy of it
};

// Size class of the general path's per-thread arrays: 0 = <8, 8>, 1 = <30, 36>, 2 = <58, 64>.
inline int generic_size_class(const HostModel& m) {
  if (m.nv <= 8 && m.njoints <= 8) return 0;
  if (m.nv <= 36 && m.njoints <= 30) return 1;
  return 2;
}

// Lanes-per-instance variants of the sub-warp chain kernel: 1 and 2 at every <NJ, NFT>; 4 and 8
// (UR5-class study variants) at <6, 1> only.
constexpr bool coop_has_variant(int nj, int nft, int lanes) {
  return lanes == 1 || lanes == 2 || ((lanes == 4 || lanes == 8) && nj == 6 && nft == 1);
}

inline Selection select_kernel(const HostModel& m, const DevProblem& P, const HostExtras& hx, const SelectOptions& o) {
  Selection s;
  const bool chain = o.use_chain && chain_eligible(m, P, hx.present && !hx.box_only());
  bool tree_ok = false;
  s.plan = make_tree_plan(m, P, &tree_ok, hx.present ? &hx.X : nullptr);
  s.path = chain ? kPathChain : (o.use_tree && tree_ok) ? kPathTree : kPathGeneral;
  s.generic_class = generic_size_class(m);
  if (chain) {
    s.nj = m.njoints;
    for (int t = 0; t < P.ntasks; ++t) s.nft += P.tasks[t].type == PK_TASK_FRAME;
    s.lanes = coop_has_variant(s.nj, s.nft, o.chain_lanes) ? o.chain_lanes : 0;
    s.pdl_row_fits = P.target_stride <= chain_row_words(s.nj, s.nft);
  }
  return s;
}

// A task mask of pk_converge_prepared (bit t: P.tasks[t]) in the chain kernels' slots: the frame
// tasks are compacted into ft[] in task order (bit k: ft[k]), the posture task is bit nft.
inline unsigned chain_task_mask(const DevProblem& P, unsigned mask, int nft) {
  unsigned out = 0u;
  int f = 0;
  for (int t = 0; t < P.ntasks; ++t) {
    const bool on = (mask >> t) & 1u;
    if (P.tasks[t].type == PK_TASK_FRAME) {
      if (on) out |= 1u << f;
      ++f;
    } else if (on) {
      out |= 1u << nft;
    }
  }
  return out;
}

// Solve to a tolerance on joint trees (pk_converge_prepared): a warp's workspace is the plan's
// words, then the step's v (4-word aligned).
struct ConvergeTreeLayout {
  TreePlan plan;  // plan.words: the whole per-warp workspace
  int o_v;
};
inline ConvergeTreeLayout converge_tree_layout(const TreePlan& plan) {
  ConvergeTreeLayout T{plan, plan.words};
  T.plan.words += (plan.nv + 3) & ~3;
  return T;
}

// Multi-start on joint trees (pk_converge_multistart_prepared): one target per CTA, one seed per
// warp.  A warp's workspace is converge's, then the seed's q (4-word aligned); after the S
// workspaces come the group's slots, two rounds of S errors and S failed flags.  The CTA's
// dynamic shared memory is capped at kCtaSmemBytes, the opt-in limit of sm_90.
constexpr int kTreeMaxSeeds = 8;
constexpr size_t kCtaSmemBytes = 227 * 1024;
struct MultistartTreeLayout : ConvergeTreeLayout {
  int o_q;
  size_t smem_bytes(int S) const { return ((size_t)plan.words * S + 4 * (size_t)S) * 4; }
};
inline MultistartTreeLayout multistart_tree_layout(const TreePlan& plan) {
  MultistartTreeLayout T{converge_tree_layout(plan), 0};
  T.o_q = T.plan.words;
  T.plan.words += (plan.nq + 3) & ~3;
  return T;
}

// Arguments of pk_converge_multistart_prepared beyond check_converge_args; "" when valid.
inline std::string check_multistart_seeds(const Selection& sel, int S) {
  if (!valid_num_seeds(S)) return "num_seeds must be 1, 2, 4, 8, 16 or 32";
  if (sel.path == kPathTree) {
    if (S > kTreeMaxSeeds) return "num_seeds must be at most 8 on the tree kernel (one warp per seed in one CTA)";
    const size_t bytes = multistart_tree_layout(sel.plan).smem_bytes(S);
    if (bytes > kCtaSmemBytes)
      return "num_seeds = " + std::to_string(S) + " needs " + std::to_string(bytes) +
             " B of shared memory on the tree kernel, more than one CTA's " + std::to_string(kCtaSmemBytes) + " B";
  }
  return "";
}

// f(std::integral_constant<int, N>) for the run-time value: the chain kernels' joint count
// (2..7, chain_eligible), frame-task count (0..2), sub-warp lanes (a coop_has_variant), the
// general path's <NJMAX, NVMAX>.
template <class F>
decltype(auto) with_nj(int nj, F&& f) {
  assert(nj >= 2 && nj <= 7);
  switch (nj) {
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 6: return f(std::integral_constant<int, 6>{});
    default: return f(std::integral_constant<int, 7>{});
  }
}

template <class F>
decltype(auto) with_nft(int nft, F&& f) {
  assert(nft >= 0 && nft <= kChainMaxFrameTasks);
  switch (nft) {
    case 0: return f(std::integral_constant<int, 0>{});
    case 1: return f(std::integral_constant<int, 1>{});
    default: return f(std::integral_constant<int, 2>{});
  }
}

// f(<NJ>, <NFT>) for a chain selection
template <class F>
decltype(auto) with_chain(const Selection& sel, F&& f) {
  return with_nj(sel.nj, [&](auto nj) { return with_nft(sel.nft, [&](auto nft) { return f(nj, nft); }); });
}

template <int NJ, int NFT, class F>
decltype(auto) with_lanes(int lanes, F&& f) {
  assert(coop_has_variant(NJ, NFT, lanes));
  if constexpr (coop_has_variant(NJ, NFT, 8))
    if (lanes == 8) return f(std::integral_constant<int, 8>{});
  if constexpr (coop_has_variant(NJ, NFT, 4))
    if (lanes == 4) return f(std::integral_constant<int, 4>{});
  if (lanes == 2) return f(std::integral_constant<int, 2>{});
  return f(std::integral_constant<int, 1>{});
}

template <class F>
decltype(auto) with_generic(int size_class, F&& f) {
  if (size_class == 0) return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 8>{});
  if (size_class == 1) return f(std::integral_constant<int, 30>{}, std::integral_constant<int, 36>{});
  return f(std::integral_constant<int, PK_MAX_JOINTS>{}, std::integral_constant<int, PK_MAX_NV>{});
}

}  // namespace pk
