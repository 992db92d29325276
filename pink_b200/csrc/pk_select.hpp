// Kernel selection shared by the CUDA library (pk_cabi.cu) and its host build (tests/hostsim):
// which kernel, instantiation and variant runs a (model, problem), and the dispatch from the
// run-time shape to the compile-time one.  Plain C++, no CUDA calls.
#pragma once

#include <algorithm>
#include <cassert>
#include <cstdint>
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

// CTAs of a launch of the PDL chain kernel (ik_chain_kernel<NJ, NFT, true>) that prefetch the
// whole grid's q and targets rows into L2 before their own loads; 0: no prefetch.  Under PDL the
// next grid's lowest-index CTAs take the slots this grid leaves free and sit there until their
// griddepcontrol.wait, while the rest of that grid starts together once this one retires; the
// prefetch lets that burst load from L2 instead of HBM.  `resident`: CTAs the device holds at
// once (occupancy per SM times the SM count).  Off when the grid is more than one wave (its
// later CTAs start as earlier ones end, not together) or when the inputs take more than a
// quarter of the L2 (they would evict one another, and whatever the running grid uses, before
// the burst reads them).  Otherwise one CTA per slot left free, at least one, at most 32 and at
// most the grid.
constexpr int kChainL2PrefetchMaxCtas = 32;
inline int chain_l2_prefetch_ctas(int64_t grid, int64_t resident, int64_t input_bytes, int64_t l2_bytes) {
  if (grid <= 0 || grid > resident || input_bytes > l2_bytes / 4) return 0;
  return (int)std::min<int64_t>({std::max<int64_t>(resident - grid, 1), kChainL2PrefetchMaxCtas, grid});
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

// The axes the separate-tolerance test (pk_converge_pose_tol_prepared) checks on the chain
// kernels, per frame slot: bit 6 f + r when frame task f is in `mask` and weighs row r (cost > 0),
// the rotation rows only for a finite orientation_tol.  Computed once per launch, so that the
// step tests no cost.
inline unsigned chain_axis_mask(const DevProblem& P, unsigned mask, float orientation_tol) {
  unsigned out = 0u;
  int f = 0;
  for (int t = 0; t < P.ntasks; ++t) {
    if (P.tasks[t].type != PK_TASK_FRAME) continue;
    if ((mask >> t) & 1u)
      for (int r = 0; r < 6; ++r)
        if (P.tasks[t].cost[r] > 0.f && (r < 3 || orientation_tol < INFINITY)) out |= 1u << (6 * f + r);
    ++f;
  }
  return out;
}

// Warps (instances) per CTA of the one-instance-per-warp tree kernels.
constexpr int kTreeWarpsPerBlock = 2;

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

// Goal-set and multi-start solves on joint trees (pk_converge_goalset_prepared): one instance per
// CTA, one member (goal, seed) per warp.  A warp's workspace is converge's, then the member's q
// (4-word aligned); after the workspaces of the S members (goals x seeds) come the group's
// slots, two rounds of S errors and S failed flags.  The CTA's dynamic shared memory is capped at
// kCtaSmemBytes, the opt-in limit of sm_90.
constexpr int kTreeMaxSeeds = 8;  // members per CTA
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

// Arguments of pk_converge_multistart_prepared beyond check_converge_args; "" when valid.  `what`
// names S in the messages (the members of a goal set, check_goalset_members).
inline std::string check_multistart_seeds(const Selection& sel, int S, const std::string& what = "num_seeds") {
  if (!valid_num_seeds(S)) return what + " must be 1, 2, 4, 8, 16 or 32";
  if (sel.path == kPathTree) {
    if (S > kTreeMaxSeeds) return what + " must be at most 8 on the tree kernel (one warp each in one CTA)";
    const size_t bytes = multistart_tree_layout(sel.plan).smem_bytes(S);
    if (bytes > kCtaSmemBytes)
      return what + " = " + std::to_string(S) + " needs " + std::to_string(bytes) +
             " B of shared memory on the tree kernel, more than one CTA's " + std::to_string(kCtaSmemBytes) + " B";
  }
  return "";
}

// Arguments of pk_converge_goalset_prepared beyond check_converge_args: G goals and S seeds, each
// a power of two, whose G S members form one multi-start group; "" when valid.
inline std::string check_goalset_members(const Selection& sel, int G, int S) {
  if (G == 1) return check_multistart_seeds(sel, S);
  if (!valid_num_seeds(G)) return "num_goals must be 1, 2, 4, 8, 16 or 32";
  if (!valid_num_seeds(S)) return "num_seeds must be 1, 2, 4, 8, 16 or 32";
  return check_multistart_seeds(sel, G * S, "num_goals * num_seeds");
}

// Problems pk_converge_vjp_prepared differentiates: tasks, the box limits and FloatingBaseVelocityLimit
// (velocity bounds cannot be active at a fixed point); "" when supported.  Barriers, equality
// constraints and AccelerationLimit would need rows of the KKT system the gradient does not carry.
inline std::string check_vjp_problem(const HostExtras& hx) {
  if (!hx.present) return "";
  if (hx.X.nbarriers) return "gradients of converge do not support barriers";
  if (hx.X.nconstraints) return "gradients of converge do not support equality constraints";
  if (hx.X.acc_enabled) return "gradients of converge do not support AccelerationLimit";
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
