// CPU build of the kernel bodies (pink_b200/csrc) for the test suite ONLY: lets
// `pytest -m "not gpu"` exercise the exact fp32 arithmetic and control flow of the
// CUDA kernels against the fp64 oracle on machines without a GPU.  Each entry makes the
// problem, selects (pk_select.hpp) and loops over the instances with the per-instance body
// the selected kernel calls.  It is never loaded by the product package (pink_b200/_cabi.py
// loads libpink_b200.so and nothing else) and is not a fallback.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/pink_b200.h"
#include "../../pink_b200/csrc/pk_select.hpp"
#include "../../pink_b200/csrc/pk_dualqp.cuh"

namespace {
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return 1; }

// make_dev_problem + host image of the optional parts, wired through P.ext
std::string make_problem(const pk::HostModel& hm, const PkProblemDesc* prob, pk::DevProblem* P, pk::HostExtras* hx) {
  const std::string e = pk::make_dev_problem(hm, prob, P, hx);
  if (e.empty() && hx->present) P->ext = &hx->X;
  return e;
}

// The CUDA library's kernel selection (pk_select.hpp) for `path`: 0 the library's default options,
// 1 PK_FORCE_GENERIC=1, 2 without the chain kernels (the tree kernel body on a chain),
// 11 / 12 / 14 / 18 PK_CHAIN_LANES = 1 / 2 / 4 / 8 (the problem must take a chain kernel) when
// `sub_warp`, the tree kernel or the general path otherwise.  sel_out: path (pk::KernelPath), nj,
// nft, the general path's <NJMAX, NVMAX>, lanes, PDL row fits, tree task rows K.  Returns the
// error of a path the problem does not fit, or "".
std::string select(const pk::HostModel& hm, const pk::DevProblem& P, const pk::HostExtras& hx, int path,
                   bool sub_warp, int* sel_out, pk::Selection* sel) {
  const bool lanes = sub_warp && path > 10;
  pk::SelectOptions o;
  o.use_chain = path == 0 || lanes;
  o.use_tree = path != 1;
  o.chain_lanes = lanes ? path - 10 : 0;
  const pk::Selection& s = *sel = pk::select_kernel(hm, P, hx, o);
  const int report[] = {s.path, s.nj, s.nft, 0, 0, s.lanes, s.pdl_row_fits, s.plan.K};
  std::memcpy(sel_out, report, sizeof(report));
  pk::with_generic(s.generic_class, [&](auto nj, auto nv) { sel_out[3] = nj; sel_out[4] = nv; });
  if (lanes && s.path != pk::kPathChain) return "problem does not fit the chain kernel";
  if (path == 2 && s.path != pk::kPathTree) return "problem does not fit the tree kernel";
  return "";
}

// A tree kernel's workspace of `words` floats in W, 8-byte aligned: the dual method keeps doubles in it.
float* tree_workspace(std::vector<float>& W, int words) {
  W.assign(words + 8, 0.f);
  float* p = W.data();
  return ((uintptr_t)p & 7) != 0 ? p + 1 : p;
}

// The chain kernel a chain selection names, at its <NJ, NFT>: chain(nj, nft, C) with the
// thread-per-instance kernel's parameter block, or coop(nj, nft, G, C, jc) with the sub-warp
// kernel's (a group of lanes emulated by loops).
template <class Chain, class Coop>
void with_chain_kernel(const pk::HostModel& hm, const pk::DevProblem& P, const pk::Selection& sel, Chain chain,
                       Coop coop) {
  pk::with_chain(sel, [&](auto nj, auto nft) {
    constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
    if (!sel.lanes) {
      pk::ChainParams<NJ> C;
      pk::make_chain_params<NJ>(hm, P, &C, P.ext);
      return chain(nj, nft, C);
    }
    pk::with_lanes<NJ, NFT>(sel.lanes, [&](auto lanes) {
      constexpr int L = decltype(lanes)::value;
      typename pk::CoopStep<NJ, NFT, L>::Params C;
      pk::make_coop_params<NJ, L>(hm, P, &C, P.ext);
      coop(nj, nft, pk::Group<L>{}, C, [&](int j) -> const pk::CoopJoint& { return C.joint[j]; });
    });
  });
}

// ik_generic_kernel's body at the instantiation the CUDA library launches for this model
void run_generic(const pk::HostModel& hm, const pk::DevProblem& P, const pk::GenericArgs& A, int64_t B) {
  const pk::DevModel M = hm.host_view();
  pk::with_generic(pk::generic_size_class(hm), [&](auto nj, auto nv) {
    static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
    for (int64_t i = 0; i < B; ++i)
      G.step(M, P, A.q + i * M.nq, A.targets ? A.targets + i * (int64_t)P.target_stride : nullptr,
             pk::generic_out(M, A, i));
  });
}

// One multi-start group of S seeds.  error(j) -> err(q_j); advance(j) -> the step of seed j, false
// when it fails (q_j unchanged), its status ORed into st_all[j].  Returns the winner; e, steps out.
template <class Error, class Advance>
int run_group(int S, float tol, int max_steps, Error error, Advance advance, std::vector<float>& e, int& steps) {
  std::vector<char> failed(S, 0);
  int s = 0;
  for (;; ++s) {
    bool hit = false, all_failed = true;
    for (int j = 0; j < S; ++j) {
      if (!failed[j]) e[j] = error(j);
      hit = hit || e[j] <= tol;
      all_failed = all_failed && failed[j];
    }
    if (hit || s == max_steps || all_failed) break;
    for (int j = 0; j < S; ++j)
      if (!failed[j] && !advance(j)) failed[j] = 1;
  }
  steps = s;
  int w = 0;
  for (int j = 1; j < S; ++j)
    if (pk::seed_before(e[j], j, e[w], w)) w = j;
  return w;
}
}  // namespace

extern "C" {

const char* hs_last_error(void) { return g_err.c_str(); }

int hs_model_create(const PkModelDesc* d, void** out) {
  pk::HostModel* m = new pk::HostModel();
  const std::string e = pk::build_host_model(d, m);
  if (!e.empty()) { delete m; return fail(e); }
  *out = m;
  return 0;
}
void hs_model_destroy(void* m) { delete (pk::HostModel*)m; }

// The kernel body the CUDA library's selection names for this problem; path and sel_out: see select.
int hs_solve_ik(void* model, const PkProblemDesc* prob, const float* q, const float* targets, float* v,
                int32_t* status, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, true, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  if (sel.path == pk::kPathChain) {
    with_chain_kernel(
        hm, P, sel,
        [&](auto nj, auto nft, const auto& C) {
          constexpr int NJ = decltype(nj)::value;
          for (int64_t i = 0; i < B; ++i) {
            float qi[NJ], vi[NJ];
            for (int k = 0; k < NJ; ++k) qi[k] = q[i * NJ + k];
            int st = 0;
            pk::ik_step_chain<NJ, decltype(nft)::value>(C, qi, targets + i * (int64_t)P.target_stride, vi, st);
            for (int k = 0; k < NJ; ++k) v[i * NJ + k] = vi[k];
            if (status) status[i] = st;
          }
        },
        [&](auto nj, auto nft, auto G, const auto& C, auto jc) {
          for (int64_t i = 0; i < B; ++i)
            pk::coop_instance<decltype(nj)::value, decltype(nft)::value>(G, C, jc, q, targets, v, status, B, 1, nullptr,
                                                                         pk::Trajectory{}, i);
        });
  } else if (sel.path == pk::kPathTree) {
    const pk::DevModel M = hm.host_view();
    std::vector<float> W;
    float* Wp = tree_workspace(W, sel.plan.words);
    for (int64_t i = 0; i < B; ++i) pk::TreeStep::solve_instance(M, P, sel.plan, q, targets, Wp, v, status, i);
  } else {
    pk::GenericArgs A{};
    A.q = q; A.targets = targets; A.v = v; A.status = status; A.task_index = -1;
    run_generic(hm, P, A, B);
  }
  return 0;
}

// Trajectory rollout (pk_rollout_trajectory_prepared) with the loop of the body the selection names:
// rollout_chain, rollout_coop (path 11 / 12 / 14 / 18), TreeStep::rollout or rollout_generic.
// targets [B][target_stride] for step 0, step s target_step floats further; q_traj / v_traj /
// status_traj: the step-major records, or null.  path and sel_out as hs_solve_ik.
int hs_rollout(void* model, const PkProblemDesc* prob, const float* q, const float* targets, int64_t target_step,
               int n_steps, float* q_out, float* v, int32_t* status, float* q_traj, float* v_traj,
               int32_t* status_traj, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, true, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  const pk::Trajectory T{target_step, q_traj, v_traj, status_traj};
  const pk::DevModel M = hm.host_view();
  if (sel.path == pk::kPathChain) {
    with_chain_kernel(
        hm, P, sel,
        [&](auto nj, auto nft, const auto& C) {
          constexpr int NJ = decltype(nj)::value;
          for (int64_t i = 0; i < B; ++i) {
            float qi[NJ], vi[NJ];
            for (int k = 0; k < NJ; ++k) qi[k] = q[i * NJ + k];
            const int st_all = pk::rollout_chain<NJ, decltype(nft)::value, true>(
                C, qi, targets + i * (int64_t)P.target_stride, vi, n_steps, true, 0, T, B, i);
            for (int k = 0; k < NJ; ++k) { q_out[i * NJ + k] = qi[k]; v[i * NJ + k] = vi[k]; }
            if (status) status[i] = st_all;
          }
        },
        [&](auto nj, auto nft, auto G, const auto& C, auto jc) {
          for (int64_t i = 0; i < B; ++i)
            pk::coop_instance<decltype(nj)::value, decltype(nft)::value>(G, C, jc, q, targets, v, status, B, n_steps,
                                                                         q_out, T, i);
        });
  } else if (sel.path == pk::kPathTree) {
    std::vector<float> W;
    float* Wp = tree_workspace(W, sel.plan.words);
    for (int64_t i = 0; i < B; ++i)
      pk::TreeStep::rollout_instance(M, P, sel.plan, q, targets, n_steps, q_out, Wp, v, status, T, B, i);
  } else {
    pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
      static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
      for (int64_t i = 0; i < B; ++i) pk::rollout_generic_instance(G, M, P, q, targets, n_steps, q_out, v, status, T, B, i);
    });
  }
  return 0;
}

// Solve to a tolerance (pk_converge_prepared) with the converge loop of the body the selection
// names: converge_chain (always the thread-per-instance kernel), TreeStep::converge or
// converge_generic.  path and sel_out as hs_solve_ik.  q_out may alias q.
int hs_converge(void* model, const PkProblemDesc* prob, const float* q, const float* targets, uint32_t mask,
                float tol, int max_steps, float* q_out, float* err, int32_t* steps, int32_t* status, int64_t B,
                int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  const std::string aerr = pk::check_converge_args(P, mask, tol, max_steps);
  if (!aerr.empty()) return fail(aerr);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, true, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  const pk::DevModel M = hm.host_view();
  if (sel.path == pk::kPathChain) {
    const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
    pk::with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value;
      pk::ChainParams<NJ> C;
      pk::make_chain_params<NJ>(hm, P, &C, P.ext);
      for (int64_t i = 0; i < B; ++i)
        pk::converge_chain_instance<NJ, decltype(nft)::value>(C, q, targets, emask, tol, max_steps, q_out, err, steps,
                                                              status, i);
    });
  } else if (sel.path == pk::kPathTree) {
    const pk::ConvergeTreeLayout T = pk::converge_tree_layout(sel.plan);
    std::vector<float> W;
    float* Wp = tree_workspace(W, T.plan.words);
    for (int64_t i = 0; i < B; ++i)
      pk::TreeStep::converge_instance(M, P, T.plan, T.o_v, q, targets, mask, tol, max_steps, q_out, Wp, err, steps,
                                      status, i);
  } else {
    pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
      static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
      for (int64_t i = 0; i < B; ++i)
        pk::converge_generic_instance(G, M, P, q, targets, mask, tol, max_steps, q_out, err, steps, status, i);
    });
  }
  return 0;
}

// Multi-start solve to a tolerance (pk_converge_multistart_prepared) with the bodies the selection
// names; q_seeds [B S][nq], the outputs [B].  path as hs_converge without the sub-warp kernel.
// A host thread cannot suspend inside a step body to wait for the other seeds of its group, so
// each round runs in two passes over the group: first every seed's error, from the step body
// with its stop forced (it returns before the QP); then the group's decision, and the step of
// every seed that goes on.  The bodies (ChainStep::assemble<true> with converge_chain_advance,
// TreeStep::run<true>, Generic::step<true>) and the winner's order (seed_before) are those the
// CUDA library runs.
int hs_converge_multistart(void* model, const PkProblemDesc* prob, const float* q_seeds, int S,
                           const float* targets, uint32_t mask, float tol, int max_steps, float* q_out, float* err,
                           int32_t* seed, int32_t* steps, int32_t* status, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  const std::string aerr = pk::check_converge_args(P, mask, tol, max_steps);
  if (!aerr.empty()) return fail(aerr);
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, false, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  const std::string kerr = pk::check_multistart_seeds(sel, S);
  if (!kerr.empty()) return fail(kerr);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  const pk::DevModel M = hm.host_view();
  const int nq = hm.nq;
  // the forced stop of the first pass, and the test of the second (never stops: err >= 0)
  const pk::ConvergeTest probe{mask, tol, true, 0.f, false, 0};
  const pk::ConvergeTest go{mask, -INFINITY, false, 0.f, false, 0};
  std::vector<float> qs((size_t)S * nq), es(S);
  std::vector<int> st_all(S);
  for (int64_t b = 0; b < B; ++b) {
    const float* trow = targets ? targets + b * (int64_t)P.target_stride : nullptr;
    std::memcpy(qs.data(), q_seeds + b * S * nq, sizeof(float) * S * nq);
    std::fill(st_all.begin(), st_all.end(), 0);
    int w = 0, n = 0;
    if (sel.path == pk::kPathChain) {
      const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
      pk::with_chain(sel, [&](auto nj, auto nft) {
        constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
        pk::ChainParams<NJ> C;
        pk::make_chain_params<NJ>(hm, P, &C, P.ext);
        auto qj = [&](int j) -> float(&)[NJ] { return *reinterpret_cast<float(*)[NJ]>(qs.data() + j * NJ); };
        auto error = [&](int j) {
          pk::ChainStep<NJ, NFT> Cs;
          bool skip;
          float ej;
          Cs.template assemble<true>(C, qj(j), trow, skip, emask, &ej);
          return ej;
        };
        auto advance = [&](int j) {
          pk::ChainStep<NJ, NFT> Cs;
          bool skip;
          float ej;
          const int st = Cs.template assemble<true>(C, qj(j), trow, skip, emask, &ej);
          return pk::converge_chain_advance(C, Cs, st, skip, qj(j), st_all[j], 0);
        };
        w = run_group(S, tol, max_steps, error, advance, es, n);
      });
    } else if (sel.path == pk::kPathTree) {
      const pk::TreePlan& L = sel.plan;
      std::vector<float> W, v(hm.nv);
      float* Wp = tree_workspace(W, L.words);
      auto error = [&](int j) {
        pk::ConvergeTest ct = probe;
        pk::TreeStep::run<true>(M, P, L, qs.data() + j * nq, trow, Wp, v.data(), nullptr, &ct);
        return ct.err;
      };
      auto advance = [&](int j) {
        float* q = qs.data() + j * nq;
        pk::ConvergeTest ct = go;
        pk::TreeStep::run<true>(M, P, L, q, trow, Wp, v.data(), nullptr, &ct);
        st_all[j] |= ct.status;
        if (pk::step_failed(st_all[j], P.safety_break)) return false;
        pk::integrate_configuration(nq, M.free_flyer, q, v.data(), P.dt, q);
        return true;
      };
      w = run_group(S, tol, max_steps, error, advance, es, n);
    } else {
      pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
        static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
        float v[decltype(nv)::value];
        int32_t st = 0;
        pk::GenericOut out{};
        out.v = v;
        out.status = &st;
        out.task_index = -1;
        auto error = [&](int j) {
          pk::ConvergeTest ct = probe;
          G.template step<true>(M, P, qs.data() + j * nq, trow, out, &ct);
          return ct.err;
        };
        auto advance = [&](int j) {
          float* q = qs.data() + j * nq;
          pk::ConvergeTest ct = go;
          G.template step<true>(M, P, q, trow, out, &ct);
          st_all[j] |= st;
          if (pk::step_failed(st_all[j], P.safety_break)) return false;
          pk::integrate_configuration(nq, M.free_flyer, q, v, P.dt, q);
          return true;
        };
        w = run_group(S, tol, max_steps, error, advance, es, n);
      });
    }
    std::memcpy(q_out + b * nq, qs.data() + w * nq, sizeof(float) * nq);
    if (err) err[b] = es[w];
    if (seed) seed[b] = w;
    if (steps) steps[b] = n;
    if (status) status[b] = st_all[w];
  }
  return 0;
}

int hs_build_ik(void* model, const PkProblemDesc* prob, const float* q, const float* targets, float* H, float* c,
                float* h, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  pk::GenericArgs A{};
  A.q = q; A.targets = targets; A.H = H; A.c = c; A.h = h; A.task_index = -1;
  run_generic(hm, P, A, B);
  return 0;
}

int hs_constraint_rows(void* model, const PkProblemDesc* prob, const float* q, const float* targets, float* G,
                       float* hG, float* E, float* f, float* lo, float* hi, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  pk::GenericArgs A{};
  A.q = q; A.targets = targets; A.G = G; A.hG = hG; A.E = E; A.f = f; A.lo = lo; A.hi = hi; A.task_index = -1;
  run_generic(hm, P, A, B);
  return 0;
}

int hs_task_terms(void* model, const PkProblemDesc* prob, int task_index, const float* q, const float* targets,
                  float* eo, float* J, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  if (task_index < 0 || task_index >= P.ntasks) return fail("task_index out of range");
  pk::GenericArgs A{};
  A.q = q; A.targets = targets; A.e = eo; A.J = J; A.task_index = task_index;
  A.task_k = pk::task_terms_rows(hm, P.tasks[task_index]);
  run_generic(hm, P, A, B);
  return 0;
}

int hs_forward_kinematics(void* model, const float* q, float* oMf, float* com, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::GenericArgs A{};
  A.q = q; A.oMf = oMf; A.com = com; A.task_index = -1;
  run_generic(hm, pk::kinematics_problem(), A, B);
  return 0;
}

int hs_frame_jacobian(void* model, int frame, const float* q, float* J, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  if (frame < 0 || frame >= hm.nframes) return fail("frame index out of range");
  pk::GenericArgs A{};
  A.q = q; A.Jf = J; A.jac_frame = frame; A.task_index = -1;
  run_generic(hm, pk::kinematics_problem(), A, B);
  return 0;
}

// q (+) v dt with the body of integrate_kernel (pk_math.cuh)
int hs_integrate(void* model, const float* q, const float* v, float dt, float* q_out, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  for (int64_t i = 0; i < B; ++i)
    pk::integrate_configuration(hm.nq, hm.free_flyer, q + i * hm.nq, v + i * hm.nv, dt, q_out + i * hm.nq);
  return 0;
}

// Direct access to the dual active-set QP (pk_dualqp.cuh) for unit tests:
//   min 1/2 |A x + b|^2 + 1/2 sum (d_i x_i + beta_i)^2,  lo <= x <= hi,  G x <= h,  E x = f
// A[K][n], G[p][n], E[meq][n] row-major; returns the solver's status bits.
int hs_dual_qp(int K, int n, int p, int meq, const float* A, const float* b, const float* d, const float* beta,
               const float* lo, const float* hi, const float* G, const float* h, const float* E, const float* f,
               float* x) {
  using QP = pk::DualQP<pk::kGenericMaxRows, PK_MAX_NV, PK_MAX_INEQ_ROWS, PK_MAX_EQ_ROWS>;
  if (K > pk::kGenericMaxRows || n > PK_MAX_NV || p > PK_MAX_INEQ_ROWS || meq > PK_MAX_EQ_ROWS) return -1;
  static thread_local float Aa[pk::kGenericMaxRows][PK_MAX_NV], Ga[PK_MAX_INEQ_ROWS][PK_MAX_NV], Ea[PK_MAX_EQ_ROWS][PK_MAX_NV];
  for (int r = 0; r < K; ++r) for (int c = 0; c < n; ++c) Aa[r][c] = A[r * n + c];
  for (int r = 0; r < p; ++r) for (int c = 0; c < n; ++c) Ga[r][c] = G[r * n + c];
  for (int r = 0; r < meq; ++r) for (int c = 0; c < n; ++c) Ea[r][c] = E[r * n + c];
  QP::Problem P{Aa, b, d, beta, lo, hi, Ga, h, Ea, f, K, n, p, meq};
  float xs[PK_MAX_NV];
  const int st = QP::run(P, xs);
  for (int i = 0; i < n; ++i) x[i] = xs[i];
  return st;
}

// Direct access to the warp-cooperative dual QP (pk_treedual.cuh) for unit tests; same
// problem as hs_dual_qp without equalities.
int hs_tree_dual_qp(int K, int n, int p, int meq, const float* A, const float* b, const float* d, const float* beta,
                    const float* lo, const float* hi, const float* G, const float* h, const float* E, const float* f,
                    float* x) {
  pk::TreePlan L;
  memset(&L, 0, sizeof(L));
  L.nj = 1; L.nq = n; L.nv = n; L.K = K; L.p = p; L.meq = meq; L.npairs = 0;
  pk::tree_layout(L, 1, 0);
  std::vector<float> W;
  float* Wp = tree_workspace(W, L.words);
  for (int r = 0; r < K; ++r) {
    for (int c = 0; c < n; ++c) Wp[L.o_A + r * L.lda + c] = A[r * n + c];
    Wp[L.o_b + r] = b[r];
  }
  for (int r = 0; r < p; ++r) {
    for (int c = 0; c < n; ++c) Wp[L.o_G + r * L.lda + c] = G[r * n + c];
    Wp[L.o_hg + r] = h[r];
  }
  for (int r = 0; r < meq; ++r) {
    for (int c = 0; c < n; ++c) Wp[L.o_E + r * L.lda + c] = E[r * n + c];
    Wp[L.o_fe + r] = f[r];
  }
  for (int i = 0; i < n; ++i) {
    Wp[L.o_d + i] = d[i]; Wp[L.o_beta + i] = beta[i]; Wp[L.o_lo + i] = lo[i]; Wp[L.o_hi + i] = hi[i];
  }
  const int st = pk::TreeDual::solve(Wp, L);
  for (int i = 0; i < n; ++i) x[i] = Wp[L.o_x + i];
  return st;
}
}
