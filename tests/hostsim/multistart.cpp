// CPU build of the multi-start loop (pk_converge_multistart_prepared, pk_multistart.cuh) for the
// test suite ONLY, next to converge.cpp and built the same way (tests/hostsim/multistart.py).
// A host thread cannot suspend inside a step body to wait for the other seeds of its group, so
// each round runs in two passes over the group: first every seed's error, from the step body
// with its stop forced (it returns before the QP); then the group's decision, and the step of
// every seed that goes on.  The bodies (ChainStep::assemble<true> with converge_chain_advance,
// TreeStep::run<true>, Generic::step<true>), the winner's order (seed_before) and the selection
// (pk_select.hpp) are those the CUDA library runs.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/pink_b200.h"
#include "../../pink_b200/csrc/pk_select.hpp"

namespace {
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return 1; }

std::string make_problem(const pk::HostModel& hm, const PkProblemDesc* prob, pk::DevProblem* P, pk::HostExtras* hx) {
  const std::string e = pk::make_dev_problem(hm, prob, P, hx);
  if (e.empty() && hx->present) P->ext = &hx->X;
  return e;
}

// One group of S seeds.  error(j) -> err(q_j); advance(j) -> the step of seed j, false when it
// fails (q_j unchanged), its status ORed into st_all[j].  Returns the winner; e, steps out.
template <class Error, class Advance>
int run_group(int S, float tol, int max_steps, Error error, Advance advance, std::vector<float>& e,
              std::vector<int>& st_all, int& steps) {
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

const char* hs_multistart_last_error(void) { return g_err.c_str(); }

// Multi-start solve to a tolerance (pk_converge_multistart_prepared) with the bodies the selection
// names; q_seeds [B S][nq], the outputs [B].  path and sel_out as hs_converge.
int hs_converge_multistart(const PkModelDesc* model, const PkProblemDesc* prob, const float* q_seeds, int S,
                           const float* targets, uint32_t mask, float tol, int max_steps, float* q_out, float* err,
                           int32_t* seed, int32_t* steps, int32_t* status, int64_t B, int path, int* sel_out) {
  pk::HostModel hm;
  const std::string me = pk::build_host_model(model, &hm);
  if (!me.empty()) return fail(me);
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  const std::string aerr = pk::check_converge_args(P, mask, tol, max_steps);
  if (!aerr.empty()) return fail(aerr);
  pk::SelectOptions o;
  o.use_chain = path == 0;
  o.use_tree = path != 1;
  const pk::Selection sel = pk::select_kernel(hm, P, hx, o);
  const int report[] = {sel.path, sel.nj, sel.nft, 0, 0, sel.lanes, sel.pdl_row_fits, sel.plan.K};
  std::memcpy(sel_out, report, sizeof(report));
  pk::with_generic(sel.generic_class, [&](auto nj, auto nv) { sel_out[3] = nj; sel_out[4] = nv; });
  if (path == 2 && sel.path != pk::kPathTree) return fail("problem does not fit the tree kernel");
  const std::string serr = pk::check_multistart_seeds(sel, S);
  if (!serr.empty()) return fail(serr);
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
      pk::with_nj(sel.nj, [&](auto nj) {
        constexpr int NJ = decltype(nj)::value;
        pk::ChainParams<NJ> C;
        pk::make_chain_params<NJ>(hm, P, &C, P.ext);
        const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
        pk::with_nft(sel.nft, [&](auto nft) {
          constexpr int NFT = decltype(nft)::value;
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
          w = run_group(S, tol, max_steps, error, advance, es, st_all, n);
        });
      });
    } else if (sel.path == pk::kPathTree) {
      const pk::TreePlan& L = sel.plan;
      std::vector<float> W(L.words + 8);
      float* Wp = W.data();
      if (((uintptr_t)Wp & 7) != 0) ++Wp;  // the dual method keeps doubles in the workspace
      std::vector<float> v(hm.nv);
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
      w = run_group(S, tol, max_steps, error, advance, es, st_all, n);
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
        w = run_group(S, tol, max_steps, error, advance, es, st_all, n);
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

}
