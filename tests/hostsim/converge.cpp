// CPU build of the converge loops of the kernel bodies (converge_chain in pk_chain.cuh,
// TreeStep::converge in pk_tree.cuh, converge_generic in pk_generic.cuh) for the test suite
// ONLY, next to hostsim.cpp and built the same way (tests/hostsim/converge.py).  It runs the
// loop at the instantiation the CUDA library's selection (pk_select.hpp) names, so that
// `pytest -m "not gpu"` checks pk_converge_prepared's arithmetic and control flow without a GPU.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/pink_b200.h"
#include "../../pink_b200/csrc/pk_select.hpp"

namespace {
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return 1; }

// make_dev_problem + host image of the optional parts, wired through P.ext (as hostsim.cpp)
std::string make_problem(const pk::HostModel& hm, const PkProblemDesc* prob, pk::DevProblem* P, pk::HostExtras* hx) {
  const std::string e = pk::make_dev_problem(hm, prob, P, hx);
  if (e.empty() && hx->present) P->ext = &hx->X;
  return e;
}
}  // namespace

extern "C" {

const char* hs_converge_last_error(void) { return g_err.c_str(); }

// Solve to a tolerance (pk_converge_prepared) with the converge loop of the body the selection
// names: converge_chain (always the thread-per-instance kernel), TreeStep::converge or
// converge_generic.  path and sel_out as hs_solve_ik (hostsim.cpp).  q_out may alias q.
int hs_converge(const PkModelDesc* model, const PkProblemDesc* prob, const float* q, const float* targets, uint32_t mask, float tol,
                int max_steps, float* q_out, float* err, int32_t* steps, int32_t* status, int64_t B, int path,
                int* sel_out) {
  pk::HostModel hm;
  const std::string me = pk::build_host_model(model, &hm);
  if (!me.empty()) return fail(me);
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  const std::string aerr = pk::check_converge_args(P, mask, tol, max_steps);
  if (!aerr.empty()) return fail(aerr);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  pk::SelectOptions o;
  o.use_chain = path == 0 || path > 10;
  o.use_tree = path != 1;
  o.chain_lanes = path > 10 ? path - 10 : 0;
  const pk::Selection sel = pk::select_kernel(hm, P, hx, o);
  const int report[] = {sel.path, sel.nj, sel.nft, 0, 0, sel.lanes, sel.pdl_row_fits, sel.plan.K};
  std::memcpy(sel_out, report, sizeof(report));
  pk::with_generic(sel.generic_class, [&](auto nj, auto nv) { sel_out[3] = nj; sel_out[4] = nv; });
  if (path > 10 && sel.path != pk::kPathChain) return fail("problem does not fit the chain kernel");
  if (path == 2 && sel.path != pk::kPathTree) return fail("problem does not fit the tree kernel");
  const pk::DevModel M = hm.host_view();
  const int nq = hm.nq;
  auto trow = [&](int64_t i) { return targets ? targets + i * (int64_t)P.target_stride : nullptr; };
  auto store = [&](int64_t i, float ei, int n, int st) {
    if (err) err[i] = ei;
    if (steps) steps[i] = n;
    if (status) status[i] = st;
  };
  if (sel.path == pk::kPathChain) {
    pk::with_nj(sel.nj, [&](auto nj) {
      constexpr int NJ = decltype(nj)::value;
      pk::ChainParams<NJ> C;
      pk::make_chain_params<NJ>(hm, P, &C, P.ext);
      const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
      pk::with_nft(sel.nft, [&](auto nft) {
        for (int64_t i = 0; i < B; ++i) {
          float qi[NJ];
          for (int k = 0; k < NJ; ++k) qi[k] = q[i * NJ + k];
          float ei;
          int n, st;
          pk::converge_chain<NJ, decltype(nft)::value>(C, qi, trow(i), emask, tol, max_steps, ei, n, st);
          for (int k = 0; k < NJ; ++k) q_out[i * NJ + k] = qi[k];
          store(i, ei, n, st);
        }
      });
    });
  } else if (sel.path == pk::kPathTree) {
    const pk::TreePlan& L = sel.plan;
    std::vector<float> W(L.words + 8);
    float* Wp = W.data();
    if (((uintptr_t)Wp & 7) != 0) ++Wp;  // the dual method keeps doubles in the workspace
    std::vector<float> v(hm.nv);
    for (int64_t i = 0; i < B; ++i) {
      float* qrow = q_out + i * nq;
      if (qrow != q + i * nq) std::memcpy(qrow, q + i * nq, sizeof(float) * nq);
      float ei;
      int n, st;
      pk::TreeStep::converge(M, P, L, qrow, trow(i), Wp, v.data(), mask, tol, max_steps, ei, n, st);
      store(i, ei, n, st);
    }
  } else {
    pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
      static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
      float v[decltype(nv)::value];
      for (int64_t i = 0; i < B; ++i) {
        float* qrow = q_out + i * nq;
        if (qrow != q + i * nq) std::memcpy(qrow, q + i * nq, sizeof(float) * nq);
        float ei;
        int n, st;
        pk::converge_generic(G, M, P, qrow, trow(i), v, mask, tol, max_steps, ei, n, st);
        store(i, ei, n, st);
      }
    });
  }
  return 0;
}

}
