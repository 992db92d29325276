// CPU build of the gradient body of pk_converge_vjp_prepared (Generic::solution_vjp in
// pink_b200/csrc/pk_generic.cuh) for the test suite ONLY, beside the host build of the other
// kernel bodies (tests/hostsim): the same source, the same fp32 arithmetic, checked against the
// fp64 oracle without a GPU.  Never loaded by the product package and not a fallback.
#include <cstdint>
#include <string>

#include "../../include/pink_b200.h"
#include "../../pink_b200/csrc/pk_select.hpp"

namespace {
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return 1; }
}  // namespace

extern "C" {

const char* hv_last_error(void) { return g_err.c_str(); }

int hv_model_create(const PkModelDesc* d, void** out) {
  pk::HostModel* m = new pk::HostModel();
  const std::string e = pk::build_host_model(d, m);
  if (!e.empty()) { delete m; return fail(e); }
  *out = m;
  return 0;
}
void hv_model_destroy(void* m) { delete (pk::HostModel*)m; }

// Gradient with respect to the targets at converged solutions, with solution_vjp_instance at the
// instantiation ik_generic_solution_vjp_kernel launches for this model (generic_size_class), after
// the argument checks of pk_converge_vjp_prepared.
int hv_converge_vjp(void* model, const PkProblemDesc* prob, const float* q_star, const float* targets,
                    const float* grad_q, float* grad_targets, int32_t* status, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = pk::make_dev_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
  if (hx.present) P.ext = &hx.X;
  const std::string verr = pk::check_vjp_problem(hx);
  if (!verr.empty()) return fail(verr);
  if (B > 0 && !grad_q) return fail("null grad_q");
  if (B > 0 && P.target_stride > 0 && (!targets || !grad_targets)) return fail("null targets or grad_targets");
  const pk::DevModel M = hm.host_view();
  pk::with_generic(pk::generic_size_class(hm), [&](auto nj, auto nv) {
    static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
    for (int64_t i = 0; i < B; ++i) pk::solution_vjp_instance(G, M, P, q_star, targets, grad_q, grad_targets, status, i);
  });
  return 0;
}
}
