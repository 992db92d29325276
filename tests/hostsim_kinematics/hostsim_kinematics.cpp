// CPU build of the differentiable forward kinematics (pk_frame_placements_batched and
// pk_frame_placements_vjp_batched, pink_b200/csrc/pk_kinematics.cuh) for the test suite ONLY,
// beside the host builds of the other kernel bodies: the same source, the same fp32 arithmetic,
// checked against the fp64 oracle without a GPU.  Never loaded by the product package and not a
// fallback.
#include <cstdint>
#include <string>

#include "../../include/pink_b200.h"
#include "../../pink_b200/csrc/pk_kinematics.cuh"
#include "../../pink_b200/csrc/pk_select.hpp"

namespace {
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return 1; }
}  // namespace

extern "C" {

const char* hk_last_error(void) { return g_err.c_str(); }

int hk_model_create(const PkModelDesc* d, void** out) {
  pk::HostModel* m = new pk::HostModel();
  const std::string e = pk::build_host_model(d, m);
  if (!e.empty()) { delete m; return fail(e); }
  *out = m;
  return 0;
}
void hk_model_destroy(void* m) { delete (pk::HostModel*)m; }

// Frame placements and CoM with frame_placements_instance, and their gradient with
// frame_placements_vjp_instance, at the instantiation the kernels launch for this model
// (generic_size_class), after the argument checks of pk_frame_placements_batched / _vjp_batched.
int hk_frame_placements(void* model, const int32_t* frames, int32_t num_frames, const float* q, float* oMf,
                        float* com, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::FrameList L;
  const std::string e = pk::make_frame_list(hm, frames, num_frames, com != nullptr, &L);
  if (!e.empty()) return fail(e);
  if (B > 0 && !q) return fail("null q");
  if (B > 0 && num_frames > 0 && !oMf) return fail("null oMf");
  const pk::DevModel M = hm.host_view();
  pk::with_generic(pk::generic_size_class(hm), [&](auto nj, auto nv) {
    static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> G;
    for (int64_t i = 0; i < B; ++i) pk::frame_placements_instance(G, M, L, q, oMf, com, i);
  });
  return 0;
}

int hk_frame_placements_vjp(void* model, const int32_t* frames, int32_t num_frames, const float* q,
                            const float* grad_oMf, const float* grad_com, float* grad_q, int64_t B) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::FrameList L;
  const std::string e = pk::make_frame_list(hm, frames, num_frames, grad_com != nullptr, &L);
  if (!e.empty()) return fail(e);
  if (B > 0 && !q) return fail("null q");
  if (B > 0 && !grad_q) return fail("null grad_q");
  const pk::DevModel M = hm.host_view();
  pk::with_generic(pk::generic_size_class(hm), [&](auto nj, auto nv) {
    static thread_local pk::FramePlacementsVjp<decltype(nj)::value, decltype(nv)::value> K;
    for (int64_t i = 0; i < B; ++i) pk::frame_placements_vjp_instance(K, M, L, q, grad_oMf, grad_com, grad_q, i);
  });
  return 0;
}
}
