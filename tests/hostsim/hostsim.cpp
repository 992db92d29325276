// CPU build of the kernel bodies (pk_chain.cuh / pk_generic.cuh) for the test
// suite ONLY: lets `pytest -m "not gpu"` exercise the exact fp32 arithmetic and
// control flow of the CUDA kernels against the fp64 oracle on machines without
// a GPU.  It is never loaded by the product package (pink_b200/_cabi.py loads
// libpink_b200.so and nothing else) and is not a fallback.
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

// The bodies of the kernels a chain selection names, lanes emulated by loops in the sub-warp one.
template <int NJ, int NFT>
void run_chain(const pk::HostModel& hm, const pk::DevProblem& P, const pk::Selection& sel, const float* q,
               const float* targets, float* v, int32_t* status, int64_t B) {
  if (!sel.lanes) {
    pk::ChainParams<NJ> C;
    pk::make_chain_params<NJ>(hm, P, &C, P.ext);
    for (int64_t i = 0; i < B; ++i) {
      float qi[NJ], vi[NJ];
      for (int k = 0; k < NJ; ++k) qi[k] = q[i * NJ + k];
      int st = 0;
      pk::ik_step_chain<NJ, NFT>(C, qi, targets + i * (int64_t)P.target_stride, vi, st);
      for (int k = 0; k < NJ; ++k) v[i * NJ + k] = vi[k];
      if (status) status[i] = st;
    }
    return;
  }
  pk::with_lanes<NJ, NFT>(sel.lanes, [&](auto lanes) {
    constexpr int L = decltype(lanes)::value;
    using Step = pk::CoopStep<NJ, NFT, L>;
    typename Step::Params C;
    pk::make_coop_params<NJ, L>(hm, P, &C, P.ext);
    const pk::Group<L> G{};
    auto jc = [&](int j) -> const pk::CoopJoint& { return C.joint[j]; };
    for (int64_t i = 0; i < B; ++i) {
      pk::GVar<typename Step::Lane, L> S;
      for (int h = 0; h < L; ++h)
        for (int k = 0; k < Step::NC; ++k) {
          const int j = h * Step::NC + k;
          S[h].q[k] = j < NJ ? q[i * NJ + j] : 0.f;
        }
      int st = 0;
      pk::ik_step_coop<NJ, NFT, L>(G, C, jc, targets + i * (int64_t)P.target_stride, S, st);
      for (int h = 0; h < L; ++h)
        for (int k = 0; k < Step::NC; ++k) {
          const int j = h * Step::NC + k;
          if (j < NJ) v[i * NJ + j] = S[h].x[k];
        }
      if (status) status[i] = st;
    }
  });
}

// make_dev_problem + host image of the optional parts, wired through P.ext
std::string make_problem(const pk::HostModel& hm, const PkProblemDesc* prob, pk::DevProblem* P, pk::HostExtras* hx) {
  const std::string e = pk::make_dev_problem(hm, prob, P, hx);
  if (e.empty() && hx->present) P->ext = &hx->X;
  return e;
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

// The kernel body the CUDA library's selection (pk_select.hpp) names for this problem.
// path: 0 the library's default options, 1 PK_FORCE_GENERIC=1, 2 without the chain kernels (the
// tree kernel body on a chain), 11 / 12 / 14 / 18 PK_CHAIN_LANES = 1 / 2 / 4 / 8 (the problem must
// take a chain kernel).  sel_out: path (pk::KernelPath), nj, nft, the general path's <NJMAX, NVMAX>,
// lanes, PDL row fits, tree task rows K.
int hs_solve_ik(void* model, const PkProblemDesc* prob, const float* q, const float* targets, float* v,
                int32_t* status, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  const std::string e = make_problem(hm, prob, &P, &hx);
  if (!e.empty()) return fail(e);
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
  if (sel.path == pk::kPathChain) {
    pk::with_nj(sel.nj, [&](auto nj) {
      pk::with_nft(sel.nft, [&](auto nft) {
        run_chain<decltype(nj)::value, decltype(nft)::value>(hm, P, sel, q, targets, v, status, B);
      });
    });
  } else if (sel.path == pk::kPathTree) {
    const pk::TreePlan& L = sel.plan;
    const pk::DevModel M = hm.host_view();
    std::vector<float> W(L.words + 8);
    float* Wp = W.data();
    if (((uintptr_t)Wp & 7) != 0) ++Wp;  // the dual method keeps doubles in the workspace
    for (int64_t i = 0; i < B; ++i)
      pk::TreeStep::run(M, P, L, q + i * L.nq, targets ? targets + i * (int64_t)L.stride : nullptr, Wp,
                        v + i * L.nv, status ? status + i : nullptr);
  } else {
    pk::GenericArgs A{};
    A.q = q; A.targets = targets; A.v = v; A.status = status; A.task_index = -1;
    run_generic(hm, P, A, B);
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
  std::vector<float> W(L.words + 8, 0.f);
  float* Wp = W.data();
  if (((uintptr_t)Wp & 7) != 0) ++Wp;  // doubles in the workspace
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
