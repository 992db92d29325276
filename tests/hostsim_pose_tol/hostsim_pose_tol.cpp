// CPU build of the separate-tolerance solves (pk_converge_pose_tol_prepared and
// pk_converge_goalset_pose_tol_prepared) for the test suite ONLY: the host build of the kernel
// bodies (tests/hostsim/hostsim.cpp, compiled into this library as it is) plus
// hs_converge_pose_tol and hs_converge_goalset_pose_tol, which run the pose-tolerance
// instantiations of the bodies the selection names (ChainStep::assemble<true, true>,
// PoseTolTest), with the test arguments the CUDA library passes (rot_scale = tol /
// orientation_tol, chain_axis_mask).  Never loaded by the product package and not a fallback.
#include "../hostsim/hostsim.cpp"

namespace {

// The validation and rot_scale of the CUDA library's separate-tolerance entries.
std::string pose_tol_problem(const pk::HostModel& hm, const PkProblemDesc* prob, uint32_t mask, float tol,
                             float orientation_tol, int max_steps, pk::DevProblem* P, pk::HostExtras* hx,
                             float* rscale) {
  std::string e = make_problem(hm, prob, P, hx);
  if (e.empty()) e = pk::check_converge_args(*P, mask, tol, max_steps);
  if (e.empty()) e = pk::check_pose_tol_args(*P, mask, tol, orientation_tol);
  *rscale = orientation_tol < INFINITY ? tol / orientation_tol : 0.f;
  return e;
}

}  // namespace

extern "C" {

// Solve to separate tolerances with the converge loop of the body the selection names:
// converge_chain<NJ, NFT, true>, TreeStep::converge<true> or converge_generic<..., true>.
// Arguments as hs_converge, plus orientation_tol.
int hs_converge_pose_tol(void* model, const PkProblemDesc* prob, const float* q, const float* targets, uint32_t mask,
                         float tol, float orientation_tol, int max_steps, float* q_out, float* err, int32_t* steps,
                         int32_t* status, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  float rs;
  const std::string e = pose_tol_problem(hm, prob, mask, tol, orientation_tol, max_steps, &P, &hx, &rs);
  if (!e.empty()) return fail(e);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, true, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  const pk::DevModel M = hm.host_view();
  if (sel.path == pk::kPathChain) {
    const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
    const unsigned amask = pk::chain_axis_mask(P, mask, orientation_tol);
    pk::with_chain(sel, [&](auto nj, auto nft) {
      constexpr int NJ = decltype(nj)::value;
      pk::ChainParams<NJ> C;
      pk::make_chain_params<NJ>(hm, P, &C, P.ext);
      for (int64_t i = 0; i < B; ++i)
        pk::converge_chain_instance<NJ, decltype(nft)::value, true>(C, q, targets, emask, tol, max_steps, q_out, err,
                                                                    steps, status, i, amask, rs);
    });
  } else if (sel.path == pk::kPathTree) {
    const pk::ConvergeTreeLayout T = pk::converge_tree_layout(sel.plan);
    std::vector<float> W;
    float* Wp = tree_workspace(W, T.plan.words);
    for (int64_t i = 0; i < B; ++i)
      pk::TreeStep::converge_instance<true>(M, P, T.plan, T.o_v, q, targets, mask, tol, max_steps, q_out, Wp, err,
                                            steps, status, i, rs);
  } else {
    pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
      constexpr int NJ = decltype(nj)::value, NV = decltype(nv)::value;
      static thread_local pk::Generic<NJ, NV> G;
      for (int64_t i = 0; i < B; ++i)
        pk::converge_generic_instance<NJ, NV, true>(G, M, P, q, targets, mask, tol, max_steps, q_out, err, steps,
                                                    status, i, rs);
    });
  }
  return 0;
}

// Goal-set solve to separate tolerances: hs_converge_goalset (tests/hostsim_goalset) with the
// pose-tolerance instantiations of its bodies.  Arguments as hs_converge_goalset, plus orientation_tol;
// G = 1 is multi-start, as on the device.
int hs_converge_goalset_pose_tol(void* model, const PkProblemDesc* prob, const float* q_seeds, int S,
                                 const float* targets, int G, uint32_t mask, float tol, float orientation_tol,
                                 int max_steps, float* q_out, float* err, int32_t* goal, int32_t* seed, int32_t* steps,
                                 int32_t* status, int64_t B, int path, int* sel_out) {
  const pk::HostModel& hm = *(pk::HostModel*)model;
  pk::DevProblem P;
  pk::HostExtras hx;
  float rs;
  const std::string e = pose_tol_problem(hm, prob, mask, tol, orientation_tol, max_steps, &P, &hx, &rs);
  if (!e.empty()) return fail(e);
  pk::Selection sel;
  const std::string serr = select(hm, P, hx, path, false, sel_out, &sel);
  if (!serr.empty()) return fail(serr);
  const std::string kerr = pk::check_goalset_members(sel, G, S);
  if (!kerr.empty()) return fail(kerr);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  const pk::DevModel M = hm.host_view();
  const int nq = hm.nq, GS = G * S;
  // the forced stop of the first pass, and the test of the second (never stops: err >= 0)
  const pk::PoseTolTest<pk::ConvergeTest> probe{{mask, tol, true, 0.f, false, 0}, rs};
  const pk::PoseTolTest<pk::ConvergeTest> go{{mask, -INFINITY, false, 0.f, false, 0}, rs};
  std::vector<float> qs((size_t)GS * nq), es(GS);
  std::vector<int> st_all(GS);
  for (int64_t b = 0; b < B; ++b) {
    auto trow = [&](int j) { return targets ? targets + (b * G + j / S) * (int64_t)P.target_stride : nullptr; };
    for (int g = 0; g < G; ++g)
      std::memcpy(qs.data() + (size_t)g * S * nq, q_seeds + b * S * nq, sizeof(float) * S * nq);
    std::fill(st_all.begin(), st_all.end(), 0);
    int w = 0, n = 0;
    if (sel.path == pk::kPathChain) {
      const unsigned emask = pk::chain_task_mask(P, mask, sel.nft);
      const unsigned amask = pk::chain_axis_mask(P, mask, orientation_tol);
      pk::with_chain(sel, [&](auto nj, auto nft) {
        constexpr int NJ = decltype(nj)::value, NFT = decltype(nft)::value;
        pk::ChainParams<NJ> C;
        pk::make_chain_params<NJ>(hm, P, &C, P.ext);
        auto qj = [&](int j) -> float(&)[NJ] { return *reinterpret_cast<float(*)[NJ]>(qs.data() + j * NJ); };
        auto error = [&](int j) {
          pk::ChainStep<NJ, NFT> Cs;
          bool skip;
          float ej;
          Cs.template assemble<true, true>(C, qj(j), trow(j), skip, emask, &ej, amask, rs);
          return ej;
        };
        auto advance = [&](int j) {
          pk::ChainStep<NJ, NFT> Cs;
          bool skip;
          float ej;
          const int st = Cs.template assemble<true, true>(C, qj(j), trow(j), skip, emask, &ej, amask, rs);
          return pk::converge_chain_advance(C, Cs, st, skip, qj(j), st_all[j], 0);
        };
        w = run_group(GS, tol, max_steps, error, advance, es, n);
      });
    } else if (sel.path == pk::kPathTree) {
      const pk::TreePlan& L = sel.plan;
      std::vector<float> W, v(hm.nv);
      float* Wp = tree_workspace(W, L.words);
      auto error = [&](int j) {
        auto ct = probe;
        pk::TreeStep::run<true>(M, P, L, qs.data() + j * nq, trow(j), Wp, v.data(), nullptr, &ct);
        return ct.err;
      };
      auto advance = [&](int j) {
        float* q = qs.data() + j * nq;
        auto ct = go;
        pk::TreeStep::run<true>(M, P, L, q, trow(j), Wp, v.data(), nullptr, &ct);
        st_all[j] |= ct.status;
        if (pk::step_failed(st_all[j], P.safety_break)) return false;
        pk::integrate_configuration(nq, M.free_flyer, q, v.data(), P.dt, q);
        return true;
      };
      w = run_group(GS, tol, max_steps, error, advance, es, n);
    } else {
      pk::with_generic(sel.generic_class, [&](auto nj, auto nv) {
        static thread_local pk::Generic<decltype(nj)::value, decltype(nv)::value> Gs;
        float v[decltype(nv)::value];
        int32_t st = 0;
        pk::GenericOut out{};
        out.v = v;
        out.status = &st;
        out.task_index = -1;
        auto error = [&](int j) {
          auto ct = probe;
          Gs.template step<true>(M, P, qs.data() + j * nq, trow(j), out, &ct);
          return ct.err;
        };
        auto advance = [&](int j) {
          float* q = qs.data() + j * nq;
          auto ct = go;
          Gs.template step<true>(M, P, q, trow(j), out, &ct);
          st_all[j] |= st;
          if (pk::step_failed(st_all[j], P.safety_break)) return false;
          pk::integrate_configuration(nq, M.free_flyer, q, v, P.dt, q);
          return true;
        };
        w = run_group(GS, tol, max_steps, error, advance, es, n);
      });
    }
    std::memcpy(q_out + b * nq, qs.data() + w * nq, sizeof(float) * nq);
    if (err) err[b] = es[w];
    if (goal) goal[b] = w / S;
    if (seed) seed[b] = w % S;
    if (steps) steps[b] = n;
    if (status) status[b] = st_all[w];
  }
  return 0;
}

}  // extern "C"
