// CPU build of the goal-set solve (pk_converge_goalset_prepared) for the test suite ONLY: the host
// build of the kernel bodies (tests/hostsim/hostsim.cpp, compiled into this library as it is) plus
// hs_converge_goalset, a sibling of hs_converge_multistart that shares its two-pass rounds
// (run_group), its selection and its step bodies, with the G S members of an instance indexed as
// on the device.  Never loaded by the product package and not a fallback.
#include "../hostsim/hostsim.cpp"

extern "C" {

// Goal-set solve to a tolerance (pk_converge_goalset_prepared) with the bodies the selection
// names; q_seeds [B S][nq], targets [B G][target_stride], the outputs [B].  Member j = g S + s of
// instance b starts at seed row b S + s and reads targets row b G + g, as on the device.  path as
// hs_converge without the sub-warp kernel.  A host thread cannot suspend inside a step body to
// wait for the other members of its group, so each round runs in two passes over the group:
// first every member's error, from the step body with its stop forced (it returns before the
// QP); then the group's decision, and the step of every member that goes on.  The bodies
// (ChainStep::assemble<true> with converge_chain_advance, TreeStep::run<true>,
// Generic::step<true>) and the winner's order (seed_before) are those the CUDA library runs.
int hs_converge_goalset(void* model, const PkProblemDesc* prob, const float* q_seeds, int S, const float* targets,
                        int G, uint32_t mask, float tol, int max_steps, float* q_out, float* err, int32_t* goal,
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
  const std::string kerr = pk::check_goalset_members(sel, G, S);
  if (!kerr.empty()) return fail(kerr);
  if (B > 0 && P.target_stride > 0 && !targets) return fail("null targets");
  const pk::DevModel M = hm.host_view();
  const int nq = hm.nq, GS = G * S;
  // the forced stop of the first pass, and the test of the second (never stops: err >= 0)
  const pk::ConvergeTest probe{mask, tol, true, 0.f, false, 0};
  const pk::ConvergeTest go{mask, -INFINITY, false, 0.f, false, 0};
  std::vector<float> qs((size_t)GS * nq), es(GS);
  std::vector<int> st_all(GS);
  for (int64_t b = 0; b < B; ++b) {
    // member j's targets row
    auto trow = [&](int j) { return targets ? targets + (b * G + j / S) * (int64_t)P.target_stride : nullptr; };
    for (int g = 0; g < G; ++g)
      std::memcpy(qs.data() + (size_t)g * S * nq, q_seeds + b * S * nq, sizeof(float) * S * nq);
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
          Cs.template assemble<true>(C, qj(j), trow(j), skip, emask, &ej);
          return ej;
        };
        auto advance = [&](int j) {
          pk::ChainStep<NJ, NFT> Cs;
          bool skip;
          float ej;
          const int st = Cs.template assemble<true>(C, qj(j), trow(j), skip, emask, &ej);
          return pk::converge_chain_advance(C, Cs, st, skip, qj(j), st_all[j], 0);
        };
        w = run_group(GS, tol, max_steps, error, advance, es, n);
      });
    } else if (sel.path == pk::kPathTree) {
      const pk::TreePlan& L = sel.plan;
      std::vector<float> W, v(hm.nv);
      float* Wp = tree_workspace(W, L.words);
      auto error = [&](int j) {
        pk::ConvergeTest ct = probe;
        pk::TreeStep::run<true>(M, P, L, qs.data() + j * nq, trow(j), Wp, v.data(), nullptr, &ct);
        return ct.err;
      };
      auto advance = [&](int j) {
        float* q = qs.data() + j * nq;
        pk::ConvergeTest ct = go;
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
          pk::ConvergeTest ct = probe;
          Gs.template step<true>(M, P, qs.data() + j * nq, trow(j), out, &ct);
          return ct.err;
        };
        auto advance = [&](int j) {
          float* q = qs.data() + j * nq;
          pk::ConvergeTest ct = go;
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
