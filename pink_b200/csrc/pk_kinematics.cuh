// Differentiable forward kinematics of selected frames and the CoM (pk_frame_placements_batched,
// pk_frame_placements_vjp_batched, DESIGN.md section 3.2i): one instance per thread, shared by
// the kernels of pk_kinematics.cu and the host build (tests/hostsim_kinematics).
//
// The forward half runs Generic::forward_kinematics, body_placement and center_of_mass, so the
// placements and the CoM are bitwise those of pk_forward_kinematics_batched.  The reverse half
// recomputes the forward at q and sweeps the tree once, leaves to root: each requested frame's
// gradient [G_R | g_p] becomes a world force F = g_p and a moment about the origin
// N = vee(G_R R^T - R G_R^T) + p x g_p, the CoM gradient g_c puts F = (m_b / M) g_c at each body's
// CoM x_b (N = x_b x F), the pairs are summed over subtrees, and joint j reads its derivative
// off its subtree's sum: a_j . (N - o_j x F) (revolute) or a_j . F (prismatic), with the world
// axis a_j and origin o_j of frame_jac_col.
#pragma once

#include <string>

#include "pk_marshal.hpp"

namespace pk {

// The frames of one call, copied into the launch's parameters (no allocation, graph-capturable).
struct FrameList {
  int n;
  int32_t f[PK_MAX_FRAMES];
};

// The frames and CoM request of pk_frame_placements_batched / _vjp_batched into L; "" when valid.
inline std::string make_frame_list(const HostModel& m, const int32_t* frames, int32_t n, bool com, FrameList* L) {
  *L = FrameList{};
  if (n < 0 || n > PK_MAX_FRAMES) return "num_frames must be in [0, " + std::to_string(PK_MAX_FRAMES) + "]";
  if (n > 0 && !frames) return "null frames";
  for (int k = 0; k < n; ++k) {
    if (frames[k] < 0 || frames[k] >= m.nframes)
      return "frame index " + std::to_string(frames[k]) + " out of range [0, " + std::to_string(m.nframes) + ")";
    L->f[k] = frames[k];
  }
  L->n = n;
  if (com && !(m.total_mass > 0.f)) return "the model's total mass is 0: it has no centre of mass";
  return "";
}

// World placement of frame f after G.forward_kinematics.
template <int NJMAX, int NVMAX>
PK_HD SE3f frame_placement(const Generic<NJMAX, NVMAX>& G, const DevModel& M, int f) {
  return compose(G.body_placement(M.frame_body[f]), load_se3(M.fX + 12 * f));
}

// oMf [L.n][12] (row-major [R | p]) and com [3] unless null, at q.
template <int NJMAX, int NVMAX>
PK_HD void frame_placements(Generic<NJMAX, NVMAX>& G, const DevModel& M, const FrameList& L, const float* q,
                            float* oMf, float* com) {
  G.forward_kinematics(M, q);
  for (int k = 0; k < L.n; ++k) store_se3(frame_placement(G, M, L.f[k]), oMf + 12 * k);
  if (com) {
    const V3 c = G.center_of_mass(M);
    com[0] = c.x; com[1] = c.y; com[2] = c.z;
  }
}

// The reverse sweep's state: the forward's placements and, per joint, the force and moment about
// the world origin on its subtree.
template <int NJMAX, int NVMAX>
struct FramePlacementsVjp {
  Generic<NJMAX, NVMAX> G;
  V3 F[NJMAX], N[NJMAX];

  // A world force and moment on `body` (-1: the root body, moved only by a free-flyer).
  PK_HD void add(const DevModel& M, int body, V3 f, V3 n, V3& Fr, V3& Nr) {
    if (body >= 0) {
      F[body] = F[body] + f;
      N[body] = N[body] + n;
    } else if (body == -1 && M.free_flyer) {
      Fr = Fr + f;
      Nr = Nr + n;
    }
  }

  // gq [nq] = (d (oMf, com) / d q)^T (gF, gc), fully written; gF [L.n][12] or null, gc [3] or null
  // (null: that term is zero).
  PK_HD void vjp(const DevModel& M, const FrameList& L, const float* q, const float* gF, const float* gc, float* gq) {
    G.forward_kinematics(M, q);
    const int nj = M.njoints;
    const int rq = M.free_flyer ? 7 : 0;
    const V3 zero = v3(0.f, 0.f, 0.f);
    for (int j = 0; j < nj; ++j) F[j] = N[j] = zero;
    V3 Fr = zero, Nr = zero;
    if (gF) {
      for (int k = 0; k < L.n; ++k) {
        const int f = L.f[k];
        const SE3f T = frame_placement(G, M, f);
        const float* g = gF + 12 * k;
        // S = G_R R^T; the moment of the rotation part is vee(S - S^T)
        float S[9];
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 3; ++b)
            S[3 * a + b] =
                fmaf(g[4 * a], T.R.m[3 * b], fmaf(g[4 * a + 1], T.R.m[3 * b + 1], g[4 * a + 2] * T.R.m[3 * b + 2]));
        const V3 gp = v3(g[3], g[7], g[11]);
        const V3 n = v3(S[7] - S[5], S[2] - S[6], S[3] - S[1]) + cross(T.p, gp);
        add(M, M.frame_body[f], gp, n, Fr, Nr);
      }
    }
    if (gc) {
      const V3 gcv = v3(gc[0], gc[1], gc[2]);
      for (int b = -1; b < nj; ++b) {
        const float m = M.mass[b + 1];
        if (m == 0.f) continue;
        const SE3f T = G.body_placement(b);
        const V3 x = mul(T.R, v3(M.com[3 * (b + 1)], M.com[3 * (b + 1) + 1], M.com[3 * (b + 1) + 2])) + T.p;
        const V3 f = (m / M.total_mass) * gcv;
        add(M, b, f, cross(x, f), Fr, Nr);
      }
    }
    for (int j = nj - 1; j >= 0; --j) {
      const V3 aw = mul(G.Tw[j].R, v3(M.axis[3 * j], M.axis[3 * j + 1], M.axis[3 * j + 2]));
      gq[rq + j] = M.jtype[j] == PK_JOINT_REVOLUTE ? dot(aw, N[j] - cross(G.Tw[j].p, F[j])) : dot(aw, F[j]);
      add(M, M.parent[j], F[j], N[j], Fr, Nr);
    }
    if (M.free_flyer) {
      gq[0] = Fr.x; gq[1] = Fr.y; gq[2] = Fr.z;
      // u = quat / |quat| rotates the tree about the root origin by dw = 2 (u_w du_v - du_w u_v + u_v x du_v)
      // (world frame); with the moment t about that origin, dL = t . dw and du = (I - u u^T) dquat / |quat|.
      // The gradient in u, [2 (u_w t + t x u_v), -2 t . u_v], is orthogonal to u: the radial part is 0.
      const V3 t = Nr - cross(G.root.p, Fr);
      const float r = 1.f / sqrtf(fmaf(q[3], q[3], fmaf(q[4], q[4], fmaf(q[5], q[5], q[6] * q[6]))));
      const V3 uv = v3(q[3] * r, q[4] * r, q[5] * r);
      const float uw = q[6] * r;
      const V3 gv = (2.f * r) * (uw * t + cross(t, uv));
      gq[3] = gv.x; gq[4] = gv.y; gq[5] = gv.z;
      gq[6] = -2.f * r * dot(t, uv);
    }
  }
};

// Instance i of frame_placements_kernel: rows i of q, oMf [B][L.n][12] and com [B][3] (unless null).
template <int NJMAX, int NVMAX>
PK_HD void frame_placements_instance(Generic<NJMAX, NVMAX>& G, const DevModel& M, const FrameList& L,
                                     const float* __restrict__ q, float* __restrict__ oMf, float* __restrict__ com,
                                     int64_t i) {
  frame_placements(G, M, L, q + i * M.nq, oMf ? oMf + i * 12 * L.n : nullptr, com ? com + 3 * i : nullptr);
}

// Instance i of frame_placements_vjp_kernel: rows i of q, grad_oMf and grad_com (unless null), grad_q.
template <int NJMAX, int NVMAX>
PK_HD void frame_placements_vjp_instance(FramePlacementsVjp<NJMAX, NVMAX>& K, const DevModel& M, const FrameList& L,
                                         const float* __restrict__ q, const float* __restrict__ grad_oMf,
                                         const float* __restrict__ grad_com, float* __restrict__ grad_q, int64_t i) {
  K.vjp(M, L, q + i * M.nq, grad_oMf ? grad_oMf + i * 12 * L.n : nullptr, grad_com ? grad_com + 3 * i : nullptr,
        grad_q + i * M.nq);
}

}  // namespace pk
