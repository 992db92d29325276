// fp32 SO(3)/SE(3) helpers shared by every kernel of the IK path.
//
// Semantics follow Pinocchio's as used by the reference (see SURVEY.md section 9 and
// pink/tasks/frame_task.py:176-226): SE3 = (R, p), twists are
// [linear; angular], log6 returns a body twist, Jlog6 is the right Jacobian
// inverse.  Formulas are re-derived for fp32: angles come from atan2 (never
// acos), the scalar coefficient functions switch between Bernoulli-series
// polynomials and closed forms where cancellation would cost digits, and the
// rotation vector near pi is recovered from a quaternion.
//
// Everything is PK_HD so that tests/hostsim can compile the same bodies for the
// host CPU (test harness only; the product has no CPU path).
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PK_HD __host__ __device__ __forceinline__
#define PK_D __device__ __forceinline__
#else
#define PK_HD inline
#define PK_D inline
#endif

#if !defined(__CUDACC__)
// host-only build (tests/hostsim): glibc has no rsqrtf, and no CUDA vector types
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
#endif

namespace pk {

struct V3 {
  float x, y, z;
};
struct M3 {
  float m[9];  // row-major
};
struct SE3f {
  M3 R;
  V3 p;
};

PK_HD V3 v3(float x, float y, float z) {
  V3 r;
  r.x = x; r.y = y; r.z = z;
  return r;
}
PK_HD V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
PK_HD V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
PK_HD V3 operator*(float s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
PK_HD float dot(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
PK_HD V3 cross(V3 a, V3 b) {
  return v3(fmaf(a.y, b.z, -a.z * b.y), fmaf(a.z, b.x, -a.x * b.z), fmaf(a.x, b.y, -a.y * b.x));
}
PK_HD float idx(V3 a, int k) { return k == 0 ? a.x : (k == 1 ? a.y : a.z); }

PK_HD V3 mul(const M3& R, V3 v) {
  return v3(fmaf(R.m[0], v.x, fmaf(R.m[1], v.y, R.m[2] * v.z)),
            fmaf(R.m[3], v.x, fmaf(R.m[4], v.y, R.m[5] * v.z)),
            fmaf(R.m[6], v.x, fmaf(R.m[7], v.y, R.m[8] * v.z)));
}
PK_HD V3 mulT(const M3& R, V3 v) {  // R^T v
  return v3(fmaf(R.m[0], v.x, fmaf(R.m[3], v.y, R.m[6] * v.z)),
            fmaf(R.m[1], v.x, fmaf(R.m[4], v.y, R.m[7] * v.z)),
            fmaf(R.m[2], v.x, fmaf(R.m[5], v.y, R.m[8] * v.z)));
}
PK_HD M3 mul(const M3& A, const M3& B) {
  M3 C;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C.m[3 * i + j] = fmaf(A.m[3 * i], B.m[j], fmaf(A.m[3 * i + 1], B.m[3 + j], A.m[3 * i + 2] * B.m[6 + j]));
  return C;
}
PK_HD M3 mulTN(const M3& A, const M3& B) {  // A^T B
  M3 C;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C.m[3 * i + j] = fmaf(A.m[i], B.m[j], fmaf(A.m[3 + i], B.m[3 + j], A.m[6 + i] * B.m[6 + j]));
  return C;
}
PK_HD M3 mulNT(const M3& A, const M3& B) {  // A B^T
  M3 C;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C.m[3 * i + j] = fmaf(A.m[3 * i], B.m[3 * j], fmaf(A.m[3 * i + 1], B.m[3 * j + 1], A.m[3 * i + 2] * B.m[3 * j + 2]));
  return C;
}
PK_HD M3 identity3() {
  M3 I;
#pragma unroll
  for (int i = 0; i < 9; ++i) I.m[i] = (i % 4 == 0) ? 1.f : 0.f;
  return I;
}
PK_HD SE3f identity_se3() {
  SE3f T;
  T.R = identity3();
  T.p = v3(0.f, 0.f, 0.f);
  return T;
}
PK_HD SE3f compose(const SE3f& a, const SE3f& b) {  // a * b
  SE3f r;
  r.R = mul(a.R, b.R);
  r.p = mul(a.R, b.p) + a.p;
  return r;
}
PK_HD SE3f act_inv(const SE3f& a, const SE3f& b) {  // a^-1 * b
  SE3f r;
  r.R = mulTN(a.R, b.R);
  r.p = mulT(a.R, b.p - a.p);
  return r;
}
PK_HD SE3f load_se3(const float* t) {  // 12 floats, row-major [R | p]
  SE3f T;
  T.R.m[0] = t[0]; T.R.m[1] = t[1]; T.R.m[2] = t[2];  T.p.x = t[3];
  T.R.m[3] = t[4]; T.R.m[4] = t[5]; T.R.m[5] = t[6];  T.p.y = t[7];
  T.R.m[6] = t[8]; T.R.m[7] = t[9]; T.R.m[8] = t[10]; T.p.z = t[11];
  return T;
}
// *p for an input the kernel never writes: through the read-only data cache on the device
template <class T>
PK_HD T load_ro(const T* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// 12 floats; `vec4`: the address is 16-byte aligned (three 128-bit read-only loads instead
// of twelve scalar ones when it is in global memory)
PK_HD SE3f load_se3_vec4(const float* t, bool vec4) {
#if defined(__CUDA_ARCH__)
  // the caller's `vec4` covers stride and offsets; the base pointer is checked here (a
  // sliced tensor may start anywhere).  __ldg only reads global memory: a row the chain
  // kernel copied to local memory takes the plain loads (resolved at compile time).
  if (vec4 && __isGlobal(t) && (reinterpret_cast<uintptr_t>(t) & 15u) == 0u) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(t));
    const float4 b = __ldg(reinterpret_cast<const float4*>(t) + 1);
    const float4 c = __ldg(reinterpret_cast<const float4*>(t) + 2);
    SE3f T;
    T.R.m[0] = a.x; T.R.m[1] = a.y; T.R.m[2] = a.z; T.p.x = a.w;
    T.R.m[3] = b.x; T.R.m[4] = b.y; T.R.m[5] = b.z; T.p.y = b.w;
    T.R.m[6] = c.x; T.R.m[7] = c.y; T.R.m[8] = c.z; T.p.z = c.w;
    return T;
  }
#else
  (void)vec4;
#endif
  return load_se3(t);
}

PK_HD void store_se3(const SE3f& T, float* t) {
  t[0] = T.R.m[0]; t[1] = T.R.m[1]; t[2] = T.R.m[2];  t[3] = T.p.x;
  t[4] = T.R.m[3]; t[5] = T.R.m[4]; t[6] = T.R.m[5];  t[7] = T.p.y;
  t[8] = T.R.m[6]; t[9] = T.R.m[7]; t[10] = T.R.m[8]; t[11] = T.p.z;
}

// correctly rounded reciprocal without the slow path of the IEEE division
PK_HD float rcp_f(float x) {
#if defined(__CUDA_ARCH__)
  return __frcp_rn(x);
#else
  return 1.0f / x;
#endif
}

PK_HD void sincos_f(float x, float* s, float* c) {
#if defined(__CUDA_ARCH__)
  sincosf(x, s, c);
#else
  *s = sinf(x);
  *c = cosf(x);
#endif
}

// Rotation about a unit axis: R = c I + s [a]x + (1 - c) a a^T.
PK_HD M3 rot_axis(V3 a, float s, float c) {
  const float t = 1.f - c;
  M3 R;
  R.m[0] = fmaf(t * a.x, a.x, c);
  R.m[1] = fmaf(t * a.x, a.y, -s * a.z);
  R.m[2] = fmaf(t * a.x, a.z, s * a.y);
  R.m[3] = fmaf(t * a.x, a.y, s * a.z);
  R.m[4] = fmaf(t * a.y, a.y, c);
  R.m[5] = fmaf(t * a.y, a.z, -s * a.x);
  R.m[6] = fmaf(t * a.x, a.z, -s * a.y);
  R.m[7] = fmaf(t * a.y, a.z, s * a.x);
  R.m[8] = fmaf(t * a.z, a.z, c);
  return R;
}

// Unit quaternion [x y z w] -> rotation (input normalised first, as the oracle).
PK_HD M3 quat_to_matrix(float x, float y, float z, float w) {
  const float n = 1.f / sqrtf(fmaf(x, x, fmaf(y, y, fmaf(z, z, w * w))));
  x *= n; y *= n; z *= n; w *= n;
  M3 R;
  R.m[0] = 1.f - 2.f * (y * y + z * z);
  R.m[1] = 2.f * (x * y - z * w);
  R.m[2] = 2.f * (x * z + y * w);
  R.m[3] = 2.f * (x * y + z * w);
  R.m[4] = 1.f - 2.f * (x * x + z * z);
  R.m[5] = 2.f * (y * z - x * w);
  R.m[6] = 2.f * (x * z - y * w);
  R.m[7] = 2.f * (y * z + x * w);
  R.m[8] = 1.f - 2.f * (x * x + y * y);
  return R;
}

// Result of the SO(3) log with the scalars the SE(3) maps need.
struct Log3 {
  V3 w;         // rotation vector
  float theta;  // |w|
  float a;      // a(theta) = 1/theta^2 - sin/(2 theta (1 - cos))  (= Jlog3 "alpha", log6 "beta")
  float adot;   // (1/theta) da/dtheta                               (= Jlog6 "beta dot")
};

// a(x = theta^2) = sum_n |B_{2n+2}| x^n / (2n+2)!   (radius of convergence (2 pi)^2)
PK_HD float series_a(float x) {
  float r = 3.3896803e-13f;
  r = fmaf(r, x, 1.3382537e-11f);
  r = fmaf(r, x, 5.2841901e-10f);
  r = fmaf(r, x, 2.0876757e-8f);
  r = fmaf(r, x, 8.2671958e-7f);
  r = fmaf(r, x, 3.3068783e-5f);
  r = fmaf(r, x, 1.3888889e-3f);
  r = fmaf(r, x, 8.3333333e-2f);
  return r;
}
// adot(x) = 2 da/dx
PK_HD float series_adot(float x) {
  float r = 7.f * 3.3896803e-13f;
  r = fmaf(r, x, 6.f * 1.3382537e-11f);
  r = fmaf(r, x, 5.f * 5.2841901e-10f);
  r = fmaf(r, x, 4.f * 2.0876757e-8f);
  r = fmaf(r, x, 3.f * 8.2671958e-7f);
  r = fmaf(r, x, 2.f * 3.3068783e-5f);
  r = fmaf(r, x, 1.3888889e-3f);
  return 2.f * r;
}

PK_HD Log3 log3(const M3& R) {
  Log3 L;
  // sin(theta) axis and cos(theta)
  const V3 sv = v3(0.5f * (R.m[7] - R.m[5]), 0.5f * (R.m[2] - R.m[6]), 0.5f * (R.m[3] - R.m[1]));
  const float s = sqrtf(dot(sv, sv));
  const float c = 0.5f * (R.m[0] + R.m[4] + R.m[8] - 1.f);
  const float theta = atan2f(s, c);
  L.theta = theta;
  const float x = theta * theta;
  if (c > -0.9f) {
    // theta / sin(theta), series when sin is tiny
    const float k = (s < 2e-2f) ? fmaf(x, fmaf(x, 7.f / 360.f, 1.f / 6.f), 1.f) : theta / s;
    L.w = k * sv;
  } else {
    // near pi: sin(theta) axis loses its direction; use the quaternion whose
    // largest vector component is taken from the diagonal (Shepperd).
    const float d0 = R.m[0], d1 = R.m[4], d2 = R.m[8];
    float qx, qy, qz, qw;
    if (d0 >= d1 && d0 >= d2) {
      const float r = sqrtf(fmaxf(1.f + d0 - d1 - d2, 0.f));
      const float f = 0.5f / r;
      qx = 0.5f * r; qy = (R.m[1] + R.m[3]) * f; qz = (R.m[2] + R.m[6]) * f; qw = (R.m[7] - R.m[5]) * f;
    } else if (d1 >= d2) {
      const float r = sqrtf(fmaxf(1.f - d0 + d1 - d2, 0.f));
      const float f = 0.5f / r;
      qx = (R.m[1] + R.m[3]) * f; qy = 0.5f * r; qz = (R.m[5] + R.m[7]) * f; qw = (R.m[2] - R.m[6]) * f;
    } else {
      const float r = sqrtf(fmaxf(1.f - d0 - d1 + d2, 0.f));
      const float f = 0.5f / r;
      qx = (R.m[2] + R.m[6]) * f; qy = (R.m[5] + R.m[7]) * f; qz = 0.5f * r; qw = (R.m[3] - R.m[1]) * f;
    }
    if (qw < 0.f) { qx = -qx; qy = -qy; qz = -qz; qw = -qw; }
    const float nv = sqrtf(fmaf(qx, qx, fmaf(qy, qy, qz * qz)));
    const float th = 2.f * atan2f(nv, qw);
    const float k = th / nv;
    L.w = v3(k * qx, k * qy, k * qz);
    L.theta = th;
  }
  if (theta < 2.f) {
    L.a = series_a(x);
    L.adot = series_adot(x);
  } else {
    const float th = L.theta;
    const float x2 = th * th;
    const float cot_half = s / (1.f - c);  // cot(theta/2)
    L.a = (1.f - 0.5f * th * cot_half) / x2;
    // -2/theta^4 + (1 + sin/theta) / (2 theta^2 (1 - cos))
    L.adot = -2.f / (x2 * x2) + (1.f + s / th) / (2.f * x2 * (1.f - c));
  }
  return L;
}

// log6: body twist e = [v; w] of T, v = alpha p - 1/2 w x p + a (w.p) w with
// alpha = 1 - theta^2 a.
PK_HD void log6(const SE3f& T, const Log3& L, float e[6]) {
  const float alpha = fmaf(-L.theta * L.theta, L.a, 1.f);
  const float wp = dot(L.w, T.p);
  const V3 v = alpha * T.p - 0.5f * cross(L.w, T.p) + (L.a * wp) * L.w;
  e[0] = v.x; e[1] = v.y; e[2] = v.z;
  e[3] = L.w.x; e[4] = L.w.y; e[5] = L.w.z;
}

// Jlog6(T) = [[A, B], [0, A]], A = a w w^T + (1 - theta^2 a) I + 1/2 [w]x, B = C A,
// C = v3 w^T + a w p^T + a (w.p) I + 1/2 [p]x, v3 = adot (w.p) w - (theta^2 adot + 2 a) p.
PK_HD void jlog6_ac(const SE3f& T, const Log3& L, M3& A, M3& C);
PK_HD void jlog6(const SE3f& T, const Log3& L, M3& A, M3& B) {
  M3 C;
  jlog6_ac(T, L, A, C);
  B = mul(C, A);
}
// The factors A and C of Jlog6 (B = C A), for callers that fold C into their own products.
PK_HD void jlog6_ac(const SE3f& T, const Log3& L, M3& A, M3& C) {
  const V3 w = L.w, p = T.p;
  const float x = L.theta * L.theta;
  const float d = fmaf(-x, L.a, 1.f);
  A.m[0] = fmaf(L.a * w.x, w.x, d);
  A.m[1] = fmaf(L.a * w.x, w.y, -0.5f * w.z);
  A.m[2] = fmaf(L.a * w.x, w.z, 0.5f * w.y);
  A.m[3] = fmaf(L.a * w.y, w.x, 0.5f * w.z);
  A.m[4] = fmaf(L.a * w.y, w.y, d);
  A.m[5] = fmaf(L.a * w.y, w.z, -0.5f * w.x);
  A.m[6] = fmaf(L.a * w.z, w.x, -0.5f * w.y);
  A.m[7] = fmaf(L.a * w.z, w.y, 0.5f * w.x);
  A.m[8] = fmaf(L.a * w.z, w.z, d);
  const float wp = dot(w, p);
  const V3 v3_ = (L.adot * wp) * w - fmaf(x, L.adot, 2.f * L.a) * p;
  const float di = L.a * wp;
  C.m[0] = fmaf(v3_.x, w.x, fmaf(L.a * w.x, p.x, di));
  C.m[1] = fmaf(v3_.x, w.y, fmaf(L.a * w.x, p.y, -0.5f * p.z));
  C.m[2] = fmaf(v3_.x, w.z, fmaf(L.a * w.x, p.z, 0.5f * p.y));
  C.m[3] = fmaf(v3_.y, w.x, fmaf(L.a * w.y, p.x, 0.5f * p.z));
  C.m[4] = fmaf(v3_.y, w.y, fmaf(L.a * w.y, p.y, di));
  C.m[5] = fmaf(v3_.y, w.z, fmaf(L.a * w.y, p.z, -0.5f * p.x));
  C.m[6] = fmaf(v3_.z, w.x, fmaf(L.a * w.z, p.x, -0.5f * p.y));
  C.m[7] = fmaf(v3_.z, w.y, fmaf(L.a * w.z, p.y, 0.5f * p.x));
  C.m[8] = fmaf(v3_.z, w.z, fmaf(L.a * w.z, p.z, di));
}

// q (+) v dt of one instance (Configuration.integrate, pink/configuration.py:273-283):
// free-flyer root on SE(3) (Pinocchio's [p, quaternion] convention), the joints after it
// on R.  `o` may alias `qi`.
PK_HD void integrate_configuration(int nq, int free_flyer, const float* qi,
                                   const float* vi, float dt, float* o) {
  int rq = 0, rv = 0;
  if (free_flyer) {
    rq = 7; rv = 6;
    // M <- M exp6(v dt): translation += R V(w) vlin, quaternion <- quaternion * exp(w/2)
    const M3 R = quat_to_matrix(qi[3], qi[4], qi[5], qi[6]);
    const V3 vl = dt * v3(vi[0], vi[1], vi[2]);
    const V3 w = dt * v3(vi[3], vi[4], vi[5]);
    const float x = dot(w, w);
    const float th = sqrtf(x);
    float b, c;  // (1 - cos)/th^2, (th - sin)/th^3
    if (th < 1e-2f) {
      b = 0.5f - x / 24.f + x * x / 720.f;
      c = 1.f / 6.f - x / 120.f + x * x / 5040.f;
    } else {
      float s, co;
      sincos_f(th, &s, &co);
      b = (1.f - co) / x;
      c = (th - s) / (x * th);
    }
    const V3 wv = cross(w, vl);
    const V3 t = vl + b * wv + c * cross(w, wv);
    const V3 p = mul(R, t);
    o[0] = qi[0] + p.x; o[1] = qi[1] + p.y; o[2] = qi[2] + p.z;
    float sh, ch;
    sincos_f(0.5f * th, &sh, &ch);
    const float k = th < 1e-4f ? 0.5f : sh / th;
    const float dx = k * w.x, dy = k * w.y, dz = k * w.z, dw = ch;
    const float n0 = rsqrtf(qi[3] * qi[3] + qi[4] * qi[4] + qi[5] * qi[5] + qi[6] * qi[6]);
    const float ax = qi[3] * n0, ay = qi[4] * n0, az = qi[5] * n0, aw = qi[6] * n0;
    float rx = aw * dx + ax * dw + ay * dz - az * dy;
    float ry = aw * dy - ax * dz + ay * dw + az * dx;
    float rz = aw * dz + ax * dy - ay * dx + az * dw;
    float rw = aw * dw - ax * dx - ay * dy - az * dz;
    const float n1 = rsqrtf(rx * rx + ry * ry + rz * rz + rw * rw);
    o[3] = rx * n1; o[4] = ry * n1; o[5] = rz * n1; o[6] = rw * n1;
  }
  for (int j = 0; j < nq - rq; ++j) o[rq + j] = fmaf(vi[rv + j], dt, qi[rq + j]);
}

// Per-step targets and records of a trajectory rollout (pk_rollout_trajectory_prepared); all
// zero for the fixed-target rollout.  The records are step-major: the row of instance i at
// step s is row s B + i.
struct Trajectory {
  int64_t target_step;  // floats from one step's targets rows to the next (0: the same rows)
  float* q;             // [n_steps][B][nq] q after each step, or null
  float* v;             // [n_steps][B][nv] velocity of each step (0 once frozen), or null
  int32_t* status;      // [n_steps][B] OR of the statuses up to each step, or null
};

// Records of step s of a trajectory from an instance's q / v rows (`n` threads from `lane`).
PK_HD void record_rows(const Trajectory& T, int s, int64_t B, int64_t i, int nq, int nv, const float* qrow,
                       const float* vrow, int st_all, bool frozen, int lane, int n) {
  const int64_t r = (int64_t)s * B + i;
  if (T.q)
    for (int k = lane; k < nq; k += n) T.q[r * nq + k] = qrow[k];
  if (T.v)
    for (int k = lane; k < nv; k += n) T.v[r * nv + k] = frozen ? 0.f : vrow[k];
  if (T.status && lane == 0) T.status[r] = st_all;
}

// The freeze rule of the rollouts: an instance whose statuses so far have one of these bits
// takes no further step.
PK_HD bool step_failed(int st_all, int safety_break) {
  return (st_all & (PK_STATUS_NO_SOLUTION | PK_STATUS_NOT_POSDEF)) || ((st_all & PK_STATUS_OUT_OF_LIMITS) && safety_break);
}

// Phase clocks of the chain kernel (compile-time switch PK_CHAIN_PHASE_CLOCKS, off in the
// product build, where PK_PHASE / PK_PHASE_FLAG expand to nothing).  Every warp keeps one
// record: %globaltimer (ns) and clock64 at each phase boundary, the largest value over its
// lanes (lanes that leave a stage early pass the next mark first), the SM it ran on and the
// stages at least one of its lanes entered.  CTAs take consecutive record slots in the order
// they start, so the records of consecutive launches (which overlap under PDL) never share a
// slot and come out grouped by launch.  Read back and reset by pk_chain_phase_records
// (scripts/chain_phases.py).
enum ChainPhase {
  kPhaseEntry = 0,     // kernel entry
  kPhaseAssembled,     // after ChainStep::assemble (limit check, FK, task rows, box)
  kPhaseCorner,        // after the corner test of BoxLSQChol::corner_start
  kPhaseClosedForm,    // after the closed-form releases (corner_start returned)
  kPhaseRounds,        // after the Cholesky rounds and polish
  kPhaseWaited,        // after griddepcontrol.wait and the re-read of the inputs
  kPhaseStored,        // after the last store
  kPhaseCount
};
enum ChainPhaseFlag { kFlagRelease1 = 1, kFlagRelease2 = 2, kFlagRounds = 4 };
struct ChainPhaseRecord {
  unsigned long long ns[kPhaseCount];
  unsigned long long clk[kPhaseCount];
  unsigned smid, flags;
};
constexpr int kChainPhaseMaxWarps = 65536;
#if defined(PK_CHAIN_PHASE_CLOCKS) && defined(__CUDACC__)
__device__ ChainPhaseRecord g_chain_phase[kChainPhaseMaxWarps];
__device__ unsigned g_chain_phase_ctas;  // CTAs that took a slot since the last read
#endif
#if defined(PK_CHAIN_PHASE_CLOCKS) && defined(__CUDA_ARCH__)
__device__ __forceinline__ unsigned& chain_phase_cta() {
  __shared__ unsigned slot;
  return slot;
}
__device__ __forceinline__ ChainPhaseRecord* chain_phase_record() {
  const unsigned w = chain_phase_cta() * ((blockDim.x + 31) / 32) + threadIdx.x / 32;
  return w < kChainPhaseMaxWarps ? &g_chain_phase[w] : nullptr;
}
// leader of the lanes active here
__device__ __forceinline__ bool chain_phase_leader() { return (threadIdx.x & 31) == (unsigned)(__ffs(__activemask()) - 1); }
__device__ __forceinline__ void chain_phase_mark(int k) {
  if (k == kPhaseEntry) {  // every thread of the CTA, before any returns
    if (threadIdx.x == 0) chain_phase_cta() = atomicAdd(&g_chain_phase_ctas, 1u);
    __syncthreads();
  }
  ChainPhaseRecord* r = chain_phase_record();
  if (!r || !chain_phase_leader()) return;
  unsigned long long ns, clk;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
  clk = clock64();
  if (k == kPhaseEntry) {
    unsigned sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    for (int j = 1; j < kPhaseCount; ++j) r->ns[j] = r->clk[j] = 0ull;
    r->ns[0] = ns;
    r->clk[0] = clk;
    r->smid = sm;
    r->flags = 0u;
    __threadfence_block();
  } else {
    atomicMax(&r->ns[k], ns);
    atomicMax(&r->clk[k], clk);
  }
}
__device__ __forceinline__ void chain_phase_flag(unsigned f) {
  ChainPhaseRecord* r = chain_phase_record();
  if (r && chain_phase_leader()) atomicOr(&r->flags, f);
}
#define PK_PHASE(k) ::pk::chain_phase_mark(::pk::k)
#define PK_PHASE_FLAG(f) ::pk::chain_phase_flag(::pk::f)
#else
#define PK_PHASE(k) ((void)0)
#define PK_PHASE_FLAG(f) ((void)0)
#endif

// max(m, n) that keeps a NaN: a NaN task error makes the whole error NaN (never <= tol).
PK_HD float err_max(float m, float n) { return (n > m || n != n) ? n : m; }

// Stop test of one step of a converge loop (pk_converge_prepared), for the step bodies that
// take it: in mask (bit t: task t of the problem), tol, last (s == max_steps); out the error,
// max over the tasks of mask of |e_t|_2 (unweighted, gain-free), whether the loop stops here
// (the step then returns before its QP), and the step's status (the same on every lane).
// The bodies take the test type as a template parameter: decide() is the stop rule, called
// where the error is known (the multi-start kernels pass a test that decides for a group).
struct ConvergeTest {
  unsigned mask;
  float tol;
  bool last;
  float err;
  bool stop;
  int status;
  PK_HD void decide(float e) {
    err = e;
    stop = e <= tol || last;
  }
};

// Order of the seeds of a multi-start group (pk_converge_multistart_prepared): seed a (error ea)
// comes before seed b when its error is smaller, a NaN error counting as +inf, ties going to the
// lower seed index.  The winner is the first seed in this order.
PK_HD bool seed_before(float ea, int a, float eb, int b) {
  ea = ea != ea ? INFINITY : ea;
  eb = eb != eb ? INFINITY : eb;
  return ea < eb || (ea == eb && a < b);
}

}  // namespace pk
