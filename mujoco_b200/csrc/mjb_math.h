// Small fixed-size fp64 algebra for the batched mj_step path.
//
// Everything here is __host__ __device__ so that the very same source is compiled by nvcc for
// sm_90a (the product) and by g++ for the test-only host emulation (tests/hostemu).
// The ORDER of floating-point operations is part of the contract: parity with the reference is
// defined against the operation order of reference src/engine/engine_inline.h and
// src/engine/engine_util_spatial.c (cited per function); builds use -fmad=false /
// -ffp-contract=off so no fused multiply-adds are introduced.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define MJB_HD __host__ __device__ __forceinline__
#define MJB_HDN __host__ __device__ __noinline__
#else
#define MJB_HD inline
#define MJB_HDN
#endif

namespace mjb {

constexpr double kMinVal = 1e-15;   // mjMINVAL  (reference include/mujoco/mjtype.h:27)
constexpr double kMaxVal = 1e10;    // mjMAXVAL
constexpr double kPi = 3.14159265358979323846;
constexpr double kMinMu = 1e-5;     // mjMINMU   (include/mujoco/mjmodel.h:25-32)
constexpr double kMinImp = 0.0001;  // mjMINIMP
constexpr double kMaxImp = 0.9999;  // mjMAXIMP

struct V3 { double x, y, z; };
struct Q4 { double w, x, y, z; };
struct M3 { double m[9]; };         // row-major rotation / frame
struct S6 { double v[6]; };         // spatial vector (rotation : translation)
struct I10 { double v[10]; };       // spatial inertia in the reference's 10-vector packing

MJB_HD double dmax(double a, double b) { return a > b ? a : b; }   // mju_max
MJB_HD double dmin(double a, double b) { return a < b ? a : b; }   // mju_min
MJB_HD double dclip(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }
MJB_HD bool is_bad(double x) { return (x != x) || x > kMaxVal || x < -kMaxVal; }  // mju_isBad

MJB_HD V3 v3(double x, double y, double z) { return V3{x, y, z}; }
MJB_HD V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
MJB_HD V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
MJB_HD V3 operator*(V3 a, double s) { return V3{a.x * s, a.y * s, a.z * s}; }
MJB_HD V3 neg(V3 a) { return V3{-a.x, -a.y, -a.z}; }
// a + b*s   (mji_addScl3)
MJB_HD V3 addscl(V3 a, V3 b, double s) { return V3{a.x + s * b.x, a.y + s * b.y, a.z + s * b.z}; }
MJB_HD double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
MJB_HD V3 cross(V3 a, V3 b) {
  return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
MJB_HD double get(V3 a, int k) { return k == 0 ? a.x : (k == 1 ? a.y : a.z); }

// normalise in place, return the length before normalisation; degenerate -> (1,0,0)
// (engine_inline.h:125-139 mji__normalize3 / engine_util_blas.c mju_normalize3)
MJB_HD double normalize(V3& a) {
  double n = sqrt(a.x * a.x + a.y * a.y + a.z * a.z);
  if (n < kMinVal) {
    a = V3{1, 0, 0};
  } else {
    double inv = 1 / n;
    a.x *= inv; a.y *= inv; a.z *= inv;
  }
  return n;
}

// quaternion normalise: identity when degenerate, untouched when already unit to 1e-15
// (engine_inline.h:228-247)
MJB_HD double normalize(Q4& q) {
  double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  if (n < kMinVal) {
    q = Q4{1, 0, 0, 0};
  } else if (fabs(n - 1) > kMinVal) {
    double inv = 1 / n;
    q.w *= inv; q.x *= inv; q.y *= inv; q.z *= inv;
  }
  return n;
}

MJB_HD bool is_identity(Q4 q) { return q.w == 1 && q.x == 0 && q.y == 0 && q.z == 0; }

// rotate vector by quaternion (engine_inline.h:252-272)
MJB_HD V3 rotate(V3 v, Q4 q) {
  if (is_identity(q)) return v;
  V3 t;
  t.x = q.w * v.x + q.y * v.z - q.z * v.y;
  t.y = q.w * v.y + q.z * v.x - q.x * v.z;
  t.z = q.w * v.z + q.x * v.y - q.y * v.x;
  V3 r;
  r.x = v.x + 2 * (q.y * t.z - q.z * t.y);
  r.y = v.y + 2 * (q.z * t.x - q.x * t.z);
  r.z = v.z + 2 * (q.x * t.y - q.y * t.x);
  return r;
}

// quaternion product (engine_inline.h:286-294)
MJB_HD Q4 qmul(Q4 a, Q4 b) {
  Q4 r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
  r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
  return r;
}
MJB_HD Q4 qconj(Q4 q) { return Q4{q.w, -q.x, -q.y, -q.z}; }

// axis-angle -> quaternion (engine_inline.h:308-326)
MJB_HD Q4 axis_angle(V3 axis, double angle) {
  if (angle == 0) return Q4{1, 0, 0, 0};
  double s = sin(angle * 0.5);
  Q4 r;
  r.w = cos(angle * 0.5);
  r.x = axis.x * s; r.y = axis.y * s; r.z = axis.z * s;
  return r;
}

// orientation difference quaternion -> 3-D velocity over dt (engine_inline.h:330-343)
MJB_HD V3 quat2vel(Q4 q, double dt) {
  V3 axis{q.x, q.y, q.z};
  double s = normalize(axis);
  double speed = 2 * atan2(s, q.w);
  if (speed > kPi) speed -= 2 * kPi;
  speed /= dt;
  return axis * speed;
}
// qb * quat(res) = qa   (engine_inline.h:347-356)
MJB_HD V3 qsub(Q4 qa, Q4 qb) { return quat2vel(qmul(qconj(qb), qa), 1); }

// integrate a unit quaternion by angular velocity * scale (engine_inline.h:400-414)
MJB_HD Q4 qintegrate(Q4 q, V3 vel, double scale) {
  V3 ax = vel;
  double angle = scale * normalize(ax);
  Q4 qrot = axis_angle(ax, angle);
  normalize(q);
  return qmul(q, qrot);
}

// quaternion -> rotation matrix (engine_util_spatial.c:145-183)
MJB_HD M3 quat2mat(Q4 q) {
  M3 r;
  if (is_identity(q)) {
    r.m[0] = 1; r.m[1] = 0; r.m[2] = 0; r.m[3] = 0; r.m[4] = 1; r.m[5] = 0; r.m[6] = 0; r.m[7] = 0; r.m[8] = 1;
    return r;
  }
  double q00 = q.w * q.w, q01 = q.w * q.x, q02 = q.w * q.y, q03 = q.w * q.z;
  double q11 = q.x * q.x, q12 = q.x * q.y, q13 = q.x * q.z;
  double q22 = q.y * q.y, q23 = q.y * q.z, q33 = q.z * q.z;
  r.m[0] = q00 + q11 - q22 - q33;
  r.m[4] = q00 - q11 + q22 - q33;
  r.m[8] = q00 - q11 - q22 + q33;
  r.m[1] = 2 * (q12 - q03);
  r.m[2] = 2 * (q13 + q02);
  r.m[3] = 2 * (q12 + q03);
  r.m[5] = 2 * (q23 - q01);
  r.m[6] = 2 * (q13 - q02);
  r.m[7] = 2 * (q23 + q01);
  return r;
}

// mat * vec  (engine_inline.h:147-153)
MJB_HD V3 mulmv(const M3& a, V3 v) {
  return V3{a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z,
            a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z,
            a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z};
}
MJB_HD V3 col(const M3& a, int k) { return V3{a.m[k], a.m[3 + k], a.m[6 + k]}; }
MJB_HD V3 row(const M3& a, int k) { return V3{a.m[3 * k], a.m[3 * k + 1], a.m[3 * k + 2]}; }

// spatial inertia about an offset point (engine_util_spatial.c:405-435 mju_inertCom)
MJB_HD I10 inert_com(V3 inertia, const M3& R, V3 dif, double mass) {
  const double* mat = R.m;
  double t[9] = {mat[0] * inertia.x, mat[3] * inertia.x, mat[6] * inertia.x,
                 mat[1] * inertia.y, mat[4] * inertia.y, mat[7] * inertia.y,
                 mat[2] * inertia.z, mat[5] * inertia.z, mat[8] * inertia.z};
  I10 r;
  r.v[0] = mat[0] * t[0] + mat[1] * t[3] + mat[2] * t[6];
  r.v[1] = mat[3] * t[1] + mat[4] * t[4] + mat[5] * t[7];
  r.v[2] = mat[6] * t[2] + mat[7] * t[5] + mat[8] * t[8];
  r.v[3] = mat[0] * t[1] + mat[1] * t[4] + mat[2] * t[7];
  r.v[4] = mat[0] * t[2] + mat[1] * t[5] + mat[2] * t[8];
  r.v[5] = mat[3] * t[2] + mat[4] * t[5] + mat[5] * t[8];
  r.v[0] += mass * (dif.y * dif.y + dif.z * dif.z);
  r.v[1] += mass * (dif.x * dif.x + dif.z * dif.z);
  r.v[2] += mass * (dif.x * dif.x + dif.y * dif.y);
  r.v[3] -= mass * dif.x * dif.y;
  r.v[4] -= mass * dif.x * dif.z;
  r.v[5] -= mass * dif.y * dif.z;
  r.v[6] = mass * dif.x;
  r.v[7] = mass * dif.y;
  r.v[8] = mass * dif.z;
  r.v[9] = mass;
  return r;
}

// 10-vector inertia times spatial vector (engine_util_spatial.c:439-446)
MJB_HD S6 mul_inert(const I10& I, const S6& s) {
  const double* i = I.v; const double* v = s.v;
  S6 r;
  r.v[0] = i[0] * v[0] + i[3] * v[1] + i[4] * v[2] - i[8] * v[4] + i[7] * v[5];
  r.v[1] = i[3] * v[0] + i[1] * v[1] + i[5] * v[2] + i[8] * v[3] - i[6] * v[5];
  r.v[2] = i[4] * v[0] + i[5] * v[1] + i[2] * v[2] - i[7] * v[3] + i[6] * v[4];
  r.v[3] = i[8] * v[1] - i[7] * v[2] + i[9] * v[3];
  r.v[4] = i[6] * v[2] - i[8] * v[0] + i[9] * v[4];
  r.v[5] = i[7] * v[0] - i[6] * v[1] + i[9] * v[5];
  return r;
}

// 6-D dot in mju_dot's accumulation order (engine_inline.h:462-468)
MJB_HD double dot6(const S6& a, const S6& b) {
  return ((a.v[0] * b.v[0] + a.v[2] * b.v[2]) + (a.v[1] * b.v[1] + a.v[3] * b.v[3])) +
         (a.v[4] * b.v[4] + a.v[5] * b.v[5]);
}

// spatial motion cross product vel x v (engine_inline.h:428-441)
MJB_HD S6 cross_motion(const S6& a, const S6& b) {
  const double* vel = a.v; const double* v = b.v;
  S6 r;
  r.v[0] = -vel[2] * v[1] + vel[1] * v[2];
  r.v[1] = vel[2] * v[0] - vel[0] * v[2];
  r.v[2] = -vel[1] * v[0] + vel[0] * v[1];
  r.v[3] = -vel[2] * v[4] + vel[1] * v[5];
  r.v[4] = vel[2] * v[3] - vel[0] * v[5];
  r.v[5] = -vel[1] * v[3] + vel[0] * v[4];
  r.v[3] += -vel[5] * v[1] + vel[4] * v[2];
  r.v[4] += vel[5] * v[0] - vel[3] * v[2];
  r.v[5] += -vel[4] * v[0] + vel[3] * v[1];
  return r;
}

// spatial force cross product vel x* f (engine_inline.h:445-458)
MJB_HD S6 cross_force(const S6& a, const S6& b) {
  const double* vel = a.v; const double* f = b.v;
  S6 r;
  r.v[0] = -vel[2] * f[1] + vel[1] * f[2];
  r.v[1] = vel[2] * f[0] - vel[0] * f[2];
  r.v[2] = -vel[1] * f[0] + vel[0] * f[1];
  r.v[3] = -vel[2] * f[4] + vel[1] * f[5];
  r.v[4] = vel[2] * f[3] - vel[0] * f[5];
  r.v[5] = -vel[1] * f[3] + vel[0] * f[4];
  r.v[0] += -vel[5] * f[4] + vel[4] * f[5];
  r.v[1] += vel[5] * f[3] - vel[3] * f[5];
  r.v[2] += -vel[4] * f[3] + vel[3] * f[4];
  return r;
}

// complete a contact frame whose first row is the normal and second row an optional tangent hint
// (engine_util_spatial.c:512-538 mju_makeFrame)
MJB_HD void make_frame(M3& f) {
  V3 xa = row(f, 0);
  normalize(xa);
  V3 ya = row(f, 1);
  if (dot(ya, ya) < 0.25) {
    ya = V3{0, 0, 0};
    if (xa.y < 0.5 && xa.y > -0.5) ya.y = 1; else ya.z = 1;
  }
  V3 t = xa * dot(xa, ya);
  ya = ya - t;
  normalize(ya);
  V3 za = cross(xa, ya);
  f.m[0] = xa.x; f.m[1] = xa.y; f.m[2] = xa.z;
  f.m[3] = ya.x; f.m[4] = ya.y; f.m[5] = ya.z;
  f.m[6] = za.x; f.m[7] = za.y; f.m[8] = za.z;
}

// polynomial spring/damper coefficient and its x-derivative (engine_util_misc.c:2311-2340)
MJB_HD double poly_force(double linear, const double* poly, int n, double x, bool odd) {
  x = odd ? fabs(x) : x;
  double res = linear, xp = 1;
  for (int i = 0; i < n; i++) { xp *= x; res += poly[i] * xp; }
  return res;
}
MJB_HD double d_xpoly_force(double linear, const double* poly, int n, double x, bool odd) {
  x = odd ? fabs(x) : x;
  double res = linear, xp = 1;
  for (int i = 0; i < n; i++) { xp *= x; res += (i + 2) * poly[i] * xp; }
  return res;
}

// mju_round (engine_util_misc.c:1752): nearest integer, halves away from zero, saturating at the int range
MJB_HD int round_int(double x) {
  if (x > 2147483647.0) return 2147483647;
  if (x < -2147483648.0) return (-2147483647 - 1);
  return (int)round(x);
}

// mju_mulQuatAxis / mju_derivQuat (engine_util_spatial.c:81-92, :225-230)
MJB_HD Q4 qmul_axis(Q4 q, V3 a) {
  return Q4{-q.x * a.x - q.y * a.y - q.z * a.z, q.w * a.x + q.y * a.z - q.z * a.y,
            q.w * a.y + q.z * a.x - q.x * a.z, q.w * a.z + q.x * a.y - q.y * a.x};
}
MJB_HD Q4 deriv_quat(Q4 q, V3 v) {
  return Q4{0.5 * (-v.x * q.x - v.y * q.y - v.z * q.z), 0.5 * (v.x * q.w + v.y * q.z - v.z * q.y),
            0.5 * (-v.x * q.z + v.y * q.w + v.z * q.x), 0.5 * (v.x * q.y - v.y * q.x + v.z * q.w)};
}

// PCG32 (engine_solver.c:240-255): the PGS sweep order must match the reference draw for draw
struct Pcg32 { uint64_t state, inc; };
MJB_HD uint32_t pcg32_next(Pcg32& r) {
  uint64_t old = r.state;
  r.state = old * 6364136223846793005ULL + (r.inc | 1);
  uint32_t xs = (uint32_t)(((old >> 18u) ^ old) >> 27u);
  uint32_t rot = (uint32_t)(old >> 59u);
  return (xs >> rot) | (xs << ((0u - rot) & 31));
}

}  // namespace mjb
