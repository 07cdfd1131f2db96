// Convex narrow phase of the batched mj_step path: the reference's native GJK / EPA
// (src/engine/engine_collision_gjk.c) with the support functions and the contact drivers of
// src/engine/engine_collision_convex.c, for the primitive pairs the reference dispatches to mjc_Convex and
// mjc_PlaneConvex (engine_collision_driver.c:45-56): plane-ellipsoid, and sphere / capsule / ellipsoid /
// cylinder / box against an ellipsoid, capsule / cylinder / box against a cylinder.
//
// Restated in this library's idiom, operation for operation (fp64, no FMA contraction), so the results are the
// reference's bit for bit.  Representation differences:
//   - the support function is chosen by a switch on the geom type, not through function pointers;
//   - the polytope lives in a per-environment scratch slot (Env::ccd_poly) and refers to faces by index;
//   - the horizon walk (engine_collision_gjk.c:1285-1305, recursive there) keeps its own explicit stack;
//   - the status holds one witness pair: for these pairs mjc_Convex asks for one contact per call
//     (maxContacts, engine_collision_convex.c:855-877), so multicontact is never reached;
//   - the horizon arrays, a fixed 24 entries in the reference, hold 6N like the face map, so a wide horizon cannot
//     overrun them;
//   - neither operand of these pairs is a mesh and a box only ever meets a smooth geom, so the "discrete geoms"
//     branches (zero GJK tolerance, repeated-vertex test in EPA) never apply and are left out.
//
// Included by mjb_collision.h after PreCon and mulmTv3, which it uses.
#pragma once
#include "mjb_types.h"

namespace mjb {

constexpr double kMaxLimit = 1.7976931348623157e308;   // mjMAX_LIMIT (DBL_MAX), engine_collision_gjk.h:39
constexpr double kMinVal2 = kMinVal * kMinVal;           // mjMINVAL2 = mjMINDIST2/3/4 in double precision
constexpr double kMaxVal2 = kMaxVal * kMaxVal;
constexpr int kCcdSlots = 4;   // polytope slots per environment: convex candidates run in rounds of this many lanes

// doubles of one polytope slot at N = ccd_iterations: (5+N) vertices of 9 doubles, 6N faces of 7 doubles, and 4 int
// arrays of 6N (face map, horizon faces, horizon edges, horizon-walk stack) = 12N doubles.  18000 bytes at N = 35.
MJB_HD long ccd_slot_doubles(int n) { return 9L * (5 + n) + 42L * n + 12L * n; }
constexpr int kCcdConDbl = 1 + 5 * 7;   // stored pre-contacts of one convex candidate: count, then (dist, pos, normal) x 5

// a point of the Minkowski difference and the two support points it came from (Vertex, engine_collision_gjk.h:63-69)
struct CcdVert { V3 vert, vert1, vert2; };
// a polytope face (Face, engine_collision_gjk.c:74-80): vertex indices packed 10 bits each, adjacent faces per edge,
// the projection of the origin on the face, its squared norm, and the position in the face map (-1: not in the map,
// -2: deleted)
struct CcdFace { V3 v; double dist2; int verts; int adj[3]; int index; int pad; };

// a geom as the convex solver sees it (mjCCDObj, engine_collision_convex.c:726-810); `shape` is the support
// function: the geom's own, or the point / segment a sphere / capsule shrinks to (mjc_ccd, engine_collision_gjk.c:2330-2356)
enum { CCD_GEOM = 0, CCD_POINT = 1, CCD_LINE = 2 };
struct CcdObj { V3 pos; M3 mat; const double* size; int type; int shape; double margin; };

struct CcdStatus {
  CcdVert simplex[4];
  int nsimplex, nx, separated, iters, max_iterations;
  double tolerance, dist_cutoff, dist;
  V3 x1, x2;
};

// scratch polytope (Polytope, engine_collision_gjk.c:90-105) over one slot of Env::ccd_poly
struct CcdPoly {
  CcdVert* verts;
  CcdFace* faces;
  int *map, *hidx, *hedge, *stack;
  int nverts, nfaces, maxfaces, nmap, nedges;
  V3 center;
  V3 w;   // the point the horizon is seen from
};

MJB_HD double det3(V3 a, V3 b, V3 c) {
  return a.x * (b.y * c.z - b.z * c.y) + a.y * (b.z * c.x - b.x * c.z) + a.z * (b.x * c.y - b.y * c.x);
}
MJB_HD V3 scl(V3 a, double s) { return V3{s * a.x, s * a.y, s * a.z}; }

// ---- support functions (engine_collision_convex.c:200-344) ---------------------------------------------------------
MJB_HD V3 ccd_support_geom(const CcdObj& o, V3 dir) {
  const M3& m = o.mat;
  const double* s = o.size;
  if (o.shape == CCD_POINT) return o.pos;
  if (o.shape == CCD_LINE) {
    const double d = m.m[2] * dir.x + m.m[5] * dir.y + m.m[8] * dir.z;
    const double sc = d >= 0 ? s[1] : -s[1];
    return V3{m.m[2] * sc + o.pos.x, m.m[5] * sc + o.pos.y, m.m[8] * sc + o.pos.z};
  }
  if (o.type == GEOM_SPHERE) return V3{s[0] * dir.x + o.pos.x, s[0] * dir.y + o.pos.y, s[0] * dir.z + o.pos.z};
  const V3 ld = mulmTv3(m, dir);
  V3 ls;
  if (o.type == GEOM_CAPSULE) {
    ls = V3{ld.x * s[0], ld.y * s[0], ld.z * s[0]};
    ls.z += (ld.z >= 0 ? s[1] : -s[1]);
  } else if (o.type == GEOM_ELLIPSOID) {
    ls = V3{ld.x * s[0], ld.y * s[1], ld.z * s[2]};
    const double n2 = ls.x * ls.x + ls.y * ls.y + ls.z * ls.z;
    if (n2 < kMinVal2) return V3{m.m[0] * s[0] + o.pos.x, m.m[3] * s[0] + o.pos.y, m.m[6] * s[0] + o.pos.z};
    const double inv = 1 / sqrt(n2);
    ls.x *= inv * s[0]; ls.y *= inv * s[1]; ls.z *= inv * s[2];
  } else if (o.type == GEOM_CYLINDER) {
    const double n2 = ld.x * ld.x + ld.y * ld.y;
    const double sc = n2 >= kMinVal2 ? s[0] / sqrt(n2) : 0;
    ls = V3{sc * ld.x, sc * ld.y, ld.z >= 0 ? s[1] : -s[1]};
  } else {   // box
    ls = V3{ld.x >= 0 ? s[0] : -s[0], ld.y >= 0 ? s[1] : -s[1], ld.z >= 0 ? s[2] : -s[2]};
  }
  return mulmv(m, ls) + o.pos;
}

// support point of the Minkowski difference, each geom inflated by half the margin (engine_collision_gjk.c:336-362)
MJB_HD CcdVert ccd_support(const CcdObj& o1, const CcdObj& o2, V3 dir, V3 dir_neg) {
  CcdVert v;
  v.vert1 = ccd_support_geom(o1, dir);
  if (o1.margin > 0) { const double h = 0.5 * o1.margin; v.vert1.x += dir.x * h; v.vert1.y += dir.y * h; v.vert1.z += dir.z * h; }
  v.vert2 = ccd_support_geom(o2, dir_neg);
  if (o2.margin > 0) { const double h = 0.5 * o2.margin; v.vert2.x += dir_neg.x * h; v.vert2.y += dir_neg.y * h; v.vert2.z += dir_neg.z * h; }
  v.vert = v.vert1 - v.vert2;
  return v;
}

// ---- GJK distance sub-algorithm (Montanari et al.; engine_collision_gjk.c:481-849) -------------------------------
MJB_HD V3 lincomb(const double* c, int n, V3 a, V3 b, V3 e, V3 f) {
  switch (n) {
    case 1: return V3{c[0] * a.x, c[0] * a.y, c[0] * a.z};
    case 2: return V3{c[0] * a.x + c[1] * b.x, c[0] * a.y + c[1] * b.y, c[0] * a.z + c[1] * b.z};
    case 3: return V3{c[0] * a.x + c[1] * b.x + c[2] * e.x, c[0] * a.y + c[1] * b.y + c[2] * e.y,
                      c[0] * a.z + c[1] * b.z + c[2] * e.z};
    case 4: return V3{c[0] * a.x + c[1] * b.x + c[2] * e.x + c[3] * f.x, c[0] * a.y + c[1] * b.y + c[2] * e.y + c[3] * f.y,
                      c[0] * a.z + c[1] * b.z + c[2] * e.z + c[3] * f.z};
  }
  return V3{0, 0, 0};
}

// projection of the origin on the plane through v1, v2, v3; 1 when the triangle is degenerate
MJB_HD int project_origin_plane(V3& res, V3 v1, V3 v2, V3 v3) {
  const V3 d21 = v2 - v1, d31 = v3 - v1, d32 = v3 - v2;
  V3 n = cross(d32, d21);
  double nv = dot(n, v2), nn = dot(n, n);
  if (nn == 0) return 1;
  if (nv != 0 && nn > kMinVal) { res = scl(n, nv / nn); return 0; }
  n = cross(d21, d31);
  nv = dot(n, v1); nn = dot(n, n);
  if (nn == 0) return 1;
  if (nv != 0 && nn > kMinVal) { res = scl(n, nv / nn); return 0; }
  n = cross(d31, d32);
  nv = dot(n, v3); nn = dot(n, n);
  res = scl(n, nv / nn);
  return 0;
}

MJB_HD int same_sign(double a, double b) { return (a > 0 && b > 0) ? 1 : ((a < 0 && b < 0) ? -1 : 0); }

MJB_HD void gjk_s1d(double* lam, V3 s1, V3 s2) {
  const V3 diff = s2 - s1;
  const double sc = -(dot(s2, diff) / dot(diff, diff));
  const V3 p{s2.x + sc * diff.x, s2.y + sc * diff.y, s2.z + sc * diff.z};
  double mu_max = s1.x - s2.x;
  int idx = 0;
  double mu = s1.y - s2.y;
  if (fabs(mu) >= fabs(mu_max)) { mu_max = mu; idx = 1; }
  mu = s1.z - s2.z;
  if (fabs(mu) >= fabs(mu_max)) { mu_max = mu; idx = 2; }
  const double c1 = get(p, idx) - get(s2, idx), c2 = get(s1, idx) - get(p, idx);
  const bool in = same_sign(mu_max, c1) && same_sign(mu_max, c2);
  lam[0] = in ? c1 / mu_max : 0;
  lam[1] = in ? c2 / mu_max : 1;
}

// signed area of the 2-D triangle (p, a, b) as the reference expands it
MJB_HD double area2(double px, double py, double ax, double ay, double bx, double by) {
  return px * ay + py * bx + ax * by - px * by - py * ax - bx * ay;
}

// the two coordinates kept when the triangle s1 s2 s3 is projected on its largest shadow, and that shadow's minor
MJB_HD double tri_minor(V3 s1, V3 s2, V3 s3, int& x, int& y) {
  const double m14 = s2.y * s3.z - s2.z * s3.y - s1.y * s3.z + s1.z * s3.y + s1.y * s2.z - s1.z * s2.y;
  const double m24 = s2.x * s3.z - s2.z * s3.x - s1.x * s3.z + s1.z * s3.x + s1.x * s2.z - s1.z * s2.x;
  const double m34 = s2.x * s3.y - s2.y * s3.x - s1.x * s3.y + s1.y * s3.x + s1.x * s2.y - s1.y * s2.x;
  const double mu1 = fabs(m14), mu2 = fabs(m24), mu3 = fabs(m34);
  if (mu1 >= mu2 && mu1 >= mu3) { x = 1; y = 2; return m14; }
  if (mu2 >= mu3) { x = 0; y = 2; return m24; }
  x = 0; y = 1; return m34;
}

MJB_HD void gjk_s2d(double* lam, V3 s1, V3 s2, V3 s3) {
  V3 p;
  if (project_origin_plane(p, s1, s2, s3)) { gjk_s1d(lam, s1, s2); lam[2] = 0; return; }
  int x, y;
  const double mmax = tri_minor(s1, s2, s3, x, y);
  const double px = get(p, x), py = get(p, y);
  const double c31 = area2(px, py, get(s2, x), get(s2, y), get(s3, x), get(s3, y));
  const double c32 = area2(px, py, get(s3, x), get(s3, y), get(s1, x), get(s1, y));
  const double c33 = area2(px, py, get(s1, x), get(s1, y), get(s2, x), get(s2, y));
  const int k1 = same_sign(mmax, c31), k2 = same_sign(mmax, c32), k3 = same_sign(mmax, c33);
  if (k1 && k2 && k3) { lam[0] = c31 / mmax; lam[1] = c32 / mmax; lam[2] = c33 / mmax; return; }
  double dmin = kMaxLimit, l[2];
  if (!k1) {
    gjk_s1d(l, s2, s3);
    const V3 q = lincomb(l, 2, s2, s3, s3, s3);
    lam[0] = 0; lam[1] = l[0]; lam[2] = l[1];
    dmin = dot(q, q);
  }
  if (!k2) {
    gjk_s1d(l, s1, s3);
    const V3 q = lincomb(l, 2, s1, s3, s3, s3);
    const double dd = dot(q, q);
    if (dd < dmin) { lam[0] = l[0]; lam[1] = 0; lam[2] = l[1]; dmin = dd; }
  }
  if (!k3) {
    gjk_s1d(l, s1, s2);
    const V3 q = lincomb(l, 2, s1, s2, s2, s2);
    const double dd = dot(q, q);
    if (dd < dmin) { lam[0] = l[0]; lam[1] = l[1]; lam[2] = 0; }
  }
}

MJB_HD void gjk_s3d(double* lam, V3 s1, V3 s2, V3 s3, V3 s4) {
  const double c41 = -det3(s2, s3, s4), c42 = det3(s1, s3, s4), c43 = -det3(s1, s2, s4), c44 = det3(s1, s2, s3);
  const double mdet = c41 + c42 + c43 + c44;
  const int k1 = same_sign(mdet, c41), k2 = same_sign(mdet, c42), k3 = same_sign(mdet, c43), k4 = same_sign(mdet, c44);
  if (k1 && k2 && k3 && k4) { lam[0] = c41 / mdet; lam[1] = c42 / mdet; lam[2] = c43 / mdet; lam[3] = c44 / mdet; return; }
  double dmin = kMaxLimit, l[3];
  if (!k1) {
    gjk_s2d(l, s2, s3, s4);
    const V3 q = lincomb(l, 3, s2, s3, s4, s4);
    lam[0] = 0; lam[1] = l[0]; lam[2] = l[1]; lam[3] = l[2];
    dmin = dot(q, q);
  }
  if (!k2) {
    gjk_s2d(l, s1, s3, s4);
    const V3 q = lincomb(l, 3, s1, s3, s4, s4);
    const double dd = dot(q, q);
    if (dd < dmin) { lam[0] = l[0]; lam[1] = 0; lam[2] = l[1]; lam[3] = l[2]; dmin = dd; }
  }
  if (!k3) {
    gjk_s2d(l, s1, s2, s4);
    const V3 q = lincomb(l, 3, s1, s2, s4, s4);
    const double dd = dot(q, q);
    if (dd < dmin) { lam[0] = l[0]; lam[1] = l[1]; lam[2] = 0; lam[3] = l[2]; dmin = dd; }
  }
  if (!k4) {
    gjk_s2d(l, s1, s2, s3);
    const V3 q = lincomb(l, 3, s1, s2, s3, s3);
    const double dd = dot(q, q);
    if (dd < dmin) { lam[0] = l[0]; lam[1] = l[1]; lam[2] = l[2]; lam[3] = 0; }
  }
}

MJB_HD void gjk_subdistance(double* lam, int n, const CcdVert* s) {
  lam[0] = lam[1] = lam[2] = lam[3] = 0;
  if (n == 4) gjk_s3d(lam, s[0].vert, s[1].vert, s[2].vert, s[3].vert);
  else if (n == 3) gjk_s2d(lam, s[0].vert, s[1].vert, s[2].vert);
  else if (n == 2) gjk_s1d(lam, s[0].vert, s[1].vert);
  else lam[0] = 1;
}

// ---- GJK (engine_collision_gjk.c:198-332) and its tetrahedron intersection fallback (:406-477) -------------------
MJB_HD CcdVert gjk_support(const CcdObj& o1, const CcdObj& o2, V3 xk, double xnorm) {
  const V3 dn = scl(xk, 1 / xnorm);
  return ccd_support(o1, o2, scl(dn, -1), dn);
}

// signed distance of the face (v1, v2, v3) to the origin along its unit normal; kMaxLimit when degenerate
MJB_HD double face_signed_dist(V3& n, V3 v1, V3 v2, V3 v3) {
  n = cross(v3 - v1, v2 - v1);
  const double n2 = dot(n, n);
  if (n2 > kMinVal2 && n2 < kMaxVal2) { n = scl(n, 1 / sqrt(n2)); return dot(n, v1); }
  return kMaxLimit;
}

// 1: contact, 0: separated, -1: inconclusive
MJB_HD int gjk_intersect(CcdStatus& st, const CcdObj& o1, const CcdObj& o2) {
  CcdVert s[4] = {st.simplex[0], st.simplex[1], st.simplex[2], st.simplex[3]};
  int ix[4] = {0, 1, 2, 3};
  int k = st.iters;
  for (; k < st.max_iterations; k++) {
    double dist[4];
    V3 nrm[4];
    dist[0] = face_signed_dist(nrm[0], s[ix[2]].vert, s[ix[1]].vert, s[ix[3]].vert);
    dist[1] = face_signed_dist(nrm[1], s[ix[0]].vert, s[ix[2]].vert, s[ix[3]].vert);
    dist[2] = face_signed_dist(nrm[2], s[ix[1]].vert, s[ix[0]].vert, s[ix[3]].vert);
    dist[3] = face_signed_dist(nrm[3], s[ix[0]].vert, s[ix[1]].vert, s[ix[2]].vert);
    if (!dist[3] || !dist[2] || !dist[1] || !dist[0]) { st.iters = k; return -1; }
    int i = (dist[0] < dist[1]) ? 0 : 1;
    int j = (dist[2] < dist[3]) ? 2 : 3;
    const int best = (dist[i] < dist[j]) ? i : j;
    if (dist[best] > 0) {
      st.nsimplex = 4;
      for (int q = 0; q < 4; q++) st.simplex[q] = s[ix[q]];
      st.iters = k;
      return 1;
    }
    s[ix[best]] = ccd_support(o1, o2, nrm[best], neg(nrm[best]));
    if (dot(nrm[best], s[ix[best]].vert) < 0) { st.nsimplex = 0; st.iters = k; return 0; }
    i = (best + 1) & 3;
    j = (best + 2) & 3;
    const int t = ix[i]; ix[i] = ix[j]; ix[j] = t;
  }
  st.iters = k;
  return -1;
}

MJB_HD void gjk(CcdStatus& st, const CcdObj& o1, const CcdObj& o2) {
  const bool get_dist = st.dist_cutoff > 0;
  bool backup = !get_dist;
  CcdVert* sx = st.simplex;
  int n = 0, k = 0;
  double lam[4] = {0, 0, 0, 0};
  const double tol2 = st.tolerance * st.tolerance;
  st.separated = 0;
  const double eps = 0.5 * tol2, min_norm = st.tolerance;
  V3 xk = st.x1 - st.x2;
  double xnorm = sqrt(dot(xk, xk)), xnorm_prev = 0;
  for (; k < st.max_iterations; k++) {
    if (xnorm < min_norm || fabs(xnorm_prev - xnorm) < kMinVal) break;
    sx[n] = gjk_support(o1, o2, xk, xnorm);
    const V3 sk = sx[n].vert;
    if (dot(xk, xk - sk) < eps) break;
    const double lower = dot(xk, sk);
    if (!get_dist) {
      if (lower > 0) { st.separated = 1; st.iters = k; st.nsimplex = 0; st.nx = 0; st.dist = kMaxLimit; return; }
    } else if (st.dist_cutoff < kMaxLimit) {
      if (lower > 0 && lower >= st.dist_cutoff * xnorm) {
        st.separated = 1; st.iters = k; st.nsimplex = 0; st.nx = 0; st.dist = kMaxLimit; return;
      }
    }
    if (n == 3 && backup) {
      st.iters = k;
      const int r = gjk_intersect(st, o1, o2);
      if (r != -1) { st.nx = 0; st.separated = r == 0; st.dist = r > 0 ? 0 : kMaxLimit; return; }
      k = st.iters;
      backup = false;
    }
    gjk_subdistance(lam, n + 1, sx);
    n = 0;
    for (int i = 0; i < 4; i++) {
      if (!lam[i]) continue;
      sx[n] = sx[i];
      lam[n++] = lam[i];
    }
    if (n < 1) { st.iters = k; st.nsimplex = 0; st.nx = 0; st.dist = kMaxLimit; st.separated = 1; return; }
    xk = lincomb(lam, n, sx[0].vert, sx[1].vert, sx[2].vert, sx[3].vert);
    xnorm_prev = xnorm;
    xnorm = sqrt(dot(xk, xk));
    if (n == 4) break;
  }
  if (n > 0) {
    st.x1 = lincomb(lam, n, sx[0].vert1, sx[1].vert1, sx[2].vert1, sx[3].vert1);
    st.x2 = lincomb(lam, n, sx[0].vert2, sx[1].vert2, sx[2].vert2, sx[3].vert2);
  }
  const CcdVert t = gjk_support(o1, o2, xk, xnorm);   // final separation check
  if (dot(xk, t.vert) > 0) st.separated = 1;
  st.nx = 1;
  st.iters = k;
  st.nsimplex = n;
  st.dist = (n == 4 && !st.separated) ? 0 : xnorm;
}

// ---- EPA polytope (engine_collision_gjk.c:855-1305) ----------------------------------------------------------------
MJB_HD int poly_support(CcdPoly& pt, const CcdObj& o1, const CcdObj& o2, V3 d, double dnorm) {
  V3 dir{1, 0, 0}, dneg{-1, 0, 0};
  if (dnorm > kMinVal) { dir = V3{d.x / dnorm, d.y / dnorm, d.z / dnorm}; dneg = scl(dir, -1); }
  const int n = pt.nverts++;
  pt.verts[n] = ccd_support(o1, o2, dir, dneg);
  return n;
}
MJB_HD int poly_insert(CcdPoly& pt, const CcdVert& v) { const int n = pt.nverts++; pt.verts[n] = v; return n; }

// attach the face (v1, v2, v3) with its three neighbours; its squared distance to the origin (0: degenerate)
MJB_HD double poly_attach(CcdPoly& pt, int v1, int v2, int v3, int a1, int a2, int a3) {
  CcdFace& f = pt.faces[pt.nfaces++];
  f.verts = v1 + (v2 << 10) + (v3 << 20);
  f.adj[0] = a1; f.adj[1] = a2; f.adj[2] = a3;
  if (project_origin_plane(f.v, pt.verts[v3].vert, pt.verts[v2].vert, pt.verts[v1].vert)) return 0;
  if (dot(f.v, pt.verts[v1].vert - pt.center) < 0) f.v = scl(f.v, -1);
  f.dist2 = dot(f.v, f.v);
  f.index = -1;
  return f.dist2;
}
MJB_HD int face_vert(int packed, int k) { return (packed >> (10 * k)) & 0x3FF; }

MJB_HD void poly_map_all(CcdPoly& pt, int n) {
  for (int i = 0; i < n; i++) { pt.map[i] = i; pt.faces[i].index = i; }
  pt.nmap = n;
}

MJB_HD void poly_reset_to_triangle(CcdPoly& pt, CcdStatus& st, int a, int b, int c) {
  st.nsimplex = 3;
  st.simplex[0] = pt.verts[a]; st.simplex[1] = pt.verts[b]; st.simplex[2] = pt.verts[c];
  pt.nfaces = 0; pt.nverts = 0; pt.nmap = 0;
}

MJB_HD int same_side(V3 p0, V3 p1, V3 p2, V3 p3) {
  const V3 n = cross(p1 - p0, p2 - p0);
  const double d1 = dot(n, p3 - p0), d2 = dot(n, scl(p0, -1));
  return (d1 > 0 && d2 > 0) || (d1 < 0 && d2 < 0);
}
MJB_HD int origin_in_tetra(V3 p0, V3 p1, V3 p2, V3 p3) {
  return same_side(p0, p1, p2, p3) && same_side(p1, p2, p3, p0) && same_side(p2, p3, p0, p1) && same_side(p3, p0, p1, p2);
}

// affine coordinates of p on the triangle v1 v2 v3 (:1022-1063)
MJB_HD void tri_affine(double* lam, V3 v1, V3 v2, V3 v3, V3 p) {
  int x, y;
  const double mmax = tri_minor(v1, v2, v3, x, y);
  const double px = get(p, x), py = get(p, y);
  lam[0] = area2(px, py, get(v2, x), get(v2, y), get(v3, x), get(v3, y)) / mmax;
  lam[1] = area2(px, py, get(v3, x), get(v3, y), get(v1, x), get(v1, y)) / mmax;
  lam[2] = area2(px, py, get(v1, x), get(v1, y), get(v2, x), get(v2, y)) / mmax;
}
MJB_HD int tri_point(V3 v1, V3 v2, V3 v3, V3 p) {
  double l[3];
  tri_affine(l, v1, v2, v3, p);
  if (l[0] < 0 || l[1] < 0 || l[2] < 0) return 0;
  const V3 pr{v1.x * l[0] + v2.x * l[1] + v3.x * l[2], v1.y * l[0] + v2.y * l[1] + v3.y * l[2],
              v1.z * l[0] + v2.z * l[1] + v3.z * l[2]};
  const V3 df = pr - p;
  return sqrt(dot(df, df)) < kMinVal;
}

// hexahedron around a 2-simplex (:1084-1164); 0 on success
MJB_HD int polytope3(CcdPoly& pt, CcdStatus& st, const CcdObj& o1, const CcdObj& o2) {
  const V3 v1 = st.simplex[0].vert, v2 = st.simplex[1].vert, v3 = st.simplex[2].vert;
  pt.center = scl((v1 + v2) + v3, 1.0 / 3.0);
  const V3 n = cross(v2 - v1, v3 - v1);
  const double nn = sqrt(dot(n, n));
  if (nn < kMinVal) return 3;
  const V3 nneg = scl(n, -1);
  const int i1 = poly_insert(pt, st.simplex[0]), i2 = poly_insert(pt, st.simplex[1]), i3 = poly_insert(pt, st.simplex[2]);
  const int i5 = poly_support(pt, o1, o2, nneg, nn);
  const int i4 = poly_support(pt, o1, o2, n, nn);
  const V3 v4 = pt.verts[i4].vert, v5 = pt.verts[i5].vert;
  if (tri_point(v1, v2, v3, v4)) return 4;
  if (tri_point(v1, v2, v3, v5)) return 5;
  if (st.dist > 10 * kMinVal && !origin_in_tetra(v1, v2, v3, v4) && !origin_in_tetra(v1, v2, v3, v5)) return 6;
  if (poly_attach(pt, i4, i1, i2, 1, 3, 2) < kMinVal2) return 7;
  if (poly_attach(pt, i4, i3, i1, 2, 4, 0) < kMinVal2) return 7;
  if (poly_attach(pt, i4, i2, i3, 0, 5, 1) < kMinVal2) return 7;
  if (poly_attach(pt, i5, i2, i1, 5, 0, 4) < kMinVal2) return 7;
  if (poly_attach(pt, i5, i1, i3, 3, 1, 5) < kMinVal2) return 7;
  if (poly_attach(pt, i5, i3, i2, 4, 2, 3) < kMinVal2) return 7;
  poly_map_all(pt, 6);
  return 0;
}

// 120-degree rotation about an axis (:899-913)
MJB_HD M3 rot120(V3 axis) {
  const double n = sqrt(dot(axis, axis));
  const double u1 = axis.x / n, u2 = axis.y / n, u3 = axis.z / n;
  const double sn = 0.86602540378, cs = -0.5;
  M3 r;
  r.m[0] = cs + u1 * u1 * (1 - cs); r.m[1] = u1 * u2 * (1 - cs) - u3 * sn; r.m[2] = u1 * u3 * (1 - cs) + u2 * sn;
  r.m[3] = u2 * u1 * (1 - cs) + u3 * sn; r.m[4] = cs + u2 * u2 * (1 - cs); r.m[5] = u2 * u3 * (1 - cs) - u1 * sn;
  r.m[6] = u1 * u3 * (1 - cs) - u2 * sn; r.m[7] = u2 * u3 * (1 - cs) + u1 * sn; r.m[8] = cs + u3 * u3 * (1 - cs);
  return r;
}

MJB_HD int ray_triangle(V3 v1, V3 v2, V3 v3, V3 v4, V3 v5) {
  const V3 d12 = v2 - v1, d13 = v3 - v1, d14 = v4 - v1, d15 = v5 - v1;
  const double a = det3(d13, d14, d12), b = det3(d14, d15, d12), c = det3(d15, d13, d12);
  if (a >= 0 && b >= 0 && c >= 0) return 1;
  if (a <= 0 && b <= 0 && c <= 0) return -1;
  return 0;
}

// hexahedron around a 1-simplex (:936-1018), falling back to polytope3 when the origin lies on a face
MJB_HD int polytope2(CcdPoly& pt, CcdStatus& st, const CcdObj& o1, const CcdObj& o2) {
  const V3 v1 = st.simplex[0].vert, v2 = st.simplex[1].vert;
  pt.center = scl(v1 + v2, 0.5);
  const V3 diff = v2 - v1;
  double value = kMaxLimit;
  int idx = 0;
  for (int i = 0; i < 3; i++) if (fabs(get(diff, i)) < value) { value = fabs(get(diff, i)); idx = i; }
  const V3 e{idx == 0 ? 1.0 : 0.0, idx == 1 ? 1.0 : 0.0, idx == 2 ? 1.0 : 0.0};
  const V3 d1 = cross(e, diff);
  const M3 R = rot120(diff);
  const V3 d2 = mulmv(R, d1), d3 = mulmv(R, d2);
  const int i1 = poly_insert(pt, st.simplex[0]), i2 = poly_insert(pt, st.simplex[1]);
  const int i3 = poly_support(pt, o1, o2, d1, sqrt(dot(d1, d1)));
  const int i4 = poly_support(pt, o1, o2, d2, sqrt(dot(d2, d2)));
  const int i5 = poly_support(pt, o1, o2, d3, sqrt(dot(d3, d3)));
  const V3 v3 = pt.verts[i3].vert, v4 = pt.verts[i4].vert, v5 = pt.verts[i5].vert;
  const int fv[6][6] = {{i1, i3, i4, 1, 3, 2}, {i1, i5, i3, 2, 4, 0}, {i1, i4, i5, 0, 5, 1},
                        {i2, i4, i3, 5, 0, 4}, {i2, i3, i5, 3, 1, 5}, {i2, i5, i4, 4, 2, 3}};
  for (int f = 0; f < 6; f++) {
    if (poly_attach(pt, fv[f][0], fv[f][1], fv[f][2], fv[f][3], fv[f][4], fv[f][5]) < kMinVal2) {
      poly_reset_to_triangle(pt, st, fv[f][0], fv[f][1], fv[f][2]);
      return polytope3(pt, st, o1, o2);
    }
  }
  if (!ray_triangle(v1, v2, v3, v4, v5)) return 2;
  poly_map_all(pt, 6);
  return 0;
}

// tetrahedron of a 3-simplex (:1168-1210), falling back to polytope3 when the origin lies on a face
MJB_HD int polytope4(CcdPoly& pt, CcdStatus& st, const CcdObj& o1, const CcdObj& o2) {
  const int a = poly_insert(pt, st.simplex[0]), b = poly_insert(pt, st.simplex[1]);
  const int c = poly_insert(pt, st.simplex[2]), e = poly_insert(pt, st.simplex[3]);
  pt.center = scl(((pt.verts[a].vert + pt.verts[b].vert) + pt.verts[c].vert) + pt.verts[e].vert, 0.25);
  const int fv[4][6] = {{a, b, c, 1, 3, 2}, {a, e, b, 2, 3, 0}, {a, c, e, 0, 3, 1}, {e, c, b, 2, 0, 1}};
  for (int f = 0; f < 4; f++) {
    if (poly_attach(pt, fv[f][0], fv[f][1], fv[f][2], fv[f][3], fv[f][4], fv[f][5]) < kMinVal2) {
      poly_reset_to_triangle(pt, st, fv[f][0], fv[f][1], fv[f][2]);
      return polytope3(pt, st, o1, o2);
    }
  }
  if (!origin_in_tetra(pt.verts[a].vert, pt.verts[b].vert, pt.verts[c].vert, pt.verts[e].vert)) return 8;
  poly_map_all(pt, 4);
  return 0;
}

MJB_HD void poly_delete(CcdPoly& pt, int f) {
  CcdFace& face = pt.faces[f];
  if (face.index >= 0) {
    pt.map[face.index] = pt.map[--pt.nmap];
    pt.faces[pt.map[face.index]].index = face.index;
  }
  face.index = -2;
}
MJB_HD void poly_add_edge(CcdPoly& pt, int f, int e) { pt.hedge[pt.nedges] = e; pt.hidx[pt.nedges++] = f; }
MJB_HD int edge_of(const CcdFace& f, int v) { return face_vert(f.verts, 0) == v ? 0 : (face_vert(f.verts, 1) == v ? 1 : 2); }
MJB_HD bool poly_visible(const CcdPoly& pt, int f) { return dot(pt.faces[f].v, pt.w) - pt.faces[f].dist2 > kMinVal; }

// horizonRec (:1285-1305) with an explicit stack: a visible face is deleted and its two other edges are walked in
// order, each neighbour that is not visible contributing a horizon edge; 1 when f0 was visible
MJB_HD int poly_horizon_walk(CcdPoly& pt, int f0, int e0) {
  if (!poly_visible(pt, f0)) return 0;
  poly_delete(pt, f0);
  int sp = 0;
  pt.stack[sp++] = (f0 << 4) | (e0 << 2) | 1;   // face, the edge it was entered by, next k in {1, 2, 3 = done}
  while (sp > 0) {
    const int top = pt.stack[sp - 1];
    const int f = top >> 4, e = (top >> 2) & 3, k = top & 3;
    if (k == 3) {
      sp--;
      if (sp > 0) pt.stack[sp - 1]++;   // the child was visible: no edge, the parent moves to its next edge
      continue;
    }
    const int i = (e + k) % 3;
    const int adj = pt.faces[f].adj[i];
    if (pt.faces[adj].index > -2) {
      const int ae = edge_of(pt.faces[adj], face_vert(pt.faces[f].verts, (i + 1) % 3));
      if (poly_visible(pt, adj)) {
        poly_delete(pt, adj);
        pt.stack[sp++] = (adj << 4) | (ae << 2) | 1;
        continue;
      }
      poly_add_edge(pt, adj, ae);
    }
    pt.stack[sp - 1]++;
  }
  return 1;
}

MJB_HD void poly_horizon(CcdPoly& pt, int f) {
  poly_delete(pt, f);
  const int packed = pt.faces[f].verts;
  int adj = pt.faces[f].adj[0];
  int ae = edge_of(pt.faces[adj], face_vert(packed, 1));
  if (!poly_horizon_walk(pt, adj, ae)) poly_add_edge(pt, adj, ae);
  adj = pt.faces[f].adj[1];
  ae = edge_of(pt.faces[adj], face_vert(packed, 2));
  if (pt.faces[adj].index > -2 && !poly_horizon_walk(pt, adj, ae)) poly_add_edge(pt, adj, ae);
  adj = pt.faces[f].adj[2];
  ae = edge_of(pt.faces[adj], face_vert(packed, 0));
  if (pt.faces[adj].index > -2 && !poly_horizon_walk(pt, adj, ae)) poly_add_edge(pt, adj, ae);
}

// EPA (:1358-1505): expand towards the face nearest the origin until its support bound closes; the witness points of
// that face go to st.x1 / st.x2 and minus its distance to st.dist
MJB_HD void epa(CcdStatus& st, CcdPoly& pt, const CcdObj& o1, const CcdObj& o2) {
  double upper = kMaxLimit, upper2 = kMaxLimit, lower2;
  int face = -1, pface = -1;
  const double tol = st.tolerance;
  const int kmax = st.max_iterations < 1000 ? st.max_iterations : 1000;
  for (int k = 0; k < kmax; k++) {
    pface = face;
    lower2 = kMaxLimit;
    for (int i = 0; i < pt.nmap; i++) {
      if (pt.faces[pt.map[i]].dist2 < lower2) { face = pt.map[i]; lower2 = pt.faces[face].dist2; }
    }
    if (lower2 > upper2 || face < 0) { face = pface; break; }
    if (lower2 <= 0) break;   // origin on the affine hull of a face (the reference warns)
    const double lower = sqrt(lower2);
    const int wi = poly_support(pt, o1, o2, pt.faces[face].v, lower);
    const double upper_k = dot(pt.faces[face].v, pt.verts[wi].vert) / lower;
    if (upper_k < upper) { upper = upper_k; upper2 = upper * upper; }
    if (upper - lower < tol) {
      if (k == 0 && upper < lower - 1e-10) face = -1;
      break;
    }
    pt.w = pt.verts[wi].vert;
    poly_horizon(pt, face);
    if (pt.nedges < 3) { face = -1; break; }
    const int nfaces = pt.nfaces, nedges = pt.nedges;
    if (nedges > pt.maxfaces - pt.nfaces) break;   // out of face memory (the reference warns)
    for (int i = 0; i < nedges; i++) {
      const int cur = nfaces + i;
      const int prev = i == 0 ? nfaces + nedges - 1 : cur - 1;
      const int next = nfaces + (i + 1) % nedges;
      const int hf = pt.hidx[i], he = pt.hedge[i];
      const int hv = pt.faces[hf].verts;
      const int a = face_vert(hv, he), b = face_vert(hv, (he + 1) % 3);
      pt.faces[hf].adj[he] = cur;
      const double d2 = poly_attach(pt, wi, b, a, prev, hf, next);
      if (d2 == 0) { face = -1; break; }
      if (d2 >= lower2 && d2 <= upper2) {
        const int m = pt.nmap++;
        pt.map[m] = pt.nfaces - 1;
        pt.faces[pt.nfaces - 1].index = m;
      }
    }
    pt.nedges = 0;
    if (!pt.nmap || face < 0) break;
  }
  if (face >= 0) {
    const CcdFace& f = pt.faces[face];
    const CcdVert& a = pt.verts[face_vert(f.verts, 0)];
    const CcdVert& b = pt.verts[face_vert(f.verts, 1)];
    const CcdVert& c = pt.verts[face_vert(f.verts, 2)];
    double lam[3];
    tri_affine(lam, a.vert, b.vert, c.vert, f.v);
    st.x1 = lincomb(lam, 3, a.vert1, b.vert1, c.vert1, c.vert1);
    st.x2 = lincomb(lam, 3, a.vert2, b.vert2, c.vert2, c.vert2);
    st.dist = -sqrt(f.dist2);
    st.nx = 1;
  } else {
    st.nx = 0;
    st.dist = 0;
  }
}

// ---- mjc_ccd (engine_collision_gjk.c:2318-2442) with one contact requested ------------------------------------------
MJB_HD double ccd(CcdStatus& st, CcdObj& o1, CcdObj& o2, double* scratch, int niter, double tolerance) {
  st.x1 = o1.pos;
  st.x2 = o2.pos;
  st.iters = 0;
  st.tolerance = tolerance;
  st.max_iterations = niter;
  st.dist_cutoff = 0;
  st.nx = 0;
  st.nsimplex = 0;
  const bool shrink1 = o1.type == GEOM_SPHERE || o1.type == GEOM_CAPSULE;
  const bool shrink2 = o2.type == GEOM_SPHERE || o2.type == GEOM_CAPSULE;
  if (shrink1 || shrink2) {   // sphere -> point, capsule -> segment, their radius (+ half margin) added afterwards
    const double m1 = o1.margin, m2 = o2.margin;
    double full1 = 0, full2 = 0;
    if (shrink1) { full1 = o1.size[0] + 0.5 * m1; o1.shape = o1.type == GEOM_SPHERE ? CCD_POINT : CCD_LINE; o1.margin = 0; }
    if (shrink2) { full2 = o2.size[0] + 0.5 * m2; o2.shape = o2.type == GEOM_SPHERE ? CCD_POINT : CCD_LINE; o2.margin = 0; }
    st.dist_cutoff += full1 + full2;
    gjk(st, o1, o2);
    st.dist_cutoff = 0;
    o1.margin = m1; o2.margin = m2;
    o1.shape = CCD_GEOM; o2.shape = CCD_GEOM;
    if (st.dist > st.tolerance) {   // shallow: inflate the witness points (:2272-2287)
      V3 n = st.x2 - st.x1;
      normalize(n);
      if (full1) { st.x1.x += full1 * n.x; st.x1.y += full1 * n.y; st.x1.z += full1 * n.z; }
      if (full2) { st.x2.x -= full2 * n.x; st.x2.y -= full2 * n.y; st.x2.z -= full2 * n.z; }
      st.dist -= (full1 + full2);
      if (st.dist > st.dist_cutoff) st.dist = kMaxLimit;
      return st.dist;
    }
    st.iters = 0;   // deep penetration: GJK again on the full shapes
    st.x1 = o1.pos;
    st.x2 = o2.pos;
  }
  gjk(st, o1, o2);
  if (st.dist <= tolerance && st.nsimplex > 1 && !st.separated) {
    st.dist = 0;
    CcdPoly pt;
    pt.nfaces = pt.nmap = pt.nverts = pt.nedges = 0;
    pt.maxfaces = 6 * niter;
    pt.verts = (CcdVert*)scratch;
    pt.faces = (CcdFace*)(scratch + 9L * (5 + niter));
    int* ip = (int*)(scratch + 9L * (5 + niter) + 42L * niter);
    pt.map = ip; pt.hidx = ip + 6 * niter; pt.hedge = ip + 12 * niter; pt.stack = ip + 18 * niter;
    int ret;
    if (st.nsimplex == 2) ret = polytope2(pt, st, o1, o2);
    else if (st.nsimplex == 3) ret = polytope3(pt, st, o1, o2);
    else ret = polytope4(pt, st, o1, o2);
    if (!ret) epa(st, pt, o1, o2);
  }
  return st.dist;
}

// mjc_penetration, native branch (engine_collision_convex.c:87-133): at most one pre-contact
MJB_HD int ccd_penetration(PreCon& c, CcdObj& o1, CcdObj& o2, double margin, double* scratch, const DModel& m) {
  CcdStatus st;
  const double dist = ccd(st, o1, o2, scratch, m.opt.ccd_iterations, m.opt.ccd_tolerance);
  if (!(dist < 0) || st.nx < 1) return 0;
  c.dist = margin + st.dist;
  c.pos = st.x1 + st.x2;
  c.pos = scl(c.pos, 0.5);
  c.normal = st.x1 - st.x2;
  normalize(c.normal);
  c.tangent = V3{0, 0, 0};
  return 1;
}

// in-place rotation of a frame about a point (mju_rotateFrame, engine_collision_convex.c:834-851)
MJB_HD void rotate_frame(V3 origin, const M3& rot, M3& xmat, V3& xpos) {
  M3 r;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      r.m[3 * i + j] = rot.m[3 * i] * xmat.m[j] + rot.m[3 * i + 1] * xmat.m[3 + j] + rot.m[3 * i + 2] * xmat.m[6 + j];
  xmat = r;
  const V3 rel = origin - xpos;
  V3 vec = mulmv(rot, rel);
  vec = vec - rel;
  xpos = xpos - vec;
}

// mjc_Convex (engine_collision_convex.c:881-962) for pair p of the candidate table: the first contact, then - unless
// mjDSBL_MULTICCD is set or a sphere / ellipsoid takes part - up to four more from the geoms rotated by +-1e-3 rad
// about the contact's tangent axes, each kept only when it is distinct from every earlier point
MJB_HD int collide_convex(PreCon* c, const DModel& m, int g1, int g2, V3 p1, const M3& m1, V3 p2, const M3& m2,
                          double margin, double* scratch) {
  const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  CcdObj o1{p1, m1, m.geom_size + 3 * g1, t1, CCD_GEOM, margin};
  CcdObj o2{p2, m2, m.geom_size + 3 * g2, t2, CCD_GEOM, margin};
  int ncon = ccd_penetration(c[0], o1, o2, margin, scratch, m);
  if (ncon != 1 || (m.opt.disableflags & DSBL_MULTICCD) || t1 == GEOM_ELLIPSOID || t1 == GEOM_SPHERE ||
      t2 == GEOM_ELLIPSOID || t2 == GEOM_SPHERE)
    return ncon;
  M3 fr;
  fr.m[0] = c[0].normal.x; fr.m[1] = c[0].normal.y; fr.m[2] = c[0].normal.z;
  for (int k = 3; k < 9; k++) fr.m[k] = 0;
  make_frame(fr);
  const double tol = 1e-3 * dmin(m.geom_rbound[g1], m.geom_rbound[g2]);
  for (int ax = 0; ax < 2; ax++) {
    for (int an = 0; an < 2; an++) {
      const V3 axis = row(fr, 1 + ax);
      const M3 rot = quat2mat(axis_angle(axis, an ? 1e-3 : -1e-3));
      M3 inv;
      for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) inv.m[3 * i + j] = rot.m[3 * j + i];
      rotate_frame(c[0].pos, rot, o1.mat, o1.pos);
      rotate_frame(c[0].pos, inv, o2.mat, o2.pos);
      const int n = ccd_penetration(c[ncon], o1, o2, margin, scratch, m);
      bool distinct = n != 0;
      for (int i = 0; distinct && i < ncon; i++) {
        const V3 df = c[i].pos - c[ncon].pos;
        if (sqrt(df.x * df.x + df.y * df.y + df.z * df.z) <= tol) distinct = false;
      }
      if (distinct) { c[ncon].dist = c[0].dist; ncon++; }
      o1.pos = p1; o1.mat = m1; o2.pos = p2; o2.mat = m2;
    }
  }
  return ncon;
}

// mjc_PlaneConvex for an ellipsoid (engine_collision_convex.c:1004-1041): the ellipsoid's support point along the
// plane's -normal (mjccd_support, :518-721, with zero margin), one contact
MJB_HD int collide_plane_ellipsoid(PreCon& c, double margin, V3 p1, const M3& m1, V3 p2, const M3& m2, const double* s) {
  const V3 normal{m1.m[2], m1.m[5], m1.m[8]};
  const V3 dir{-m1.m[2], -m1.m[5], -m1.m[8]};
  const V3 ld = mulmTv3(m2, dir);
  V3 r{ld.x * s[0], ld.y * s[1], ld.z * s[2]};
  normalize(r);
  r.x *= s[0]; r.y *= s[1]; r.z *= s[2];
  r.x += ld.x * 0.0 / 2; r.y += ld.y * 0.0 / 2; r.z += ld.z * 0.0 / 2;   // + local_dir * margin / 2, margin 0
  r = mulmv(m2, r);
  r = r + p2;
  const V3 dif = r - p1;
  c.dist = dot(normal, dif);
  if (c.dist > margin) return 0;
  c.pos = r;
  c.pos.x += normal.x * (-0.5 * c.dist); c.pos.y += normal.y * (-0.5 * c.dist); c.pos.z += normal.z * (-0.5 * c.dist);
  c.normal = normal;
  c.tangent = V3{0, 0, 0};
  return 1;
}

// the pairs (t1 <= t2) that go through GJK / EPA
MJB_HD bool pair_gjk(int t1, int t2) {
  if (t2 == GEOM_ELLIPSOID) return t1 == GEOM_SPHERE || t1 == GEOM_CAPSULE || t1 == GEOM_ELLIPSOID;
  if (t2 == GEOM_CYLINDER) return t1 == GEOM_CAPSULE || t1 == GEOM_ELLIPSOID || t1 == GEOM_CYLINDER;
  if (t2 == GEOM_BOX) return t1 == GEOM_ELLIPSOID || t1 == GEOM_CYLINDER;
  return false;
}

}  // namespace mjb
