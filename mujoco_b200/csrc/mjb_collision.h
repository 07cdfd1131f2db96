// Collision detection of the batched mj_step path, one environment per call.
//
// The reference runs broadphase (PCA frame + sweep-and-prune), midphase (BVH/OBB) and narrowphase
// per step (src/engine/engine_collision_driver.c:595-886).  Every pruning stage there is
// conservative with respect to the final `dist < margin` decision, and the ORDER in which contacts
// are emitted is a pure function of the model (body-pair signature order, then the per-pair geom
// order, :637-745,410-443).  This implementation therefore walks a STATIC, host-precomputed
// candidate table (mjb_model.cc) in that order and applies, per candidate, exactly the
// reference's per-pair filter (bounding sphere / plane distance, :267-284,547-591) followed by the
// same closed-form colliders (src/engine/engine_collision_primitive.c:28-530) and mj_setContact
// (:1839-1875).  All environments of a warp walk the same table: no divergence in control flow
// except the hit/miss branches.
#pragma once
#include "mjb_types.h"

namespace mjb {

struct PreCon { double dist; V3 pos, normal, tangent; };

// plane : sphere, shared by plane-capsule  (engine_collision_primitive.c:28-50)
MJB_HD int raw_plane_sphere(PreCon& c, double margin, V3 ppos, const M3& pmat, V3 spos, double radius) {
  c.normal = V3{pmat.m[2], pmat.m[5], pmat.m[8]};
  V3 t = spos - ppos;
  double cdist = dot(t, c.normal);
  if (cdist > margin + radius) return 0;
  c.dist = cdist - radius;
  t = c.normal * (-c.dist / 2 - radius);
  c.pos = spos + t;
  c.tangent = V3{0, 0, 0};
  return 1;
}

// sphere : sphere kernel shared by the capsule colliders (engine_collision_primitive.c:246-285)
MJB_HD int raw_sphere_sphere(PreCon& c, double margin, V3 p1, const M3& m1, double r1, V3 p2, const M3& m2, double r2) {
  V3 dif = p1 - p2;
  double d2 = dot(dif, dif);
  double mind = margin + r1 + r2;
  if (d2 > mind * mind) return 0;
  c.dist = sqrt(d2) - r1 - r2;
  c.normal = p2 - p1;
  double len = normalize(c.normal);
  if (len < kMinVal) {
    V3 a1{m1.m[2], m1.m[5], m1.m[8]}, a2{m2.m[2], m2.m[5], m2.m[8]};
    c.normal = cross(a1, a2);
    normalize(c.normal);
  }
  c.pos = c.normal * (r1 + c.dist / 2);
  c.pos = c.pos + p1;
  c.tangent = V3{0, 0, 0};
  return 1;
}

MJB_HD int collide_plane_capsule(PreCon* c, double margin, V3 p1, const M3& m1, V3 p2, const M3& m2, const double* size2) {
  V3 axis{m2.m[2], m2.m[5], m2.m[8]};
  V3 seg{size2[1] * axis.x, size2[1] * axis.y, size2[1] * axis.z};
  int n1 = raw_plane_sphere(c[0], margin, p1, m1, p2 + seg, size2[0]);
  int n2 = raw_plane_sphere(c[n1], margin, p1, m1, p2 - seg, size2[0]);
  if (n1) c[0].tangent = axis;
  if (n2) c[n1].tangent = axis;
  return n1 + n2;
}

MJB_HD int collide_sphere_capsule(PreCon* c, double margin, V3 p1, const M3& m1, const double* size1,
                                  V3 p2, const M3& m2, const double* size2) {
  double len = size2[1];
  V3 axis{m2.m[2], m2.m[5], m2.m[8]};
  V3 vec = p1 - p2;
  double x = dclip(dot(axis, vec), -len, len);
  vec = axis * x;
  vec = vec + p2;
  return raw_sphere_sphere(c[0], margin, p1, m1, size1[0], vec, m2, size2[0]);
}

// capsule : capsule (engine_collision_primitive.c:431-518)
MJB_HD int collide_capsule_capsule(PreCon* c, double margin, V3 p1, const M3& m1, const double* size1,
                                   V3 p2, const M3& m2, const double* size2) {
  V3 ax1{m1.m[2] * size1[1], m1.m[5] * size1[1], m1.m[8] * size1[1]};
  V3 ax2{m2.m[2] * size2[1], m2.m[5] * size2[1], m2.m[8] * size2[1]};
  V3 dif = p1 - p2;
  double ma = dot(ax1, ax1), mb = -dot(ax1, ax2), mc = dot(ax2, ax2);
  double u = -dot(ax1, dif), v = dot(ax2, dif);
  double det = ma * mc - mb * mb;
  const double r1 = size1[0], r2 = size2[0];
  if (fabs(det) >= kMinVal) {
    double x1 = (mc * u - mb * v) / det;
    double x2 = (ma * v - mb * u) / det;
    if (x1 > 1) { x1 = 1; x2 = (v - mb) / mc; }
    else if (x1 < -1) { x1 = -1; x2 = (v + mb) / mc; }
    if (x2 > 1) { x2 = 1; x1 = dclip((u - mb) / ma, -1, 1); }
    else if (x2 < -1) { x2 = -1; x1 = dclip((u + mb) / ma, -1, 1); }
    V3 v1 = ax1 * x1; v1 = v1 + p1;
    V3 v2 = ax2 * x2; v2 = v2 + p2;
    return raw_sphere_sphere(c[0], margin, v1, m1, r1, v2, m2, r2);
  }
  // parallel axes: up to two contacts from the four end-point projections
  V3 v1 = p1 + ax1;
  double x2 = dclip((v - mb) / mc, -1, 1);
  V3 v2 = ax2 * x2; v2 = v2 + p2;
  int n1 = raw_sphere_sphere(c[0], margin, v1, m1, r1, v2, m2, r2);
  v1 = p1 - ax1;
  x2 = dclip((v + mb) / mc, -1, 1);
  v2 = ax2 * x2; v2 = v2 + p2;
  int n2 = raw_sphere_sphere(c[n1], margin, v1, m1, r1, v2, m2, r2);
  if (n1 + n2 >= 2) return n1 + n2;
  v2 = p2 + ax2;
  double x1 = dclip((u - mb) / ma, -1, 1);
  v1 = ax1 * x1; v1 = v1 + p1;
  int n3 = raw_sphere_sphere(c[n1 + n2], margin, v1, m1, r1, v2, m2, r2);
  if (n1 + n2 + n3 >= 2) return n1 + n2 + n3;
  v2 = p2 - ax2;
  x1 = dclip((u + mb) / ma, -1, 1);
  v1 = ax1 * x1; v1 = v1 + p1;
  int n4 = raw_sphere_sphere(c[n1 + n2 + n3], margin, v1, m1, r1, v2, m2, r2);
  return n1 + n2 + n3 + n4;
}

// ---- cylinder and box colliders (only in kernels compiled with FEAT_COLBOX) ------------------------------------
MJB_HD V3 mulmTv3(const M3& a, V3 v) {   // mji_mulMatTVec3
  return V3{a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z,
            a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z};
}

// plane : cylinder (engine_collision_primitive.c:101-208): the rim point nearest to the plane on either disk, plus
// two points at +-60 degrees on the nearer disk; up to four contacts
MJB_HD int collide_plane_cylinder(PreCon* c, double margin, V3 p1, const M3& m1, V3 p2, const M3& m2, const double* size2) {
  const V3 normal{m1.m[2], m1.m[5], m1.m[8]};
  V3 axis{m2.m[2], m2.m[5], m2.m[8]};
  double prjaxis = dot(normal, axis);
  if (prjaxis > 0) { axis = axis * -1.0; prjaxis = -prjaxis; }   // the axis points towards the plane
  V3 vec = p2 - p1;
  const double dist0 = dot(vec, normal);
  vec = axis * prjaxis;        // - normal, without its component along the axis
  vec = vec - normal;
  const double len_sqr = dot(vec, vec);
  if (len_sqr >= kMinVal * kMinVal) {
    const double scl = size2[0] / sqrt(len_sqr);
    vec.x *= scl; vec.y *= scl; vec.z *= scl;
  } else {                     // disk parallel to the plane: the cylinder's x axis
    vec = V3{m2.m[0] * size2[0], m2.m[3] * size2[0], m2.m[6] * size2[0]};
  }
  const double prjvec = dot(vec, normal);
  axis = axis * size2[1];
  prjaxis *= size2[1];
  int cnt = 0;
  auto put = [&](double dist, V3 pos) {
    c[cnt].dist = dist;
    pos.x += normal.x * (-dist * 0.5); pos.y += normal.y * (-dist * 0.5); pos.z += normal.z * (-dist * 0.5);
    c[cnt].pos = pos;
    c[cnt].normal = normal;
    c[cnt].tangent = V3{0, 0, 0};
    cnt++;
  };
  if (dist0 + prjaxis + prjvec <= margin) put(dist0 + prjaxis + prjvec, (p2 + vec) + axis);
  else return 0;
  if (dist0 - prjaxis + prjvec <= margin) put(dist0 - prjaxis + prjvec, (p2 + vec) - axis);
  const double prjvec1 = -prjvec * 0.5;
  if (dist0 + prjaxis + prjvec1 <= margin) {
    V3 vec1 = cross(vec, axis);
    normalize(vec1);
    vec1 = vec1 * (size2[0] * sqrt(3.0) / 2);
    const double dist = dist0 + prjaxis + prjvec1;
    V3 pa = (p2 + vec1) + axis;
    pa.x += vec.x * -0.5; pa.y += vec.y * -0.5; pa.z += vec.z * -0.5;
    put(dist, pa);
    V3 pb = (p2 - vec1) + axis;
    pb.x += vec.x * -0.5; pb.y += vec.y * -0.5; pb.z += vec.z * -0.5;
    put(dist, pb);
  }
  return cnt;
}

// plane : box (engine_collision_primitive.c:210-258): the corners below the margin that point down, at most four
MJB_HD int collide_plane_box(PreCon* c, double margin, V3 p1, const M3& m1, V3 p2, const M3& m2, const double* size2) {
  const V3 norm{m1.m[2], m1.m[5], m1.m[8]};
  const V3 dif = p2 - p1;
  const double dist = dot(dif, norm);
  int cnt = 0;
  for (int i = 0; i < 8; i++) {
    const V3 vec{(i & 1) ? size2[0] : -size2[0], (i & 2) ? size2[1] : -size2[1], (i & 4) ? size2[2] : -size2[2]};
    V3 corner = mulmv(m2, vec);
    const double ldist = dot(norm, corner);
    if (dist + ldist > margin || ldist > 0) continue;
    c[cnt].dist = dist + ldist;
    c[cnt].normal = norm;
    corner = corner + p2;
    c[cnt].pos = corner + norm * (-c[cnt].dist / 2);
    c[cnt].tangent = V3{0, 0, 0};
    if (++cnt >= 4) return 4;
  }
  return cnt;
}

// sphere : cylinder (engine_collision_primitive.c:345-423): side (sphere-sphere against the axis point), cap
// (plane-sphere against the cap plane) or rim (sphere-sphere against the rim point)
MJB_HD int collide_sphere_cylinder(PreCon* c, double margin, V3 p1, const M3& m1, const double* size1,
                                   V3 p2, const M3& m2, const double* size2) {
  const double radius = size2[0], height = size2[1];
  const V3 axis{m2.m[2], m2.m[5], m2.m[8]};
  V3 vec = p1 - p2;
  const double x = dot(axis, vec);
  V3 a_proj = axis * x;
  V3 p_proj = vec - a_proj;
  const double p_proj_sqr = dot(p_proj, p_proj);
  bool collide_side = fabs(x) < height;
  bool collide_cap = p_proj_sqr < radius * radius;
  if (collide_side && collide_cap) {   // centre inside the cylinder: keep the shallower exit
    const double dist_cap = height - fabs(x);
    const double dist_radius = radius - sqrt(p_proj_sqr);
    if (dist_cap < dist_radius) collide_side = false; else collide_cap = false;
  }
  if (collide_side) {
    a_proj = a_proj + p2;
    return raw_sphere_sphere(c[0], margin, p1, m1, size1[0], a_proj, m2, size2[0]);
  }
  if (collide_cap) {
    V3 pos_cap;
    M3 mat_cap = m2;
    if (x > 0) pos_cap = addscl(p2, axis, height);
    else {
      pos_cap = addscl(p2, axis, -height);
      mat_cap.m[0] = -m2.m[0]; mat_cap.m[2] = -m2.m[2]; mat_cap.m[3] = -m2.m[3]; mat_cap.m[5] = -m2.m[5];
      mat_cap.m[6] = -m2.m[6]; mat_cap.m[8] = -m2.m[8];
    }
    const int n = raw_plane_sphere(c[0], margin, pos_cap, mat_cap, p1, size1[0]);
    if (n) c[0].normal = c[0].normal * -1.0;   // the pair is (sphere, cylinder): the normal points from the sphere
    return n;
  }
  p_proj = p_proj * (size2[0] / sqrt(p_proj_sqr));
  vec = axis * (x > 0 ? height : -height);
  vec = vec + p_proj;
  vec = vec + p2;
  return raw_sphere_sphere(c[0], margin, p1, m1, size1[0], vec, m2, 0.0);
}

// sphere : box (engine_collision_box.c:35-95)
MJB_HD int raw_sphere_box(PreCon& c, double margin, V3 p1, double r1, V3 p2, const M3& m2, const double* size2) {
  V3 tmp = p1 - p2;
  const V3 center = mulmTv3(m2, tmp);
  V3 clamped = center;
  if (size2[0] > 0) clamped.x = dclip(clamped.x, -size2[0], size2[0]);
  if (size2[1] > 0) clamped.y = dclip(clamped.y, -size2[1], size2[1]);
  if (size2[2] > 0) clamped.z = dclip(clamped.z, -size2[2], size2[2]);
  V3 deepest = center;
  tmp = clamped - center;
  double dist = normalize(tmp);
  if (dist - r1 > margin) return 0;
  V3 pos;
  if (dist <= kMinVal) {   // sphere centre inside the box: leave through the nearest face
    double closest = (size2[0] + size2[1] + size2[2]) * 2;
    int k = 0;
    for (int i = 0; i < 6; i++) {
      const double v = fabs(((i % 2) ? 1 : -1) * size2[i / 2] - get(center, i / 2));
      if (closest > v) { closest = v; k = i; }
    }
    V3 nearest{0, 0, 0};
    const double sgn = (k % 2) ? -1 : 1;
    if (k / 2 == 0) nearest.x = sgn; else if (k / 2 == 1) nearest.y = sgn; else nearest.z = sgn;
    pos = center;
    const double s = (r1 - closest) / 2;
    pos.x += nearest.x * s; pos.y += nearest.y * s; pos.z += nearest.z * s;
    c.normal = mulmv(m2, nearest);
    dist = -closest;
  } else {
    deepest.x += tmp.x * r1; deepest.y += tmp.y * r1; deepest.z += tmp.z * r1;
    pos = V3{0, 0, 0};
    pos.x += clamped.x * 0.5; pos.y += clamped.y * 0.5; pos.z += clamped.z * 0.5;
    pos.x += deepest.x * 0.5; pos.y += deepest.y * 0.5; pos.z += deepest.z * 0.5;
    c.normal = mulmv(m2, tmp);
  }
  tmp = mulmv(m2, pos);
  c.pos = tmp + p2;
  c.dist = dist - r1;
  c.tangent = V3{0, 0, 0};
  return 1;
}

// capsule : box (engine_collision_box.c:110-590).  In the box frame: the point of the capsule's segment closest to
// the box (against the faces, then against the twelve edges by segment-segment distance), a sphere-box contact
// there, and - when the segment runs along a face or an edge - a second sphere-box contact at the far point of the
// segment that is still above the box.
MJB_HD int collide_capsule_box(PreCon* c, double margin, V3 p1, const M3& m1, const double* size1,
                               V3 p2, const M3& m2, const double* size2) {
  double tmp1[3], tmp2[3], tmp3[3], halfaxis[3], axis[3], dif[3], pos[3];
  const double halflength = size1[1];
  double secondpos = -4;   // no second contact (valid values are in [-1, 1])
  double bestsegmentpos, bestboxpos = 0, bestdist, dist, mul = 0, e1, e2, dp = 0, de = 0;
  int cltype = -4, clface = -1, clcorner = 0, cledge = 0, c1, c2, ax = 0, ax1 = 0, ax2 = 0;
  {
    const V3 t = mulmTv3(m2, p1 - p2);          // capsule centre in the box frame
    pos[0] = t.x; pos[1] = t.y; pos[2] = t.z;
    const V3 a = mulmTv3(m2, V3{m1.m[2], m1.m[5], m1.m[8]});
    axis[0] = a.x; axis[1] = a.y; axis[2] = a.z;
    for (int k = 0; k < 3; k++) halfaxis[k] = axis[k] * halflength;
  }
  int axisdir = 0;
  if (halfaxis[0] > 0) axisdir += 1;
  if (halfaxis[1] > 0) axisdir += 2;
  if (halfaxis[2] > 0) axisdir += 4;
  const double bestdistmax = margin + 2 * (size1[0] + halflength + size2[0] + size2[1] + size2[2]);
  bestdist = bestdistmax;
  bestsegmentpos = 0;
  // is an end of the segment closest to a face of the box?
  for (int i = -1; i <= 1; i += 2) {
    for (int k = 0; k < 3; k++) { tmp1[k] = pos[k]; tmp1[k] += halfaxis[k] * i; tmp2[k] = tmp1[k]; }
    c1 = 0; c2 = -1;
    for (int j = 0; j < 3; j++) {
      if (tmp1[j] < -size2[j]) { c1++; c2 = j; tmp1[j] = -size2[j]; }
      else if (tmp1[j] > size2[j]) { c1++; c2 = j; tmp1[j] = size2[j]; }
    }
    if (c1 > 1) continue;
    for (int k = 0; k < 3; k++) tmp1[k] -= tmp2[k];
    dist = tmp1[0] * tmp1[0] + tmp1[1] * tmp1[1] + tmp1[2] * tmp1[2];
    if (dist < bestdist) { bestdist = dist; bestsegmentpos = i; cltype = -2 + i; clface = c2; }
  }
  // the twelve edges: edge along axis j through the corner i (bit j of i clear)
  for (int j = 0; j < 3; j++) {
    for (int i = 0; i < 8; i++) {
      if ((i & (1 << j)) != 0) continue;
      tmp3[0] = ((i & 1) ? 1 : -1) * size2[0];
      tmp3[1] = ((i & 2) ? 1 : -1) * size2[1];
      tmp3[2] = ((i & 4) ? 1 : -1) * size2[2];
      tmp3[j] = 0;
      for (int k = 0; k < 3; k++) dif[k] = tmp3[k] - pos[k];
      const double ma = size2[j] * size2[j];
      const double mb = -size2[j] * halfaxis[j];
      const double mc = size1[1] * size1[1];
      const double u = -size2[j] * dif[j];
      const double v = halfaxis[0] * dif[0] + halfaxis[1] * dif[1] + halfaxis[2] * dif[2];
      const double det = ma * mc - mb * mb;
      if (fabs(det) < kMinVal) continue;
      const double idet = 1 / det;
      double x1 = (mc * u - mb * v) * idet;
      double x2 = (ma * v - mb * u) * idet;
      int s1 = 1, s2 = 1;   // 1: inside the segment, 0 / 2: clamped to an end
      if (x1 > 1) { x1 = 1; s1 = 2; x2 = (v - mb) * (1 / mc); }
      else if (x1 < -1) { x1 = -1; s1 = 0; x2 = (v + mb) * (1 / mc); }
      if (x2 > 1) {
        x2 = 1; s2 = 2;
        x1 = (u - mb) * (1 / ma);
        if (x1 > 1) { x1 = 1; s1 = 2; } else if (x1 < -1) { x1 = -1; s1 = 0; }
      } else if (x2 < -1) {
        x2 = -1; s2 = 0;
        x1 = (u + mb) * (1 / ma);
        if (x1 > 1) { x1 = 1; s1 = 2; } else if (x1 < -1) { x1 = -1; s1 = 0; }
      }
      for (int k = 0; k < 3; k++) { dif[k] = tmp3[k] - pos[k]; dif[k] += halfaxis[k] * (-x2); }
      dif[j] += size2[j] * x1;
      const double d2 = dif[0] * dif[0] + dif[1] * dif[1] + dif[2] * dif[2];
      c1 = s1 * 3 + s2;
      if (d2 < bestdist - kMinVal) {
        bestdist = d2;
        bestsegmentpos = x2;
        bestboxpos = x1;
        c2 = c1 / 6;                       // the upper end of the edge is the closest
        clcorner = i + (1 << j) * c2;
        cledge = j;
        cltype = c1;
      }
    }
  }
  if (cltype == -4) return 0;
  bool skip = false;
  if (cltype >= 0 && cltype / 3 != 1) {   // closest to a corner of the box
    c1 = axisdir ^ clcorner;
    if (c1 == 0 || c1 == 7) skip = true;   // pointing to or away from the corner: no second contact
    else {
      if (c1 == 1 || c1 == 2 || c1 == 4) { mul = 1; de = 1 - bestsegmentpos; dp = 1 + bestsegmentpos; }
      if (c1 == 3 || c1 == 5 || c1 == 6) { mul = -1; c1 = 7 - c1; dp = 1 - bestsegmentpos; de = 1 + bestsegmentpos; }
      if (c1 == 1) { ax = 0; ax1 = 1; ax2 = 2; }
      if (c1 == 2) { ax = 1; ax1 = 2; ax2 = 0; }
      if (c1 == 4) { ax = 2; ax1 = 0; ax2 = 1; }
      if (axis[ax] * axis[ax] > 0.5) {     // second point along the edge of the box
        secondpos = de;
        e1 = 2 * size2[ax] / fabs(halfaxis[ax]);
        if (e1 < secondpos) secondpos = e1;
        secondpos *= mul;
      } else {                             // second point along a face of the box
        secondpos = dp;
        e1 = 2 * size2[ax1] / fabs(halfaxis[ax1]);
        if (e1 < secondpos) secondpos = e1;
        e1 = 2 * size2[ax2] / fabs(halfaxis[ax2]);
        if (e1 < secondpos) secondpos = e1;
        secondpos *= -mul;
      }
    }
  } else if (cltype >= 0 && cltype / 3 == 1) {   // closest to the inside of an edge
    c1 = axisdir ^ clcorner;
    c1 &= 7 - (1 << cledge);
    if (c1 != 1 && c1 != 2 && c1 != 4) skip = true;   // T configuration: no second contact
    else {
      if (cledge == 0) { ax1 = 1; ax2 = 2; }
      if (cledge == 1) { ax1 = 2; ax2 = 0; }
      if (cledge == 2) { ax1 = 0; ax2 = 1; }
      ax = cledge;
      if (fabs(axis[ax1]) > fabs(axis[ax2])) ax1 = ax2;   // the face the capsule makes the lower angle with
      ax2 = 3 - ax - ax1;
      if (c1 & (1 << ax2)) { mul = 1; secondpos = 1 - bestsegmentpos; }
      else { mul = -1; secondpos = 1 + bestsegmentpos; }
      e1 = 2 * size2[ax2] / fabs(halfaxis[ax2]);
      if (e1 < secondpos) secondpos = e1;
      if (((axisdir & (1 << ax)) != 0) == ((c1 & (1 << ax2)) != 0)) e2 = 1 - bestboxpos;
      else e2 = 1 + bestboxpos;
      e1 = size2[ax] * e2 / fabs(halfaxis[ax]);
      if (e1 < secondpos) secondpos = e1;
      secondpos *= mul;
    }
  } else if (cltype < 0) {                 // an end of the capsule is closest to a face
    if (clface == -1) skip = true;         // the closest point is inside the box
    else {
      mul = (cltype == -3) ? 1 : -1;
      secondpos = 2;
      for (int k = 0; k < 3; k++) { tmp1[k] = pos[k]; tmp1[k] += halfaxis[k] * (-mul); }
      for (int i = 0; i < 3; i++) {
        if (i == clface) continue;
        e1 = (size2[i] - tmp1[i]) / halfaxis[i] * mul;
        if (e1 > 0 && e1 < secondpos) secondpos = e1;
        e1 = (-size2[i] - tmp1[i]) / halfaxis[i] * mul;
        if (e1 > 0 && e1 < secondpos) secondpos = e1;
      }
      secondpos *= mul;
    }
  }
  (void)skip;
  // sphere at the first contact point, back in the world frame
  for (int k = 0; k < 3; k++) { tmp1[k] = pos[k]; tmp1[k] += halfaxis[k] * bestsegmentpos; }
  V3 w = mulmv(m2, V3{tmp1[0], tmp1[1], tmp1[2]});
  w = w + p2;
  int n = raw_sphere_box(c[0], margin, w, size1[0], p2, m2, size2);
  if (secondpos > -3) {
    for (int k = 0; k < 3; k++) { tmp1[k] = pos[k]; tmp1[k] += halfaxis[k] * (secondpos + bestsegmentpos); }
    w = mulmv(m2, V3{tmp1[0], tmp1[1], tmp1[2]});
    w = w + p2;
    n += raw_sphere_box(c[n], margin, w, size1[0], p2, m2, size2);
  }
  return n;
}

// ---- box : box (engine_collision_box.c:592-1068): separating-axis test over the 15 candidate axes, then a face
// manifold (the incident face clipped against the side planes of the reference face) or one edge-edge contact
constexpr double kBoxSepEps = 1e-13, kBoxParEps = 1e-16, kBoxSgnEps = 1e-9, kBoxDupEps = 1e-14, kBoxEdgeBias = 1e-6;
constexpr int kBoxMaxVert = 12;

// clip polygon `cur` against sign * v[coord] <= limit (Sutherland-Hodgman, z interpolated); untouched when every
// vertex is inside, otherwise written to `spare` and the buffers swap (engine_collision_box.c:655-697)
MJB_HD int box_clip(int nin, double (*&cur)[3], double (*&spare)[3], int coord, double sign, double limit) {
  double (*in)[3] = cur;
  double dd[kBoxMaxVert];
  bool all_inside = true;
  for (int k = 0; k < nin; k++) { dd[k] = sign * in[k][coord] - limit; all_inside = all_inside && dd[k] <= 0; }
  if (all_inside) return nin;
  double (*out)[3] = spare;
  int nout = 0;
  for (int k = 0; k < nin; k++) {
    const double* p = in[k];
    const int k1 = (k + 1 == nin) ? 0 : k + 1;
    const double dpv = dd[k], dq = dd[k1];
    if (dpv <= 0 && nout < kBoxMaxVert) { out[nout][0] = p[0]; out[nout][1] = p[1]; out[nout][2] = p[2]; nout++; }
    if (((dpv < 0 && dq > 0) || (dpv > 0 && dq < 0)) && nout < kBoxMaxVert) {
      const double* q = in[k1];
      const double t = dpv / (dpv - dq);
      out[nout][0] = p[0] + t * (q[0] - p[0]);
      out[nout][1] = p[1] + t * (q[1] - p[1]);
      out[nout][2] = p[2] + t * (q[2] - p[2]);
      nout++;
    }
  }
  cur = out;
  spare = in;
  return nout;
}

MJB_HD int collide_box_box(PreCon* c, double margin, V3 p1, const M3& m1, const double* size1,
                           V3 p2, const M3& m2, const double* size2) {
  double rot[9], rotabs[9], pos21[3], pos12[3];
  {
    const V3 a = mulmTv3(m1, p2 - p1), b = mulmTv3(m2, p1 - p2);
    pos21[0] = a.x; pos21[1] = a.y; pos21[2] = a.z;
    pos12[0] = b.x; pos12[1] = b.y; pos12[2] = b.z;
    for (int r = 0; r < 3; r++)        // rot = mat1' * mat2: the axes of box 2 in the frame of box 1
      for (int q = 0; q < 3; q++) rot[3 * r + q] = m1.m[r] * m2.m[q] + m1.m[3 + r] * m2.m[3 + q] + m1.m[6 + r] * m2.m[6 + q];
    for (int i = 0; i < 9; i++) rotabs[i] = fabs(rot[i]);
  }
  // ---- stage 1: separating-axis test
  const double septol = margin + kBoxSepEps * (size1[0] + size1[1] + size1[2] + size2[0] + size2[1] + size2[2]);
  double sep_best = -kMaxVal, sep_face;
  int code = -1;
  for (int i = 0; i < 3; i++) {
    const double radius2 = rotabs[3 * i + 0] * size2[0] + rotabs[3 * i + 1] * size2[1] + rotabs[3 * i + 2] * size2[2];
    const double sep = fabs(pos21[i]) - size1[i] - radius2;
    if (sep > septol) return 0;
    if (sep > sep_best) { sep_best = sep; code = i; }
  }
  for (int j = 0; j < 3; j++) {
    const double radius1 = rotabs[0 + j] * size1[0] + rotabs[3 + j] * size1[1] + rotabs[6 + j] * size1[2];
    const double sep = fabs(pos12[j]) - size2[j] - radius1;
    if (sep > septol) return 0;
    if (sep > sep_best) { sep_best = sep; code = 3 + j; }
  }
  sep_face = sep_best;
  const int code_face = code;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
      double ax1 = -rot[3 * i2 + j];
      double ax2 = rot[3 * i1 + j];
      const double norm2 = ax1 * ax1 + ax2 * ax2;
      if (norm2 < kBoxParEps) continue;
      const double inv = 1 / sqrt(norm2);
      ax1 *= inv;
      ax2 *= inv;
      const double radius1 = size1[i1] * fabs(ax1) + size1[i2] * fabs(ax2);
      const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      const double a2_1 = ax1 * rot[3 * i1 + j1] + ax2 * rot[3 * i2 + j1];
      const double a2_2 = ax1 * rot[3 * i1 + j2] + ax2 * rot[3 * i2 + j2];
      const double radius2 = size2[j1] * fabs(a2_1) + size2[j2] * fabs(a2_2);
      const double sep = fabs(ax1 * pos21[i1] + ax2 * pos21[i2]) - radius1 - radius2;
      if (sep > septol) return 0;
      if (sep - kBoxEdgeBias * fabs(sep) > sep_best && sep > sep_face) { sep_best = sep; code = 6 + 3 * i + j; }
    }
  }
  if (code < 0) return 0;
  auto edge_axis = [&](int i, int j, double* axis) {   // unit cross product of e_i and column j of rot
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
    axis[i] = 0;
    axis[i1] = -rot[3 * i2 + j];
    axis[i2] = rot[3 * i1 + j];
    V3 v{axis[0], axis[1], axis[2]};
    normalize(v);
    axis[0] = v.x; axis[1] = v.y; axis[2] = v.z;
  };
  if (code >= 6) {   // an edge axis nearly parallel to the best face axis gives way to the face
    double axis[3];
    edge_axis((code - 6) / 3, (code - 6) % 3, axis);
    double face_dot;
    if (code_face < 3) face_dot = fabs(axis[code_face]);
    else {
      const int f = code_face - 3;
      face_dot = fabs(axis[0] * rot[0 + f] + axis[1] * rot[3 + f] + axis[2] * rot[6 + f]);
    }
    if (face_dot > 0.99 && sep_best < sep_face + 0.05 * fabs(sep_face) + kMinVal) { code = code_face; sep_best = sep_face; }
  }
  // ---- stage 2a: edge-edge contact
  if (code >= 6) {
    const int i = (code - 6) / 3, j = (code - 6) % 3;
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    double axis[3];
    edge_axis(i, j, axis);
    if (axis[0] * pos21[0] + axis[1] * pos21[1] + axis[2] * pos21[2] < 0) { axis[0] = -axis[0]; axis[1] = -axis[1]; axis[2] = -axis[2]; }
    const double a2[3] = {axis[0] * rot[0 + 0] + axis[1] * rot[3 + 0] + axis[2] * rot[6 + 0],
                          axis[0] * rot[0 + 1] + axis[1] * rot[3 + 1] + axis[2] * rot[6 + 1],
                          axis[0] * rot[0 + 2] + axis[1] * rot[3 + 2] + axis[2] * rot[6 + 2]};
    int amb1 = -1, amb2 = -1;
    if (fabs(axis[i1]) < kBoxSgnEps) amb1 = i1; else if (fabs(axis[i2]) < kBoxSgnEps) amb1 = i2;
    if (fabs(a2[j1]) < kBoxSgnEps) amb2 = j1; else if (fabs(a2[j2]) < kBoxSgnEps) amb2 = j2;
    const double d2[3] = {rot[0 + j], rot[3 + j], rot[6 + j]};
    const double b = d2[i];
    const double denom = 1 - b * b;
    double w1[3] = {0, 0, 0}, w2[3] = {0, 0, 0};
    double best_d2 = kMaxVal;
    for (int v1 = 0; v1 < (amb1 >= 0 ? 2 : 1); v1++) {
      for (int v2 = 0; v2 < (amb2 >= 0 ? 2 : 1); v2++) {
        double c1[3], cc[3], c2[3], e[3];
        c1[i] = 0;
        c1[i1] = axis[i1] >= 0 ? size1[i1] : -size1[i1];
        c1[i2] = axis[i2] >= 0 ? size1[i2] : -size1[i2];
        if (amb1 >= 0 && v1) c1[amb1] = -c1[amb1];
        cc[j] = 0;
        cc[j1] = a2[j1] >= 0 ? -size2[j1] : size2[j1];
        cc[j2] = a2[j2] >= 0 ? -size2[j2] : size2[j2];
        if (amb2 >= 0 && v2) cc[amb2] = -cc[amb2];
        for (int r = 0; r < 3; r++) c2[r] = rot[3 * r] * cc[0] + rot[3 * r + 1] * cc[1] + rot[3 * r + 2] * cc[2];
        for (int r = 0; r < 3; r++) c2[r] += pos21[r];
        for (int r = 0; r < 3; r++) e[r] = c2[r] - c1[r];
        const double d1e = e[i];
        const double d2e = d2[0] * e[0] + d2[1] * e[1] + d2[2] * e[2];
        double sp = denom < kMinVal ? 0 : (d1e - b * d2e) / denom;
        sp = dclip(sp, -size1[i], size1[i]);
        const double t = dclip(b * sp - d2e, -size2[j], size2[j]);
        sp = dclip(d1e + b * t, -size1[i], size1[i]);
        double q1[3] = {c1[0], c1[1], c1[2]}, q2[3] = {c2[0], c2[1], c2[2]};
        q1[i] += sp;
        for (int r = 0; r < 3; r++) q2[r] += d2[r] * t;
        const double g0 = q2[0] - q1[0], g1 = q2[1] - q1[1], g2 = q2[2] - q1[2];
        const double gap2 = g0 * g0 + g1 * g1 + g2 * g2;
        if (gap2 < best_d2) { best_d2 = gap2; for (int r = 0; r < 3; r++) { w1[r] = q1[r]; w2[r] = q2[r]; } }
      }
    }
    const double dist = (w2[0] - w1[0]) * axis[0] + (w2[1] - w1[1]) * axis[1] + (w2[2] - w1[2]) * axis[2];
    if (dist > septol) return 0;
    const V3 mid{0.5 * (w1[0] + w2[0]), 0.5 * (w1[1] + w2[1]), 0.5 * (w1[2] + w2[2])};
    c[0].dist = dist;
    c[0].pos = mulmv(m1, mid) + p1;
    c[0].normal = mulmv(m1, V3{axis[0], axis[1], axis[2]});
    c[0].tangent = V3{0, 0, 0};
    return 1;
  }
  // ---- stage 2b: face contact
  const bool ref1 = code < 3;
  const int a = ref1 ? code : code - 3;
  const double* sizeref = ref1 ? size1 : size2;
  const double* sizeinc = ref1 ? size2 : size1;
  const V3 posref = ref1 ? p1 : p2;
  const M3& matref = ref1 ? m1 : m2;
  const double* posoi = ref1 ? pos21 : pos12;
  double rinc[9];   // incident axes in the reference frame
  if (ref1) { for (int k = 0; k < 9; k++) rinc[k] = rot[k]; }
  else { for (int r = 0; r < 3; r++) for (int q = 0; q < 3; q++) rinc[3 * q + r] = rot[3 * r + q]; }
  const double sgn = posoi[a] >= 0 ? 1 : -1;
  int binc = 0;
  for (int k = 1; k < 3; k++) if (fabs(rinc[3 * a + k]) > fabs(rinc[3 * a + binc])) binc = k;
  const double tinc = sgn * rinc[3 * a + binc] > 0 ? -1 : 1;
  const int ax = (a + 1) % 3, ay = (a + 2) % 3, bu = (binc + 1) % 3, bv = (binc + 2) % 3;
  double poly[2][kBoxMaxVert][3];
  double cx[3], du[3], dv[3];
  for (int r = 0; r < 3; r++) {
    const int cc = r == 0 ? ax : (r == 1 ? ay : a);
    cx[r] = posoi[cc] + tinc * sizeinc[binc] * rinc[3 * cc + binc];
    du[r] = sizeinc[bu] * rinc[3 * cc + bu];
    dv[r] = sizeinc[bv] * rinc[3 * cc + bv];
  }
  cx[2] = sgn * cx[2] - sizeref[a];
  du[2] *= sgn;
  dv[2] *= sgn;
  for (int k = 0; k < 4; k++) {
    const double su = (k == 0 || k == 3) ? 1 : -1, sv = (k < 2) ? 1 : -1;
    poly[0][k][0] = cx[0] + su * du[0] + sv * dv[0];
    poly[0][k][1] = cx[1] + su * du[1] + sv * dv[1];
    poly[0][k][2] = cx[2] + su * du[2] + sv * dv[2];
  }
  int nvert = 4;
  double (*cur)[3] = poly[0];
  double (*spare)[3] = poly[1];
  nvert = box_clip(nvert, cur, spare, 0, 1, sizeref[ax]);
  nvert = box_clip(nvert, cur, spare, 0, -1, sizeref[ax]);
  nvert = box_clip(nvert, cur, spare, 1, 1, sizeref[ay]);
  nvert = box_clip(nvert, cur, spare, 1, -1, sizeref[ay]);
  double accepted[kBoxMaxVert][3];
  int naccept = 0;
  const double dupe2 = kBoxDupEps * (sizeref[ax] * sizeref[ax] + sizeref[ay] * sizeref[ay]);
  for (int k = 0; k < nvert; k++) {
    if (cur[k][2] > margin) continue;
    bool dupe = false;
    for (int q = 0; q < naccept; q++) {
      const double dx = accepted[q][0] - cur[k][0], dy = accepted[q][1] - cur[k][1];
      if (dx * dx + dy * dy < dupe2) { dupe = true; break; }
    }
    if (!dupe) { accepted[naccept][0] = cur[k][0]; accepted[naccept][1] = cur[k][1]; accepted[naccept][2] = cur[k][2]; naccept++; }
  }
  if (naccept == 0) return 0;
  if (naccept > 8) naccept = 8;   // a quadrilateral clipped by four half-planes has at most eight vertices
  const double nsign = ref1 ? sgn : -sgn;
  const V3 normal{nsign * matref.m[3 * 0 + a], nsign * matref.m[3 * 1 + a], nsign * matref.m[3 * 2 + a]};
  for (int k = 0; k < naccept; k++) {
    const double* v = accepted[k];
    double posc[3];
    posc[ax] = v[0];
    posc[ay] = v[1];
    posc[a] = sgn * (sizeref[a] + 0.5 * v[2]);
    c[k].dist = v[2];
    c[k].pos = mulmv(matref, V3{posc[0], posc[1], posc[2]}) + posref;
    c[k].normal = normal;
    c[k].tangent = V3{0, 0, 0};
  }
  return naccept;
}

}  // namespace mjb

// convex narrow phase (GJK / EPA, plane-ellipsoid), only in kernels compiled with FEAT_CONVEX
#include "mjb_convex.h"

namespace mjb {

// filter + narrowphase of candidate pair p; returns the number of pre-contacts written to pc[]
MJB_HD int pair_collide(const Env& d, int p, PreCon* pc) {
  const DModel& m = d.m;
  FD gx = d.geom_xpos(), gm = d.geom_xmat();
  const int g1 = m.pair_geom1[p], g2 = m.pair_geom2[p];
  const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  const double margin = m.pair_margin[p];
  const double rb1 = m.geom_rbound[g1], rb2 = m.geom_rbound[g2];
  V3 p1 = ld3(gx, 3 * g1), p2 = ld3(gx, 3 * g2);
  // per-pair filter (mj_filterSphere)
  if (rb1 > 0 && rb2 > 0) {
    V3 dif = p1 - p2;
    double dsq = dif.x * dif.x + dif.y * dif.y + dif.z * dif.z;
    double bound = rb1 + rb2 + margin;
    if (dsq > bound * bound) return 0;
  } else if (t1 == GEOM_PLANE && rb2 > 0) {
    V3 nrm{gm[9 * g1 + 2], gm[9 * g1 + 5], gm[9 * g1 + 8]};
    V3 dif = p2 - p1;
    if (dot(dif, nrm) > margin + rb2) return 0;
  }
  M3 m1 = ld9(gm, 9 * g1), m2 = ld9(gm, 9 * g2);
  const double* s1 = m.geom_size + 3 * g1;
  const double* s2 = m.geom_size + 3 * g2;
  if (t1 == GEOM_PLANE && t2 == GEOM_SPHERE) return raw_plane_sphere(pc[0], margin, p1, m1, p2, s2[0]);
  if (t1 == GEOM_PLANE && t2 == GEOM_CAPSULE) return collide_plane_capsule(pc, margin, p1, m1, p2, m2, s2);
  if (t1 == GEOM_SPHERE && t2 == GEOM_SPHERE) return raw_sphere_sphere(pc[0], margin, p1, m1, s1[0], p2, m2, s2[0]);
  if (t1 == GEOM_SPHERE && t2 == GEOM_CAPSULE) return collide_sphere_capsule(pc, margin, p1, m1, s1, p2, m2, s2);
  if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) return collide_capsule_capsule(pc, margin, p1, m1, s1, p2, m2, s2);
  if (d.feat & FEAT_COLBOX) {
    if (t1 == GEOM_PLANE && t2 == GEOM_CYLINDER) return collide_plane_cylinder(pc, margin, p1, m1, p2, m2, s2);
    if (t1 == GEOM_PLANE && t2 == GEOM_BOX) return collide_plane_box(pc, margin, p1, m1, p2, m2, s2);
    if (t1 == GEOM_SPHERE && t2 == GEOM_CYLINDER) return collide_sphere_cylinder(pc, margin, p1, m1, s1, p2, m2, s2);
    if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) return raw_sphere_box(pc[0], margin, p1, s1[0], p2, m2, s2);
    if (t1 == GEOM_CAPSULE && t2 == GEOM_BOX) return collide_capsule_box(pc, margin, p1, m1, s1, p2, m2, s2);
    if (t1 == GEOM_BOX && t2 == GEOM_BOX) return collide_box_box(pc, margin, p1, m1, s1, p2, m2, s2);
  }
  return 0;
}

// ordinal of GJK candidate p among the GJK candidates of the table (its entry in the pre-contact store ccd_con)
MJB_HD int gjk_ordinal(const DModel& m, int p) {
  int c = 0;
  for (int q = 0; q < p; q++) c += pair_gjk(m.geom_type[m.pair_geom1[q]], m.geom_type[m.pair_geom2[q]]) ? 1 : 0;
  return c;
}

// GJK / EPA candidates, before the count pass: the first K lanes of the environment each take every K-th GJK candidate
// in table order, with their own polytope slot (K = the environment's slots, at most its lanes), and store the
// candidate's pre-contacts, so that neither pass of collision_t evaluates it again
MJB_HD void convex_pass(const Env& d) {
  const DModel& m = d.m;
  const int npair = m.sz.npair;
  int K = kCcdSlots < d.nlane ? kCcdSlots : d.nlane;
  if (m.sz.ccdslots < K) K = m.sz.ccdslots;
  if (d.lane < K) {
    double* slot = &d.ccd_poly()[(long)d.lane * m.sz.ccdslot];
    FD store = d.ccd_con();
    FD gx = d.geom_xpos(), gm = d.geom_xmat();
    int c = 0;
    for (int p = 0; p < npair; p++) {
      const int g1 = m.pair_geom1[p], g2 = m.pair_geom2[p];
      if (!pair_gjk(m.geom_type[g1], m.geom_type[g2])) continue;
      if (c++ % K != d.lane) continue;
      const long base = 36L * (c - 1);
      const double margin = m.pair_margin[p];
      const V3 p1 = ld3(gx, 3 * g1), p2 = ld3(gx, 3 * g2);
      const V3 dif = p1 - p2;   // bounding-sphere filter (mj_filterSphere); neither geom is a plane
      const double dsq = dif.x * dif.x + dif.y * dif.y + dif.z * dif.z;
      const double bound = m.geom_rbound[g1] + m.geom_rbound[g2] + margin;
      int n = 0;
      PreCon pc[5];
      if (!(dsq > bound * bound)) n = collide_convex(pc, m, g1, g2, p1, ld9(gm, 9 * g1), p2, ld9(gm, 9 * g2), margin, slot);
      store[base] = n;
      for (int k = 0; k < n; k++) {
        const long o = base + 1 + 7 * k;
        store[o] = pc[k].dist;
        st3(store, o + 1, pc[k].pos);
        st3(store, o + 4, pc[k].normal);
      }
    }
  }
  MJB_PSYNC();
}

// pre-contacts of GJK candidate p stored by convex_pass; returns their number
MJB_HD int convex_load(const Env& d, int p, PreCon* pc);

// candidate p in a FEAT_CONVEX kernel: GJK candidates from the store of convex_pass, plane-ellipsoid (after the plane
// filter of mj_filterSphere), every other pair through pair_collide
MJB_HD int pair_collide_convex(const Env& d, int p, PreCon* pc) {
  const DModel& m = d.m;
  const int g1 = m.pair_geom1[p], g2 = m.pair_geom2[p];
  const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  if (pair_gjk(t1, t2)) return convex_load(d, p, pc);
  if (t1 != GEOM_PLANE || t2 != GEOM_ELLIPSOID) return pair_collide(d, p, pc);
  FD gx = d.geom_xpos(), gm = d.geom_xmat();
  const double margin = m.pair_margin[p];
  const V3 p1 = ld3(gx, 3 * g1), p2 = ld3(gx, 3 * g2);
  if (m.geom_rbound[g2] > 0) {
    const V3 nrm{gm[9 * g1 + 2], gm[9 * g1 + 5], gm[9 * g1 + 8]};
    if (dot(p2 - p1, nrm) > margin + m.geom_rbound[g2]) return 0;
  }
  return collide_plane_ellipsoid(pc[0], margin, p1, ld9(gm, 9 * g1), p2, ld9(gm, 9 * g2), m.geom_size + 3 * g2);
}

MJB_HD int convex_load(const Env& d, int p, PreCon* pc) {
  FD store = d.ccd_con();
  const long base = 36L * gjk_ordinal(d.m, p);
  const int n = (int)store[base];
  for (int k = 0; k < n; k++) {
    const long o = base + 1 + 7 * k;
    pc[k].dist = store[o];
    pc[k].pos = ld3(store, o + 1);
    pc[k].normal = ld3(store, o + 4);
    pc[k].tangent = V3{0, 0, 0};
  }
  return n;
}

// walk the static candidate table cooperatively in two passes: (1) every lane counts the
// pre-contacts of its candidates, (2) after a serial scan that assigns contact slots IN TABLE ORDER
// (the reference's emission order) the few hitting pairs are evaluated again and written in place.
template <int MAXC, bool CONVEX = false>
MJB_HD void collision_t(const Env& d) {
  const DModel& m = d.m;
  FI ncon_f = d.ncon();
  if (m.opt.disableflags & (DSBL_CONSTRAINT | DSBL_CONTACT)) {
    MJB_LANE0 ncon_f[0] = 0;
    MJB_PSYNC();
    return;
  }
  FI cnt = d.scr_ipair();        // per pair: number of pre-contacts, then packed (offset | n << 24)
  const int npair = m.sz.npair, nconmax = m.sz.nconmax;
  if constexpr (CONVEX) convex_pass(d);
  MJB_PFOR(p, npair) {
    PreCon pc[MAXC];
    if constexpr (CONVEX) cnt[p] = pair_collide_convex(d, p, pc);
    else cnt[p] = pair_collide(d, p, pc);
  }
  MJB_PSYNC();
  MJB_LANE0 {   // exclusive scan in table order, capped at nconmax
    int total = 0;
    bool full = false;
    for (int p = 0; p < npair; p++) {
      int n = cnt[p];
      if (total + n > nconmax) { n = nconmax - total; full = true; }
      cnt[p] = total | (n << 24);
      total += n;
    }
    if (full) d.warning()[WARN_CONTACTFULL] += 1;
    ncon_f[0] = total;
  }
  MJB_PSYNC();
  FD cdist = d.con_dist(), cpos = d.con_pos(), cframe = d.con_frame(), cinc = d.con_includemargin();
  FD cfri = d.con_friction(), csolref = d.con_solref(), csolimp = d.con_solimp(), cmu = d.con_mu();
  FI cg1 = d.con_geom1(), cg2 = d.con_geom2(), cdim = d.con_dim(), cexc = d.con_exclude(), cadr = d.con_efcadr();
  FI cpair = d.con_pair();
  MJB_PFOR(p, npair) {
    const int off = cnt[p] & 0xFFFFFF, n = cnt[p] >> 24;
    if (!n) continue;
    PreCon pc[MAXC];
    if constexpr (CONVEX) pair_collide_convex(d, p, pc);
    else pair_collide(d, p, pc);
    for (int k = 0; k < n; k++) {
      const int c = off + k;
      const double dist = pc[k].dist;
      cdist[c] = dist;
      st3(cpos, 3 * c, pc[k].pos);
      M3 fr;
      fr.m[0] = pc[k].normal.x; fr.m[1] = pc[k].normal.y; fr.m[2] = pc[k].normal.z;
      fr.m[3] = pc[k].tangent.x; fr.m[4] = pc[k].tangent.y; fr.m[5] = pc[k].tangent.z;
      fr.m[6] = 0; fr.m[7] = 0; fr.m[8] = 0;
      make_frame(fr);
      st9(cframe, 9 * c, fr);
      cg1[c] = m.pair_geom1[p]; cg2[c] = m.pair_geom2[p];
      cpair[c] = p;
      cdim[c] = m.pair_dim[p];
      const double inc = m.pair_includemargin[p];
      cinc[c] = inc;
      for (int j = 0; j < 5; j++) cfri[5 * c + j] = m.pair_friction[5 * p + j];
      for (int j = 0; j < 2; j++) csolref[2 * c + j] = m.pair_solref[2 * p + j];
      for (int j = 0; j < 5; j++) csolimp[5 * c + j] = m.pair_solimp[5 * p + j];
      cexc[c] = (dist >= inc) ? 1 : 0;
      cadr[c] = -1;
      cmu[c] = 0;
    }
  }
  MJB_PSYNC();
}

// pairs of the sphere / capsule / plane family give at most two contacts; the cylinder and box colliders up to
// eight, the convex pairs up to five (kernels without FEAT_COLBOX / FEAT_CONVEX do not carry their code or the larger
// pre-contact array)
// On the device the convex branch is compiled only in the translation unit that defines MJB_CONVEX_UNIT (the
// FEAT_CONVEX instantiations, mjb_kstep_convex32.cu): in every other kernel collision() is the same code as without the
// convex narrow phase, so their inlining and stack layout do not see GJK / EPA at all.  Host compilations (the
// emulation of the device path) always carry it.
MJB_HD void collision(const Env& d) {
#if defined(MJB_CONVEX_UNIT) || !defined(__CUDA_ARCH__)
  if (d.feat & FEAT_CONVEX) { collision_t<8, true>(d); return; }
#endif
  if (d.feat & FEAT_COLBOX) collision_t<8>(d); else collision_t<2>(d);
}

}  // namespace mjb
