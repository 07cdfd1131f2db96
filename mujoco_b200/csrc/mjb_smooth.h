// Smooth dynamics of the batched mj_step path for ONE environment, executed cooperatively by the
// lanes that own it (32 lanes of a warp in the fused kernel, 1 lane in lane-per-env mode).
//
// Replaces (reference file:line)  src/engine/engine_core_smooth.c  mj_kinematics :40-242,
// mj_comPos :246-350, mj_tendon (fixed tendons) :927-985, mj_transmission (joint) :1265-1330,
// mj_crb/mj_tendonArmature :1845-1971, mj_factorI :1997-2029, mj_solveLD :2033-2117,
// mj_comVel :2179-2245, mj_rne :2328-2390;  src/engine/engine_passive.c mj_springdamper :655-842.
//
// Parallel structure: the tree recursions run level by level (MJB_PFOR over the bodies / dofs of a
// level, MJB_PSYNC between levels).  Every output element is still produced by ONE lane with the
// reference's operation order — backward accumulations use host-built child / descendant lists in
// the order in which the serial loops of the reference would have added them — so results are
// bit-identical to the serial restatement whatever the lane count.
#pragma once
#include "mjb_types.h"

namespace mjb {

// ------------------------------------------------------------------------------------------------
// forward kinematics: body frames level by level, then inertial and geom frames
MJB_HD void kinematics(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody;
  FD qpos = d.qpos(), xpos = d.xpos(), xquat = d.xquat(), xmat = d.xmat();
  FD xipos = d.xipos(), ximat = d.ximat(), xanchor = d.xanchor(), xaxis = d.xaxis();

  MJB_LANE0 {   // world body
    st3(xpos, 0, V3{0, 0, 0});
    st4(xquat, 0, Q4{1, 0, 0, 0});
    st3(xipos, 0, V3{0, 0, 0});
    for (int k = 0; k < 9; k++) { xmat[k] = (k % 4 == 0) ? 1.0 : 0.0; ximat[k] = (k % 4 == 0) ? 1.0 : 0.0; }
  }
  MJB_PSYNC();

  for (int l = 1; l < m.sz.nlevel; l++) {
    const int adr = m.lvl_adr[l], cnt = m.lvl_adr[l + 1] - adr;
    MJB_PFOR(k_, cnt) {
      const int i = m.lvl_body[adr + k_];
      V3 p; Q4 q;
      const int jadr = m.body_jntadr[i], jnum = m.body_jntnum[i];
      if (jnum == 1 && m.jnt_type[jadr] == JNT_FREE) {
        const int qa = m.jnt_qposadr[jadr];
        p = ld3(qpos, qa);
        q = ld4(qpos, qa + 3);
        normalize(q);
        st3(xanchor, 3 * jadr, p);
        st3(xaxis, 3 * jadr, ldc3(m.jnt_axis, 3 * jadr));
      } else {
        const int pid = m.body_parentid[i];
        V3 bpos = ldc3(m.body_pos, 3 * i);
        Q4 bquat = ldc4(m.body_quat, 4 * i);
        if (m.sz.nmocap && m.body_mocapid[i] >= 0) {   // mocap body: pose from mjData (engine_core_smooth.c:84-90)
          const int mid = m.body_mocapid[i];
          bpos = ld3(d.mocap_pos(), 3 * mid);
          bquat = ld4(d.mocap_quat(), 4 * mid);
          normalize(bquat);
        }
        if (pid) {
          p = mulmv(ld9(xmat, 9 * pid), bpos);
          p = p + ld3(xpos, 3 * pid);
          q = qmul(ld4(xquat, 4 * pid), bquat);
        } else {
          p = bpos;
          q = bquat;
        }
        for (int j = 0; j < jnum; j++) {
          const int jid = jadr + j, qa = m.jnt_qposadr[jid], jt = m.jnt_type[jid];
          V3 jaxis = ldc3(m.jnt_axis, 3 * jid), jpos = ldc3(m.jnt_pos, 3 * jid);
          V3 ax = rotate(jaxis, q);
          V3 an = rotate(jpos, q);
          an = an + p;
          if (jt == JNT_SLIDE) {
            p = addscl(p, ax, qpos[qa] - m.qpos0[qa]);
          } else {  // ball or hinge
            Q4 ql;
            if (jt == JNT_BALL) {
              ql = ld4(qpos, qa);
              normalize(ql);
            } else {
              ql = axis_angle(jaxis, qpos[qa] - m.qpos0[qa]);
            }
            q = qmul(q, ql);
            V3 off = rotate(jpos, q);
            p = an - off;
          }
          st3(xanchor, 3 * jid, an);
          st3(xaxis, 3 * jid, ax);
        }
      }
      normalize(q);
      st4(xquat, 4 * i, q);
      st3(xpos, 3 * i, p);
      st9(xmat, 9 * i, quat2mat(q));
    }
    MJB_PSYNC();
  }

  // inertial frames (mj_local2Global, engine_core_util.c) and geom frames: independent items
  FD gpos = d.geom_xpos(), gmat = d.geom_xmat();
  const int ngeom = m.sz.ngeom;
  MJB_PFOR(i_, nbody - 1) {
    const int i = i_ + 1;
    const int sf = m.body_sameframe[i];
    V3 bp = ld3(xpos, 3 * i);
    M3 bm = ld9(xmat, 9 * i);
    if (sf == SAMEFRAME_BODY) st3(xipos, 3 * i, bp);
    else st3(xipos, 3 * i, mulmv(bm, ldc3(m.body_ipos, 3 * i)) + bp);
    if (sf == SAMEFRAME_NONE) st9(ximat, 9 * i, quat2mat(qmul(ld4(xquat, 4 * i), ldc4(m.body_iquat, 4 * i))));
    else st9(ximat, 9 * i, bm);
  }
  MJB_PSYNC();
  MJB_PFOR(g, ngeom) {
    const int b = m.geom_bodyid[g], sf = m.geom_sameframe[g];
    V3 bp = ld3(xpos, 3 * b);
    if (sf == SAMEFRAME_BODY) st3(gpos, 3 * g, bp);
    else if (sf == SAMEFRAME_INERTIA) st3(gpos, 3 * g, ld3(xipos, 3 * b));
    else st3(gpos, 3 * g, mulmv(ld9(xmat, 9 * b), ldc3(m.geom_pos, 3 * g)) + bp);
    if (sf == SAMEFRAME_NONE) st9(gmat, 9 * g, quat2mat(qmul(ld4(xquat, 4 * b), ldc4(m.geom_quat, 4 * g))));
    else if (sf == SAMEFRAME_BODY || sf == SAMEFRAME_BODYROT) st9(gmat, 9 * g, ld9(xmat, 9 * b));
    else st9(gmat, 9 * g, ld9(ximat, 9 * b));
  }
  // sites: same local-to-global rule (mj_kinematics, engine_core_smooth.c:222-233)
  FD spos = d.site_xpos(), smat = d.site_xmat();
  MJB_PFOR(s_, m.sz.nsite) {
    const int b = m.site_bodyid[s_], sf = m.site_sameframe[s_];
    V3 bp = ld3(xpos, 3 * b);
    if (sf == SAMEFRAME_BODY) st3(spos, 3 * s_, bp);
    else if (sf == SAMEFRAME_INERTIA) st3(spos, 3 * s_, ld3(xipos, 3 * b));
    else st3(spos, 3 * s_, mulmv(ld9(xmat, 9 * b), ldc3(m.site_pos, 3 * s_)) + bp);
    if (sf == SAMEFRAME_NONE) st9(smat, 9 * s_, quat2mat(qmul(ld4(xquat, 4 * b), ldc4(m.site_quat, 4 * s_))));
    else if (sf == SAMEFRAME_BODY || sf == SAMEFRAME_BODYROT) st9(smat, 9 * s_, ld9(xmat, 9 * b));
    else st9(smat, 9 * s_, ld9(ximat, 9 * b));
  }
  MJB_PSYNC();
}

// backward accumulation over the body tree: acc[parent] += acc[child] for `width` components,
// children added in descending id order, deepest level first (== serial loop i = nbody-1..1).
// skip_world: do not accumulate into the world body (mj_crb) / do (mj_comPos, mj_rne)
MJB_HD void tree_accumulate(const Env& d, FD acc, int width, bool skip_world) {
  const DModel& m = d.m;
  for (int l = m.sz.nlevel - 2; l >= (skip_world ? 1 : 0); l--) {
    const int adr = m.lvl_adr[l], cnt = m.lvl_adr[l + 1] - adr;
    MJB_PFOR(it, cnt * width) {
      const int p = m.lvl_body[adr + it / width], k = it % width;
      const int ca = m.child_adr[p], cn = m.child_adr[p + 1] - ca;
      if (cn) {
        double s = acc[(long)width * p + k];
        for (int c = 0; c < cn; c++) s += acc[(long)width * m.child_id[ca + c] + k];
        acc[(long)width * p + k] = s;
      }
    }
    MJB_PSYNC();
  }
}

// ------------------------------------------------------------------------------------------------
// subtree centres of mass, com-frame inertias (cinert) and motion axes (cdof)
MJB_HD void com_pos(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody;
  FD sc = d.subtree_com(), xipos = d.xipos(), ximat = d.ximat(), xmat = d.xmat();
  FD cinert = d.cinert(), cdof = d.cdof(), xanchor = d.xanchor(), xaxis = d.xaxis();

  MJB_PFOR(i, nbody) st3(sc, 3 * i, ld3(xipos, 3 * i) * m.body_mass[i]);
  MJB_PSYNC();
  tree_accumulate(d, sc, 3, false);
  MJB_PFOR(i, nbody) {
    if (m.body_subtreemass[i] < kMinVal) st3(sc, 3 * i, ld3(xipos, 3 * i));
    else st3(sc, 3 * i, ld3(sc, 3 * i) * (1.0 / m.body_subtreemass[i]));
  }
  MJB_PSYNC();

  MJB_PFOR(i, nbody) {
    if (i == 0) { for (int k = 0; k < 10; k++) cinert[k] = 0; }
    else {
      V3 off = ld3(xipos, 3 * i) - ld3(sc, 3 * m.body_rootid[i]);
      st10(cinert, 10 * i, inert_com(ldc3(m.body_inertia, 3 * i), ld9(ximat, 9 * i), off, m.body_mass[i]));
    }
  }
  MJB_PFOR(j, m.sz.njnt) {
    const int i = m.jnt_bodyid[j];
    V3 root = ld3(sc, 3 * m.body_rootid[i]);
    int da = 6 * m.jnt_dofadr[j];
    V3 off = root - ld3(xanchor, 3 * j);
    const int jt = m.jnt_type[j];
    if (jt == JNT_FREE || jt == JNT_BALL) {
      if (jt == JNT_FREE) {
        for (int k = 0; k < 18; k++) cdof[da + k] = 0;
        cdof[da + 3] = 1; cdof[da + 10] = 1; cdof[da + 17] = 1;
        da += 18;
      }
      for (int k = 0; k < 3; k++) {
        V3 ax{xmat[9 * i + k], xmat[9 * i + k + 3], xmat[9 * i + k + 6]};
        st3(cdof, da + 6 * k, ax);
        st3(cdof, da + 6 * k + 3, cross(ax, off));
      }
    } else if (jt == JNT_SLIDE) {
      st3(cdof, da, V3{0, 0, 0});
      st3(cdof, da + 3, ld3(xaxis, 3 * j));
    } else {
      V3 ax = ld3(xaxis, 3 * j);
      st3(cdof, da, ax);
      st3(cdof, da + 3, cross(ax, off));
    }
  }
  MJB_PSYNC();
}

#if defined(MJB_SPATIAL_UNIT) || !defined(__CUDA_ARCH__)
// ------------------------------------------------------------------------------------------------
// spatial tendons (FEAT_SPATIAL): compiled on the device only in mjb_kstep_spatial32.cu, so that every other kernel
// keeps its code.  Wrapping: mju_wrap, wrap_circle, wrap_inside, is_intersect, length_circle
// (engine_util_misc.c:35-417); 2D vectors are double[2], dot products in mju_dot's order.
MJB_HD double dot2(const double* a, const double* b) {
  return dot_ref(2, [&](int i) { return a[i]; }, [&](int i) { return b[i]; });
}
MJB_HD double normalize2(double* v) {   // mju_normalize, n = 2
  const double n = sqrt(dot2(v, v));
  if (n < kMinVal) { v[0] = 1; v[1] = 0; }
  else { const double inv = 1 / n; v[0] *= inv; v[1] *= inv; }
  return n;
}
MJB_HD bool wrap_is_intersect(const double* p1, const double* p2, const double* p3, const double* p4) {
  const double det = (p4[1] - p3[1]) * (p2[0] - p1[0]) - (p4[0] - p3[0]) * (p2[1] - p1[1]);
  if (fabs(det) < kMinVal) return false;
  const double a = ((p4[0] - p3[0]) * (p1[1] - p3[1]) - (p4[1] - p3[1]) * (p1[0] - p3[0])) / det;
  const double b = ((p2[0] - p1[0]) * (p1[1] - p3[1]) - (p2[1] - p1[1]) * (p1[0] - p3[0])) / det;
  return a >= 0 && a <= 1 && b >= 0 && b <= 1;
}
MJB_HD double wrap_length_circle(const double* p0, const double* p1, int ind, double radius) {
  double p0n[2] = {p0[0], p0[1]}, p1n[2] = {p1[0], p1[1]};
  normalize2(p0n);
  normalize2(p1n);
  double angle = acos(dot2(p0n, p1n));
  const double cr = p0[1] * p1[0] - p0[0] * p1[1];
  if ((cr > 0 && ind) || (cr < 0 && !ind)) angle = 2 * kPi - angle;
  return radius * angle;
}
// circle wrap of the 2D segment end[0..1] - end[2..3]; side: optional 2D side point.  Length or -1 (no wrap)
MJB_HD double wrap_circle(double* pnt, const double* end, const double* side, double radius) {
  const double sqlen0 = end[0] * end[0] + end[1] * end[1];
  const double sqlen1 = end[2] * end[2] + end[3] * end[3];
  const double sqrad = radius * radius;
  if (sqlen0 < sqrad || sqlen1 < sqrad || radius < kMinVal) return -1;
  const double dif[2] = {end[2] - end[0], end[3] - end[1]};
  const double dd = dif[0] * dif[0] + dif[1] * dif[1];
  if (dd < kMinVal) return -1;
  double a = -(dif[0] * end[0] + dif[1] * end[1]) / dd;
  if (a < 0) a = 0;
  else if (a > 1) a = 1;
  double tmp[2] = {a * dif[0] + end[0], a * dif[1] + end[1]};
  if (tmp[0] * tmp[0] + tmp[1] * tmp[1] > sqrad && (!side || dot2(side, tmp) >= 0)) return -1;
  const double sqrt0 = sqrt(sqlen0 - sqrad), sqrt1 = sqrt(sqlen1 - sqrad);
  double sol[2][2][2], good[2];
  for (int i = 0; i < 2; i++) {
    const double sgn = (i == 0 ? 1 : -1);
    sol[i][0][0] = (end[0] * sqrad + sgn * radius * end[1] * sqrt0) / sqlen0;
    sol[i][0][1] = (end[1] * sqrad - sgn * radius * end[0] * sqrt0) / sqlen0;
    sol[i][1][0] = (end[2] * sqrad - sgn * radius * end[3] * sqrt1) / sqlen1;
    sol[i][1][1] = (end[3] * sqrad + sgn * radius * end[2] * sqrt1) / sqlen1;
    if (side) {
      tmp[0] = sol[i][0][0] + sol[i][1][0]; tmp[1] = sol[i][0][1] + sol[i][1][1];
      normalize2(tmp);
      good[i] = dot2(tmp, side);
    } else {
      tmp[0] = sol[i][0][0] - sol[i][1][0]; tmp[1] = sol[i][0][1] - sol[i][1][1];
      good[i] = -dot2(tmp, tmp);
    }
    if (wrap_is_intersect(end, sol[i][0], end + 2, sol[i][1])) good[i] = -10000;
  }
  const int i = (good[0] > good[1] ? 0 : 1);
  pnt[0] = sol[i][0][0]; pnt[1] = sol[i][0][1]; pnt[2] = sol[i][1][0]; pnt[3] = sol[i][1][1];
  if (wrap_is_intersect(end, pnt, end + 2, pnt + 2)) return -1;
  return wrap_length_circle(sol[i][0], sol[i][1], i, radius);
}
// wrap with the side site inside the circle: Newton iteration on asin(A z) + asin(B z) - 2 asin(z) + G = 0.
// 0 (both points at the same tangent point) or -1 (no wrap)
MJB_HD double wrap_inside(double* pnt, const double* end, double radius) {
  const int maxiter = 20;
  const double zinit = 1 - 1e-7, tolerance = 1e-6;
  const double len0 = sqrt(dot2(end, end)), len1 = sqrt(dot2(end + 2, end + 2));
  const double dif[2] = {end[2] - end[0], end[3] - end[1]};
  const double dd = dif[0] * dif[0] + dif[1] * dif[1];
  if (len0 <= radius || len1 <= radius || radius < kMinVal || len0 < kMinVal || len1 < kMinVal) return -1;
  if (dd > kMinVal) {
    const double a = -(dif[0] * end[0] + dif[1] * end[1]) / dd;
    if (a > 0 && a < 1) {
      const double tmp[2] = {end[0] + dif[0] * a, end[1] + dif[1] * a};
      if (sqrt(dot2(tmp, tmp)) <= radius) return -1;
    }
  }
  pnt[0] = 0.5 * (end[0] + end[2]);
  pnt[1] = 0.5 * (end[1] + end[3]);
  normalize2(pnt);
  pnt[0] = pnt[0] * radius; pnt[1] = pnt[1] * radius;
  pnt[2] = pnt[0]; pnt[3] = pnt[1];
  const double A = radius / len0, B = radius / len1;
  const double cosG = (len0 * len0 + len1 * len1 - dd) / (2 * len0 * len1);
  if (cosG < -1 + kMinVal) return -1;
  else if (cosG > 1 - kMinVal) return 0;
  const double G = acos(cosG);
  double z = zinit;
  double f = asin(A * z) + asin(B * z) - 2 * asin(z) + G;
  if (f > 0) return 0;
  int iter;
  for (iter = 0; iter < maxiter && fabs(f) > tolerance; iter++) {
    const double df = A / dmax(kMinVal, sqrt(1 - z * z * A * A)) + B / dmax(kMinVal, sqrt(1 - z * z * B * B)) -
                      2 / dmax(kMinVal, sqrt(1 - z * z));
    if (df > -kMinVal) return 0;
    const double z1 = z - f / df;
    if (z1 > z) return 0;
    z = z1;
    f = asin(A * z) + asin(B * z) - 2 * asin(z) + G;
    if (f > tolerance) return 0;
  }
  if (iter >= maxiter) return 0;
  double vec[2], ang;
  if (end[0] * end[3] - end[1] * end[2] > 0) { vec[0] = end[0]; vec[1] = end[1]; ang = asin(z) - asin(A * z); }
  else { vec[0] = end[2]; vec[1] = end[3]; ang = asin(z) - asin(B * z); }
  normalize2(vec);
  pnt[0] = radius * (cos(ang) * vec[0] - sin(ang) * vec[1]);
  pnt[1] = radius * (sin(ang) * vec[0] + cos(ang) * vec[1]);
  pnt[2] = pnt[0]; pnt[3] = pnt[1];
  return 0;
}
MJB_HD V3 mul_mat_t(const M3& a, V3 v) {   // mju_mulMatTVec3
  return V3{a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z,
            a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z};
}
// mju_wrap: the path x0 -> x1 around a sphere / cylinder (geom frame xpos, xmat), optional side site.  Returns the
// wrap length and the two tangent points w0, w1, or -1 when the straight segment does not touch the geom
MJB_HD double wrap_geom(V3& w0, V3& w1, V3 x0, V3 x1, V3 xpos, const M3& xmat, double radius, int type,
                        const V3* side) {
  const V3 p0 = mul_mat_t(xmat, x0 - xpos), p1 = mul_mat_t(xmat, x1 - xpos);
  if (sqrt(dot(p0, p0)) < kMinVal || sqrt(dot(p1, p1)) < kMinVal) return -1;
  V3 ax0, ax1;
  if (type == WRAP_SPHERE) {
    ax0 = p0;
    normalize(ax0);
    V3 normal = cross(p0, p1);
    const double nrm = normalize(normal);
    if (nrm < kMinVal) {   // p0, p1 parallel
      int i = 0;
      if (fabs(ax0.y) > fabs(ax0.x) && fabs(ax0.y) > fabs(ax0.z)) i = 1;
      if (fabs(ax0.z) > fabs(ax0.x) && fabs(ax0.z) > fabs(ax0.y)) i = 2;
      ax1 = V3{i == 0 ? 0.0 : 1.0, i == 1 ? 0.0 : 1.0, i == 2 ? 0.0 : 1.0};
      normal = cross(ax0, ax1);
      normalize(normal);
    }
    ax1 = cross(normal, ax0);
    normalize(ax1);
  } else {
    ax0 = V3{1, 0, 0};
    ax1 = V3{0, 1, 0};
  }
  const double dd[4] = {dot(p0, ax0), dot(p0, ax1), dot(p1, ax0), dot(p1, ax1)};
  V3 s{0, 0, 0};
  double sd[2] = {0, 0};
  if (side) {
    s = mul_mat_t(xmat, *side - xpos);
    sd[0] = dot(s, ax0); sd[1] = dot(s, ax1);
    normalize2(sd);
    sd[0] = sd[0] * radius; sd[1] = sd[1] * radius;
  }
  double wlen, pnt[4];
  if (side && sqrt(dot(s, s)) < radius) wlen = wrap_inside(pnt, dd, radius);
  else wlen = wrap_circle(pnt, dd, side ? sd : nullptr, radius);
  if (wlen < 0) return -1;
  V3 r0 = ax0 * pnt[0], r1 = ax0 * pnt[2];
  r0 = r0 + ax1 * pnt[1];
  r1 = r1 + ax1 * pnt[3];
  if (type == WRAP_CYLINDER) {
    const double L0 = sqrt((p0.x - r0.x) * (p0.x - r0.x) + (p0.y - r0.y) * (p0.y - r0.y));
    const double L1 = sqrt((p1.x - r1.x) * (p1.x - r1.x) + (p1.y - r1.y) * (p1.y - r1.y));
    r0.z = p0.z + (p1.z - p0.z) * L0 / (L0 + wlen + L1);
    r1.z = p0.z + (p1.z - p0.z) * (L0 + wlen) / (L0 + wlen + L1);
    const double height = fabs(r1.z - r0.z);
    wlen = sqrt(wlen * wlen + height * height);
  }
  w0 = mulmv(xmat, r0) + xpos;
  w1 = mulmv(xmat, r1) + xpos;
  return wlen;
}
MJB_HD double jac_elem(const Env& d, V3 pt, int body, int k, int c);   // mjb_constraint.h
MJB_HD double dist3(V3 a, V3 b) { const V3 d = a - b; return sqrt(d.x * d.x + d.y * d.y + d.z * d.z); }

// phase 1, one lane per spatial tendon: walk the path (mj_tendon, engine_core_smooth.c:985-1109) for the length and
// the path points.  The points go to the tendon's own slot (tendon_slotadr) in wrap_xpos / wrap_obj, since the running
// count ten_wrapadr depends on which wraps of the earlier tendons are active; ten_wrapnum holds the count.
MJB_HD void tendon_path(const Env& d, int i) {
  const DModel& m = d.m;
  FD sx = d.site_xpos(), gx = d.geom_xpos(), gm = d.geom_xmat(), wx = d.wrap_xpos();
  FI wo = d.wrap_obj();
  const int adr = m.tendon_adr[i], num = m.tendon_num[i], w0 = m.tendon_slotadr[i];
  int w = w0, j = 0;
  double len = 0, divisor = 1;
  while (j < num - 1) {
    int t1 = m.wrap_type[adr + j + 1], id1 = m.wrap_objid[adr + j + 1];
    const int t0 = m.wrap_type[adr + j], id0 = m.wrap_objid[adr + j];
    if (t0 == WRAP_PULLEY || t1 == WRAP_PULLEY) {
      if (t0 == WRAP_PULLEY) {
        divisor = m.wrap_prm[adr + j];
        st3(wx, 3 * w, V3{0, 0, 0});
        wo[w++] = -2;
      }
      j++;
      continue;
    }
    const V3 p0 = ld3(sx, 3 * id0);
    double wlen = -1;
    int wrapid = -1;
    const bool geom = (t1 == WRAP_SPHERE || t1 == WRAP_CYLINDER);
    V3 a, b;
    if (geom) {
      wrapid = id1;
      id1 = m.wrap_objid[adr + j + 2];
      const int sideid = round_int(m.wrap_prm[adr + j + 1]);
      const V3 side = sideid >= 0 ? ld3(sx, 3 * sideid) : V3{0, 0, 0};
      wlen = wrap_geom(a, b, p0, ld3(sx, 3 * id1), ld3(gx, 3 * wrapid), ld9(gm, 9 * wrapid), m.geom_size[3 * wrapid], t1,
                       sideid >= 0 ? &side : nullptr);
    }
    const V3 p1 = ld3(sx, 3 * id1);
    if (wlen < 0) len += dist3(p0, p1) / divisor;
    else len += (dist3(p0, a) + wlen + dist3(b, p1)) / divisor;
    st3(wx, 3 * w, p0);
    wo[w] = -1;
    if (wlen >= 0) {
      st3(wx, 3 * (w + 1), a);
      st3(wx, 3 * (w + 2), b);
      wo[w + 1] = wrapid; wo[w + 2] = wrapid;
    }
    w += (wlen < 0 ? 1 : 3);
    j += (geom ? 2 : 1);
    if (j == num - 1 || m.wrap_type[adr + j + 1] == WRAP_PULLEY) {   // last site before a pulley or the end
      st3(wx, 3 * w, p1);
      wo[w++] = -1;
    }
  }
  d.ten_length()[i] = len;
  d.ten_wrapnum()[i] = w - w0;
}

// tendon Jacobian entry (tendon i, row element a, column c) from one path segment q1 (body b1) -> q2 (body b2): the
// chain rule of mj_tendon with mj_jacDifPair (engine_core_util.c:437-516, issparse = 1), mju_mulMatTVec and
// mju_combineSparseInc (engine_util_sparse.c:309), for this one element.  J is the element so far; scl = 1/divisor.
MJB_HD double segment_entry(const Env& d, int i, int a, int c, double J, V3 q1, int b1, V3 q2, int b2, double scl) {
  const DModel& m = d.m;
  const int nv = m.sz.nv;
  V3 dif = q2 - q1;
  normalize(dif);
  const bool simple = m.body_simple[b1] && m.body_simple[b2];
  // the merged dof chain (mj_mergeChainSimple / mj_mergeChain), increasing: NV and membership
  auto in_chain = [&](int k) -> bool {
    if (simple) return (k >= m.body_dofadr[b1] && k < m.body_dofadr[b1] + m.body_dofnum[b1]) ||
                       (k >= m.body_dofadr[b2] && k < m.body_dofadr[b2] + m.body_dofnum[b2]);
    return m.body_dofanc[(long)b1 * nv + k] || m.body_dofanc[(long)b2 * nv + k];
  };
  int NV = 0;
  if (simple) NV = m.body_dofnum[b1] + m.body_dofnum[b2];
  else for (int k = 0; k < nv; k++) NV += in_chain(k);
  if (!NV) return J;
  // column k of (jac2 - jac1) . dif, zero components of dif skipped.  Simple bodies write -(first) and +(second)
  // straight into the difference (mj_jacSparseSimple); otherwise jac2 - jac1 of the two chain Jacobians.
  auto chain_rule = [&](int k) -> double {
    double jd[3];
    if (simple) {
      const bool second = k >= m.body_dofadr[b2] && k < m.body_dofadr[b2] + m.body_dofnum[b2];
      const V3 pt = second ? q2 : q1;
      const int body = second ? b2 : b1;
      const V3 off = pt - ld3(d.subtree_com(), 3 * m.body_rootid[body]);
      const V3 t = cross(ld3(d.cdof(), 6 * k), off);
      for (int r = 0; r < 3; r++) {
        const double v = d.cdof()[6 * k + 3 + r] + get(t, r);
        jd[r] = second ? v : -v;
      }
    } else {
      for (int r = 0; r < 3; r++) jd[r] = jac_elem(d, q2, b2, r, k) - jac_elem(d, q1, b1, r, k);
    }
    double res = 0;
    for (int r = 0; r < 3; r++) { const double s = get(dif, r); if (s) res += jd[r] * s; }
    return res;
  };
  const int radr = m.ten_J_rowadr[i], rnnz = m.ten_J_rownnz[i];
  bool same = (NV == rnnz);
  for (int e = 0; e < rnnz && same; e++) same = in_chain(m.ten_J_colind[radr + e]);
  if (same) {   // identical pattern: dst = 1*dst + scl*src, element for element (mju_addToSclScl)
    int k = 0, n = -1;   // the a-th dof of the chain
    for (; k < nv; k++) if (in_chain(k) && ++n == a) break;
    return J * 1.0 + chain_rule(k) * scl;
  }
  if (!in_chain(c)) return J;   // merge: only common indices change
  return J + scl * chain_rule(c);
}

// phase 2, one lane per element of a spatial tendon's ten_J row: the element's segments in path order, with the
// points of phase 1 (sites from site_xpos, tangent points from the tendon's slot)
MJB_HD void tendon_jacobian(const Env& d) {
  const DModel& m = d.m;
  FD J = d.ten_J(), sx = d.site_xpos(), wx = d.wrap_xpos();
  FI wo = d.wrap_obj();
  MJB_PFOR(q, m.sz.nJten) {
    int i = 0;
    while (i + 1 < m.sz.ntendon && m.ten_J_rowadr[i + 1] <= q) i++;
    const int adr = m.tendon_adr[i], num = m.tendon_num[i];
    if (m.wrap_type[adr] == WRAP_JOINT) continue;
    const int a = q - m.ten_J_rowadr[i], c = m.ten_J_colind[q];
    double val = 0, divisor = 1;
    int w = m.tendon_slotadr[i], j = 0;
    while (j < num - 1) {
      const int t0 = m.wrap_type[adr + j], t1 = m.wrap_type[adr + j + 1];
      if (t0 == WRAP_PULLEY || t1 == WRAP_PULLEY) {
        if (t0 == WRAP_PULLEY) { divisor = m.wrap_prm[adr + j]; w++; }
        j++;
        continue;
      }
      const bool geom = (t1 == WRAP_SPHERE || t1 == WRAP_CYLINDER);
      const int id0 = m.wrap_objid[adr + j], id1 = m.wrap_objid[adr + j + (geom ? 2 : 1)];
      const bool wrapped = geom && wo[w + 1] >= 0;
      V3 pt[4];
      int bd[4];
      pt[0] = ld3(sx, 3 * id0); bd[0] = m.site_bodyid[id0];
      const int np = wrapped ? 4 : 2;
      if (wrapped) {
        pt[1] = ld3(wx, 3 * (w + 1)); pt[2] = ld3(wx, 3 * (w + 2));
        bd[1] = bd[2] = m.geom_bodyid[m.wrap_objid[adr + j + 1]];
      }
      pt[np - 1] = ld3(sx, 3 * id1); bd[np - 1] = m.site_bodyid[id1];
      for (int k = 0; k + 1 < np; k++)
        if (bd[k] != bd[k + 1]) val = segment_entry(d, i, a, c, val, pt[k], bd[k], pt[k + 1], bd[k + 1], 1 / divisor);
      w += wrapped ? 3 : 1;
      j += geom ? 2 : 1;
      if (j == num - 1 || m.wrap_type[adr + j + 1] == WRAP_PULLEY) w++;
    }
    J[q] = val;
  }
}

// ten_wrapadr as the running count over the tendons, and each spatial tendon's points packed from its slot to there
// (slots never start before the packed position, so one forward pass moves them in place)
MJB_HD void tendon_pack(const Env& d) {
  const DModel& m = d.m;
  MJB_LANE0 {
    FD wx = d.wrap_xpos();
    FI wo = d.wrap_obj(), wadr = d.ten_wrapadr(), wnum = d.ten_wrapnum();
    int cnt = 0;
    for (int i = 0; i < m.sz.ntendon; i++) {
      const bool spatial = m.wrap_type[m.tendon_adr[i]] != WRAP_JOINT;
      const int n = spatial ? wnum[i] : 0, s = m.tendon_slotadr[i];
      wadr[i] = cnt;
      wnum[i] = n;
      for (int k = 0; k < n; k++) {
        for (int r = 0; r < 3; r++) wx[3 * (cnt + k) + r] = wx[3 * (s + k) + r];
        wo[cnt + k] = wo[s + k];
      }
      cnt += n;
    }
  }
  MJB_PSYNC();
}
#endif

// ------------------------------------------------------------------------------------------------
// tendons: length and sparse Jacobian.  Fixed tendons: constant pattern, one lane per tendon.  Spatial tendons
// (FEAT_SPATIAL): path walk per tendon, then the Jacobian elements spread over the lanes, then the path packing.
MJB_HD void tendon(const Env& d) {
  const DModel& m = d.m;
  const int nt = m.sz.ntendon;
  if (!nt) return;
  FD L = d.ten_length(), J = d.ten_J(), qpos = d.qpos();
  MJB_PFOR(i, nt) {
    const int adr = m.tendon_adr[i], num = m.tendon_num[i];
#if defined(MJB_SPATIAL_UNIT) || !defined(__CUDA_ARCH__)
    if ((d.feat & FEAT_SPATIAL) && m.wrap_type[adr] != WRAP_JOINT) { tendon_path(d, i); continue; }
#endif
    const int radr = m.ten_J_rowadr[i], rnnz = m.ten_J_rownnz[i];
    double len = 0;
    for (int a = 0; a < rnnz; a++) J[radr + a] = 0;
    for (int j = 0; j < num; j++) {
      const int k = m.wrap_objid[adr + j];
      const double c = m.wrap_prm[adr + j];
      len += c * qpos[m.jnt_qposadr[k]];
      // J(row i, col dofadr) = 1*J + c*1   (mju_combineSparseInc with a single source entry)
      const int dof = m.jnt_dofadr[k];
      for (int a = 0; a < rnnz; a++) {
        if (m.ten_J_colind[radr + a] == dof) { J[radr + a] = 1.0 * J[radr + a] + c * 1.0; break; }
      }
    }
    L[i] = len;
  }
  MJB_PSYNC();
#if defined(MJB_SPATIAL_UNIT) || !defined(__CUDA_ARCH__)
  if (d.feat & FEAT_SPATIAL) {
    tendon_jacobian(d);
    MJB_PSYNC();
    tendon_pack(d);
  }
#endif
}

// ------------------------------------------------------------------------------------------------
// transmissions (mj_transmission, engine_core_smooth.c:1380-1480): scalar joints — actuator_length and the
// single moment entry; fixed tendons — length = ten_length * gear, moment row = ten_J row * gear (the row
// values are re-formed as ten_J * gear where they are used, actuator_moment keeps the gear)
MJB_HD void transmission(const Env& d) {
  const DModel& m = d.m;
  FD len = d.actuator_length(), mom = d.actuator_moment(), qpos = d.qpos();
  MJB_PFOR(i, m.sz.nu) {
    const int j = m.actuator_trnjnt[i];
    const double g = m.actuator_gear0[i];
    const int tt = (d.feat & FEAT_ACT) ? m.actuator_trntype[i] : TRN_JOINT;
    if (tt == TRN_TENDON) len[i] = d.ten_length()[j] * g;
    else if (tt == TRN_BALL || tt == TRN_FREE) {   // 3D / 6D gear (engine_core_smooth.c:1331-1393)
      const double* gear = m.actuator_gear6 + 6 * i;
      FD m6 = d.actuator_mom6();
      Q4 q = ld4(qpos, m.jnt_qposadr[j] + (tt == TRN_FREE ? 3 : 0));
      normalize(q);
      V3 ga{gear[tt == TRN_FREE ? 3 : 0], gear[tt == TRN_FREE ? 4 : 1], gear[tt == TRN_FREE ? 5 : 2]};
      if (m.actuator_inparent[i]) ga = rotate(ga, Q4{q.w, -q.x, -q.y, -q.z});
      if (tt == TRN_BALL) {
        const V3 axis = quat2vel(q, 1);
        len[i] = axis.x * ga.x + axis.y * ga.y + axis.z * ga.z;
        m6[6 * i] = ga.x; m6[6 * i + 1] = ga.y; m6[6 * i + 2] = ga.z;
      } else {
        len[i] = 0;
        m6[6 * i] = gear[0]; m6[6 * i + 1] = gear[1]; m6[6 * i + 2] = gear[2];
        m6[6 * i + 3] = ga.x; m6[6 * i + 4] = ga.y; m6[6 * i + 5] = ga.z;
      }
    }
    else if (tt >= TRN_SITE) len[i] = 0;   // length and moment row: site_moment(), after the site poses exist
    else len[i] = qpos[m.jnt_qposadr[j]] * g;
    mom[i] = g;
  }
  MJB_PSYNC();
}

// ------------------------------------------------------------------------------------------------
// composite rigid body algorithm -> tree-sparse M, plus tendon armature
MJB_HD void make_M(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody, nv = m.sz.nv;
  FD crb = d.crb(), cinert = d.cinert(), cdof = d.cdof(), M = d.M();
  MJB_PFOR(i, 10 * nbody) crb[i] = cinert[i];
  MJB_PFOR(i, m.sz.nC) M[i] = 0;
  MJB_PSYNC();
  tree_accumulate(d, crb, 10, true);
  MJB_PFOR(i, nv) {
    const int adr = m.M_rowadr[i];
    if (m.dof_simplenum[i]) { M[adr] = m.dof_M0[i]; }
    else {
      int a = adr + m.M_rownnz[i] - 1;
      double acc = m.dof_armature_eff[i];
      S6 buf = mul_inert(ld10(crb, 10 * m.dof_bodyid[i]), ld6(cdof, 6 * i));
      for (int j = i; j >= 0; j = m.dof_parentid[j]) {
        M[a] = acc + dot6(ld6(cdof, 6 * j), buf);
        acc = 0;
        a--;
      }
    }
  }
  MJB_PSYNC();
  // tendon armature: M += armature * J' J  over the tendon's sparsity pattern (rare; serial)
  bool any = false;
  for (int k = 0; k < m.sz.ntendon; k++) any = any || (m.tendon_armature_eff[k] != 0);
  if (any) {
    MJB_LANE0 {
      FD tJ = d.ten_J();
      for (int k = 0; k < m.sz.ntendon; k++) {
        const double arm = m.tendon_armature_eff[k];
        if (!arm) continue;
        const int jadr = m.ten_J_rowadr[k], jnnz = m.ten_J_rownnz[k];
        for (int j = 0; j < jnnz; j++) {
          const double Ji = tJ[jadr + j];
          if (!Ji) continue;
          const int i = m.ten_J_colind[jadr + j];
          const int madr = m.M_rowadr[i], mnnz = m.M_rownnz[i];
          const double scl = arm * Ji;
          int a = 0, b = 0;   // walk both sorted index lists (mju_addToSclSparseInc)
          while (a < mnnz && b < jnnz) {
            const int ca = m.M_colind[madr + a], cb = m.ten_J_colind[jadr + b];
            if (ca == cb) { M[madr + a] += scl * tJ[jadr + b]; a++; b++; }
            else if (ca < cb) a++;
            else b++;
          }
        }
      }
    }
    MJB_PSYNC();
  }
}

// ------------------------------------------------------------------------------------------------
// in-place sparse L'DL of a tree-sparse matrix in M's CSR pattern.  Pivot rows are processed
// serially (nv-1..0) as in the reference; the element updates of one pivot are independent and
// come from the host-built program (fac_*).
MJB_HD void factor_I(const Env& d, FD mat, FD diaginv) {
  const DModel& m = d.m;
  const int nv = m.sz.nv;
  for (int k = nv - 1; k >= 0; k--) {
    const int start = m.M_rowadr[k];
    const int diag = m.M_rownnz[k] - 1;
    const double invD = 1 / mat[start + diag];
    MJB_LANE0 diaginv[k] = invD;
    if (diag == 0) continue;
    const int pa = m.fac_adr[k], pn = m.fac_adr[k + 1] - pa;
    MJB_PFOR(t, pn) {
      const int dst = m.fac_dst[pa + t];
      mat[dst] += mat[m.fac_src[pa + t]] * (-mat[m.fac_cf[pa + t]] * invD);
    }
    MJB_PSYNC();
    MJB_PFOR(c, diag) mat[start + c] = mat[start + c] * invD;
    MJB_PSYNC();
  }
  MJB_PSYNC();
}

// in-place x <- (L'DL)^-1 x for one right-hand side, by dof-tree levels
MJB_HD void solve_LD(const Env& d, FD x, FD qLD, FD qLDiagInv) {
  const DModel& m = d.m;
  const int nv = m.sz.nv;
  // x <- L^-T x : deepest dofs are final; each dof then gathers its descendants' contributions in
  // descending descendant order (the order of the serial scatter loop)
  for (int l = m.sz.ndlevel - 2; l >= 0; l--) {
    const int adr = m.dlvl_adr[l], cnt = m.dlvl_adr[l + 1] - adr;
    MJB_PFOR(t, cnt) {
      const int j = m.dlvl_dof[adr + t];
      const int a0 = m.mt_adr[j], an = m.mt_adr[j + 1] - a0;
      if (an) {
        double s = x[j];
        for (int c = 0; c < an; c++) {
          const double xi = x[m.mt_dof[a0 + c]];
          if (xi != 0) s -= qLD[m.mt_qadr[a0 + c]] * xi;
        }
        x[j] = s;
      }
    }
    MJB_PSYNC();
  }
  MJB_PFOR(i, nv) x[i] *= qLDiagInv[i];
  MJB_PSYNC();
  // x <- L^-1 x : shallow dofs are final first
  for (int l = 1; l < m.sz.ndlevel; l++) {
    const int adr = m.dlvl_adr[l], cnt = m.dlvl_adr[l + 1] - adr;
    MJB_PFOR(t, cnt) {
      const int i = m.dlvl_dof[adr + t];
      const int ra = m.M_rowadr[i], dn = m.M_rownnz[i] - 1;
      x[i] -= dot_sparse_ref(dn, [&](int c) { return qLD[ra + c]; },
                             [&](int c) { return x[m.M_colind[ra + c]]; });
    }
    MJB_PSYNC();
  }
}

// ------------------------------------------------------------------------------------------------
// com-frame body velocities and time derivatives of the motion axes, level by level
MJB_HD void com_vel(const Env& d) {
  const DModel& m = d.m;
  FD cvel = d.cvel(), cdof = d.cdof(), cdd = d.cdof_dot(), qvel = d.qvel();
  MJB_LANE0 { for (int k = 0; k < 6; k++) cvel[k] = 0; }
  MJB_PSYNC();
  for (int l = 1; l < m.sz.nlevel; l++) {
    const int ladr = m.lvl_adr[l], cnt = m.lvl_adr[l + 1] - ladr;
    MJB_PFOR(k_, cnt) {
      const int i = m.lvl_body[ladr + k_];
      S6 cv = ld6(cvel, 6 * m.body_parentid[i]);
      const int dn = m.body_dofnum[i], bda = m.body_dofadr[i];
      for (int j = 0; j < dn; j++) {
        const int jt = m.jnt_type[m.dof_jntid[bda + j]];
        if (jt == JNT_FREE || jt == JNT_BALL) {
          if (jt == JNT_FREE) {
            for (int k = 0; k < 18; k++) cdd[6 * bda + k] = 0;
            // cvel += cdof[0..2]' * qvel[0..2]   (mju_mulMatTVec: skip exact zeros, row by row)
            S6 t; for (int k = 0; k < 6; k++) t.v[k] = 0;
            for (int r = 0; r < 3; r++) {
              const double s = qvel[bda + r];
              if (s != 0) for (int k = 0; k < 6; k++) t.v[k] += cdof[6 * (bda + r) + k] * s;
            }
            for (int k = 0; k < 6; k++) cv.v[k] += t.v[k];
            j += 3;
          }
          for (int r = 0; r < 3; r++) st6(cdd, 6 * (bda + j + r), cross_motion(cv, ld6(cdof, 6 * (bda + j + r))));
          S6 t; for (int k = 0; k < 6; k++) t.v[k] = 0;
          for (int r = 0; r < 3; r++) {
            const double s = qvel[bda + j + r];
            if (s != 0) for (int k = 0; k < 6; k++) t.v[k] += cdof[6 * (bda + j + r) + k] * s;
          }
          for (int k = 0; k < 6; k++) cv.v[k] += t.v[k];
          j += 2;
        } else {
          S6 cd = ld6(cdof, 6 * (bda + j));
          st6(cdd, 6 * (bda + j), cross_motion(cv, cd));
          const double s = qvel[bda + j];
          for (int k = 0; k < 6; k++) cv.v[k] += cd.v[k] * s;
        }
      }
      st6(cvel, 6 * i, cv);
    }
    MJB_PSYNC();
  }
}

// res = sum_r dof[r] * vec[r] over n dofs (mju_mulDofVec, engine_util_spatial.c:466-474)
MJB_HD S6 mul_dof_vec(FD dof, FD vec, int n) {
  S6 r;
  if (n == 1) {
    for (int k = 0; k < 6; k++) r.v[k] = dof[k] * vec[0];
  } else {
    for (int k = 0; k < 6; k++) r.v[k] = 0;
    for (int a = 0; a < n; a++) {
      const double s = vec[a];
      if (s != 0) for (int k = 0; k < 6; k++) r.v[k] += dof[6 * a + k] * s;
    }
  }
  return r;
}

// bias forces by recursive Newton-Euler without the acceleration term (flg_acc = 0)
MJB_HD void rne_bias(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody, nv = m.sz.nv;
  FD cacc = d.scr_body(), cfrc = d.scr_body() + 6 * nbody;
  FD cinert = d.cinert(), cvel = d.cvel(), cdof = d.cdof(), cdd = d.cdof_dot(), qvel = d.qvel();
  MJB_LANE0 {
    for (int k = 0; k < 6; k++) { cacc[k] = 0; cfrc[k] = 0; }
    if (!(m.opt.disableflags & DSBL_GRAVITY)) {
      cacc[3] = m.opt.gravity[0] * -1; cacc[4] = m.opt.gravity[1] * -1; cacc[5] = m.opt.gravity[2] * -1;
    }
  }
  MJB_PSYNC();
  for (int l = 1; l < m.sz.nlevel; l++) {
    const int ladr = m.lvl_adr[l], cnt = m.lvl_adr[l + 1] - ladr;
    MJB_PFOR(k_, cnt) {
      const int i = m.lvl_body[ladr + k_];
      const int bda = m.body_dofadr[i];
      S6 t = mul_dof_vec(cdd + 6 * bda, qvel + bda, m.body_dofnum[i]);
      S6 a = ld6(cacc, 6 * m.body_parentid[i]);
      for (int k = 0; k < 6; k++) a.v[k] = a.v[k] + t.v[k];
      st6(cacc, 6 * i, a);
      I10 I = ld10(cinert, 10 * i);
      S6 f = mul_inert(I, a);
      S6 v = ld6(cvel, 6 * i);
      S6 Iv = mul_inert(I, v);
      S6 c = cross_force(v, Iv);
      for (int k = 0; k < 6; k++) f.v[k] += c.v[k];
      st6(cfrc, 6 * i, f);
    }
    MJB_PSYNC();
  }
  // backward accumulation; the reference zeroes the world force first and never adds into it
  tree_accumulate(d, cfrc, 6, true);
  FD out = d.qfrc_bias();
  MJB_PFOR(i, nv) out[i] = dot6(ld6(cdof, 6 * i), ld6(cfrc, 6 * m.dof_bodyid[i]));
  MJB_PSYNC();
}

// ------------------------------------------------------------------------------------------------
// passive forces: joint springs, dof dampers, tendon spring-dampers
MJB_HD void passive(const Env& d) {
  const DModel& m = d.m;
  const int nv = m.sz.nv;
  FD fs = d.qfrc_spring(), fd = d.qfrc_damper(), fp = d.qfrc_passive(), qpos = d.qpos(), qvel = d.qvel();
  MJB_PFOR(i, nv) { fs[i] = 0; fd[i] = 0; fp[i] = 0; }
  MJB_PSYNC();
  const bool spring = !(m.opt.disableflags & DSBL_SPRING), damper = !(m.opt.disableflags & DSBL_DAMPER);
  if (!spring && !damper) return;
  if (spring) {
    MJB_PFOR(j, m.sz.njnt) {
      const double k0 = m.jnt_stiffness[j];
      const double* sp = m.jnt_stiffnesspoly + kNPoly * j;
      if (k0 == 0 && sp[0] == 0 && sp[1] == 0) continue;
      int pa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
      const int jt = m.jnt_type[j];
      if (jt == JNT_FREE || jt == JNT_BALL) {
        if (jt == JNT_FREE) {
          V3 dif = ld3(qpos, pa) - ldc3(m.qpos_spring, pa);
          double r = sqrt(dot(dif, dif));
          double k = poly_force(k0, sp, kNPoly, r, false);
          st3(fs, da, addscl(ld3(fs, da), dif, -k));
          da += 3; pa += 3;
        }
        Q4 q = ld4(qpos, pa);
        normalize(q);
        V3 dif = qsub(q, ldc4(m.qpos_spring, pa));
        double r = sqrt(dot(dif, dif));
        double k = poly_force(k0, sp, kNPoly, r, false);
        st3(fs, da, addscl(ld3(fs, da), dif, -k));
      } else {
        const double x = qpos[pa] - m.qpos_spring[pa];
        fs[da] = -x * poly_force(k0, sp, kNPoly, x, false);
      }
    }
  }
  if (damper) {
    MJB_PFOR(i, nv) {
      const double b = m.dof_damping_eff[i];
      const double* bp = m.dof_dampingpoly_eff + kNPoly * i;
      if (b != 0 || bp[0] != 0 || bp[1] != 0) {
        const double v = qvel[i];
        fd[i] = -v * poly_force(b, bp, kNPoly, v, true);
      }
    }
  }
  MJB_PSYNC();
  if (m.sz.ntendon) {
    MJB_LANE0 {   // tendons may share dofs: keep the reference's serial accumulation order
      FD tl = d.ten_length(), tv = d.ten_velocity(), tJ = d.ten_J();
      for (int i = 0; i < m.sz.ntendon; i++) {
        double k0 = 0, b0 = 0;
        const double* sp = m.tendon_stiffnesspoly + kNPoly * i;
        double dp[kNPoly] = {0, 0};
        if (spring) k0 = m.tendon_stiffness[i];
        if (damper) { b0 = m.tendon_damping_eff[i]; dp[0] = m.tendon_dampingpoly_eff[kNPoly * i]; dp[1] = m.tendon_dampingpoly_eff[kNPoly * i + 1]; }
        if (k0 == 0 && (!spring || (sp[0] == 0 && sp[1] == 0)) && b0 == 0 && dp[0] == 0 && dp[1] == 0) continue;
        const double len = tl[i], lo = m.tendon_lengthspring[2 * i], hi = m.tendon_lengthspring[2 * i + 1];
        const double x = (len > hi) ? len - hi : (len < lo) ? len - lo : 0;
        const double f_s = spring ? -x * poly_force(k0, sp, kNPoly, x, false) : 0;
        const double v = tv[i];
        const double f_d = damper ? -v * poly_force(b0, dp, kNPoly, v, true) : 0;
        if (f_s || f_d) {
          const int adr = m.ten_J_rowadr[i], end = adr + m.ten_J_rownnz[i];
          for (int j = adr; j < end; j++) {
            const int k = m.ten_J_colind[j];
            const double Jv = tJ[j];
            fs[k] += Jv * f_s;
            fd[k] += Jv * f_d;
          }
        }
      }
    }
    MJB_PSYNC();
  }
  MJB_PFOR(i, nv) fp[i] = fs[i] + fd[i];
  MJB_PSYNC();
}

}  // namespace mjb
