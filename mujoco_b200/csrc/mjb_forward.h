// Pipeline driver of the batched mj_step path for ONE environment (cooperative lanes).
//
// Replaces (reference file:line) src/engine/engine_forward.c: mj_checkPos/Vel/Acc :54-113,
// mj_fwdPosition :131-177, mj_fwdVelocity :181-225, mj_fwdActuation :353-1003 (motor / affine
// gain-bias family on hinge and slide joints), mj_fwdAcceleration :1007-1052, mj_fwdConstraint
// :1148-1252, mj_EulerSkip :1398-1476, mj_advance :1261-1395, mj_step :1846-1880; and
// src/engine/engine_support.c mj_integratePos :639-680.
//
// Stages (ids used by mjb_run_stages and the kernels):
//   0 position   checks, kinematics, com, tendon, M, L'DL, collision, constraint rows, dual
//                projection (PGS), transmission
//   1 velocity   velocity, passive, reference, bias, actuation, smooth acceleration, efc_b and the
//                solver start point (warmstart)
//   2 solve      PGS (or Newton) iterations
//   3 integrate  dual finish, acceleration check, semi-implicit Euler, advance
//   4 finish     dual finish only (mj_forward)
#pragma once
#include "mjb_prof.h"
#include "mjb_collision.h"
#include "mjb_constraint.h"
#include "mjb_newton.h"
#include "mjb_history.h"

namespace mjb {

// history buffers as mj_resetData leaves them (engine_io.c:1404-1454): control samples at -n*dt .. -dt, zero; sensor
// samples on the same grid, or with an interval at its ticks before the first one rounded up to the timestep grid,
// the last tick in the user slot (-period for phase 0, else the phase).  Serial (one lane).
MJB_HD void reset_history(const Env& d) {
  const DModel& m = d.m;
  const double dt = m.opt.timestep;
  FD h = d.history();
  for (int i = 0; i < m.sz.nu; i++) {
    const int n = m.actuator_history[2 * i];
    if (n <= 0) continue;
    FD buf = h + m.actuator_historyadr[i];
    buf[0] = 0;
    buf[1] = n - 1;
    for (int j = 0; j < n; j++) buf[2 + j] = -(n - j) * dt;
    for (int j = 0; j < n; j++) buf[2 + n + j] = 0;
  }
  for (int i = 0; i < m.sz.nsensor; i++) {
    const int n = m.sensor_history[2 * i];
    if (n <= 0) continue;
    const int dim = m.sensor_dim[i];
    const double period = m.sensor_interval[2 * i], phase = m.sensor_interval[2 * i + 1];
    FD buf = h + m.sensor_historyadr[i];
    buf[0] = (period > 0) ? (phase == 0 ? -period : phase) : -dt;
    buf[1] = n - 1;
    if (period > 0) {
      const double t0 = (phase == 0) ? -period : phase;
      for (int j = 0; j < n; j++) {
        const double ct = t0 - (n - 1 - j) * period;
        buf[2 + j] = ceil(ct / dt) * dt;
      }
    } else {
      for (int j = 0; j < n; j++) buf[2 + j] = -(n - j) * dt;
    }
    for (int j = 0; j < n * dim; j++) buf[2 + n + j] = 0;
  }
  d.hist_flg()[0] = 0;
  d.hist_flg()[1] = 0;
}

// mj_readCtrl (engine_support.c:886-908): a delayed actuator's control at time - delay, read from its buffer
MJB_HD double read_ctrl(const Env& d, int i) {
  const DModel& m = d.m;
  double c;
  hist_read(d.history() + m.actuator_historyadr[i], m.actuator_history[2 * i], 1, &c, d.time()[0] - m.actuator_delay[i],
            m.actuator_history[2 * i + 1]);
  return c;
}

// mj_resetData for one environment: qpos0, zero velocities/controls/warmstart/time/warnings
MJB_HD void reset_env(const Env& d, bool clear_warnings) {
  const DModel& m = d.m;
  FD qpos = d.qpos(), qvel = d.qvel(), ctrl = d.ctrl(), ws = d.qacc_warmstart(), qa = d.qfrc_applied();
  for (int i = 0; i < m.sz.nq; i++) qpos[i] = m.qpos0[i];
  for (int i = 0; i < m.sz.nv; i++) { qvel[i] = 0; ws[i] = 0; qa[i] = 0; d.qacc()[i] = 0; }
  for (int i = 0; i < m.sz.nu; i++) ctrl[i] = 0;
  for (int i = 0; i < m.sz.na; i++) { d.act()[i] = 0; d.act_dot()[i] = 0; }
  for (int i = 0; i < 6 * m.sz.nbody; i++) d.xfrc_applied()[i] = 0;
  for (int i = 0; i < m.sz.neq; i++) d.eq_active()[i] = m.eq_active0[i];
  if (m.sz.nmocap) {   // mj_resetData: mocap poses from the model (engine_io.c:1531-1540)
    for (int i = 0; i < m.sz.nbody; i++) {
      const int mid = m.body_mocapid[i];
      if (mid < 0) continue;
      for (int k = 0; k < 3; k++) d.mocap_pos()[3 * mid + k] = m.body_pos[3 * i + k];
      for (int k = 0; k < 4; k++) d.mocap_quat()[4 * mid + k] = m.body_quat[4 * i + k];
    }
  }
  d.time()[0] = 0;
  d.ncon()[0] = 0; d.nefc()[0] = 0; d.ne()[0] = 0; d.nf()[0] = 0; d.nl()[0] = 0; for (int k = 0; k < NISLAND; k++) d.solver_niter()[k] = 0;
  if (clear_warnings) for (int i = 0; i < NWARNING; i++) d.warning()[i] = 0;
#if defined(MJB_HISTORY_CODE) && defined(__CUDA_ARCH__)
  if (d.feat & FEAT_HISTORY) reset_history(d);
#elif defined(MJB_HISTORY_CODE)
  if (d.m.sz.nhistory) reset_history(d);   // the host emulation is one build for every model (run_env)
#endif
}

// scan for NaN / overflow (serial, lane 0 only); on failure raise the warning and (unless
// disabled) reset the env.  result is published in scr_int[0] for the other lanes.
MJB_HD void check_vec(const Env& d, FD v, int n, int warn) {
  MJB_LANE0 {
    int bad = 0;
    for (int i = 0; i < n; i++) {
      if (is_bad(v[i])) {
        if (!(d.m.opt.disableflags & DSBL_AUTORESET)) reset_env(d, true);   // clears warnings, like mj_resetData
        d.warning()[warn] += 1;
        bad = 1;
        break;
      }
    }
    d.scr_int()[0] = bad;
  }
  MJB_PSYNC();
}

// transmissions with a dense moment row (mj_transmission, engine_core_smooth.c):
//   site without a reference site (:1573-1593): the 6D gear, expressed in the world through the site frame,
//       projected on the site's translational and rotational Jacobians; length 0;
//   site with a reference site (:1595-1700): gear in the reference site's frame, Jacobians relative to the
//       reference site, the dofs of the common ancestral chain cleared; length = offset and orientation
//       difference in the reference frame, dotted with the gear;
//   slider-crank (:1396-1465): length a'v - sqrt((a'v)^2 + r^2 - v'v) of the rod between crank and slider sites,
//       moment by the chain rule through the point and axis Jacobians.
MJB_HD void site_moment(const Env& d) {
  const DModel& m = d.m;
  if (!(d.feat & FEAT_ACT) || !m.sz.sitetrn) return;
  const int nv = m.sz.nv;
  FD row = d.actuator_momrow(), cdof = d.cdof(), len = d.actuator_length();
  auto jacr = [&](int body, int r, int j) { return m.body_dofanc[(long)body * nv + j] ? cdof[6 * j + r] : 0.0; };
  for (int u = 0; u < m.sz.nu; u++) {
    const int tt = m.actuator_trntype[u];
    if (tt < TRN_SITE) continue;
    const int sid = m.actuator_trnjnt[u], body = m.site_bodyid[sid];
    const double* gear = m.actuator_gear6 + 6 * u;
    const V3 sp = ld3(d.site_xpos(), 3 * sid);
    if (tt == TRN_SITE) {
      const M3 sm = ld9(d.site_xmat(), 9 * sid);
      const V3 wt = mulmv(sm, V3{gear[0], gear[1], gear[2]}), wr = mulmv(sm, V3{gear[3], gear[4], gear[5]});
      const double w[6] = {wt.x, wt.y, wt.z, wr.x, wr.y, wr.z};
      MJB_PFOR(j, nv) {
        double m1 = 0, m2 = 0;   // mju_mulMatTVec skips rows whose wrench component is zero
        for (int r = 0; r < 3; r++) if (w[r]) m1 += jac_elem(d, sp, body, r, j) * w[r];
        for (int r = 0; r < 3; r++) if (w[3 + r]) m2 += jacr(body, r, j) * w[3 + r];
        row[(long)u * nv + j] = m1 + m2;
      }
    } else if (tt == TRN_SITEREF) {
      const int rid = m.actuator_trnid2[u], rbody = m.site_bodyid[rid];
      const M3 rm = ld9(d.site_xmat(), 9 * rid);
      const V3 rp = ld3(d.site_xpos(), 3 * rid);
      const bool tr = gear[0] != 0 || gear[1] != 0 || gear[2] != 0, ro = gear[3] != 0 || gear[4] != 0 || gear[5] != 0;
      const V3 wt = mulmv(rm, V3{gear[0], gear[1], gear[2]}), wr = mulmv(rm, V3{gear[3], gear[4], gear[5]});
      const double w[6] = {wt.x, wt.y, wt.z, wr.x, wr.y, wr.z};
      MJB_LANE0 {
        double l = 0;
        if (tr) {
          const V3 v = mulmTv3(rm, sp - rp);
          l += v.x * gear[0] + v.y * gear[1] + v.z * gear[2];
        }
        if (ro) {   // site orientations from the parent bodies' quaternions, in the reference's (site, body) order
          const Q4 q = qmul(ldc4(m.site_quat, 4 * sid), ld4(d.xquat(), 4 * body));
          const Q4 rq = qmul(ldc4(m.site_quat, 4 * rid), ld4(d.xquat(), 4 * rbody));
          const V3 v = qsub(q, rq);
          l += v.x * gear[3] + v.y * gear[4] + v.z * gear[5];
        }
        len[u] = l;
      }
      const int* clr = m.actuator_refclear + (long)u * nv;
      MJB_PFOR(j, nv) {
        double mrow = 0;
        if (tr) {
          double m1 = 0;
          for (int r = 0; r < 3; r++) {
            const double jd = clr[j] ? 0.0 : jac_elem(d, sp, body, r, j) - jac_elem(d, rp, rbody, r, j);
            if (w[r]) m1 += jd * w[r];
          }
          mrow = m1;
        }
        if (ro) {
          double m2 = 0;
          for (int r = 0; r < 3; r++) {
            const double jd = clr[j] ? 0.0 : jacr(body, r, j) - jacr(rbody, r, j);
            if (w[3 + r]) m2 += jd * w[3 + r];
          }
          mrow += m2;
        }
        row[(long)u * nv + j] = mrow;
      }
    } else {   // slider-crank
      const int lid = m.actuator_trnid2[u], lbody = m.site_bodyid[lid];
      const double rod = m.actuator_cranklength[u], g = gear[0];
      const M3 lm = ld9(d.site_xmat(), 9 * lid);
      const V3 lp = ld3(d.site_xpos(), 3 * lid);
      const V3 axis{lm.m[2], lm.m[5], lm.m[8]};
      const V3 vec = sp - lp;
      const double av = dot(vec, axis);
      const double det = av * av + rod * rod - dot(vec, vec);
      double sdet = 0, l;
      const bool ok = det > 0;
      if (!ok) l = av; else { sdet = sqrt(det); l = av - sdet; }
      V3 dlda, dldv;
      if (ok) {
        dldv = axis * (1 - av / sdet);
        dlda = vec * (1 / sdet);
        dldv = dldv + dlda;
        dlda = vec * (1 - av / sdet);
      } else { dlda = vec; dldv = axis; }
      MJB_LANE0 len[u] = l * g;
      const double da[3] = {dlda.x, dlda.y, dlda.z}, dv[3] = {dldv.x, dldv.y, dldv.z};
      MJB_PFOR(j, nv) {
        // axis Jacobian = rotational Jacobian of the slider's body crossed with the axis; point Jacobian of the crank
        // site relative to the slider site
        const double r0 = jacr(lbody, 0, j), r1 = jacr(lbody, 1, j), r2 = jacr(lbody, 2, j);
        const double ja[3] = {r1 * axis.z - r2 * axis.y, r2 * axis.x - r0 * axis.z, r0 * axis.y - r1 * axis.x};
        double mr = 0;
        for (int k = 0; k < 3; k++) {
          const double jk = jac_elem(d, sp, body, k, j) - jac_elem(d, lp, lbody, k, j);
          mr += da[k] * ja[k] + dv[k] * jk;
        }
        row[(long)u * nv + j] = mr ? mr * g : 0.0;
      }
    }
  }
  MJB_PSYNC();
}

MJB_HD void fwd_position(const Env& d) {
  MJB_PROF_BEGIN
  kinematics(d);
  com_pos(d);
  tendon(d);
  MJB_PROF_MARK(0)
  make_M(d);
  {
    FD M = d.M(), qLD = d.qLD();
    MJB_PFOR(i, d.m.sz.nC) qLD[i] = M[i];
    MJB_PSYNC();
    factor_I(d, qLD, d.qLDiagInv());
  }
  MJB_PROF_MARK(1)
  collision(d);
  MJB_PROF_MARK(2)
  make_constraint(d);
  make_islands(d);
  MJB_PROF_MARK(3)
  project_constraint(d);
  MJB_PROF_MARK(4)
  transmission(d);
  site_moment(d);
  MJB_PROF_MARK(5)
}

MJB_HD void object_velocity(const Env& d, int kind, int id, V3& ang, V3& lin);   // defined with the sensors below
MJB_HD void history_advance(const Env& d);   // defined with the sensors below (FEAT_HISTORY)
MJB_HD V3 mulmTv(const M3& a, V3 v);

// fluid forces, inertia-box model (mj_fluid / mj_inertiaBoxFluidModel, engine_passive.c:868-903, :1154-1210):
// per body a viscous and a quadratic drag wrench from the body-local velocity relative to the wind, applied
// at the body's com through mj_applyFT; bodies in order, added to qfrc_passive before gravity compensation
MJB_HD void fluid(const Env& d) {
  const DModel& m = d.m;
  if (!(d.feat & FEAT_ACT) || !m.sz.fluid) return;
  const int nv = m.sz.nv, nbody = m.sz.nbody;
  FD ff = d.qfrc_fluid(), fp = d.qfrc_passive(), wr = d.scr_body(), cdof = d.cdof();   // wr: 6 per body (torque, force), world frame
  const bool off = (m.opt.disableflags & DSBL_SPRING) && (m.opt.disableflags & DSBL_DAMPER);
  if (off) { MJB_PFOR(j, nv) ff[j] = 0; MJB_PSYNC(); return; }
  const double visc = m.opt.viscosity, dens = m.opt.density;
  MJB_PFOR(i, nbody) {
    for (int k = 0; k < 6; k++) wr[6 * i + k] = 0;
    if (m.body_mass[i] < kMinVal) continue;
    const double* in = m.body_inertia + 3 * i;
    const double mass = m.body_mass[i];
    const double box[3] = {sqrt(dmax(kMinVal, (in[1] + in[2] - in[0])) / mass * 6.0), sqrt(dmax(kMinVal, (in[0] + in[2] - in[1])) / mass * 6.0),
                           sqrt(dmax(kMinVal, (in[0] + in[1] - in[2])) / mass * 6.0)};
    const M3 xi = ld9(d.ximat(), 9 * i);
    V3 ang, lin;
    object_velocity(d, SOBJ_BODY, i, ang, lin);
    ang = mulmTv(xi, ang); lin = mulmTv(xi, lin);          // flg_local = 1
    // wind in local coordinates (mju_transformSpatial of (0, wind): the translation leaves it unchanged)
    const V3 w0{m.opt.wind[0], m.opt.wind[1], m.opt.wind[2]};
    const V3 dif = ld3(d.xipos(), 3 * i) - ld3(d.subtree_com(), 3 * m.body_rootid[i]);
    const V3 lw = mulmTv(xi, w0 - cross(dif, V3{0, 0, 0}));
    lin = lin - lw;
    double lf[6] = {0, 0, 0, 0, 0, 0};
    const double lv[6] = {ang.x, ang.y, ang.z, lin.x, lin.y, lin.z};
    if (visc > 0) {
      const double diam = (box[0] + box[1] + box[2]) / 3.0;
      const double sa = -kPi * diam * diam * diam * visc, sl = -3.0 * kPi * diam * visc;
      for (int k = 0; k < 3; k++) { lf[k] = lv[k] * sa; lf[3 + k] = lv[3 + k] * sl; }
    }
    if (dens > 0) {
      lf[3] -= 0.5 * dens * box[1] * box[2] * fabs(lv[3]) * lv[3];
      lf[4] -= 0.5 * dens * box[0] * box[2] * fabs(lv[4]) * lv[4];
      lf[5] -= 0.5 * dens * box[0] * box[1] * fabs(lv[5]) * lv[5];
      lf[0] -= dens * box[0] * (box[1] * box[1] * box[1] * box[1] + box[2] * box[2] * box[2] * box[2]) * fabs(lv[0]) * lv[0] / 64.0;
      lf[1] -= dens * box[1] * (box[0] * box[0] * box[0] * box[0] + box[2] * box[2] * box[2] * box[2]) * fabs(lv[1]) * lv[1] / 64.0;
      lf[2] -= dens * box[2] * (box[0] * box[0] * box[0] * box[0] + box[1] * box[1] * box[1] * box[1]) * fabs(lv[2]) * lv[2] / 64.0;
    }
    const V3 bt = mulmv(xi, V3{lf[0], lf[1], lf[2]}), bf = mulmv(xi, V3{lf[3], lf[4], lf[5]});
    st3(wr, 6 * i, bt); st3(wr, 6 * i + 3, bf);
  }
  MJB_PSYNC();
  MJB_PFOR(j, nv) {
    double acc = 0;
    for (int i = 0; i < nbody; i++) {
      if (m.body_mass[i] < kMinVal) continue;
      const V3 pt = ld3(d.xipos(), 3 * i);
      const bool in = m.body_dofanc[(long)i * nv + j];
      double qf = 0, qt = 0;   // mj_applyFT: force part, then torque part; zero components are skipped
      for (int r = 0; r < 3; r++) { const double f = wr[6 * i + 3 + r]; if (f) qf += jac_elem(d, pt, i, r, j) * f; }
      acc += qf;
      for (int r = 0; r < 3; r++) { const double t = wr[6 * i + r]; if (t) qt += (in ? cdof[6 * j + r] : 0.0) * t; }
      acc += qt;
    }
    ff[j] = acc;
    fp[j] += acc;
  }
  MJB_PSYNC();
}

// gravity compensation (mj_gravcomp, engine_passive.c:846-866; mj_applyFT with a zero torque): per body an
// upward force -gravity*mass*gravcomp at the body's com, mapped through the point Jacobian; bodies in order
MJB_HD void gravcomp(const Env& d) {
  const DModel& m = d.m;
  if (!(d.feat & FEAT_ACT) || !m.sz.gravcomp) return;
  const int nv = m.sz.nv;
  FD gc = d.qfrc_gravcomp(), fp = d.qfrc_passive();
  const double* g = m.opt.gravity;
  const bool off = (m.opt.disableflags & DSBL_GRAVITY) || sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]) == 0 ||
                   ((m.opt.disableflags & DSBL_SPRING) && (m.opt.disableflags & DSBL_DAMPER));
  MJB_PFOR(j, nv) {
    double acc = 0;
    if (!off) {
      for (int i = 1; i < m.sz.nbody; i++) {
        if (!m.body_gravcomp[i]) continue;
        const double s = -(m.body_mass[i] * m.body_gravcomp[i]);
        const double f[3] = {g[0] * s, g[1] * s, g[2] * s};
        const V3 pt = ld3(d.xipos(), 3 * i);
        double q = 0;   // mju_mulMatTVec: rows with a zero force component are skipped
        for (int r = 0; r < 3; r++) if (f[r]) q += jac_elem(d, pt, i, r, j) * f[r];
        acc += q;
        acc += 0.0;     // the (zero) torque part of mj_applyFT
      }
    }
    gc[j] = acc;
    if (!off && !m.jnt_actgravcomp[m.dof_jntid[j]]) fp[j] += acc;
  }
  MJB_PSYNC();
}

#if defined(MJB_SPATIAL_UNIT) || !defined(__CUDA_ARCH__)
// d/dt(ten_J) . vec for a spatial tendon without geom wrapping (mj_tendonDot, engine_core_smooth.c:1115-1250, dense
// branch): per segment between different bodies, the Jacobian-derivative difference along the unit direction plus the
// Jacobian difference along the direction's rate of change, each dotted with vec and divided by the pulley divisor
MJB_HD double tendon_dot(const Env& d, int i, FD vec) {
  const DModel& m = d.m;
  const int nv = m.sz.nv, adr = m.tendon_adr[i], num = m.tendon_num[i];
  if (m.wrap_type[adr] == WRAP_JOINT) return 0;
  FD sx = d.site_xpos();
  double res = 0, divisor = 1;
  for (int j = 0; j < num - 1; j++) {
    const int t0 = m.wrap_type[adr + j], t1 = m.wrap_type[adr + j + 1];
    if (t0 == WRAP_PULLEY || t1 == WRAP_PULLEY) {
      if (t0 == WRAP_PULLEY) divisor = m.wrap_prm[adr + j];
      continue;
    }
    const int id0 = m.wrap_objid[adr + j], id1 = m.wrap_objid[adr + j + 1];
    const int b0 = m.site_bodyid[id0], b1 = m.site_bodyid[id1];
    if (b0 == b1) continue;
    const V3 p0 = ld3(sx, 3 * id0), p1 = ld3(sx, 3 * id1);
    V3 ang, v0, v1;
    object_velocity(d, SOBJ_SITE, id0, ang, v0);
    object_velocity(d, SOBJ_SITE, id1, ang, v1);
    V3 dp = p1 - p0;
    const double norm = normalize(dp);
    V3 dv = v1 - v0;
    dv = addscl(dv, dp, -dot(dp, dv));
    dv = dv * (norm > kMinVal ? 1 / norm : 0);
    // chain rule, first term: d/dt(jac2 - jac1) * dpnt; second term: (jac2 - jac1) * d/dt(dpnt) (mju_mulMatTVec)
    res += dot_ref(nv, [&](int c) {
      double t = 0;
      for (int r = 0; r < 3; r++) { const double s = get(dp, r); if (s) t += (jacdot_elem(d, p1, b1, r, c) - jacdot_elem(d, p0, b0, r, c)) * s; }
      return t;
    }, [&](int c) { return vec[c]; }) / divisor;
    res += dot_ref(nv, [&](int c) {
      double t = 0;
      for (int r = 0; r < 3; r++) { const double s = get(dv, r); if (s) t += (jac_elem(d, p1, b1, r, c) - jac_elem(d, p0, b0, r, c)) * s; }
      return t;
    }, [&](int c) { return vec[c]; }) / divisor;
  }
  return res;
}

// tendon-armature bias (mj_tendonBias, engine_core_smooth.c:2606-2640): qfrc_bias += ten_J * armature *
// (d/dt(ten_J) . qvel), armature = tendon armature + the armature of actuators on the tendon; tendons in order
MJB_HD void tendon_bias(const Env& d) {
  const DModel& m = d.m;
  MJB_LANE0 {
    FD qfrc = d.qfrc_bias(), tJ = d.ten_J();
    for (int i = 0; i < m.sz.ntendon; i++) {
      const double armature = m.tendon_armature_eff[i];
      if (!armature) continue;
      const double coef = armature * tendon_dot(d, i, d.qvel());
      if (coef) {
        const int adr = m.ten_J_rowadr[i], nnz = m.ten_J_rownnz[i];
        for (int j = 0; j < nnz; j++) qfrc[m.ten_J_colind[adr + j]] += coef * tJ[adr + j];
      }
    }
  }
  MJB_PSYNC();
}
#endif

MJB_HD void fwd_velocity(const Env& d) {
  const DModel& m = d.m;
#ifdef MJB_HISTORY_CODE
  if (d.feat & FEAT_HISTORY) MJB_LANE0 d.hist_flg()[1] = 0;   // mj_fwdVelocity clears flg_subtreevel (engine_forward.c:185)
#endif
  FD qvel = d.qvel();
  FD tv = d.ten_velocity(), tJ = d.ten_J();
  MJB_PFOR(i, m.sz.ntendon) {
    const int adr = m.ten_J_rowadr[i], nnz = m.ten_J_rownnz[i];
    tv[i] = dot_sparse_ref(nnz, [&](int c) { return tJ[adr + c]; }, [&](int c) { return qvel[m.ten_J_colind[adr + c]]; });
  }
  FD av = d.actuator_velocity(), mom = d.actuator_moment();
  const bool act = !(m.opt.disableflags & DSBL_ACTUATION);
  MJB_PFOR(i, m.sz.nu) {
    if (!act) av[i] = 0;
    else if ((d.feat & FEAT_ACT) && m.actuator_trntype[i] == TRN_TENDON) {
      const int t = m.actuator_trnjnt[i], adr = m.ten_J_rowadr[t], nnz = m.ten_J_rownnz[t];
      const double g = mom[i];
      av[i] = dot_sparse_ref(nnz, [&](int c) { return tJ[adr + c] * g; }, [&](int c) { return qvel[m.ten_J_colind[adr + c]]; });
    } else if ((d.feat & FEAT_ACT) && m.actuator_trntype[i] >= TRN_SITE) {   // sparse dot over the nonzero moments
      FD row = d.actuator_momrow() + (long)i * m.sz.nv;
      int idx[64], nnz = 0;
      for (int c = 0; c < m.sz.nv; c++) if (row[c]) idx[nnz++] = c;
      av[i] = dot_sparse_ref(nnz, [&](int c) { return row[idx[c]]; }, [&](int c) { return qvel[idx[c]]; });
    } else if ((d.feat & FEAT_ACT) && m.actuator_trntype[i] >= TRN_BALL) {
      const int da = m.jnt_dofadr[m.actuator_trnjnt[i]], nd = (m.actuator_trntype[i] == TRN_FREE) ? 6 : 3;
      FD m6 = d.actuator_mom6();
      av[i] = dot_sparse_ref(nd, [&](int c) { return m6[6 * i + c]; }, [&](int c) { return qvel[da + c]; });
    } else {
      const int dof = m.jnt_dofadr[m.actuator_trnjnt[i]];
      double r = 0;
      r += mom[i] * qvel[dof];
      av[i] = r;
    }
  }
  MJB_PSYNC();
  com_vel(d);
  passive(d);
  fluid(d);
  gravcomp(d);
  reference_constraint(d);
  rne_bias(d);
  // tendon-armature bias: d/dt(ten_J) is identically zero for fixed tendons, so only spatial tendons contribute
#if defined(MJB_SPATIAL_UNIT) || !defined(__CUDA_ARCH__)
  if (d.feat & FEAT_SPATIAL) tendon_bias(d);
#endif
}

// muscle model (engine_util_misc.c:1049-1190): FLV gain, passive bias, activation dynamics
MJB_HD double muscle_gain_length(double length, double lmin, double lmax) {
  if (lmin <= length && length <= lmax) {
    const double a = 0.5 * (lmin + 1), b = 0.5 * (1 + lmax);
    if (length <= a) { const double x = (length - lmin) / dmax(kMinVal, a - lmin); return 0.5 * x * x; }
    else if (length <= 1) { const double x = (1 - length) / dmax(kMinVal, 1 - a); return 1 - 0.5 * x * x; }
    else if (length <= b) { const double x = (length - 1) / dmax(kMinVal, b - 1); return 1 - 0.5 * x * x; }
    else { const double x = (lmax - length) / dmax(kMinVal, lmax - b); return 0.5 * x * x; }
  }
  return 0.0;
}
MJB_HD double muscle_gain(double len, double vel, const double* lengthrange, double acc0, const double* prm) {
  double force = prm[2];
  const double scale = prm[3], lmin = prm[4], lmax = prm[5], vmax = prm[6], fvmax = prm[8];
  if (force < 0) force = scale / dmax(kMinVal, acc0);
  const double L0 = (lengthrange[1] - lengthrange[0]) / dmax(kMinVal, prm[1] - prm[0]);
  const double L = prm[0] + (len - lengthrange[0]) / dmax(kMinVal, L0);
  const double V = vel / dmax(kMinVal, L0 * vmax);
  const double FL = muscle_gain_length(L, lmin, lmax);
  double FV;
  const double y = fvmax - 1;
  if (V <= -1) FV = 0;
  else if (V <= 0) FV = (V + 1) * (V + 1);
  else if (V <= y) FV = fvmax - (y - V) * (y - V) / dmax(kMinVal, y);
  else FV = fvmax;
  return -force * FL * FV;
}
MJB_HD double muscle_bias(double len, const double* lengthrange, double acc0, const double* prm) {
  double force = prm[2];
  const double scale = prm[3], lmax = prm[5], fpmax = prm[7];
  if (force < 0) force = scale / dmax(kMinVal, acc0);
  const double L0 = (lengthrange[1] - lengthrange[0]) / dmax(kMinVal, prm[1] - prm[0]);
  const double L = prm[0] + (len - lengthrange[0]) / dmax(kMinVal, L0);
  const double b = 0.5 * (1 + lmax);
  if (L <= 1) return 0;
  else if (L <= b) { const double x = (L - 1) / dmax(kMinVal, b - 1); return -force * fpmax * 0.5 * x * x; }
  else { const double x = (L - b) / dmax(kMinVal, b - 1); return -force * fpmax * (0.5 + x); }
}
MJB_HD double muscle_dynamics(double ctrl, double act, const double* prm) {
  const double ctrlclamp = dclip(ctrl, 0, 1), actclamp = dclip(act, 0, 1);
  const double tau_act = prm[0] * (0.5 + 1.5 * actclamp), tau_deact = prm[1] / (0.5 + 1.5 * actclamp);
  const double width = prm[2], dctrl = ctrlclamp - act;
  double tau;
  if (width < kMinVal) tau = dctrl > 0 ? tau_act : tau_deact;
  else {
    const double x = dctrl / width + 0.5;   // mju_sigmoid
    const double sg = (x <= 0) ? 0.0 : (x >= 1) ? 1.0 : x * x * x * (3 * x * (2 * x - 5) + 10);
    tau = tau_deact + (tau_act - tau_deact) * sg;
  }
  return dctrl / dmax(kMinVal, tau);
}

// mj_nextActivation (engine_support.c:706-775): activation after one timestep, clamped to actrange
MJB_HD double next_activation(const Env& d, int u, double act, double act_dot) {
  const DModel& m = d.m;
  if (m.actuator_dyntype[u] == DYN_FILTEREXACT) {
    const double tau = dmax(kMinVal, m.actuator_dynprm[kNDyn * u]);
    act = act + act_dot * tau * (1 - exp(-m.opt.timestep / tau));
  } else {
    act = act + act_dot * m.opt.timestep;
  }
  if (m.actuator_actlimited[u]) act = dclip(act, m.actuator_actrange[2 * u], m.actuator_actrange[2 * u + 1]);
  return act;
}

// advance activations (mj_advance, engine_forward.c:1316-1326) with the given act_dot
MJB_HD void advance_act(const Env& d, FD act_dot) {
  const DModel& m = d.m;
  if (!(d.feat & FEAT_ACT) || m.sz.na == 0 || (m.opt.disableflags & DSBL_ACTUATION)) return;
  FD act = d.act();
  MJB_PFOR(u, m.sz.nu) {
    const int a = m.actuator_actadr[u];
    if (a >= 0) act[a] = next_activation(d, u, act[a], act_dot[a]);
    if (a >= 0 && m.actuator_dyntype[u] == DYN_INTEGRATOR && m.actuator_wrapperiod[u] > 0) {   // engine_forward.c:1328-1340
      const double period = m.actuator_wrapperiod[u], err = act[a] - d.actuator_length()[u];
      act[a] = act[a] - period * round_int(err / period);
    }
  }
  MJB_PSYNC();
}

MJB_HD void fwd_actuation(const Env& d) {
  const DModel& m = d.m;
  const int nu = m.sz.nu, nv = m.sz.nv;
  FD force = d.actuator_force(), qfa = d.qfrc_actuator(), ctrl_in = d.ctrl();
  if (nu == 0 || (m.opt.disableflags & DSBL_ACTUATION)) {
    MJB_PFOR(i, nu) force[i] = 0;
    MJB_PFOR(i, nv) qfa[i] = 0;
    MJB_PSYNC();
    return;
  }
  FD ctrl = d.scr_nv() + 4 * nv;   // local, clamped copy (host guarantees nu <= 4*nv)
  const bool clamp = !(m.opt.disableflags & DSBL_CLAMPCTRL);
  MJB_PFOR(i, nu) {
    double c = ctrl_in[i];
#ifdef MJB_HISTORY_CODE
    if ((d.feat & FEAT_HISTORY) && m.actuator_delay[i] != 0 && m.actuator_history[2 * i] > 0) c = read_ctrl(d, i);
#endif
    if (clamp && m.actuator_ctrllimited[i]) c = dclip(c, m.actuator_ctrlrange[2 * i], m.actuator_ctrlrange[2 * i + 1]);
    ctrl[i] = c;
  }
  MJB_PSYNC();
  MJB_LANE0 {
    for (int i = 0; i < nu; i++) {
      if (is_bad(ctrl[i])) {
        d.warning()[WARN_BADCTRL] += 1;
        for (int k = 0; k < nu; k++) ctrl[k] = 0;
        break;
      }
    }
  }
  MJB_PSYNC();
  FD len = d.actuator_length(), vel = d.actuator_velocity(), mom = d.actuator_moment();
  const bool stateful = (d.feat & FEAT_ACT) != 0;
  if (stateful && m.sz.na) {   // act_dot of the stateful actuators
    FD act = d.act(), act_dot = d.act_dot();
    MJB_PFOR(i, nu) {
      const int a = m.actuator_actadr[i];
      if (a < 0) continue;
      const double* dp = m.actuator_dynprm + kNDyn * i;
      const int dt = m.actuator_dyntype[i];
      if (dt == DYN_INTEGRATOR) act_dot[a] = ctrl[i];
      else if (dt == DYN_MUSCLE) act_dot[a] = muscle_dynamics(ctrl[i], act[a], dp);
      else act_dot[a] = (ctrl[i] - act[a]) / dmax(kMinVal, dp[0]);
    }
    MJB_PSYNC();
  }
  MJB_PFOR(i, nu) {
    const double* gp = m.actuator_gainprm + kNGain * i;
    const double* bp = m.actuator_biasprm + kNGain * i;
    const int gt = m.actuator_gaintype[i], bt = m.actuator_biastype[i];
    double gain;
    if (gt == GAIN_FIXED) gain = gp[0];
    else if (stateful && gt == GAIN_MUSCLE) gain = muscle_gain(len[i], vel[i], m.actuator_lengthrange + 2 * i, m.actuator_acc0[i], gp);
    else gain = gp[0] + gp[1] * len[i] + gp[2] * vel[i];
    double in = ctrl[i];
    if (stateful && m.actuator_actadr[i] >= 0) {
      const int a = m.actuator_actadr[i];
      in = m.actuator_actearly[i] ? next_activation(d, i, d.act()[a], d.act_dot()[a]) : d.act()[a];
    }
    if (stateful && m.actuator_wrapperiod[i] > 0) {   // rotational setpoint: representative nearest the length (wrapSetpoint)
      const double period = m.actuator_wrapperiod[i], err = in - len[i];
      in = in - period * round_int(err / period);
    }
    double f = gain * in;
    double bias;
    if (bt == BIAS_NONE) bias = 0.0;
    else if (stateful && bt == BIAS_MUSCLE) bias = muscle_bias(len[i], m.actuator_lengthrange + 2 * i, m.actuator_acc0[i], bp);
    else bias = bp[0] + bp[1] * len[i] + bp[2] * vel[i];
    f += bias;
    force[i] = f;
  }
  if (stateful && m.sz.ntendon) {   // tendons with a limit on their total actuator force (engine_forward.c:955-985)
    MJB_PSYNC();
    MJB_LANE0 {
      for (int t = 0; t < m.sz.ntendon; t++) {
        if (!m.tendon_actfrclimited[t]) continue;
        double total = 0;
        for (int i = 0; i < nu; i++) if (m.actuator_trntype[i] == TRN_TENDON && m.actuator_trnjnt[i] == t) total += force[i];
        if (!total) continue;
        const double lo = m.tendon_actfrcrange[2 * t], hi = m.tendon_actfrcrange[2 * t + 1];
        for (int i = 0; i < nu; i++) {
          if (m.actuator_trntype[i] != TRN_TENDON || m.actuator_trnjnt[i] != t) continue;
          if (total < lo) force[i] *= lo / total;
          else if (total > hi) force[i] *= hi / total;
        }
      }
    }
    MJB_PSYNC();
  }
  MJB_PFOR(i, nu) {
    if (m.actuator_forcelimited[i]) force[i] = dclip(force[i], m.actuator_forcerange[2 * i], m.actuator_forcerange[2 * i + 1]);
  }
  MJB_PFOR(i, nv) qfa[i] = 0;
  MJB_PSYNC();
  MJB_LANE0 {   // several actuators may drive one dof: keep the serial accumulation order
    for (int i = 0; i < nu; i++) {
      const double s = force[i];
      if (s == 0) continue;
      if (stateful && m.actuator_trntype[i] == TRN_TENDON) {
        const int t = m.actuator_trnjnt[i], adr = m.ten_J_rowadr[t], nnz = m.ten_J_rownnz[t];
        FD tJ = d.ten_J();
        for (int c = 0; c < nnz; c++) qfa[m.ten_J_colind[adr + c]] += (tJ[adr + c] * mom[i]) * s;
        continue;
      }
      if (stateful && m.actuator_trntype[i] >= TRN_SITE) {
        FD row = d.actuator_momrow() + (long)i * nv;
        for (int c = 0; c < nv; c++) if (row[c]) qfa[c] += row[c] * s;
        continue;
      }
      if (stateful && m.actuator_trntype[i] >= TRN_BALL) {
        const int da = m.jnt_dofadr[m.actuator_trnjnt[i]], nd = (m.actuator_trntype[i] == TRN_FREE) ? 6 : 3;
        FD m6 = d.actuator_mom6();
        for (int c = 0; c < nd; c++) qfa[da + c] += m6[6 * i + c] * s;
        continue;
      }
      qfa[m.jnt_dofadr[m.actuator_trnjnt[i]]] += mom[i] * s;
    }
    if (stateful && m.sz.gravcomp && !(m.opt.disableflags & DSBL_GRAVITY)) {   // actuator-level gravity compensation
      FD gcf = d.qfrc_gravcomp();
      for (int j = 0; j < m.sz.njnt; j++) {
        if (!m.jnt_actgravcomp[j]) continue;
        const int da = m.jnt_dofadr[j], nd = (m.jnt_type[j] == JNT_FREE) ? 6 : (m.jnt_type[j] == JNT_BALL) ? 3 : 1;
        for (int k = 0; k < nd; k++) qfa[da + k] += gcf[da + k];
      }
    }
    for (int j = 0; j < m.sz.njnt; j++) {
      if (!m.jnt_actfrclimited[j]) continue;
      const int da = m.jnt_dofadr[j];
      qfa[da] = dclip(qfa[da], m.jnt_actfrcrange[2 * j], m.jnt_actfrcrange[2 * j + 1]);
    }
  }
  MJB_PSYNC();
}

MJB_HD void fwd_acceleration(const Env& d) {
  const int nv = d.m.sz.nv;
  FD qfs = d.qfrc_smooth(), qas = d.qacc_smooth();
  FD fp = d.qfrc_passive(), fb = d.qfrc_bias(), fa = d.qfrc_applied(), fact = d.qfrc_actuator();
  MJB_PFOR(i, nv) {
    double s = fp[i] - fb[i];
    s += fa[i];
    s += fact[i];
    qfs[i] = s;
    qas[i] = s;
  }
  if (d.feat & FEAT_ACT) {   // Cartesian perturbations (mj_xfrcAccumulate, engine_support.c:497-512): mj_applyFT per body
    FD xf = d.xfrc_applied(), cdof = d.cdof();
    MJB_PFOR(j, nv) {
      double acc = qfs[j];
      bool any = false;
      for (int i = 1; i < d.m.sz.nbody; i++) {
        const double* w = &xf[6 * i];
        if (w[0] == 0 && w[1] == 0 && w[2] == 0 && w[3] == 0 && w[4] == 0 && w[5] == 0) continue;
        any = true;
        const V3 pt = ld3(d.xipos(), 3 * i);
        const bool in = d.m.body_dofanc[(long)i * nv + j];
        double qf = 0, qt = 0;
        for (int r = 0; r < 3; r++) if (w[r]) qf += jac_elem(d, pt, i, r, j) * w[r];
        acc += qf;
        for (int r = 0; r < 3; r++) if (w[3 + r]) qt += (in ? cdof[6 * j + r] : 0.0) * w[3 + r];
        acc += qt;
      }
      if (any) { qfs[j] = acc; qas[j] = acc; }
    }
  }
  MJB_PSYNC();
  solve_LD(d, qas, d.qLD(), d.qLDiagInv());
}

// position integration on the configuration manifold (one lane per joint)
MJB_HD void integrate_pos(const Env& d, FD qpos, FD qvel, double dt) {
  const DModel& m = d.m;
  MJB_PFOR(j, m.sz.njnt) {
    int pa = m.jnt_qposadr[j], va = m.jnt_dofadr[j];
    const int jt = m.jnt_type[j];
    if (jt == JNT_FREE || jt == JNT_BALL) {
      if (jt == JNT_FREE) {
        for (int i = 0; i < 3; i++) qpos[pa + i] += dt * qvel[va + i];
        pa += 3; va += 3;
      }
      Q4 q = qintegrate(ld4(qpos, pa), ld3(qvel, va), dt);
      st4(qpos, pa, q);
    } else {
      qpos[pa] += dt * qvel[va];
    }
  }
  MJB_PSYNC();
}

// semi-implicit Euler with implicit joint damping, then advance state and time
MJB_HD void euler_advance(const Env& d) {
  const DModel& m = d.m;
  const int nv = m.sz.nv;
  const double h = m.opt.timestep;
  FD qacc = d.qacc(), qvel = d.qvel();
  FD acc = d.scr_nv();   // acceleration used for the velocity update
#ifdef MJB_HISTORY_CODE
  if (d.feat & FEAT_HISTORY) history_advance(d);
#endif
  if (!m.opt.eulerdamp) {
    MJB_PFOR(i, nv) acc[i] = qacc[i];
    MJB_PSYNC();
  } else {
    FD qH = d.qH(), M = d.M();
    MJB_PFOR(i, m.sz.nC) qH[i] = M[i];
    MJB_PSYNC();
    MJB_PFOR(i, nv) {
      const double dd = d_xpoly_force(m.dof_damping_eff[i], m.dof_dampingpoly_eff + kNPoly * i, kNPoly, qvel[i], true);
      qH[m.M_rowadr[i] + m.M_rownnz[i] - 1] += h * dd;
    }
    MJB_PSYNC();
    factor_I(d, qH, d.qHDiagInv());
    FD qfs = d.qfrc_smooth(), qfc = d.qfrc_constraint();
    MJB_PFOR(i, nv) acc[i] = qfs[i] + qfc[i];
    MJB_PSYNC();
    solve_LD(d, acc, qH, d.qHDiagInv());
  }
  advance_act(d, d.act_dot());
  MJB_PFOR(i, nv) qvel[i] += acc[i] * h;
  MJB_PSYNC();
  integrate_pos(d, d.qpos(), d.qvel(), h);
  FD ws = d.qacc_warmstart();
  MJB_PFOR(i, nv) ws[i] = qacc[i];
  MJB_LANE0 d.time()[0] += h;
  MJB_PSYNC();
}

// standalone free bodies under implicitfast (engine_forward.c:1742-1762): the symmetric solve drops the derivative of
// the bias (gyroscopic) force; a body that is a whole tree by itself - one free joint, no children - gets its six
// accelerations from a local unsymmetric solve instead, A = M - h dqfrc_smooth/dqvel with the bias block of
// mjd_freeBias_vel (engine_derivative.c:706-905), by the partially pivoted 6x6 LU of engine_util_solve.c:855-925.
// qHblk: the body's 6x6 lower triangle of qH = M - h qDeriv (its qDeriv block is diagonal here: the model check
// refuses actuators on such a body).  rhs -> x.
MJB_HD void free_body_implicit(const Env& d, int body, int adr, const double* qHlow, const double* rhs, double* x) {
  const DModel& m = d.m;
  const double h = m.opt.timestep, mass = m.body_mass[body];
  double R[9], Xi[9], s[3], w[3];
  FD xmat = d.xmat(), ximat = d.ximat(), xipos = d.xipos(), xpos = d.xpos(), qvel = d.qvel();
  for (int i = 0; i < 9; i++) { R[i] = xmat[9 * body + i]; Xi[i] = ximat[9 * body + i]; }
  for (int i = 0; i < 3; i++) s[i] = xipos[3 * body + i] - xpos[3 * body + i];
  const double v0 = qvel[adr + 3], v1 = qvel[adr + 4], v2 = qvel[adr + 5];
  for (int i = 0; i < 3; i++) w[i] = R[3 * i] * v0 + R[3 * i + 1] * v1 + R[3 * i + 2] * v2;
  const double* inertia = m.body_inertia + 3 * body;
  double XI[9], Iw[9];
  for (int i = 0; i < 3; i++) for (int c = 0; c < 3; c++) XI[3 * i + c] = Xi[3 * i + c] * inertia[c];
  Iw[0] = XI[0] * Xi[0] + XI[1] * Xi[1] + XI[2] * Xi[2];
  Iw[4] = XI[3] * Xi[3] + XI[4] * Xi[4] + XI[5] * Xi[5];
  Iw[8] = XI[6] * Xi[6] + XI[7] * Xi[7] + XI[8] * Xi[8];
  Iw[1] = Iw[3] = XI[0] * Xi[3] + XI[1] * Xi[4] + XI[2] * Xi[5];
  Iw[2] = Iw[6] = XI[0] * Xi[6] + XI[1] * Xi[7] + XI[2] * Xi[8];
  Iw[5] = Iw[7] = XI[3] * Xi[6] + XI[4] * Xi[7] + XI[5] * Xi[8];
  const double ws[3] = {w[1] * s[2] - w[2] * s[1], w[2] * s[0] - w[0] * s[2], w[0] * s[1] - w[1] * s[0]};
  double Iww[3];
  for (int i = 0; i < 3; i++) Iww[i] = Iw[3 * i] * w[0] + Iw[3 * i + 1] * w[1] + Iw[3 * i + 2] * w[2];
  const double wds = w[0] * s[0] + w[1] * s[1] + w[2] * s[2];
  double K[9];
  K[0] = s[0] * w[0] - wds;   K[1] = s[0] * w[1] - ws[2];  K[2] = s[0] * w[2] + ws[1];
  K[3] = s[1] * w[0] + ws[2]; K[4] = s[1] * w[1] - wds;    K[5] = s[1] * w[2] - ws[0];
  K[6] = s[2] * w[0] - ws[1]; K[7] = s[2] * w[1] + ws[0];  K[8] = s[2] * w[2] - wds;
  double lin[9], C[9], tmp[9], rot[9];
  for (int i = 0; i < 3; i++) for (int c = 0; c < 3; c++) lin[3 * i + c] = K[3 * i] * R[c] + K[3 * i + 1] * R[3 + c] + K[3 * i + 2] * R[6 + c];
  for (int c = 0; c < 3; c++) {
    const double sk0 = s[1] * K[6 + c] - s[2] * K[3 + c], sk1 = s[2] * K[c] - s[0] * K[6 + c], sk2 = s[0] * K[3 + c] - s[1] * K[c];
    const double wi0 = w[1] * Iw[6 + c] - w[2] * Iw[3 + c], wi1 = w[2] * Iw[c] - w[0] * Iw[6 + c], wi2 = w[0] * Iw[3 + c] - w[1] * Iw[c];
    C[c] = -mass * sk0 + wi0 + (c == 1 ? Iww[2] : (c == 2 ? -Iww[1] : 0));
    C[3 + c] = -mass * sk1 + wi1 + (c == 0 ? -Iww[2] : (c == 2 ? Iww[0] : 0));
    C[6 + c] = -mass * sk2 + wi2 + (c == 0 ? Iww[1] : (c == 1 ? -Iww[0] : 0));
  }
  for (int i = 0; i < 3; i++) for (int c = 0; c < 3; c++) tmp[3 * i + c] = R[i] * C[c] + R[3 + i] * C[3 + c] + R[6 + i] * C[6 + c];        // R' C
  for (int i = 0; i < 3; i++) for (int c = 0; c < 3; c++) rot[3 * i + c] = tmp[3 * i] * R[c] + tmp[3 * i + 1] * R[3 + c] + tmp[3 * i + 2] * R[6 + c];
  double A[36];
  for (int i = 0; i < 36; i++) A[i] = 0;
  for (int r = 0; r < 6; r++) {
    const int ra = m.M_rowadr[adr + r], rn = m.M_rownnz[adr + r];
    for (int k = 0; k < rn; k++) { const int c = m.M_colind[ra + k] - adr; A[6 * r + c] = qHlow[ra + k]; A[6 * c + r] = qHlow[ra + k]; }
  }
  const double hm = -h * mass;
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { A[6 * r + 3 + c] += hm * lin[3 * r + c]; A[6 * (3 + r) + 3 + c] += h * rot[3 * r + c]; }
  int pivot[6];
  for (int k = 0; k < 6; k++) {
    pivot[k] = k;
    double maxval = fabs(A[6 * k + k]);
    int maxrow = k;
    for (int i = k + 1; i < 6; i++) { const double val = fabs(A[6 * i + k]); if (val > maxval) { maxval = val; maxrow = i; } }
    if (maxval < kMinVal) return;     // singular: the symmetric solution stays
    if (maxrow != k) {
      pivot[k] = maxrow;
      for (int j = 0; j < 6; j++) { const double t = A[6 * k + j]; A[6 * k + j] = A[6 * maxrow + j]; A[6 * maxrow + j] = t; }
    }
    const double dinv = 1.0 / A[6 * k + k];
    for (int i = k + 1; i < 6; i++) {
      A[6 * i + k] *= dinv;
      const double aik = A[6 * i + k];
      for (int j = k + 1; j < 6; j++) A[6 * i + j] -= aik * A[6 * k + j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) y[i] = rhs[i];
  for (int i = 0; i < 6; i++) {
    if (pivot[i] != i) { const double t = y[i]; y[i] = y[pivot[i]]; y[pivot[i]] = t; }
    for (int j = 0; j < i; j++) y[i] -= A[6 * i + j] * y[j];
  }
  for (int i = 5; i >= 0; i--) {
    for (int j = i + 1; j < 6; j++) y[i] -= A[6 * i + j] * y[j];
    y[i] /= A[6 * i + i];
  }
  for (int i = 0; i < 6; i++) x[i] = y[i];
}

// implicitfast integrator (mj_implicitSkip, engine_forward.c:1649-1771; standalone free bodies: free_body_implicit):
// qH = M - h * d(qfrc_actuator + qfrc_passive)/d(qvel) on M's sparsity (mjd_smooth_vel with flg_bias = 0,
// engine_derivative.c:3145-3170: actuator velocity gains mjd_actuator_vel :2350-2500, then dof and tendon
// damping mjd_passive_vel :3040-3140; entries outside the tree sparsity are dropped as in the reference),
// L'DL, qacc_int = qH^-1 (qfrc_smooth + qfrc_constraint), mj_advance
MJB_HD void implicitfast_advance(const Env& d) {
  const DModel& m = d.m;
  const int nv = m.sz.nv, nu = m.sz.nu, ntendon = m.sz.ntendon;
  const double h = m.opt.timestep;
  FD qacc = d.qacc(), qvel = d.qvel(), qH = d.qH(), M = d.M();
  FD acc = d.scr_nv();
  FD tB = d.scr_nv() + nv;          // per tendon: B = -d(damping force)/d(velocity)
  FD aB = d.scr_nv() + 2 * nv;      // per actuator: d(force)/d(velocity) (0 when clamped)   [nu <= 4 nv]
  const bool act_on = !(m.opt.disableflags & DSBL_ACTUATION);
  const bool spring_off = (m.opt.disableflags & DSBL_SPRING) != 0, damper_off = (m.opt.disableflags & DSBL_DAMPER) != 0;
  const bool passive_on = !(spring_off && damper_off) && !damper_off;
  FD tv = d.ten_velocity(), tJ = d.ten_J(), mom = d.actuator_moment(), force = d.actuator_force(), ctrl = d.ctrl();
#ifdef MJB_HISTORY_CODE
  if (d.feat & FEAT_HISTORY) history_advance(d);
#endif
  MJB_PFOR(t, ntendon) {
    tB[t] = passive_on ? -d_xpoly_force(m.tendon_damping_eff[t], m.tendon_dampingpoly_eff + kNPoly * t, kNPoly, tv[t], true) : 0.0;
  }
  MJB_PFOR(u, nu) {
    double bv = 0;
    bool live = act_on;
    if (live && m.actuator_forcelimited[u]) {
      const double f = force[u];
      if (f <= m.actuator_forcerange[2 * u] || f >= m.actuator_forcerange[2 * u + 1]) live = false;
    }
    if (live) {
      if (m.actuator_biastype[u] == BIAS_AFFINE) bv = m.actuator_biasprm[kNGain * u + 2];
      const double gv = (m.actuator_gaintype[u] == GAIN_AFFINE) ? m.actuator_gainprm[kNGain * u + 2] : 0.0;
      if (gv != 0) {
        const int a = (d.feat & FEAT_ACT) ? m.actuator_actadr[u] : -1;
        if (a < 0) bv += gv * ctrl[u];
        else bv += gv * (m.actuator_actearly[u] ? next_activation(d, u, d.act()[a], d.act_dot()[a]) : d.act()[a]);
      }
    }
    aB[u] = bv;
  }
  MJB_PSYNC();
  MJB_PFOR(i, nv) {
    const int adr = m.M_rowadr[i], nnz = m.M_rownnz[i];
    for (int a = 0; a < nnz; a++) {
      const int j = m.M_colind[adr + a];
      double q = 0;
      for (int u = 0; u < nu; u++) {   // actuators in index order (mjd_actuator_vel): J'BJ of each moment row
        if (aB[u] == 0) continue;
        if ((d.feat & FEAT_ACT) && m.actuator_trntype[u] == TRN_TENDON) {   // moment row = ten_J row * gear
          const int t = m.actuator_trnjnt[u], ta = m.ten_J_rowadr[t], tn = m.ten_J_rownnz[t];
          double Ji = 0, Jj = 0;
          bool hi = false, hj = false;
          for (int c = 0; c < tn; c++) {
            const int col = m.ten_J_colind[ta + c];
            if (col == i) { Ji = tJ[ta + c] * mom[u]; hi = true; }
            if (col == j) { Jj = tJ[ta + c] * mom[u]; hj = true; }
          }
          if (hi && hj) q += Jj * (Ji * aB[u]);
        } else if ((d.feat & FEAT_ACT) && m.actuator_trntype[u] >= TRN_SITE) {
          FD row = d.actuator_momrow() + (long)u * nv;
          if (row[i] && row[j]) q += row[j] * (row[i] * aB[u]);
        } else if ((d.feat & FEAT_ACT) && m.actuator_trntype[u] >= TRN_BALL) {   // moment row on the joint's 3 / 6 dofs
          const int da = m.jnt_dofadr[m.actuator_trnjnt[u]], nd = (m.actuator_trntype[u] == TRN_FREE) ? 6 : 3;
          if (i >= da && i < da + nd && j >= da && j < da + nd) {
            FD m6 = d.actuator_mom6();
            q += m6[6 * u + (j - da)] * (m6[6 * u + (i - da)] * aB[u]);
          }
        } else if (i == j && m.jnt_dofadr[m.actuator_trnjnt[u]] == i) {
          q += mom[u] * (mom[u] * aB[u]);
        }
      }
      if (i == j) {
        if (passive_on) q -= d_xpoly_force(m.dof_damping_eff[i], m.dof_dampingpoly_eff + kNPoly * i, kNPoly, qvel[i], true);
      }
      for (int t = 0; t < ntendon; t++) {
        const double B = tB[t];
        if (B == 0) continue;
        const int ta = m.ten_J_rowadr[t], tn = m.ten_J_rownnz[t];
        double Ji = 0, Jj = 0;
        bool hi = false, hj = false;
        for (int c = 0; c < tn; c++) {
          const int col = m.ten_J_colind[ta + c];
          if (col == i) { Ji = tJ[ta + c]; hi = true; }
          if (col == j) { Jj = tJ[ta + c]; hj = true; }
        }
        if (hi && hj) q += Jj * (Ji * B);
      }
      qH[adr + a] = M[adr + a] + q * (-h);
    }
  }
  MJB_PSYNC();
  factor_I(d, qH, d.qHDiagInv());
  FD qfs = d.qfrc_smooth(), qfc = d.qfrc_constraint();
  MJB_PFOR(i, nv) acc[i] = qfs[i] + qfc[i];
  MJB_PSYNC();
  solve_LD(d, acc, qH, d.qHDiagInv());
  if (m.sz.freebody) {   // one lane per standalone free body: its six rows are decoupled from every other dof
    MJB_PFOR(j, m.sz.njnt) {
      const int body = m.jnt_bodyid[j];
      if (m.jnt_type[j] != JNT_FREE || m.body_jntnum[body] != 1 || m.body_subtreemass[body] != m.body_mass[body]) continue;
      const int adr = m.jnt_dofadr[j];
      double rhs[6], x[6];
      for (int i = 0; i < 6; i++) { rhs[i] = qfs[adr + i] + qfc[adr + i]; x[i] = acc[adr + i]; }
      free_body_implicit(d, body, adr, qH.p, rhs, x);
      for (int i = 0; i < 6; i++) acc[adr + i] = x[i];
    }
    MJB_PSYNC();
  }
  advance_act(d, d.act_dot());
  MJB_PFOR(i, nv) qvel[i] += acc[i] * h;
  MJB_PSYNC();
  integrate_pos(d, d.qpos(), d.qvel(), h);
  FD ws = d.qacc_warmstart();
  MJB_PFOR(i, nv) ws[i] = qacc[i];
  MJB_LANE0 d.time()[0] += h;
  MJB_PSYNC();
}

// ---- stages ---------------------------------------------------------------------------------------
// Every stage is entered by ALL lanes that share the environment.
MJB_HD void stage_position(const Env& d, bool is_step) {
  if (is_step) {
    check_vec(d, d.qpos(), d.m.sz.nq, WARN_BADQPOS);
    check_vec(d, d.qvel(), d.m.sz.nv, WARN_BADQVEL);
  }
  fwd_position(d);
}
MJB_HD void stage_velocity(const Env& d) {
  MJB_PROF_BEGIN
  fwd_velocity(d);
  MJB_PROF_MARK(6)
  fwd_actuation(d);
  fwd_acceleration(d);
  MJB_PROF_MARK(7)
  constraint_begin(d);
  MJB_PROF_MARK(8)
}
MJB_HD void stage_solve(const Env& d) {
  if (d.solver == SOL_PGS) solve_pgs(d);
  else solve_primal(d, d.solver == SOL_NEWTON);
  if (d.m.opt.noslip_iterations > 0) solve_noslip(d);   // engine_forward.c:1216-1243
}
MJB_HD void stage_finish_forward(const Env& d) {
  MJB_PROF_BEGIN
  if (d.solver == SOL_PGS || d.m.opt.noslip_iterations > 0) dual_finish(d);   // engine_forward.c:1247
  MJB_PROF_MARK(9)
}
// ---- sensors (engine_sensor.c: mj_computeSensorPos :525-836, Vel :839-955, Acc :958-1385, apply_cutoff
// :198-223, frame helpers :227-277; mj_objectVelocity engine_core_util.c:835-886, mju_transformSpatial
// engine_util_spatial.c).  All supported sensors read quantities that stay valid until the end of the
// forward pass, so the three stage-wise sweeps of the reference collapse into one, run after the solve.
MJB_HD void sensor_frame(const Env& d, int kind, int id, V3& pos, M3& mat) {
  if (kind == SOBJ_XBODY) { pos = ld3(d.xpos(), 3 * id); mat = ld9(d.xmat(), 9 * id); }
  else if (kind == SOBJ_BODY) { pos = ld3(d.xipos(), 3 * id); mat = ld9(d.ximat(), 9 * id); }
  else if (kind == SOBJ_GEOM) { pos = ld3(d.geom_xpos(), 3 * id); mat = ld9(d.geom_xmat(), 9 * id); }
  else { pos = ld3(d.site_xpos(), 3 * id); mat = ld9(d.site_xmat(), 9 * id); }
}
MJB_HD Q4 sensor_quat(const Env& d, int kind, int id) {
  const DModel& m = d.m;
  if (kind == SOBJ_XBODY) return ld4(d.xquat(), 4 * id);
  if (kind == SOBJ_BODY) return qmul(ld4(d.xquat(), 4 * id), ldc4(m.body_iquat, 4 * id));
  if (kind == SOBJ_GEOM) return qmul(ld4(d.xquat(), 4 * m.geom_bodyid[id]), ldc4(m.geom_quat, 4 * id));
  return qmul(ld4(d.xquat(), 4 * m.site_bodyid[id]), ldc4(m.site_quat, 4 * id));
}
MJB_HD V3 mulmTv(const M3& a, V3 v) {   // mju_mulMatTVec3
  return V3{a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z,
            a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z};
}
// 6D velocity of an object frame in the global frame (angular, linear)
MJB_HD void object_velocity(const Env& d, int kind, int id, V3& ang, V3& lin) {
  const DModel& m = d.m;
  const int body = (kind == SOBJ_GEOM) ? m.geom_bodyid[id] : (kind == SOBJ_SITE) ? m.site_bodyid[id] : id;
  if (m.body_dofnum[m.body_weldid[body]] == 0) { ang = V3{0, 0, 0}; lin = V3{0, 0, 0}; return; }
  V3 pos; M3 mat;
  sensor_frame(d, kind, id, pos, mat);
  FD cvel = d.cvel();
  ang = ld3(cvel, 6 * body);
  const V3 vl = ld3(cvel, 6 * body + 3);
  const V3 dif = pos - ld3(d.subtree_com(), 3 * m.body_rootid[body]);
  lin = vl - cross(dif, ang);
}

// mj_rnePostConstraint (engine_core_smooth.c:2394-2600): external contact forces per body (cfrc_ext), body
// accelerations (cacc) and interaction forces with the parent (cfrc_int), all in the com-based frame.
// Only run when a sensor needs it.  xfrc_applied and connect / weld rows are not part of the supported set.
MJB_HD S6 transform_force(S6 v, V3 newpos, V3 oldpos) {   // mju_transformSpatial, flg_force = 1, no rotation
  const V3 dif = newpos - oldpos;
  const V3 tq{v.v[0], v.v[1], v.v[2]}, f{v.v[3], v.v[4], v.v[5]};
  const V3 t = tq - cross(dif, f);
  return S6{{t.x, t.y, t.z, f.x, f.y, f.z}};
}
MJB_HD void rne_post(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody, ncon = d.ncon()[0];
  FD cacc = d.cacc(), cint = d.cfrc_int(), cext = d.cfrc_ext();
  FD cinert = d.cinert(), cvel = d.cvel(), cdof = d.cdof(), cdd = d.cdof_dot(), qvel = d.qvel(), qacc = d.qacc();
  FD force = d.efc_force(), cfri = d.con_friction(), cframe = d.con_frame(), cpos = d.con_pos(), sc = d.subtree_com();
  FI cadr = d.con_efcadr(), cdim = d.con_dim(), cg1 = d.con_geom1(), cg2 = d.con_geom2();
  // cfrc_ext: one lane per body, contacts in order, body 1 (subtract) before body 2 (add)
  MJB_PFOR(k, nbody) {
    S6 acc{{0, 0, 0, 0, 0, 0}};
    if (k && (d.feat & FEAT_ACT)) {   // cfrc_ext = perturbation wrench (engine_core_smooth.c:2406-2420), moved to the subtree com
      const double* w = &d.xfrc_applied()[6 * k];
      if (!(w[0] == 0 && w[1] == 0 && w[2] == 0 && w[3] == 0 && w[4] == 0 && w[5] == 0)) {
        const S6 c = transform_force(S6{{w[3], w[4], w[5], w[0], w[1], w[2]}}, ld3(sc, 3 * m.body_rootid[k]), ld3(d.xipos(), 3 * k));
        for (int q = 0; q < 6; q++) acc.v[q] += c.v[q];
      }
    }
    if (k) {
      for (int i = 0; i < ncon; i++) {
        const int a = cadr[i];
        if (a < 0) continue;
        const int b1 = m.geom_bodyid[cg1[i]], b2 = m.geom_bodyid[cg2[i]];
        if (b1 != k && b2 != k) continue;
        const int dim = cdim[i];
        double lf[6] = {0, 0, 0, 0, 0, 0};   // mj_contactForce: contact-frame force:torque (mju_decodePyramid)
        if (dim == 1) lf[0] = force[a];
        else {
          double n = 0;
          for (int q = 0; q < 2 * (dim - 1); q++) n += force[a + q];
          lf[0] = n;
          for (int q = 0; q < dim - 1; q++) lf[q + 1] = (force[a + 2 * q] - force[a + 2 * q + 1]) * cfri[5 * i + q];
        }
        lf[0] -= 0.0;   // adhesion (unsupported, zero)
        const M3 fr = ld9(cframe, 9 * i);
        const V3 tq = mulmTv(fr, V3{lf[3], lf[4], lf[5]}), ff = mulmTv(fr, V3{lf[0], lf[1], lf[2]});
        const S6 cc = transform_force(S6{{tq.x, tq.y, tq.z, ff.x, ff.y, ff.z}}, ld3(sc, 3 * m.body_rootid[k]), ld3(cpos, 3 * i));
        if (b1 == k) for (int q = 0; q < 6; q++) acc.v[q] -= cc.v[q];
        if (b2 == k) for (int q = 0; q < 6; q++) acc.v[q] += cc.v[q];
      }
    }
    if ((d.feat & FEAT_EQUALITY) && k && d.ne()[0]) {   // connect rows: force on body 1 (+) and body 2 (-), applied at the anchors
      FI ieq = d.scr_ieq();
      for (int eq = 0; eq < m.sz.neq; eq++) {
        const int r = ieq[eq];
        if (r < 0 || m.eq_kind[eq] < EQ_CONNECT) continue;
        const int o1 = m.eq_obj1id[eq], o2 = m.eq_obj2id[eq];
        if (o1 != k && o2 != k) continue;
        V3 p0, p1;
        connect_anchors(d, eq, p0, p1);
        const bool weld = m.eq_kind[eq] == EQ_WELD;   // welds also transmit a torque
        const S6 cf{{weld ? force[r + 3] : 0.0, weld ? force[r + 4] : 0.0, weld ? force[r + 5] : 0.0, force[r], force[r + 1], force[r + 2]}};
        if (o1 == k) { const S6 cc = transform_force(cf, ld3(sc, 3 * m.body_rootid[k]), p0); for (int q = 0; q < 6; q++) acc.v[q] += cc.v[q]; }
        if (o2 == k) { const S6 cc = transform_force(cf, ld3(sc, 3 * m.body_rootid[k]), p1); for (int q = 0; q < 6; q++) acc.v[q] -= cc.v[q]; }
      }
    }
    st6(cext, 6 * k, acc);
  }
  MJB_LANE0 {
    for (int k = 0; k < 6; k++) { cacc[k] = 0; cint[k] = 0; }
    if (!(m.opt.disableflags & DSBL_GRAVITY)) {
      cacc[3] = m.opt.gravity[0] * -1; cacc[4] = m.opt.gravity[1] * -1; cacc[5] = m.opt.gravity[2] * -1;
    }
  }
  MJB_PSYNC();
  for (int l = 1; l < m.sz.nlevel; l++) {
    const int ladr = m.lvl_adr[l], cnt = m.lvl_adr[l + 1] - ladr;
    MJB_PFOR(k_, cnt) {
      const int j = m.lvl_body[ladr + k_];
      const int bda = m.body_dofadr[j], dn = m.body_dofnum[j];
      S6 t = mul_dof_vec(cdd + 6 * bda, qvel + bda, dn);
      S6 a = ld6(cacc, 6 * m.body_parentid[j]);
      for (int k = 0; k < 6; k++) a.v[k] = a.v[k] + t.v[k];
      t = mul_dof_vec(cdof + 6 * bda, qacc + bda, dn);
      for (int k = 0; k < 6; k++) a.v[k] += t.v[k];
      st6(cacc, 6 * j, a);
      const I10 I = ld10(cinert, 10 * j);
      S6 f = mul_inert(I, a);
      const S6 v = ld6(cvel, 6 * j);
      const S6 c = cross_force(v, mul_inert(I, v));
      for (int k = 0; k < 6; k++) f.v[k] += c.v[k];
      const S6 e = ld6(cext, 6 * j);
      for (int k = 0; k < 6; k++) f.v[k] = f.v[k] - e.v[k];
      st6(cint, 6 * j, f);
    }
    MJB_PSYNC();
  }
  tree_accumulate(d, cint, 6, false);
}
// 6D acceleration of an object frame (mj_objectAcceleration): global frame, or the object's own frame
MJB_HD void object_acceleration(const Env& d, int kind, int id, bool local, V3& ang, V3& lin) {
  const DModel& m = d.m;
  const int body = (kind == SOBJ_GEOM) ? m.geom_bodyid[id] : (kind == SOBJ_SITE) ? m.site_bodyid[id] : id;
  if (m.body_dofnum[m.body_weldid[body]] == 0) { ang = V3{0, 0, 0}; lin = V3{0, 0, 0}; return; }
  V3 pos; M3 mat;
  sensor_frame(d, kind, id, pos, mat);
  const V3 dif = pos - ld3(d.subtree_com(), 3 * m.body_rootid[body]);
  V3 aa = ld3(d.cacc(), 6 * body), al = ld3(d.cacc(), 6 * body + 3) - cross(dif, aa);
  V3 va = ld3(d.cvel(), 6 * body), vl = ld3(d.cvel(), 6 * body + 3) - cross(dif, va);
  if (local) { aa = mulmTv(mat, aa); al = mulmTv(mat, al); va = mulmTv(mat, va); vl = mulmTv(mat, vl); }
  ang = aa;
  lin = al + cross(va, vl);
}

// ray against a sphere / box zone (engine_ray.c: ray_quad :103, ray_sphere :242, ray_box :490); only the
// distance is needed (>= 0: hit), normals are not
MJB_HD double ray_quad(double a, double b, double c, double* xx = nullptr) {
  double det = b * b - a * c;
  if (det < 0 || a < kMinVal) { if (xx) { xx[0] = -1; xx[1] = -1; } return -1; }
  det = sqrt(det);
  const double x0 = (-b - det) / a, x1 = (-b + det) / a;
  if (xx) { xx[0] = x0; xx[1] = x1; }
  if (x0 >= 0) return x0;
  if (x1 >= 0) return x1;
  return -1;
}
MJB_HD double ray_sphere(V3 pos, double dist_sqr, V3 pnt, V3 vec) {
  const V3 dif = pnt - pos;
  const double a = vec.x * vec.x + vec.y * vec.y + vec.z * vec.z;
  const double b = vec.x * dif.x + vec.y * dif.y + vec.z * dif.z;
  const double c = dif.x * dif.x + dif.y * dif.y + dif.z * dif.z - dist_sqr;
  return ray_quad(a, b, c);
}
MJB_HD double ray_plane(V3 pos, const M3& mat, const double* size, V3 pnt, V3 vec) {   // engine_ray.c:204-238
  const V3 dif = pnt - pos;
  const double lp[3] = {mat.m[0] * dif.x + mat.m[3] * dif.y + mat.m[6] * dif.z, mat.m[1] * dif.x + mat.m[4] * dif.y + mat.m[7] * dif.z,
                        mat.m[2] * dif.x + mat.m[5] * dif.y + mat.m[8] * dif.z};
  const double lv[3] = {mat.m[0] * vec.x + mat.m[3] * vec.y + mat.m[6] * vec.z, mat.m[1] * vec.x + mat.m[4] * vec.y + mat.m[7] * vec.z,
                        mat.m[2] * vec.x + mat.m[5] * vec.y + mat.m[8] * vec.z};
  if (lv[2] > -kMinVal) return -1;          // not pointing at the front face
  const double x = -lp[2] / lv[2];
  if (x < 0) return -1;
  const double p0 = lp[0] + x * lv[0], p1 = lp[1] + x * lv[1];
  if ((size[0] <= 0 || fabs(p0) <= size[0]) && (size[1] <= 0 || fabs(p1) <= size[1])) return x;   // inside the rendered rectangle
  return -1;
}
MJB_HD double ray_box(V3 pos, const M3& mat, const double* size, V3 pnt, V3 vec) {
  const double ssz = size[0] * size[0] + size[1] * size[1] + size[2] * size[2];
  if (ray_sphere(pos, ssz, pnt, vec) < 0) return -1;
  const V3 dif = pnt - pos;
  const double lp[3] = {mat.m[0] * dif.x + mat.m[3] * dif.y + mat.m[6] * dif.z, mat.m[1] * dif.x + mat.m[4] * dif.y + mat.m[7] * dif.z,
                        mat.m[2] * dif.x + mat.m[5] * dif.y + mat.m[8] * dif.z};
  const double lv[3] = {mat.m[0] * vec.x + mat.m[3] * vec.y + mat.m[6] * vec.z, mat.m[1] * vec.x + mat.m[4] * vec.y + mat.m[7] * vec.z,
                        mat.m[2] * vec.x + mat.m[5] * vec.y + mat.m[8] * vec.z};
  double x = -1;
  for (int i = 0; i < 3; i++) {
    if (fabs(lv[i]) <= kMinVal) continue;
    const int f0 = (i == 0) ? 1 : 0, f1 = (i == 2) ? 1 : 2;
    for (int side = -1; side <= 1; side += 2) {
      const double sol = (side * size[i] - lp[i]) / lv[i];
      if (sol < 0) continue;
      const double p0 = lp[f0] + sol * lv[f0], p1 = lp[f1] + sol * lv[f1];
      if (fabs(p0) <= size[f0] && fabs(p1) <= size[f1] && (x < 0 || sol < x)) x = sol;
    }
  }
  return x;
}

// local ray (ray_map, engine_ray.c:38): point and direction in the zone's frame
MJB_HD void ray_local(V3 pos, const M3& mat, V3 pnt, V3 vec, double* lp, double* lv) {
  const V3 dif = pnt - pos;
  lp[0] = mat.m[0] * dif.x + mat.m[3] * dif.y + mat.m[6] * dif.z;
  lp[1] = mat.m[1] * dif.x + mat.m[4] * dif.y + mat.m[7] * dif.z;
  lp[2] = mat.m[2] * dif.x + mat.m[5] * dif.y + mat.m[8] * dif.z;
  lv[0] = mat.m[0] * vec.x + mat.m[3] * vec.y + mat.m[6] * vec.z;
  lv[1] = mat.m[1] * vec.x + mat.m[4] * vec.y + mat.m[7] * vec.z;
  lv[2] = mat.m[2] * vec.x + mat.m[5] * vec.y + mat.m[8] * vec.z;
}
MJB_HD double ray_capsule(V3 pos, const M3& mat, const double* size, V3 pnt, V3 vec) {   // engine_ray.c:272-355
  const double ssz = size[0] + size[1];
  if (ray_sphere(pos, ssz * ssz, pnt, vec) < 0) return -1;
  double lp[3], lv[3], xx[2];
  ray_local(pos, mat, pnt, vec, lp, lv);
  double x = -1;
  double a = lv[0] * lv[0] + lv[1] * lv[1];
  double b = lv[0] * lp[0] + lv[1] * lp[1];
  double c = lp[0] * lp[0] + lp[1] * lp[1] - size[0] * size[0];
  const double sol = ray_quad(a, b, c, xx);
  if (sol >= 0 && fabs(lp[2] + sol * lv[2]) <= size[1]) { if (x < 0 || sol < x) x = sol; }
  double ld[3] = {lp[0], lp[1], lp[2] - size[1]};   // top cap
  a = lv[0] * lv[0] + lv[1] * lv[1] + lv[2] * lv[2];
  b = lv[0] * ld[0] + lv[1] * ld[1] + lv[2] * ld[2];
  c = ld[0] * ld[0] + ld[1] * ld[1] + ld[2] * ld[2] - size[0] * size[0];
  ray_quad(a, b, c, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0 && lp[2] + xx[i] * lv[2] >= size[1]) { if (x < 0 || xx[i] < x) x = xx[i]; }
  ld[2] = lp[2] + size[1];                          // bottom cap
  b = lv[0] * ld[0] + lv[1] * ld[1] + lv[2] * ld[2];
  c = ld[0] * ld[0] + ld[1] * ld[1] + ld[2] * ld[2] - size[0] * size[0];
  ray_quad(a, b, c, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0 && lp[2] + xx[i] * lv[2] <= -size[1]) { if (x < 0 || xx[i] < x) x = xx[i]; }
  return x;
}
MJB_HD double ray_ellipsoid(V3 pos, const M3& mat, const double* size, V3 pnt, V3 vec) {   // engine_ray.c:358-398
  double lp[3], lv[3];
  ray_local(pos, mat, pnt, vec, lp, lv);
  const double s[3] = {1 / (size[0] * size[0]), 1 / (size[1] * size[1]), 1 / (size[2] * size[2])};
  const double a = s[0] * lv[0] * lv[0] + s[1] * lv[1] * lv[1] + s[2] * lv[2] * lv[2];
  const double b = s[0] * lv[0] * lp[0] + s[1] * lv[1] * lp[1] + s[2] * lv[2] * lp[2];
  const double c = s[0] * lp[0] * lp[0] + s[1] * lp[1] * lp[1] + s[2] * lp[2] * lp[2] - 1;
  return ray_quad(a, b, c);
}
MJB_HD double ray_cylinder(V3 pos, const M3& mat, const double* size, V3 pnt, V3 vec) {   // engine_ray.c:401-486
  const double ssz = size[0] * size[0] + size[1] * size[1];
  if (ray_sphere(pos, ssz, pnt, vec) < 0) return -1;
  double lp[3], lv[3];
  ray_local(pos, mat, pnt, vec, lp, lv);
  double x = -1;
  if (fabs(lv[2]) > kMinVal) {
    for (int side = -1; side <= 1; side += 2) {
      const double sol = (side * size[1] - lp[2]) / lv[2];
      if (sol < 0) continue;
      const double p0 = lp[0] + sol * lv[0], p1 = lp[1] + sol * lv[1];
      if (p0 * p0 + p1 * p1 <= size[0] * size[0] && (x < 0 || sol < x)) x = sol;
    }
  }
  const double a = lv[0] * lv[0] + lv[1] * lv[1];
  const double b = lv[0] * lp[0] + lv[1] * lp[1];
  const double c = lp[0] * lp[0] + lp[1] * lp[1] - size[0] * size[0];
  const double sol = ray_quad(a, b, c);
  if (sol >= 0 && fabs(lp[2] + sol * lv[2]) <= size[1] && (x < 0 || sol < x)) x = sol;
  return x;
}

// mj_subtreeVel (engine_core_smooth.c:2249-2322): linear velocity and angular momentum of every subtree
// about its own centre of mass; serial over bodies in the reference's order (sensor models only)
MJB_HD void subtree_vel(const Env& d) {
  const DModel& m = d.m;
  const int nbody = m.sz.nbody;
  FD lv = d.subtree_linvel(), am = d.subtree_angmom(), bv = d.subtree_bvel();
  MJB_PFOR(i, nbody) {
    V3 ang, lin;
    object_velocity(d, SOBJ_BODY, i, ang, lin);
    st3(bv, 6 * i, ang); st3(bv, 6 * i + 3, lin);
    const double mass = m.body_mass[i];
    st3(lv, 3 * i, V3{lin.x * mass, lin.y * mass, lin.z * mass});
    const M3 xi = ld9(d.ximat(), 9 * i);
    V3 dv = mulmTv(xi, ang);
    dv.x *= m.body_inertia[3 * i]; dv.y *= m.body_inertia[3 * i + 1]; dv.z *= m.body_inertia[3 * i + 2];
    st3(am, 3 * i, mulmv(xi, dv));
  }
  MJB_PSYNC();
  MJB_LANE0 {
    for (int i = nbody - 1; i >= 0; i--) {
      if (i) { const int p = m.body_parentid[i]; st3(lv, 3 * p, ld3(lv, 3 * p) + ld3(lv, 3 * i)); }
      const double s = 1 / dmax(kMinVal, m.body_subtreemass[i]);
      const V3 l = ld3(lv, 3 * i);
      st3(lv, 3 * i, V3{l.x * s, l.y * s, l.z * s});
    }
    for (int i = nbody - 1; i > 0; i--) {
      const int p = m.body_parentid[i];
      V3 dx = ld3(d.xipos(), 3 * i) - ld3(d.subtree_com(), 3 * i);
      V3 dv = ld3(bv, 6 * i + 3) - ld3(lv, 3 * i);
      const double mass = m.body_mass[i];
      V3 dL = cross(dx, V3{dv.x * mass, dv.y * mass, dv.z * mass});
      st3(am, 3 * i, ld3(am, 3 * i) + dL);
      st3(am, 3 * p, ld3(am, 3 * p) + ld3(am, 3 * i));
      dx = ld3(d.subtree_com(), 3 * i) - ld3(d.subtree_com(), 3 * p);
      dv = ld3(lv, 3 * i) - ld3(lv, 3 * p);
      const double sm = m.body_subtreemass[i];
      dL = cross(dx, V3{dv.x * sm, dv.y * sm, dv.z * sm});
      st3(am, 3 * p, ld3(am, 3 * p) + dL);
    }
  }
  MJB_PSYNC();
}

// potential and kinetic energy (mj_energyPos / mj_energyVel, engine_sensor.c:1659-1779): gravity and the joint /
// tendon springs (serial sums in the reference's order, on lane 0), 0.5 qvel' M qvel.  Both depend on the position
// and velocity stages only, so they are evaluated once, after the solve, whatever stage the reference uses.
MJB_HD double poly_potential(double linear, const double* poly, double x) {   // mju_polyPotential, flg_odd = 0
  double res = 0.5 * linear * (x * x);
  double xpow = x;
  for (int i = 0; i < kNPoly; i++) {
    xpow *= x;
    res += poly[i] / (i + 3) * (xpow * x);
  }
  return res;
}
MJB_HD void energy(const Env& d) {
  const DModel& m = d.m;
  if (!(d.feat & FEAT_SENSOR)) return;   // (models with energy flags or sensors run the full kernels)
  FD en = d.energy();
  if (!m.sz.epot) { MJB_LANE0 { en[0] = 0; if (!m.sz.ekin) en[1] = 0; } }
  else {
    MJB_LANE0 {
      double e = 0;
      if (!(m.opt.disableflags & DSBL_GRAVITY)) {
        FD xi = d.xipos();
        for (int i = 1; i < m.sz.nbody; i++)
          e -= m.body_mass[i] * (m.opt.gravity[0] * xi[3 * i] + m.opt.gravity[1] * xi[3 * i + 1] + m.opt.gravity[2] * xi[3 * i + 2]);
      }
      if (!(m.opt.disableflags & DSBL_SPRING)) {
        FD qpos = d.qpos();
        for (int b = 1; b < m.sz.nbody; b++) {
          for (int j = m.body_jntadr[b]; j < m.body_jntadr[b] + m.body_jntnum[b]; j++) {
            const double k = m.jnt_stiffness[j];
            const double* poly = m.jnt_stiffnesspoly + kNPoly * j;
            bool zero = true;
            for (int c = 0; c < kNPoly; c++) if (poly[c] != 0) zero = false;
            if (k == 0 && zero) continue;
            int padr = m.jnt_qposadr[j];
            const int jt = m.jnt_type[j];
            if (jt == JNT_FREE) {
              const V3 dif = ld3(qpos, padr) - ldc3(m.qpos_spring, padr);
              e += poly_potential(k, poly, sqrt(dif.x * dif.x + dif.y * dif.y + dif.z * dif.z));
              padr += 3;
            }
            if (jt == JNT_FREE || jt == JNT_BALL) {
              const V3 dif = qsub(ld4(qpos, padr), ldc4(m.qpos_spring, padr));
              e += poly_potential(k, poly, sqrt(dif.x * dif.x + dif.y * dif.y + dif.z * dif.z));
            } else {
              e += poly_potential(k, poly, qpos[padr] - m.qpos_spring[padr]);
            }
          }
        }
        FD tl = d.ten_length();
        for (int t = 0; t < m.sz.ntendon; t++) {
          const double len = tl[t], lower = m.tendon_lengthspring[2 * t], upper = m.tendon_lengthspring[2 * t + 1];
          const double x = (len > upper) ? len - upper : (len < lower) ? len - lower : 0;
          e += poly_potential(m.tendon_stiffness[t], m.tendon_stiffnesspoly + kNPoly * t, x);
        }
      }
      en[0] = e;
    }
  }
  if (m.sz.ekin) {
    FD vec = d.scr_nv(), qvel = d.qvel();
    MJB_PSYNC();
    mul_M(d, vec, qvel);
    MJB_LANE0 en[1] = 0.5 * dot_ref(m.sz.nv, [&](int i) { return vec[i]; }, [&](int i) { return qvel[i]; });
  }
  MJB_PSYNC();
}

// ---- contact sensor (engine_sensor.c:318-470,1027-1165) -------------------------------------------------------------
// point inside a site volume (mju_insideGeom, engine_util_misc.c:452-496)
MJB_HD bool inside_geom(V3 pos, const M3& mat, const double* size, int type, V3 point) {
  const V3 vec = point - pos;
  if (type == GEOM_SPHERE) return dot(vec, vec) < size[0] * size[0];
  const V3 pl = mulmTv3(mat, vec);
  if (type == GEOM_CAPSULE) {
    const double zc = dclip(pl.z, -size[1], size[1]);
    const double zd = (pl.z - zc) * (pl.z - zc);
    return pl.x * pl.x + pl.y * pl.y + zd < size[0] * size[0];
  }
  if (type == GEOM_ELLIPSOID) return pl.x * pl.x / (size[0] * size[0]) + pl.y * pl.y / (size[1] * size[1]) + pl.z * pl.z / (size[2] * size[2]) < 1;
  if (type == GEOM_CYLINDER) return fabs(pl.z) < size[1] && pl.x * pl.x + pl.y * pl.y < size[0] * size[0];
  if (type == GEOM_BOX) return fabs(pl.x) < size[0] && fabs(pl.y) < size[1] && fabs(pl.z) < size[2];
  return false;
}
// object kinds of a contact sensor: 0 none, 1 site, 2 geom, 3 body, 4 subtree (xbody)
MJB_HD bool contact_check(const DModel& m, int body, int geom, int kind, int id) {
  if (kind == 0 || kind == 1) return true;
  if (kind == 2) return id == geom;
  if (kind == 3) return id == body;
  while (body > id) body = m.body_parentid[body];
  return body == id;
}
// 0: no match, 1: match, -1: match with the contact frame flipped (matchContact)
MJB_HD int contact_match(const Env& d, int con, int k1, int id1, int k2, int id2) {
  const DModel& m = d.m;
  if (k1 == 0 && k2 == 0) return 1;
  if (k1 == 1 && !inside_geom(ld3(d.site_xpos(), 3 * id1), ld9(d.site_xmat(), 9 * id1), m.site_size + 3 * id1, m.site_type[id1], ld3(d.con_pos(), 3 * con))) return 0;
  const int g1 = d.con_geom1()[con], g2 = d.con_geom2()[con], b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
  const bool m11 = contact_check(m, b1, g1, k1, id1), m12 = contact_check(m, b2, g2, k1, id1);
  const bool m21 = contact_check(m, b1, g1, k2, id2), m22 = contact_check(m, b2, g2, k2, id2);
  if (!m11 && !m12) return 0;
  if (!m21 && !m22) return 0;
  if (k1 != 0 && k2 != 0) {
    const bool regular = m11 && m22, reverse = m12 && m21;
    if (regular && !reverse) return 1;
    if (reverse && !regular) return -1;
    if (regular && reverse) return 1;
  } else if (k1 != 0) return m11 ? 1 : -1;
  else if (k2 != 0) return m22 ? 1 : -1;
  return 0;
}
// contact-frame force : torque of contact `con` (mj_contactForce, engine_core_util.c:1075-1095; pyramidal cones)
MJB_HD void contact_wrench(const Env& d, int con, double* lf) {
  for (int q = 0; q < 6; q++) lf[q] = 0;
  const int a = d.con_efcadr()[con];
  if (a < 0) return;
  FD force = d.efc_force(), cfri = d.con_friction();
  const int dim = d.con_dim()[con];
  if (dim == 1) lf[0] = force[a];
  else {
    double n = 0;
    for (int q = 0; q < 2 * (dim - 1); q++) n += force[a + q];
    lf[0] = n;
    for (int q = 0; q < dim - 1; q++) lf[q + 1] = (force[a + 2 * q] - force[a + 2 * q + 1]) * cfri[5 * con + q];
  }
  lf[0] -= 0.0;   // adhesion (refused by the model check: zero)
}
MJB_HD void contact_sensor(const Env& d, int i, FD out) {
  const DModel& m = d.m;
  const int spec = m.sensor_intprm0[i], reduce = m.sensor_intprm1[i], dim = m.sensor_dim[i], adr = m.sensor_adr[i];
  const int k1 = m.sensor_objraw[i], id1 = m.sensor_objid[i], k2 = m.sensor_refraw[i], id2 = m.sensor_refid[i];
  const int fsz[7] = {1, 3, 3, 1, 3, 3, 3};   // found, force, torque, dist, pos, normal, tangent
  int off[7], size = 0;
  for (int f = 0; f < 7; f++) { off[f] = (spec & (1 << f)) ? size : -1; if (spec & (1 << f)) size += fsz[f]; }
  const int num = size ? dim / size : 0, ncon = d.ncon()[0];
  for (int c = 0; c < dim; c++) out[adr + c] = 0;
  int nmatch = 0;
  for (int j = 0; j < ncon; j++) if (contact_match(d, j, k1, id1, k2, id2)) nmatch++;
  auto criterion = [&](int j) {
    if (reduce == 1) return d.con_dist()[j];
    double lf[6];
    contact_wrench(d, j, lf);
    return -(lf[0] * lf[0] + lf[1] * lf[1] + lf[2] * lf[2]);
  };
  auto fill = [&](int slot, int j, bool flip) {   // copySensorData
    const long base = adr + (long)slot * size;
    if (off[0] >= 0) out[base + off[0]] = nmatch;
    if (off[1] >= 0 || off[2] >= 0) {
      double lf[6];
      contact_wrench(d, j, lf);
      if (off[1] >= 0) { out[base + off[1]] = lf[0]; out[base + off[1] + 1] = lf[1]; out[base + off[1] + 2] = flip ? lf[2] * -1 : lf[2]; }
      if (off[2] >= 0) { out[base + off[2]] = lf[3]; out[base + off[2] + 1] = lf[4]; out[base + off[2] + 2] = flip ? lf[5] * -1 : lf[5]; }
    }
    if (off[3] >= 0) out[base + off[3]] = d.con_dist()[j];
    if (off[4] >= 0) for (int c = 0; c < 3; c++) out[base + off[4] + c] = d.con_pos()[3 * j + c];
    if (off[5] >= 0) for (int c = 0; c < 3; c++) out[base + off[5] + c] = flip ? d.con_frame()[9 * j + c] * -1 : d.con_frame()[9 * j + c];
    if (off[6] >= 0) for (int c = 0; c < 3; c++) out[base + off[6] + c] = flip ? d.con_frame()[9 * j + 3 + c] * -1 : d.con_frame()[9 * j + 3 + c];
  };
  const int nslot = num < nmatch ? num : nmatch;
  if (reduce == 0) {          // first matches in contact order
    int slot = 0;
    for (int j = 0; j < ncon && slot < nslot; j++) {
      const int mj = contact_match(d, j, k1, id1, k2, id2);
      if (mj) fill(slot++, j, mj < 0);
    }
  } else if (reduce == 1 || reduce == 2) {   // the nslot smallest by (criterion, contact id), ascending (ContactSelect)
    double lastc = 0;
    int lastj = -1;
    for (int slot = 0; slot < nslot; slot++) {
      int best = -1;
      double bestc = 0;
      for (int j = 0; j < ncon; j++) {
        if (!contact_match(d, j, k1, id1, k2, id2)) continue;
        const double cj = criterion(j);
        if (lastj >= 0 && (cj < lastc || (cj == lastc && j <= lastj))) continue;   // already emitted
        if (best < 0 || cj < bestc || (cj == bestc && j < best)) { best = j; bestc = cj; }
      }
      if (best < 0) break;
      fill(slot, best, contact_match(d, best, k1, id1, k2, id2) < 0);
      lastc = bestc; lastj = best;
    }
  } else {                    // net force about the force-weighted centroid, global frame
    V3 point{0, 0, 0};
    double total = 0;
    for (int j = 0; j < ncon; j++) {
      const int mj = contact_match(d, j, k1, id1, k2, id2);
      if (!mj) continue;
      double lf[6];
      contact_wrench(d, j, lf);
      if (mj < 0) for (int q = 0; q < 6; q++) lf[q] = lf[q] * -1;
      const double w = sqrt(lf[0] * lf[0] + lf[1] * lf[1] + lf[2] * lf[2]);
      point.x += d.con_pos()[3 * j] * w; point.y += d.con_pos()[3 * j + 1] * w; point.z += d.con_pos()[3 * j + 2] * w;
      total += w;
    }
    point = point * (1.0 / (total > kMinVal ? total : kMinVal));
    V3 force{0, 0, 0}, torque{0, 0, 0};
    for (int j = 0; j < ncon; j++) {
      const int mj = contact_match(d, j, k1, id1, k2, id2);
      if (!mj) continue;
      double lf[6];
      contact_wrench(d, j, lf);
      if (mj < 0) for (int q = 0; q < 6; q++) lf[q] = lf[q] * -1;
      const M3 fr = ld9(d.con_frame(), 9 * j);
      const V3 fj = mulmTv3(fr, V3{lf[0], lf[1], lf[2]}), tj = mulmTv3(fr, V3{lf[3], lf[4], lf[5]});
      force = force + fj;
      torque = torque + tj;
      torque = torque + cross(ld3(d.con_pos(), 3 * j) - point, fj);
    }
    if (off[0] >= 0) out[adr + off[0]] = nmatch;
    if (off[1] >= 0) { out[adr + off[1]] = force.x; out[adr + off[1] + 1] = force.y; out[adr + off[1] + 2] = force.z; }
    if (off[2] >= 0) { out[adr + off[2]] = torque.x; out[adr + off[2] + 1] = torque.y; out[adr + off[2] + 2] = torque.z; }
    if (off[3] >= 0) out[adr + off[3]] = 0;
    if (off[4] >= 0) { out[adr + off[4]] = point.x; out[adr + off[4] + 1] = point.y; out[adr + off[4] + 2] = point.z; }
    if (off[5] >= 0) out[adr + off[5]] = 1;
    if (off[6] >= 0) out[adr + off[6] + 1] = 1;
  }
}

// ---- history buffers (FEAT_HISTORY): compute_or_read_sensor (engine_sensor.c:1387-1428) and the lazy inputs ----
// whether sensor i is computed in this forward pass (else it is read from its buffer)
MJB_HD bool sensor_computes(const Env& d, int i) {
  const DModel& m = d.m;
  if (m.sensor_history[2 * i] <= 0) return true;
  if (m.sensor_delay[i] > 0) return false;
  const double interval = m.sensor_interval[2 * i];
  if (interval > 0) return d.history()[m.sensor_historyadr[i]] + interval <= d.time()[0];
  return true;
}
// whether mj_advance computes sensor i into a new sample (a delayed sensor whose interval, if any, has elapsed)
MJB_HD bool sensor_computes_in_advance(const Env& d, int i) {
  const DModel& m = d.m;
  if (m.sensor_history[2 * i] <= 0 || !(m.sensor_delay[i] > 0)) return false;
  const double interval = m.sensor_interval[2 * i];
  return !(interval > 0) || d.history()[m.sensor_historyadr[i]] + interval <= d.time()[0];
}
// mj_rnePostConstraint / mj_subtreeVel run inside the reference's per-sensor computation, once per forward pass (flags
// flg_rnepost / flg_subtreevel), and only when a sensor that needs them is computed: before the sensors of a forward
// pass (advance = false) or before the delayed sensors that mj_advance computes (advance = true)
MJB_HD void lazy_sensor_inputs(const Env& d, bool advance) {
  const DModel& m = d.m;
  bool rp = false, sv = false;
  for (int i = 0; i < m.sz.nsensor; i++) {
    if (!(advance ? sensor_computes_in_advance(d, i) : sensor_computes(d, i))) continue;
    const int t = m.sensor_type[i];
    if (t == SENS_ACCELEROMETER || t == SENS_FORCE || t == SENS_TORQUE || t == SENS_FRAMELINACC || t == SENS_FRAMEANGACC) rp = true;
    if (t == SENS_SUBTREELINVEL || t == SENS_SUBTREEANGMOM) sv = true;
  }
  FI flg = d.hist_flg();
  rp = rp && m.sz.rnepost && !flg[0];
  sv = sv && m.sz.subtreevel && !flg[1];
  MJB_PSYNC();
  if (rp) rne_post(d);
  if (sv) subtree_vel(d);
  MJB_LANE0 { if (rp) flg[0] = 1; if (sv) flg[1] = 1; }
  MJB_PSYNC();
}
// advance (FEAT_HISTORY only): the sensor part of mj_advance instead of the sensors of a forward pass - every sensor
// with a buffer records a sample at the current time (an interval sensor only once its interval has elapsed, advancing
// its tick), computed into the new slot when the sensor is delayed, else copied from sensordata
MJB_HD void sensors(const Env& d, bool advance = false) {
  const DModel& m = d.m;
#ifdef MJB_HISTORY_CODE
  if ((d.feat & FEAT_HISTORY) && !advance) {   // mj_forward clears flg_rnepost whenever it runs the sensors, disabled or not
    MJB_LANE0 d.hist_flg()[0] = 0;
    MJB_PSYNC();
  }
#endif
  if (!m.sz.nsensor || ((m.opt.disableflags & DSBL_SENSOR) && !advance)) return;
  const int nefc = d.nefc()[0], nf = d.ne()[0] + d.nf()[0];   // first row after the equality and friction rows
  FD sd = d.sensordata();
  FI etype = d.efc_type(), eid = d.efc_id();
#ifdef MJB_HISTORY_CODE
  if (d.feat & FEAT_HISTORY) lazy_sensor_inputs(d, advance);
  else
#endif
  {
    if (m.sz.rnepost) rne_post(d);
    if (m.sz.subtreevel) subtree_vel(d);
  }
  MJB_PFOR(i, m.sz.nsensor) {
    FD out = sd;   // where sensor i's values go (out[sensor_adr ...])
#ifdef MJB_HISTORY_CODE
    if (d.feat & FEAT_HISTORY) {
      const int n = m.sensor_history[2 * i], dim = m.sensor_dim[i], adr = m.sensor_adr[i];
      FD buf = d.history() + m.sensor_historyadr[i];
      const double time = d.time()[0];
      if (!advance) {   // compute_or_read_sensor: a sensor that is not computed now is read at time - delay
        if (!sensor_computes(d, i)) { hist_read(buf, n, dim, sd + adr, time - m.sensor_delay[i], m.sensor_history[2 * i + 1]); continue; }
      } else {
        if (n <= 0) continue;
        const double interval = m.sensor_interval[2 * i];
        if (interval > 0) {
          if (!(buf[0] + interval <= time)) continue;
          buf[0] += interval;
        }
        FD slot = hist_insert(buf, n, dim, time);
        if (!(m.sensor_delay[i] > 0)) { for (int k = 0; k < dim; k++) slot[k] = sd[adr + k]; continue; }
        out = slot + (-(long)adr);
      }
    }
#endif
    const int type = m.sensor_type[i], id = m.sensor_objid[i], adr = m.sensor_adr[i], dim = m.sensor_dim[i];
    const int okind = m.sensor_objtype[i], rkind = m.sensor_reftype[i], refid = m.sensor_refid[i];
    double v[4] = {0, 0, 0, 0};
    auto limit_row = [&](int ctype) {   // first limit row of this joint / tendon, -1 if inactive
      for (int j = nf; j < nefc; j++) if (etype[j] == ctype && eid[j] == id) return j;
      return -1;
    };
    switch (type) {
      case SENS_JOINTPOS: v[0] = d.qpos()[m.jnt_qposadr[id]]; break;
      case SENS_TENDONPOS: v[0] = d.ten_length()[id]; break;
      case SENS_ACTUATORPOS: v[0] = d.actuator_length()[id]; break;
      case SENS_BALLQUAT: { Q4 q = ld4(d.qpos(), m.jnt_qposadr[id]); normalize(q); v[0] = q.w; v[1] = q.x; v[2] = q.y; v[3] = q.z; break; }
      case SENS_JOINTLIMITPOS: { const int j = limit_row(CNSTR_LIMIT_JOINT); if (j >= 0) v[0] = d.efc_pos()[j] - d.efc_margin()[j]; break; }
      case SENS_TENDONLIMITPOS: { const int j = limit_row(CNSTR_LIMIT_TENDON); if (j >= 0) v[0] = d.efc_pos()[j] - d.efc_margin()[j]; break; }
      case SENS_FRAMEPOS: case SENS_FRAMEXAXIS: case SENS_FRAMEYAXIS: case SENS_FRAMEZAXIS: {
        V3 pos; M3 mat;
        sensor_frame(d, okind, id, pos, mat);
        const int off = type - SENS_FRAMEXAXIS;
        V3 r = (type == SENS_FRAMEPOS) ? pos : V3{mat.m[off], mat.m[off + 3], mat.m[off + 6]};
        if (refid >= 0) {
          V3 rpos; M3 rmat;
          sensor_frame(d, rkind, refid, rpos, rmat);
          r = mulmTv(rmat, (type == SENS_FRAMEPOS) ? pos - rpos : r);
        }
        v[0] = r.x; v[1] = r.y; v[2] = r.z;
        break;
      }
      case SENS_FRAMEQUAT: {
        Q4 q = sensor_quat(d, okind, id);
        if (refid >= 0) {
          Q4 rq = sensor_quat(d, rkind, refid);
          rq = Q4{rq.w, -rq.x, -rq.y, -rq.z};
          q = qmul(rq, q);
        }
        v[0] = q.w; v[1] = q.x; v[2] = q.y; v[3] = q.z;
        break;
      }
      case SENS_SUBTREECOM: { const V3 c = ld3(d.subtree_com(), 3 * id); v[0] = c.x; v[1] = c.y; v[2] = c.z; break; }
      case SENS_SUBTREELINVEL: { const V3 c = ld3(d.subtree_linvel(), 3 * id); v[0] = c.x; v[1] = c.y; v[2] = c.z; break; }
      case SENS_SUBTREEANGMOM: { const V3 c = ld3(d.subtree_angmom(), 3 * id); v[0] = c.x; v[1] = c.y; v[2] = c.z; break; }
      case SENS_TOUCH: {   // engine_sensor.c:980-1025: normal forces of the body's contacts whose ray meets the zone
        const int bodyid = m.site_bodyid[id], ncon = d.ncon()[0];
        FI cadr = d.con_efcadr(), cdim = d.con_dim(), g1 = d.con_geom1(), g2 = d.con_geom2();
        FD ef = d.efc_force();
        const V3 spos = ld3(d.site_xpos(), 3 * id);
        const M3 smat = ld9(d.site_xmat(), 9 * id);
        for (int j = 0; j < ncon; j++) {
          const int b1 = m.geom_bodyid[g1[j]], b2 = m.geom_bodyid[g2[j]], a = cadr[j];
          if (a < 0 || (bodyid != b1 && bodyid != b2)) continue;
          double fn = 0;   // mju_decodePyramid: normal force = sum of the pyramid forces
          if (cdim[j] == 1) fn = ef[a];
          else for (int k = 0; k < 2 * (cdim[j] - 1); k++) fn += ef[a + k];
          if (fn <= 0) continue;
          const V3 fr = ld3(d.con_frame(), 9 * j);
          V3 ray{fr.x * fn, fr.y * fn, fr.z * fn};
          normalize(ray);
          if (bodyid == b2) ray = V3{ray.x * -1, ray.y * -1, ray.z * -1};
          const V3 cp = ld3(d.con_pos(), 3 * j);
          const int st = m.site_type[id];
          const double* ssz = m.site_size + 3 * id;
          const double hit = (st == GEOM_SPHERE) ? ray_sphere(spos, ssz[0] * ssz[0], cp, ray) : (st == GEOM_BOX) ? ray_box(spos, smat, ssz, cp, ray)
                           : (st == GEOM_CAPSULE) ? ray_capsule(spos, smat, ssz, cp, ray) : (st == GEOM_ELLIPSOID) ? ray_ellipsoid(spos, smat, ssz, cp, ray)
                           : ray_cylinder(spos, smat, ssz, cp, ray);
          if (hit >= 0) v[0] += fn;
        }
        break;
      }
      case SENS_CLOCK: v[0] = d.time()[0]; break;
      case SENS_CONTACT: contact_sensor(d, i, out); continue;
      case SENS_RANGEFINDER: {   // mj_ray (engine_ray.c:1308-1351) along the site's z axis, the site's own body excluded
        const int spec = m.sensor_intprm0[i], bodyex = m.site_bodyid[id];
        const M3 smat = ld9(d.site_xmat(), 9 * id);
        const V3 org = ld3(d.site_xpos(), 3 * id), dir{smat.m[2], smat.m[5], smat.m[8]};
        double dist = -1;
        for (int g = 0; g < m.sz.ngeom; g++) {
          if (m.geom_rayskip[g] || m.geom_bodyid[g] == bodyex) continue;
          const V3 gp = ld3(d.geom_xpos(), 3 * g);
          const M3 gm = ld9(d.geom_xmat(), 9 * g);
          const double* gs = m.geom_size + 3 * g;
          const int gt = m.geom_type[g];
          const double nd = (gt == GEOM_PLANE) ? ray_plane(gp, gm, gs, org, dir) : (gt == GEOM_SPHERE) ? ray_sphere(gp, gs[0] * gs[0], org, dir)
                          : (gt == GEOM_CAPSULE) ? ray_capsule(gp, gm, gs, org, dir) : (gt == GEOM_ELLIPSOID) ? ray_ellipsoid(gp, gm, gs, org, dir)
                          : (gt == GEOM_CYLINDER) ? ray_cylinder(gp, gm, gs, org, dir) : ray_box(gp, gm, gs, org, dir);
          if (nd >= 0 && (nd < dist || dist < 0)) dist = nd;
        }
        // fill_raydata (engine_sensor.c:470-520), then the cutoff of every field
        double vv[11];
        int n = 0;
        const bool hit = dist >= 0;
        if (spec & 1) vv[n++] = dist;
        if (spec & 2) { vv[n++] = hit ? dir.x : 0; vv[n++] = hit ? dir.y : 0; vv[n++] = hit ? dir.z : 0; }
        if (spec & 4) { vv[n++] = org.x; vv[n++] = org.y; vv[n++] = org.z; }
        V3 pt{0, 0, 0};
        if ((spec & (8 | 32)) && hit) pt = addscl(org, dir, dist);
        if (spec & 8) { vv[n++] = pt.x; vv[n++] = pt.y; vv[n++] = pt.z; }
        if (spec & 32) vv[n++] = hit ? dist : -1;
        const int cmr = m.sensor_cutmode[i];
        const double cutr = m.sensor_cutoff[i];
        for (int k2 = 0; k2 < n && k2 < dim; k2++) {
          double x = vv[k2];
          if (cmr == 1) x = dclip(x, -cutr, cutr); else if (cmr == 2) x = dmin(cutr, x);
          out[adr + k2] = x;
        }
        continue;
      }
      case SENS_E_POTENTIAL: v[0] = d.energy()[0]; break;
      case SENS_E_KINETIC: v[0] = d.energy()[1]; break;
      case SENS_JOINTVEL: v[0] = d.qvel()[m.jnt_dofadr[id]]; break;
      case SENS_TENDONVEL: v[0] = d.ten_velocity()[id]; break;
      case SENS_ACTUATORVEL: v[0] = d.actuator_velocity()[id]; break;
      case SENS_BALLANGVEL: { const V3 w = ld3(d.qvel(), m.jnt_dofadr[id]); v[0] = w.x; v[1] = w.y; v[2] = w.z; break; }
      case SENS_JOINTLIMITVEL: { const int j = limit_row(CNSTR_LIMIT_JOINT); if (j >= 0) v[0] = d.efc_vel()[j]; break; }
      case SENS_TENDONLIMITVEL: { const int j = limit_row(CNSTR_LIMIT_TENDON); if (j >= 0) v[0] = d.efc_vel()[j]; break; }
      case SENS_FRAMELINVEL: case SENS_FRAMEANGVEL: {
        V3 ang, lin;
        object_velocity(d, okind, id, ang, lin);
        if (refid >= 0) {
          V3 pos, rpos, rang, rlin; M3 mat, rmat;
          sensor_frame(d, okind, id, pos, mat);
          sensor_frame(d, rkind, refid, rpos, rmat);
          object_velocity(d, rkind, refid, rang, rlin);
          V3 rel_ang = ang - rang, rel_lin = lin - rlin;
          rel_lin = rel_lin + cross(pos - rpos, rang);
          ang = mulmTv(rmat, rel_ang);
          lin = mulmTv(rmat, rel_lin);
        }
        const V3 r = (type == SENS_FRAMELINVEL) ? lin : ang;
        v[0] = r.x; v[1] = r.y; v[2] = r.z;
        break;
      }
      case SENS_VELOCIMETER: case SENS_GYRO: {   // site velocity expressed in the site frame
        V3 ang, lin, pos; M3 mat;
        object_velocity(d, SOBJ_SITE, id, ang, lin);
        sensor_frame(d, SOBJ_SITE, id, pos, mat);
        const V3 r = mulmTv(mat, (type == SENS_GYRO) ? ang : lin);
        v[0] = r.x; v[1] = r.y; v[2] = r.z;
        break;
      }
      case SENS_ACCELEROMETER: {
        V3 ang, lin;
        object_acceleration(d, SOBJ_SITE, id, true, ang, lin);
        v[0] = lin.x; v[1] = lin.y; v[2] = lin.z;
        break;
      }
      case SENS_FORCE: case SENS_TORQUE: {   // interaction force with the parent at the site, in the site frame
        V3 pos; M3 mat;
        sensor_frame(d, SOBJ_SITE, id, pos, mat);
        const int body = m.site_bodyid[id];
        const S6 t = transform_force(ld6(d.cfrc_int(), 6 * body), pos, ld3(d.subtree_com(), 3 * m.body_rootid[body]));
        const V3 r = (type == SENS_FORCE) ? mulmTv(mat, V3{t.v[3], t.v[4], t.v[5]}) : mulmTv(mat, V3{t.v[0], t.v[1], t.v[2]});
        v[0] = r.x; v[1] = r.y; v[2] = r.z;
        break;
      }
      case SENS_FRAMELINACC: case SENS_FRAMEANGACC: {
        V3 ang, lin;
        object_acceleration(d, okind, id, false, ang, lin);
        const V3 r = (type == SENS_FRAMELINACC) ? lin : ang;
        v[0] = r.x; v[1] = r.y; v[2] = r.z;
        break;
      }
      case SENS_ACTUATORFRC: v[0] = d.actuator_force()[id]; break;
      case SENS_JOINTACTFRC: v[0] = d.qfrc_actuator()[m.jnt_dofadr[id]]; break;
      case SENS_JOINTLIMITFRC: { const int j = limit_row(CNSTR_LIMIT_JOINT); if (j >= 0) v[0] = d.efc_force()[j]; break; }
      case SENS_TENDONLIMITFRC: { const int j = limit_row(CNSTR_LIMIT_TENDON); if (j >= 0) v[0] = d.efc_force()[j]; break; }
      default: break;
    }
    const int cm = m.sensor_cutmode[i];
    const double cut = m.sensor_cutoff[i];
    for (int k = 0; k < dim && k < 4; k++) {
      double x = v[k];
      if (cm == 1) x = dclip(x, -cut, cut);
      else if (cm == 2) x = dmin(cut, x);
      out[adr + k] = x;
    }
  }
  MJB_PSYNC();
}

// the history part of mj_advance (engine_forward.c:1265-1312), at the current time and before the state moves: the
// control of every actuator with a buffer is recorded, then the sensor samples (sensors, advance = true)
MJB_HD void history_advance(const Env& d) {
  const DModel& m = d.m;
  MJB_PFOR(i, m.sz.nu) {
    const int n = m.actuator_history[2 * i];
    if (n > 0) hist_insert(d.history() + m.actuator_historyadr[i], n, 1, d.time()[0])[0] = d.ctrl()[i];
  }
  MJB_PSYNC();
  sensors(d, true);
}

// explicit Runge-Kutta 4 (mj_RungeKutta, engine_forward.c:1486-1591) split into phases around the
// forward passes, which are separate launches of the fused kernel:
//   phase 1..3 (after forward #phase-1): record F[phase-1] = qacc, form X[phase] = X[0] (+) h*dX with the
//              tableau row A[phase-1], install it as the state at time T[phase-1]
//   phase 4    (after forward #3): record F[3], combine with B, restore X[0] and advance (mj_advance)
// rk_scr layout: x0 qpos[nq] | x0 qvel[nv] | X[1..3] qvel [3 nv] | F[0..3] [4 nv] | t0
MJB_HD void rk4_phase(const Env& d, int phase) {
  const DModel& m = d.m;
  const int nq = m.sz.nq, nv = m.sz.nv;
  const double h = m.opt.timestep;
  FD scr = d.rk_scr();
  FD x0q = scr, x0v = scr + nq, xv = scr + nq + nv, F = scr + nq + 4 * nv, t0 = scr + nq + 8 * nv;
  FD dXv = d.scr_nv(), dXa = d.scr_nv() + nv, dXact = d.scr_nv() + 2 * nv;
  FD qpos = d.qpos(), qvel = d.qvel(), qacc = d.qacc();
  // activations ride along as extra state (X) with act_dot as their derivative (F)
  const int na = (d.feat & FEAT_ACT) ? m.sz.na : 0;
  FD x0a = scr + nq + 8 * nv + 4, Fa = x0a + na;   // Fa[4][na]
  FD act = d.act(), act_dot = d.act_dot();
  const double A[9] = {0.5, 0, 0, 0, 0.5, 0, 0, 0, 1};
  const double B[4] = {1.0 / 6.0, 1.0 / 3.0, 1.0 / 3.0, 1.0 / 6.0};
  if (phase == 1) {
    MJB_PFOR(i, nq) x0q[i] = qpos[i];
    MJB_PFOR(i, nv) x0v[i] = qvel[i];
    MJB_PFOR(i, na) x0a[i] = act[i];
    MJB_LANE0 t0[0] = d.time()[0];
  }
  MJB_PFOR(i, nv) F[(phase - 1) * nv + i] = qacc[i];
  MJB_PFOR(i, na) Fa[(phase - 1) * na + i] = act_dot[i];
  MJB_PSYNC();
#ifdef MJB_HISTORY_CODE
  if ((d.feat & FEAT_HISTORY) && phase == 4) {   // mj_advance runs on the restored X[0] and time, stage-4 derived quantities
    MJB_PFOR(i, nq) qpos[i] = x0q[i];
    MJB_PFOR(i, nv) qvel[i] = x0v[i];
    MJB_PFOR(i, na) act[i] = x0a[i];
    MJB_LANE0 d.time()[0] = t0[0];
    MJB_PSYNC();
    history_advance(d);
  }
#endif
  auto Xv = [&](int j, int i) { return j == 0 ? x0v[i] : xv[(j - 1) * nv + i]; };
  if (phase < 4) {
    MJB_PFOR(i, nv) {
      double sv = 0, sa = 0;
      for (int j = 0; j < phase; j++) {
        const double a = A[(phase - 1) * 3 + j];
        sv += Xv(j, i) * a;
        sa += F[j * nv + i] * a;
      }
      dXv[i] = sv; dXa[i] = sa;
    }
    MJB_PFOR(i, na) {
      double sa = 0;
      for (int j = 0; j < phase; j++) sa += Fa[j * na + i] * A[(phase - 1) * 3 + j];
      act[i] = x0a[i] + sa * h;
    }
    MJB_PFOR(i, nq) qpos[i] = x0q[i];
    MJB_PSYNC();
    integrate_pos(d, qpos, dXv, h);
    MJB_PFOR(i, nv) {
      const double v = x0v[i] + dXa[i] * h;
      qvel[i] = v;
      xv[(phase - 1) * nv + i] = v;
    }
    MJB_LANE0 {
      double c = 0;
      for (int j = 0; j < phase; j++) c += A[(phase - 1) * 3 + j];
      d.time()[0] = t0[0] + c * h;
    }
    MJB_PSYNC();
  } else {
    MJB_PFOR(i, nv) {
      double sv = 0, sa = 0;
      for (int j = 0; j < 4; j++) { sv += Xv(j, i) * B[j]; sa += F[j * nv + i] * B[j]; }
      dXv[i] = sv; dXa[i] = sa;
    }
    MJB_PFOR(i, na) {
      double sa = 0;
      for (int j = 0; j < 4; j++) sa += Fa[j * na + i] * B[j];
      dXact[i] = sa;
      act[i] = x0a[i];
    }
    MJB_PFOR(i, nq) qpos[i] = x0q[i];
    MJB_PSYNC();
    if (na) advance_act(d, dXact);
    MJB_PFOR(i, nv) qvel[i] = x0v[i] + dXa[i] * h;
    integrate_pos(d, qpos, dXv, h);
    FD ws = d.qacc_warmstart();
    MJB_PFOR(i, nv) ws[i] = qacc[i];
    MJB_LANE0 d.time()[0] = t0[0] + h;
    MJB_PSYNC();
  }
}

}  // namespace mjb
