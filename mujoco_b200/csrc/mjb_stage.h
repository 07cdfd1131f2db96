// Per-environment bodies of the launchable operations; shared verbatim by the CUDA kernels
// (mjb_kernels.cu) and the test-only host emulation (tests/hostemu/hostemu_backend.cc).
#pragma once
#include "mjb_forward.h"

namespace mjb {

MJB_HD bool env_has_warning(const Env& d) {
  FI w = d.warning();
  for (int i = 0; i < NWARNING; i++) if (w[i]) return true;
  return false;
}

// stage mask bits: 1<<stage.  forward = stages 0,1,2,4 ; step = stages 0,1,2,3
constexpr int kMaskStep = 0xF, kMaskForward = 0x17;

// run the selected stages of one environment with its cooperative lanes.
// flags: bit0 = part of mj_step (qpos/qvel checks), bit1 = skip environments that raised a warning.
// shot/sint: optional staging area (shared memory) for the hot block; only with env-major storage.
// mask bits: 1 position, 2 velocity, 4 solve, 8 finish + acceleration check + Euler, 16 finish only
// (mj_forward), 32 finish + acceleration check without integration (first forward of an RK4 step).
// mj_checkAcc (engine_forward.c:99-113): a bad acceleration resets the environment and the forward
// pass is run again before integrating; that second pass is the SAME code (one loop iteration more),
// not a second inlined copy of the pipeline.
MJB_HD void run_stage_mask(const Env& d, int mask, int flags, int first_pass = 0) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int pass = first_pass; pass < 2; pass++) {
    const bool redo = pass == 1;
    if ((mask & 1) || redo) stage_position(d, (flags & 1) != 0 && !redo);
    if ((mask & 2) || redo) stage_velocity(d);
    if ((mask & 4) || redo) stage_solve(d);
    if (mask & (8 | 16 | 32)) { stage_finish_forward(d); energy(d); if ((d.feat & FEAT_SENSOR) && !(flags & 8)) sensors(d); }
    if (!(mask & (8 | 32))) return;
    if (!redo) {
      check_vec(d, d.qacc(), d.m.sz.nv, WARN_BADQACC);
      const int bad = d.scr_int()[0];
      MJB_PSYNC();
      if (bad && !(d.m.opt.disableflags & DSBL_AUTORESET)) continue;
    }
    if (mask & 8) { if ((d.feat & FEAT_IMPLICITFAST) && d.m.opt.integrator == INT_IMPLICITFAST) implicitfast_advance(d); else euler_advance(d); }
    return;
  }
}

// rollout rule (rollout.cc:127-155): an environment that carries a warning when a step BEGINS does not
// step.  flags bit1: evaluate that now (first launch of a step) and remember it in step_skip;
// flags bit2: a later launch of the same multi-launch step (RK4) reuses the remembered decision, so
// a warning raised inside the step does not cut the step short.
MJB_HD bool step_enabled(const Env& d, int flags) {
  if (flags & 2) {
    const bool skip = env_has_warning(d);
    MJB_PSYNC();
    MJB_LANE0 d.step_skip()[0] = skip ? 1 : 0;
    MJB_PSYNC();
    return !skip;
  }
  if (flags & 4) return d.step_skip()[0] == 0;
  return true;
}

// SPLIT step (the PGS solve runs as its own launch between the two parts, mjb_pgs4.cu):
//   part 1: position + velocity stages (constraint_begin included);
//   part 2: dual finish + acceleration check + integration.  A bad acceleration only MARKS the environment
//           (step_skip = 2); the redo launch of the fused kernel (flags bit4, below) then repeats the forward
//           pass on the reset state and integrates - mj_checkAcc + mj_forward, engine_forward.c:99-113 - so
//           that neither part has to carry the whole pipeline.
MJB_HD void run_part(const Env& d, int part, int flags) {
  if (part == 1) {
    stage_position(d, (flags & 1) != 0);
    stage_velocity(d);
    return;
  }
  stage_finish_forward(d);
  energy(d);
  if ((d.feat & FEAT_SENSOR) && !(flags & 8)) sensors(d);
  check_vec(d, d.qacc(), d.m.sz.nv, WARN_BADQACC);
  const int bad = d.scr_int()[0];
  MJB_PSYNC();
  if (bad && !(d.m.opt.disableflags & DSBL_AUTORESET)) {
    MJB_LANE0 d.step_skip()[0] = 2;
    MJB_PSYNC();
    return;
  }
  MJB_PROF_BEGIN
  if ((d.feat & FEAT_IMPLICITFAST) && d.m.opt.integrator == INT_IMPLICITFAST) implicitfast_advance(d); else euler_advance(d);
  MJB_PROF_MARK(10)
}

// run the selected stages of one environment with its cooperative lanes.
// flags: bit0 = part of mj_step (qpos/qvel checks), bit1/bit2 = rollout skip rule (step_enabled),
// bit4 = redo launch of a split step: only environments marked by part 2 (step_skip == 2) run, from the
// second pass of run_stage_mask (forward on the reset state, then integration).
// part: 0 = stages by mask (fused), 1 / 2 = parts of the split step.
// sm/smcap: optional per-warp shared-memory scratch (doubles) used by the latency-critical loops.
MJB_HD void run_env(const DModel& m, const Batch& b, int e, int mask, int flags, int lane, int nlane,
                    double* sm, int smcap, int solver = -1, unsigned lanes = 0xffffffffu, int feat = FEAT_ALL,
                    int part = 0) {
  Env d(m, b, e, lane, nlane);
#if !defined(__CUDA_ARCH__)
  // a host compilation of this code (the emulation of the device path) is one build for every model: a model with
  // convex collision pairs takes the convex narrow phase there too, and one with spatial tendons their paths.  Device
  // kernels fix their features per instantiation instead (FEAT_CONVEX only in mjb_kstep_convex32.cu, FEAT_SPATIAL
  // only in mjb_kstep_spatial32.cu).
  if (m.sz.convex) feat |= FEAT_CONVEX;
  if (m.sz.spatial) feat |= FEAT_SPATIAL;
  if (m.sz.nhistory) feat |= FEAT_HISTORY;
#endif
  d.sm = sm; d.smcap = smcap; d.mask = lanes; d.feat = feat;
  d.solver = solver < 0 ? m.opt.solver : solver;
  if (flags & 16) {
    const bool marked = d.step_skip()[0] == 2;
    MJB_PSYNC();
    if (!marked) return;
    MJB_LANE0 d.step_skip()[0] = 0;
    MJB_PSYNC();
    run_stage_mask(d, kMaskStep, flags, 1);
    return;
  }
  if (!step_enabled(d, flags)) return;
  if (part) run_part(d, part, flags);
  else run_stage_mask(d, mask, flags);
}

// one phase of the Runge-Kutta step (between forward launches); models with history buffers take the FEAT_HISTORY
// instantiation (mjb_kstep_history32.cu), whose last phase runs the history part of mj_advance
MJB_HD void run_rk4(const DModel& m, const Batch& b, int e, int phase, int flags, int lane, int nlane, int feat = FEAT_ALL) {
  Env d(m, b, e, lane, nlane);
#if !defined(__CUDA_ARCH__)
  if (m.sz.nhistory) feat |= FEAT_HISTORY;
#endif
  d.feat = feat;
  d.solver = m.opt.solver;
  if (!step_enabled(d, flags)) return;
  rk4_phase(d, phase);
}

// control [nenv][nstep][ncontrol] (reference layout): segments ctrl then qfrc_applied by spec bits
// skip_warned: the rollout rule (rollout.cc:127-155) - an environment that carries a warning no longer steps, so
// its controls are not written either.  Per-step callers (mjb_step_host) always write the controls.
MJB_HD void run_set_control(const DModel& m, const Batch& b, int e, const double* control, int nstep, int t,
                            unsigned spec, int ncontrol, bool skip_warned = true) {
  Env d(m, b, e);
  if (skip_warned && env_has_warning(d)) return;
  const double* src = control + ((size_t)e * nstep + t) * ncontrol;
  int k = 0;
  if (spec & (1u << 6)) { FD c = d.ctrl(); for (int i = 0; i < m.sz.nu; i++) c[i] = src[k++]; }
  if (spec & (1u << 7)) { FD q = d.qfrc_applied(); for (int i = 0; i < m.sz.nv; i++) q[i] = src[k++]; }
  if (spec & (1u << 8)) { FD q = d.xfrc_applied(); for (int i = 0; i < 6 * m.sz.nbody; i++) q[i] = src[k++]; }
  if (spec & (1u << 9)) { FD q = d.eq_active(); for (int i = 0; i < m.sz.neq; i++) q[i] = src[k++]; }
  if (spec & (1u << 10)) { FD q = d.mocap_pos(); for (int i = 0; i < 3 * m.sz.nmocap; i++) q[i] = src[k++]; }
  if (spec & (1u << 11)) { FD q = d.mocap_quat(); for (int i = 0; i < 4 * m.sz.nmocap; i++) q[i] = src[k++]; }
}

// state [nenv][nstep][nstate] = (time, qpos, qvel, act, history)  (mjSTATE_FULLPHYSICS)
MJB_HD void run_get_state(const DModel& m, const Batch& b, int e, double* state, int nstep, int t, int nstate) {
  Env d(m, b, e);
  double* dst = state + ((size_t)e * nstep + t) * nstate;
  int k = 0;
  dst[k++] = d.time()[0];
  FD qp = d.qpos(), qv = d.qvel();
  for (int i = 0; i < m.sz.nq; i++) dst[k++] = qp[i];
  for (int i = 0; i < m.sz.nv; i++) dst[k++] = qv[i];
  for (int i = 0; i < m.sz.na; i++) dst[k++] = d.act()[i];
  for (int i = 0; i < m.sz.nhistory; i++) dst[k++] = d.history()[i];
}

// sensordata [nenv][nstep][nsensordata]; a warned env repeats its last values (the reference pads likewise)
MJB_HD void run_get_sensor(const DModel& m, const Batch& b, int e, double* sens, int nstep, int t, int nsens) {
  Env d(m, b, e);
  double* dst = sens + ((size_t)e * nstep + t) * nsens;
  FD sd = d.sensordata();
  for (int i = 0; i < nsens; i++) dst[i] = sd[i];
}

// native layouts: ctrl [nstep][nu][stride], state [nstep][nstate][stride] — coalesced across envs
MJB_HD void run_set_control_native(const DModel& m, const Batch& b, int e, const double* ctrl, int t) {
  Env d(m, b, e);
  FD c = d.ctrl();
  const double* src = ctrl + (size_t)t * m.sz.nu * b.stride + e;
  for (int i = 0; i < m.sz.nu; i++) c[i] = src[(size_t)i * b.stride];
}
MJB_HD void run_get_state_native(const DModel& m, const Batch& b, int e, double* state, int t, int nstate) {
  Env d(m, b, e);
  double* dst = state + (size_t)t * nstate * b.stride + e;
  int k = 0;
  dst[(size_t)(k++) * b.stride] = d.time()[0];
  FD qp = d.qpos(), qv = d.qvel();
  for (int i = 0; i < m.sz.nq; i++) dst[(size_t)(k++) * b.stride] = qp[i];
  for (int i = 0; i < m.sz.nv; i++) dst[(size_t)(k++) * b.stride] = qv[i];
  for (int i = 0; i < m.sz.na; i++) dst[(size_t)(k++) * b.stride] = d.act()[i];
  for (int i = 0; i < m.sz.nhistory; i++) dst[(size_t)(k++) * b.stride] = d.history()[i];
}

// dense [nenv][cnt] <-> field of either layout; idx enumerates (env, elem)
MJB_HD void run_pack(const Batch& b, int is_int, long off, long cnt, void* dense, int to_dense, long idx) {
  const long e = idx / cnt, i = idx - e * cnt;
  if (is_int) {
    int* f = b.itg + (size_t)e * b.ipitch + (size_t)(off + i);
    int* dn = (int*)dense + idx;
    if (to_dense) *dn = *f; else *f = *dn;
  } else {
    double* f = b.dbl + (size_t)e * b.dpitch + (size_t)(off + i);
    double* dn = (double*)dense + idx;
    if (to_dense) *dn = *f; else *f = *dn;
  }
}
MJB_HD void run_fill_zero(const Batch& b, int is_int, long off, long cnt, long idx) {
  const long e = idx / cnt, i = idx - e * cnt;
  if (is_int) b.itg[(size_t)e * b.ipitch + (size_t)(off + i)] = 0;
  else b.dbl[(size_t)e * b.dpitch + (size_t)(off + i)] = 0;
}

}  // namespace mjb
