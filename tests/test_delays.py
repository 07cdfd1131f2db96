"""Actuator and sensor history buffers (delayed controls, delayed and sampled sensors) against the reference engine.

Fixture (tests/golden/make_delay_fixture.py): models/ant_delay.xml, the ant with delayed actuators of every
interpolation, a delay longer than its buffer, a delayed filter actuator and position servo, a buffer without delay,
delay-only / interval-only / interval-and-delay / buffer-only sensors, and a free ball (two islands).  CPU tests: the
kernel source compiled for the host (tests/hostemu) reproduces the oracle bit for bit, history segment included.
GPU tests: libmjb200 on the device against the oracle; buffer times and control samples exact, fields at 1e-9."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import mujoco_b200 as mb
from mjb_util import HOSTEMU, HUMANOID, ROOT, compare_forward, hostemu_lib, make_pair, perturbed_states
from oracle_util import Oracle, available

DELAY = os.path.join(ROOT, "tests", "golden", "ant_delay.mjb")
MINVAL = 1e-15
DSBL_SENSOR, DSBL_ISLAND = 1 << 13, 1 << 18
RNE_FIELDS = ("cacc", "cfrc_int", "cfrc_ext")

needs_hostemu = pytest.mark.skipif(not (available() and os.path.exists(HOSTEMU)), reason="oracle or hostemu not built")


def states_for(o, nenv, seed):
    """seeded states around the reset state (history buffers as mj_resetData leaves them)"""
    return perturbed_states(o, nenv, seed, qvel_std=0.5, qpos_std=0.05)


def controls_for(o, nenv, nstep, seed):
    rng = np.random.default_rng(seed + 1000)
    lo, hi = o.mfield("actuator_ctrlrange").reshape(-1, 2).T
    return rng.uniform(lo, hi, (nenv, nstep, o.size("nu")))


def hist_offset(o):
    return 1 + o.size("nq") + o.size("nv") + o.size("na")


def oracle_forward(o, state, ctrl):
    o.reset()
    o.set_state(state)
    o.dfield("ctrl")[:] = ctrl
    o.forward()


def compare_history_forward(b, o, states, ctrl, exact=True, rtol=0.0, extra=()):
    """every hot-path field after mj_forward (compare_forward), then sensordata, the history segment and the extra
    fields named (fields of the lazy mj_rnePostConstraint / mj_subtreeVel only where the forward pass computes them)"""
    compare_forward(b, o, states, ctrl, rtol=rtol, exact=exact, check_dual=False)
    names = ("sensordata",) + tuple(extra)
    got = {f: b.field(f) for f in names}
    hist = b.get_state(mb.STATE_HISTORY)
    for e in range(states.shape[0]):
        oracle_forward(o, states[e], ctrl[e])
        assert np.array_equal(hist[e], np.array(o.dfield("history"))), e   # forward does not touch the buffers
        for f in names:
            a, r = got[f][e], np.array(o.dfield(f)).reshape(-1)
            if exact:
                assert np.array_equal(a, r), (f, e, np.abs(a - r).max())
            else:
                assert np.abs(a - r).max() <= rtol * max(1.0, np.abs(r).max()), (f, e)


# ---- branch bookkeeping: the reference's insert / read decisions, restated from a buffer in a state vector --------
def _phys(cursor, n, i):
    return (cursor + 1 + i) % n


def _find(times, n, cursor, t):
    if t <= times[_phys(cursor, n, 0)]:
        return 0
    if t > times[_phys(cursor, n, n - 1)]:
        return n
    lo, hi = 0, n - 1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if times[_phys(cursor, n, mid)] < t:
            lo = mid
        else:
            hi = mid
    return hi


def insert_branch(buf, n, t):
    cursor, times = int(buf[1]), buf[2:2 + n]
    i = _find(times, n, cursor, t)
    if i < n and abs(t - times[_phys(cursor, n, i)]) < MINVAL:
        return "match"
    return "older" if i == 0 else "newer" if i == n else "shift"


def read_branch(buf, n, t, interp):
    cursor, times = int(buf[1]), buf[2:2 + n]
    if t <= times[_phys(cursor, n, 0)] + MINVAL:
        return "clamp_old"
    if t >= times[_phys(cursor, n, n - 1)] - MINVAL:
        return "clamp_new"
    i = _find(times, n, cursor, t)
    if abs(t - times[_phys(cursor, n, i)]) < MINVAL:
        return "exact"
    if interp == 0:
        return "zoh"
    if interp == 1:
        return "linear"
    return "cubic_end" if (i <= 1 or i >= n - 1) else "cubic_mid"


def branches_of(o, state):
    """insert and read branches the step from this (pre-step) state takes"""
    seen = set()
    h = state[hist_offset(o):]
    t = state[0]
    ah, aadr, adelay = o.mfield("actuator_history").reshape(-1, 2), o.mfield("actuator_historyadr"), o.mfield("actuator_delay")
    for i in range(o.size("nu")):
        n, interp = ah[i]
        if n <= 0:
            continue
        buf = h[aadr[i]:]
        if adelay[i]:
            seen.add("read_" + read_branch(buf, n, t - adelay[i], interp))
        seen.add("insert_" + insert_branch(buf, n, t))
    sh, sadr, sdelay, sint = (o.mfield("sensor_history").reshape(-1, 2), o.mfield("sensor_historyadr"),
                              o.mfield("sensor_delay"), o.mfield("sensor_interval").reshape(-1, 2))
    for i in range(o.size("nsensor")):
        n, interp = sh[i]
        if n <= 0:
            continue
        buf = h[sadr[i]:]
        due = sint[i, 0] > 0 and buf[0] + sint[i, 0] <= t
        if sdelay[i] > 0 or (sint[i, 0] > 0 and not due):
            seen.add("read_" + read_branch(buf, n, t - sdelay[i], interp))
        if sint[i, 0] <= 0 or due:
            seen.add("insert_" + insert_branch(buf, n, t))
    return seen


def edited_times(o, s0):
    """state0 rows whose time sits on the newest control sample, half a step before it and before the oldest sample:
    the insert branches that a rollout from time 0 never takes"""
    s = s0.copy()
    dt = o.opt("timestep")
    s[1, 0] = -dt
    s[2, 0] = -1.5 * dt
    s[3, 0] = -1.0
    return s


# ---- host emulation, bit for bit ------------------------------------------------------------------------------------
def rollout_bit_exact(solver, nenv=8, nstep=150, seed=7, check_every=10, edit=True, path=DELAY, extra=("subtree_linvel",),
                      **opts):
    m, b, o = make_pair(path, solver, library=hostemu_lib(), nenv=nenv, nconmax=48, njmax=200, **opts)
    s0 = states_for(o, nenv, seed)
    if edit:
        s0 = edited_times(o, s0)
    ctrl = controls_for(o, nenv, nstep, seed)
    out = b.rollout(s0, ctrl)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    assert stats[:, 3].sum() == 0 and (b.warnings() == 0).all()
    assert np.array_equal(out, ref)
    for t in range(2, nstep, check_every):
        compare_history_forward(b, o, ref[:, t, :], ctrl[:, t, :], extra=extra)
    return o, s0, ref


@needs_hostemu
@pytest.mark.parametrize("solver", [mb.SOLVER_PGS, mb.SOLVER_NEWTON, mb.SOLVER_CG])
def test_delay_forward_bit_exact(solver):
    """every field after mj_forward, sensordata and the buffers, bit for bit, along a reference rollout"""
    nenv, nstep = 8, 60
    m, b, o = make_pair(DELAY, solver, library=hostemu_lib(), nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=3)
    ctrl = controls_for(o, nenv, nstep, seed=3)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    for t in (0, 25, 59):
        compare_history_forward(b, o, ref[:, t, :], ctrl[:, t, :], extra=("subtree_linvel",))


@needs_hostemu
@pytest.mark.parametrize("solver", [mb.SOLVER_PGS, mb.SOLVER_NEWTON, mb.SOLVER_CG])
def test_delay_rollout_bit_exact(solver):
    """150-step rollouts with random controls, the history segment of every state included, bit for bit"""
    rollout_bit_exact(solver)


@needs_hostemu
@pytest.mark.parametrize("variant", ["rk4", "implicitfast", "noislands", "nosensor"])
def test_delay_variants_bit_exact(variant):
    """RK4 (stage evaluations read delayed controls at their own times; the samples mj_advance computes mix X[0] with
    stage-4 kinematics); implicitfast (velocity derivatives from the undelayed ctrl); islands off; mjDSBL_SENSOR
    (mj_advance still computes the delayed sensors and copies the stale sensordata of the others)"""
    opts = {"rk4": dict(integrator=1), "implicitfast": dict(integrator=3), "noislands": dict(disableflags=DSBL_ISLAND),
            "nosensor": dict(disableflags=DSBL_SENSOR)}[variant]
    rollout_bit_exact(mb.SOLVER_NEWTON, nenv=6, nstep=100, seed=11, check_every=13, **opts)


ACC_DELAYED = """<mujoco>
  <option timestep="0.005"{opt}/>
  <worldbody>
    <geom type="plane" size="2 2 0.1"/>
    <body pos="0 0 0.4">
      <freejoint/>
      <geom type="box" size="0.1 0.08 0.05"/>
      <site name="s" pos="0.02 0 0.03"/>
      <body pos="0.15 0 0">
        <joint name="h" type="hinge" axis="0 1 0" damping="0.1"/>
        <geom type="capsule" size="0.03" fromto="0 0 0 0.2 0 0"/>
        <site name="t" pos="0.1 0 0"/>
      </body>
    </body>
  </worldbody>
  <actuator><motor joint="h" ctrlrange="-1 1" delay="0.01" nsample="3" interp="linear"/></actuator>
  <sensor>
    <accelerometer site="s" delay="0.0075" nsample="4" interp="cubic"/>
    <force site="t" delay="0.005" nsample="2"/>
    <framelinacc objtype="site" objname="t" delay="0.01" nsample="3" interp="linear"/>
    <subtreelinvel body="world" delay="0.005" nsample="2"/>
    <jointpos joint="h"/>
  </sensor>
</mujoco>"""


@needs_hostemu
@pytest.mark.parametrize("integrator", ["euler", "rk4"])
def test_delayed_acceleration_sensors_only(integrator):
    """every acceleration sensor delayed: cacc / cfrc_int / cfrc_ext are written by mj_advance, not by mj_forward (and
    under RK4 from the fourth stage); checked after mj_forward and after mj_step"""
    opt = ' integrator="RK4"' if integrator == "rk4" else ""
    with tempfile.TemporaryDirectory() as tmp:
        xml, path = os.path.join(tmp, "acc.xml"), os.path.join(tmp, "acc.mjb")
        with open(xml, "w") as f:
            f.write(ACC_DELAYED.format(opt=opt))
        Oracle(xml).save_mjb(path)
        o, s0, ref = rollout_bit_exact(mb.SOLVER_NEWTON, nenv=4, nstep=60, seed=5, check_every=11, edit=False, path=path,
                                       extra=())
        m = mb.Model(path, library=hostemu_lib())
        b = mb.Batch(m, 1, nconmax=48, njmax=200)
        ctrl = controls_for(o, 1, 40, seed=5)[0]
        o.reset()
        o.set_state(s0[0])
        b.set_state(s0[:1])
        for t in range(40):
            o.dfield("ctrl")[:] = ctrl[t]
            b.set_field("ctrl", ctrl[t][None])
            o.step()
            b.step(1)
            assert np.array_equal(b.get_state()[0], o.get_state()), t
            for f in RNE_FIELDS + ("subtree_linvel", "sensordata"):
                assert np.array_equal(b.field(f)[0], np.array(o.dfield(f)).reshape(-1)), (t, f)


@needs_hostemu
def test_delay_branch_coverage():
    """the rollouts reach every branch of the buffers: the four insert branches, and reads that clamp before the
    oldest and after the newest sample, match a sample exactly, and interpolate by zero-order hold, linearly, and
    cubically both next to an end of the buffer and away from the ends"""
    seen = set()
    for solver in (mb.SOLVER_PGS, mb.SOLVER_NEWTON):
        o, s0, ref = rollout_bit_exact(solver, nenv=8, nstep=150, seed=7, check_every=49)
        for e in range(s0.shape[0]):
            seen |= branches_of(o, s0[e])
            for t in range(ref.shape[1] - 1):
                seen |= branches_of(o, ref[e, t])
    want = {"insert_" + k for k in ("match", "older", "newer", "shift")} | \
        {"read_" + k for k in ("clamp_old", "clamp_new", "exact", "zoh", "linear", "cubic_end", "cubic_mid")}
    assert want <= seen, want - seen


@needs_hostemu
def test_delay_auto_reset():
    """an environment whose qvel is NaN is reset within its first step, buffers included, exactly as mj_resetData does
    (the step then goes on from the reset state, with the zero controls of the reset), and the rollout pads the rest of
    its rows as the reference does"""
    nenv, nstep = 4, 30
    m, b, o = make_pair(DELAY, mb.SOLVER_NEWTON, library=hostemu_lib(), nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=9)
    s0[2, 1 + o.size("nq") + 7] = np.nan
    ctrl = controls_for(o, nenv, nstep, seed=9)
    out = b.rollout(s0, ctrl)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    assert stats[2, 3] > 0 and b.warnings()[2].sum() > 0
    assert np.array_equal(out, ref)
    o.reset()
    o.step()
    assert np.array_equal(out[2, 0], o.get_state())
    assert np.array_equal(out[2, 0, hist_offset(o):], np.array(o.dfield("history")))


SPATIAL_HISTORY = """<mujoco>
  <worldbody>
    <site name="top" pos="0 0 1"/>
    <body pos="0 0 0.3"><joint name="z" type="slide" axis="0 0 1"/><geom type="sphere" size="0.1"/><site name="s"/></body>
  </worldbody>
  <tendon><spatial name="sp"><site site="top"/><site site="s"/></spatial></tendon>
  <actuator><motor joint="z" delay="0.004" nsample="2"/></actuator>
</mujoco>"""
CONVEX_HISTORY = """<mujoco>
  <worldbody>
    <geom type="plane" size="1 1 0.1"/>
    <body pos="0 0 0.3"><freejoint/><geom type="ellipsoid" size="0.1 0.08 0.05"/><site name="s"/></body>
  </worldbody>
  <sensor><framepos objtype="site" objname="s" delay="0.004" nsample="2"/></sensor>
</mujoco>"""


@needs_hostemu
@pytest.mark.parametrize("xml,words", [(SPATIAL_HISTORY, "spatial tendons"), (CONVEX_HISTORY, "convex")])
def test_delay_refusals(xml, words):
    """no kernel carries history buffers together with spatial tendons or convex pairs: refused with a reason"""
    with tempfile.TemporaryDirectory() as tmp:
        x, path = os.path.join(tmp, "m.xml"), os.path.join(tmp, "m.mjb")
        with open(x, "w") as f:
            f.write(xml)
        Oracle(x).save_mjb(path)
        m = mb.Model(path, library=hostemu_lib())
        with pytest.raises(mb.MjbError) as err:
            mb.Batch(m, 2)
    assert "history" in str(err.value) and words in str(err.value)


@needs_hostemu
def test_delay_layout_of_other_models_unchanged():
    """models without buffers allocate no history field and their state has no history segment"""
    m = mb.Model(HUMANOID, library=hostemu_lib())
    b = mb.Batch(m, 2)
    assert b.field_size("history") == 0
    assert b.state_size(mb.STATE_HISTORY) == 0
    d = mb.Batch(mb.Model(DELAY, library=hostemu_lib()), 2)
    assert d.field_size("history") == Oracle(DELAY).size("nhistory") == d.state_size(mb.STATE_HISTORY)


@needs_hostemu
def test_delay_mj_step_symbols_and_mjdata_bridge_bit_exact():
    """mj_step / mj_step1 + mj_step2 under the reference's names, and mjb_step_mjdata, on the reference's own mjData:
    the reference's trajectory, d->history included, step for step"""
    lib = C.CDLL(HOSTEMU)
    for name in ("mj_step", "mj_step1", "mj_step2"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p]
        getattr(lib, name).restype = None
    lib.mjb_forget_model.argtypes = [C.c_void_p]
    ref, ours = Oracle(DELAY), Oracle(DELAY)
    s0 = states_for(ref, 1, seed=5)[0]
    ctrl = controls_for(ref, 1, 60, seed=5)[0]
    for o in (ref, ours):
        o.reset()
        o.set_state(s0)
    for t in range(60):
        for o in (ref, ours):
            o.dfield("ctrl")[:] = ctrl[t]
        ref.step()
        if t % 2:
            lib.mj_step(ours.m, ours.d)
        else:
            lib.mj_step1(ours.m, ours.d)
            lib.mj_step2(ours.m, ours.d)
        assert np.array_equal(ref.get_state(), ours.get_state()), t
    lib.mjb_forget_model(ours.m)

    nenv = 3
    ref = [Oracle(DELAY) for _ in range(nenv)]
    ours = [Oracle(DELAY) for _ in range(nenv)]
    b = mb.Batch(mb.Model(DELAY, library=hostemu_lib()), nenv, nconmax=48, njmax=200)
    states = states_for(ref[0], nenv, seed=6)
    ctrl = controls_for(ref[0], nenv, 40, seed=6)
    for e in range(nenv):
        for o in (ref[e], ours[e]):
            o.reset()
            o.set_state(states[e])
    for t in range(40):
        for e in range(nenv):
            for o in (ref[e], ours[e]):
                o.dfield("ctrl")[:] = ctrl[e, t]
            ref[e].step()
        b.step_mjdata([o.d for o in ours])
        for e in range(nenv):
            assert np.array_equal(ref[e].get_state(), ours[e].get_state()), (t, e)
            for f in ("history", "sensordata", "actuator_force", "cacc"):
                assert np.array_equal(np.array(ref[e].dfield(f)), np.array(ours[e].dfield(f))), (t, e, f)


# ---- on the device ---------------------------------------------------------------------------------------------------
RTOL = 1e-9


def check_history(got, ref, o, rtol=RTOL):
    """buffer bookkeeping (user slots, cursors, times) and control samples exact; sensor samples at rtol"""
    h0 = hist_offset(o)
    exact = np.zeros(o.size("nhistory"), dtype=bool)
    ah, aadr = o.mfield("actuator_history").reshape(-1, 2), o.mfield("actuator_historyadr")
    for i in range(o.size("nu")):
        n = ah[i, 0]
        if n > 0:
            exact[aadr[i]:aadr[i] + 2 + 2 * n] = True
    sh, sadr = o.mfield("sensor_history").reshape(-1, 2), o.mfield("sensor_historyadr")
    for i in range(o.size("nsensor")):
        n = sh[i, 0]
        if n > 0:
            exact[sadr[i]:sadr[i] + 2 + n] = True
    a, r = got[..., h0:], ref[..., h0:]
    assert np.array_equal(a[..., exact], r[..., exact])
    assert np.abs(a[..., ~exact] - r[..., ~exact]).max(initial=0) <= rtol * max(1.0, np.abs(r).max())
    assert np.abs(got[..., :h0] - ref[..., :h0]).max() <= rtol * max(1.0, np.abs(ref[..., :h0]).max())


@pytest.mark.gpu
@pytest.mark.parametrize("solver,warp_per_env", [(mb.SOLVER_PGS, True), (mb.SOLVER_NEWTON, True), (mb.SOLVER_CG, True),
                                                 (mb.SOLVER_NEWTON, False), (mb.SOLVER_PGS, False)])
def test_delay_forward_gpu(solver, warp_per_env):
    """forward passes on 32 lanes and on one lane per environment: contacts, rows and solver_niter exact, the buffers
    untouched, every field (sensordata and the lazy rnePost / subtreeVel fields included) at 1e-9"""
    assert available()
    nenv, nstep = 8, 40
    m, b, o = make_pair(DELAY, solver, nenv=nenv, nconmax=48, njmax=200, warp_per_env=warp_per_env)
    s0 = edited_times(o, states_for(o, nenv, seed=13))
    ctrl = controls_for(o, nenv, nstep, seed=13)
    ref, _, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1)
    for t in (0, 20, 39):
        compare_history_forward(b, o, ref[:, t, :], ctrl[:, t, :], exact=False, rtol=RTOL, extra=("subtree_linvel",))


@pytest.mark.gpu
@pytest.mark.parametrize("solver,opts", [(mb.SOLVER_PGS, {}), (mb.SOLVER_NEWTON, {}), (mb.SOLVER_CG, {}),
                                         (mb.SOLVER_NEWTON, dict(integrator=1)), (mb.SOLVER_PGS, dict(integrator=3))])
def test_delay_stepwise_gpu(solver, opts):
    """each device step against the reference's mj_step started from the device's previous state (history segment
    included) and warm start"""
    nenv, nstep = 8, 50
    m, b, o = make_pair(DELAY, solver, nenv=nenv, nconmax=48, njmax=200, **opts)
    state = states_for(o, nenv, seed=17)
    ctrl = controls_for(o, nenv, nstep, seed=17)
    b.set_state(state)
    b.set_field("qacc_warmstart", 0.0)
    warm = np.zeros((nenv, o.size("nv")))
    for t in range(nstep):
        b.set_field("ctrl", ctrl[:, t])
        b.step(1)
        assert (b.warnings() == 0).all(), t
        got, gwarm, gsens = b.get_state(), b.field("qacc_warmstart"), b.field("sensordata")
        refs = np.zeros_like(got)
        for e in range(nenv):
            o.reset()
            o.set_state(state[e])
            o.dfield("qacc_warmstart")[:] = warm[e]
            o.dfield("ctrl")[:] = ctrl[e, t]
            o.step()
            refs[e] = o.get_state()
            rw = np.array(o.dfield("qacc_warmstart"))
            assert np.abs(gwarm[e] - rw).max() <= RTOL * max(1.0, np.abs(rw).max()), (t, e)
        check_history(got, refs, o)
        state, warm = got, gwarm


@pytest.mark.gpu
def test_delay_rollout_sensordata_and_native_state_gpu():
    """mjb_rollout's states (history segment included) and sensordata against the reference's mj_step loop; the
    native-layout states of mjb_rollout_device carry the same history segment"""
    import torch
    nenv, nstep = 16, 30
    m, b, o = make_pair(DELAY, mb.SOLVER_NEWTON, nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=19)
    ctrl = controls_for(o, nenv, nstep, seed=19)
    out, sens = b.rollout(s0, ctrl, return_sensordata=True)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1)
    assert stats[:, 3].sum() == 0 and (b.warnings() == 0).all()
    assert np.array_equal(out[..., 0], ref[..., 0])
    assert np.abs(out - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max())
    for e in (0, 7, 15):
        o.reset()
        o.set_state(s0[e])
        for t in range(nstep):
            o.dfield("ctrl")[:] = ctrl[e, t]
            o.step()
            r = np.array(o.dfield("sensordata"))
            assert np.abs(sens[e, t] - r).max() <= 1e-7 * max(1.0, np.abs(r).max()), (e, t)
    # native layout: ctrl [nstep][nu][stride], state [nstep][nstate][stride]
    stride, nstate, nu = b.env_stride(), b.state_size(), o.size("nu")
    b.set_state(s0)
    b.set_field("qacc_warmstart", 0.0)
    dc = torch.zeros((nstep, nu, stride), dtype=torch.float64, device="cuda")
    dc[:, :, :nenv] = torch.from_numpy(np.ascontiguousarray(ctrl.transpose(1, 2, 0))).cuda()
    ds = torch.zeros((nstep, nstate, stride), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    b.rollout_device(nstep, dc.data_ptr(), ds.data_ptr())
    torch.cuda.ExternalStream(b.stream()).synchronize()
    native = ds[:, :, :nenv].cpu().numpy().transpose(2, 0, 1)
    assert np.array_equal(native, out)


@pytest.mark.gpu
def test_delay_4096_envs_gpu():
    """4096 environments x 200 steps: no warning the reference does not raise itself on the same states, every state
    finite, and a sample of environments matches the reference's rollout"""
    nenv, nstep = 4096, 200
    m, b, o = make_pair(DELAY, mb.SOLVER_NEWTON, nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=23)
    ctrl = controls_for(o, nenv, nstep, seed=23)
    out = b.rollout(s0, ctrl)
    w = b.warnings()
    _, stats, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1, want_state=False)
    warned = set(np.nonzero(w.sum(axis=1))[0].tolist())
    assert warned <= set(np.nonzero(stats[:, 3])[0].tolist()), warned
    assert np.isfinite(out).all()
    pick = np.arange(0, nenv, 512)
    ref, _, _ = o.rollout(s0[pick], ctrl[pick], nthread=os.cpu_count() or 1)
    assert np.array_equal(out[pick, :, 0], ref[..., 0])
    check_history(out[pick, :50], ref[:, :50], o, rtol=1e-6)   # the first 50 steps, before contacts amplify rounding


@pytest.mark.gpu
def test_delay_path_choice_gpu():
    """a history PGS batch steps with the fused kernel (no split step to profile); humanoid keeps the split step"""
    m = mb.Model(DELAY)
    m.set_option("solver", mb.SOLVER_PGS)
    b = mb.Batch(m, 64, nconmax=48, njmax=200)
    with pytest.raises(mb.MjbError):
        b.step_profile()
    h = mb.Model(HUMANOID)
    h.set_option("solver", mb.SOLVER_PGS)
    hb = mb.Batch(h, 64)
    assert len(hb.step_profile()) == 4
