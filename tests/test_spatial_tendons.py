"""Spatial tendons (site paths, sphere and cylinder wrapping, pulleys, the tendon-armature bias) against the reference
engine.

Fixtures (tests/golden/make_tendon_fixtures.py): models/tendon_paths.xml, authored here, and the reference's
tendon_arm/arm26.xml (muscles on cylinder-wrapped tendons) and replicate/newton_cradle.xml (site-to-site tendons on
free bodies).  CPU tests: the kernel source compiled for the host (tests/hostemu) reproduces the oracle bit for bit.
GPU tests: libmjb200 on the device against the oracle; the device's acos / asin / sqrt are not the host's, so fields
are held to 1e-9 and rollouts are re-synchronised on the device state every step."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import mujoco_b200 as mb
from mjb_util import HOSTEMU, HUMANOID, ROOT, compare_forward, hostemu_lib, make_pair
from oracle_util import Oracle, available

GOLDEN = os.path.join(ROOT, "tests", "golden")
PATHS = os.path.join(GOLDEN, "tendon_paths.mjb")
ARM26 = os.path.join(GOLDEN, "arm26.mjb")
CRADLE = os.path.join(GOLDEN, "newton_cradle.mjb")
FIXTURES = {"tendon_paths": PATHS, "arm26": ARM26, "newton_cradle": CRADLE}
WRAP_INTS = ("ten_wrapadr", "ten_wrapnum", "wrap_obj")
WRAP_SPHERE, WRAP_CYLINDER = 4, 5
CNSTR_FRICTION_TENDON, CNSTR_LIMIT_TENDON = 2, 4

needs_hostemu = pytest.mark.skipif(not (available() and os.path.exists(HOSTEMU)), reason="oracle or hostemu not built")


def states_for(o, nenv, seed):
    """seeded states around the model's reset state: scalar joints moved and spun; free bodies shifted, spun and
    thrown (quaternions unnormalised on purpose: the engine normalises)"""
    rng = np.random.default_rng(seed)
    o.reset()
    s0 = np.tile(o.get_state(), (nenv, 1))
    nq, nv = o.size("nq"), o.size("nv")
    jt, qa, da = o.mfield("jnt_type"), o.mfield("jnt_qposadr"), o.mfield("jnt_dofadr")
    for e in range(nenv):
        for j in range(o.size("njnt")):
            q, v = 1 + qa[j], 1 + nq + da[j]
            if jt[j] == 0:     # free: small shift, random orientation, velocity
                s0[e, q:q + 2] += rng.uniform(-0.05, 0.05, 2)
                s0[e, q + 3:q + 7] += rng.normal(0, 0.3, 4)
                s0[e, v:v + 6] = rng.normal(0, 0.8, 6)
            elif jt[j] in (2, 3):
                s0[e, q] += rng.uniform(-1.2, 1.2) if jt[j] == 3 else rng.uniform(-0.01, 0.01)
                s0[e, v] = rng.normal(0, 2.0)
    return s0


def controls_for(o, nenv, nstep, seed):
    rng = np.random.default_rng(seed + 1000)
    rng_lo, rng_hi = o.mfield("actuator_ctrlrange").reshape(-1, 2).T if o.size("nu") else (np.zeros(0), np.zeros(0))
    return rng.uniform(rng_lo, rng_hi, (nenv, nstep, o.size("nu")))


def oracle_at(o, state, ctrl):
    o.reset()
    o.set_state(state)
    o.dfield("ctrl")[:] = ctrl
    o.forward()


def compare_wrap(b, o, states, ctrl, exact=True, rtol=0.0):
    """the path points after mj_forward: ten_wrapadr / ten_wrapnum / wrap_obj exact, wrap_xpos over the points in use"""
    got = {f: b.field(f) for f in WRAP_INTS}
    gx = b.field("wrap_xpos")
    for e in range(states.shape[0]):
        oracle_at(o, states[e], ctrl[e])
        n = int(np.sum(o.dfield("ten_wrapnum")))
        for f in ("ten_wrapadr", "ten_wrapnum"):
            assert np.array_equal(got[f][e], o.dfield(f)), (f, e, got[f][e], o.dfield(f))
        assert np.array_equal(got["wrap_obj"][e, :n], np.array(o.dfield("wrap_obj")).reshape(-1)[:n]), (e, got["wrap_obj"][e, :n])
        a, r = gx[e, :3 * n], np.array(o.dfield("wrap_xpos")).reshape(-1)[:3 * n]
        if exact:
            assert np.array_equal(a, r), ("wrap_xpos", e, np.abs(a - r).max())
        else:
            assert np.abs(a - r).max() <= rtol * max(1.0, np.abs(r).max()), ("wrap_xpos", e)


class Coverage:
    """what the forward passes of a test reached: path shapes, constraint rows, islands, the armature bias"""

    def __init__(self, o):
        self.o = o
        self.seen = set()
        self.wrapnum = {}

    def add(self, b, states, ctrl):
        o = self.o
        wt, wid = o.mfield("wrap_type"), o.mfield("wrap_objid")
        cyl = {int(wid[k]) for k in range(len(wt)) if wt[k] == WRAP_CYLINDER}
        obj, num = b.field("wrap_obj"), b.field("ten_wrapnum")
        etype, nefc = b.field("efc_type"), b.field("nefc")[:, 0]
        nisland = b.field("nisland")[:, 0]
        for e in range(states.shape[0]):
            n = int(num[e].sum())
            if (obj[e, :n] == -2).any():
                self.seen.add("pulley")
            if cyl & set(obj[e, :n].tolist()):
                self.seen.add("cylinder")
            for i, k in enumerate(num[e]):
                self.wrapnum.setdefault(i, set()).add(int(k))
            t = etype[e, :nefc[e]]
            if (t == CNSTR_LIMIT_TENDON).any():
                self.seen.add("tendon_limit")
            if (t == CNSTR_FRICTION_TENDON).any():
                self.seen.add("tendon_friction")
            if nisland[e] < o.size("ntree"):
                self.seen.add("islands_merged")
        # the tendon-armature bias: qfrc_bias of the oracle with and without the armature of the tendons
        for e in range(states.shape[0]):
            oracle_at(o, states[e], ctrl[e])
            with_arm = np.array(o.dfield("qfrc_bias"))
            ta, aa = o.mfield("tendon_armature"), o.mfield("actuator_armature")
            keep = ta.copy(), aa.copy()
            ta[:], aa[:] = 0, 0
            oracle_at(o, states[e], ctrl[e])
            without = np.array(o.dfield("qfrc_bias"))
            ta[:], aa[:] = keep
            if not np.array_equal(with_arm, without):
                self.seen.add("armature_bias")

    def static(self):
        """site-side geometry of the model: a side site inside its sphere, simple and non-simple segment bodies"""
        o = self.o
        wt, wid, wprm = o.mfield("wrap_type"), o.mfield("wrap_objid"), o.mfield("wrap_prm")
        simple, sbody = o.mfield("body_simple"), o.mfield("site_bodyid")
        o.reset()
        o.forward()
        sx, gx, gs = np.array(o.dfield("site_xpos")).reshape(-1, 3), np.array(o.dfield("geom_xpos")).reshape(-1, 3), o.mfield("geom_size").reshape(-1, 3)
        for k in range(len(wt)):
            if wt[k] == WRAP_SPHERE and wprm[k] >= 0:
                side, g = int(round(wprm[k])), int(wid[k])
                if np.linalg.norm(sx[side] - gx[g]) < gs[g, 0]:
                    self.seen.add("side_inside")
        adr, num = o.mfield("tendon_adr"), o.mfield("tendon_num")
        for i in range(o.size("ntendon")):
            sites = [int(wid[adr[i] + j]) for j in range(num[i]) if wt[adr[i] + j] == 3]
            for s1, s2 in zip(sites, sites[1:]):
                b1, b2 = sbody[s1], sbody[s2]
                if b1 != b2:
                    self.seen.add("simple_pair" if simple[b1] and simple[b2] else "nonsimple_pair")


# ---- host emulation, bit for bit ------------------------------------------------------------------------------------
@needs_hostemu
@pytest.mark.parametrize("solver", [mb.SOLVER_PGS, mb.SOLVER_NEWTON, mb.SOLVER_CG])
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_spatial_forward_bit_exact(fixture, solver):
    """every mjData field after mj_forward and the path points, bit for bit, along a reference rollout"""
    path = FIXTURES[fixture]
    nenv, nstep = 8, 60
    m, b, o = make_pair(path, solver, library=hostemu_lib(), nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=3)
    ctrl = controls_for(o, nenv, nstep, seed=3)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    for t in (0, 25, 59):
        compare_forward(b, o, ref[:, t, :], ctrl[:, t, :], rtol=0, exact=True, check_dual=(solver == mb.SOLVER_PGS))
        compare_wrap(b, o, ref[:, t, :], ctrl[:, t, :])


def rollout_bit_exact(path, solver, nenv=8, nstep=150, seed=7, check_every=10, coverage=None, **opts):
    m, b, o = make_pair(path, solver, library=hostemu_lib(), nenv=nenv, nconmax=48, njmax=200, **opts)
    s0 = states_for(o, nenv, seed)
    ctrl = controls_for(o, nenv, nstep, seed)
    out = b.rollout(s0, ctrl)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    assert np.array_equal(b.warnings().sum(axis=1) > 0, stats[:, 3] > 0)
    assert np.array_equal(out, ref)
    for t in range(2, nstep, check_every):
        compare_forward(b, o, ref[:, t, :], ctrl[:, t, :], rtol=0, exact=True, check_dual=(solver == mb.SOLVER_PGS))
        compare_wrap(b, o, ref[:, t, :], ctrl[:, t, :])
        if coverage is not None:
            coverage.add(b, ref[:, t, :], ctrl[:, t, :])
    return o


@needs_hostemu
@pytest.mark.parametrize("fixture,solver", [("tendon_paths", mb.SOLVER_PGS), ("tendon_paths", mb.SOLVER_NEWTON),
                                            ("arm26", mb.SOLVER_PGS), ("arm26", mb.SOLVER_NEWTON)])
def test_spatial_rollout_bit_exact(fixture, solver):
    """150-step rollouts with random controls, bit for bit, with forward passes checked along the way"""
    rollout_bit_exact(FIXTURES[fixture], solver)


@needs_hostemu
def test_newton_cradle_rollout_bit_exact():
    """the cradle (1e-4 s step, 14 limited site-to-site tendons on free bodies) with Newton"""
    rollout_bit_exact(CRADLE, mb.SOLVER_NEWTON, nenv=4, nstep=150, check_every=37)


@needs_hostemu
@pytest.mark.parametrize("variant", ["rk4", "implicitfast", "noislands", "noslip"])
def test_spatial_variants_bit_exact(variant):
    """RK4; implicitfast (tendon damping derivatives); islands off; the noslip post-solver"""
    opts = {"rk4": dict(integrator=1), "implicitfast": dict(integrator=3), "noislands": dict(disableflags=1 << 18),
            "noslip": dict(noslip_iterations=5)}[variant]
    with tempfile.TemporaryDirectory() as tmp:
        path = PATHS
        if variant == "implicitfast":   # muscle gains have no velocity derivative here: the muscle becomes affine
            o = Oracle(PATHS)
            for f in ("actuator_gaintype", "actuator_biastype"):
                o.mfield(f)[0] = 1
            o.mfield("actuator_gainprm").reshape(o.size("nu"), -1)[0, :3] = (1, 0, 0)
            o.mfield("actuator_biasprm").reshape(o.size("nu"), -1)[0, :3] = 0
            path = os.path.join(tmp, "affine.mjb")
            o.save_mjb(path)
        rollout_bit_exact(path, mb.SOLVER_NEWTON, nenv=6, nstep=100, seed=11, check_every=13, **opts)


@needs_hostemu
def test_spatial_coverage():
    """the rollouts of tendon_paths reach every branch this feature adds: a pulley, a sphere wrap both active and
    inactive, a side site inside its sphere (wrap_inside), an active cylinder wrap, simple-body and non-simple
    segments, active tendon limit and friction rows, two trees joined into one island by a tendon, and a non-zero
    tendon-armature bias"""
    o = Oracle(PATHS)
    cov = Coverage(o)
    cov.static()
    for solver in (mb.SOLVER_PGS, mb.SOLVER_NEWTON):
        rollout_bit_exact(PATHS, solver, nenv=8, nstep=150, seed=7, check_every=10, coverage=cov)
    want = {"pulley", "cylinder", "side_inside", "simple_pair", "nonsimple_pair", "tendon_limit", "tendon_friction",
            "islands_merged", "armature_bias"}
    assert want <= cov.seen, want - cov.seen
    wt, wprm, adr, num = o.mfield("wrap_type"), o.mfield("wrap_prm"), o.mfield("tendon_adr"), o.mfield("tendon_num")
    sphere_no_side = [i for i in range(o.size("ntendon"))
                      if any(wt[adr[i] + j] == WRAP_SPHERE and wprm[adr[i] + j] < 0 for j in range(num[i]))]
    assert sphere_no_side and all(len(cov.wrapnum[i]) > 1 for i in sphere_no_side), cov.wrapnum   # on and off


@needs_hostemu
def test_spatial_mj_step_symbols_and_mjdata_bridge_bit_exact():
    """mj_step / mj_step1 + mj_step2 under the reference's names, and mjb_step_mjdata, on the reference's own mjData
    of arm26: the reference's trajectory and path points step for step"""
    lib = C.CDLL(HOSTEMU)
    for name in ("mj_step", "mj_step1", "mj_step2"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p]
        getattr(lib, name).restype = None
    lib.mjb_forget_model.argtypes = [C.c_void_p]
    ref, ours = Oracle(ARM26), Oracle(ARM26)
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
        assert np.array_equal(np.array(ref.dfield("ten_length")), np.array(ours.dfield("ten_length")))
    lib.mjb_forget_model(ours.m)

    nenv = 3
    ref = [Oracle(ARM26) for _ in range(nenv)]
    ours = [Oracle(ARM26) for _ in range(nenv)]
    m = mb.Model(ARM26, library=hostemu_lib())
    b = mb.Batch(m, nenv)
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
            n = int(np.sum(ref[e].dfield("ten_wrapnum")))
            for f in ("ten_length", "qfrc_bias", "qfrc_passive", "actuator_force", "ten_wrapadr", "ten_wrapnum"):
                assert np.array_equal(np.array(ref[e].dfield(f)), np.array(ours[e].dfield(f))), (t, e, f)
            assert np.array_equal(np.array(ref[e].dfield("wrap_obj")).reshape(-1)[:n],
                                  np.array(ours[e].dfield("wrap_obj")).reshape(-1)[:n]), (t, e)
            assert np.array_equal(np.array(ref[e].dfield("wrap_xpos")).reshape(-1)[:3 * n],
                                  np.array(ours[e].dfield("wrap_xpos")).reshape(-1)[:3 * n]), (t, e)


SPATIAL_CONVEX = """<mujoco>
  <worldbody>
    <geom type="plane" size="1 1 0.1"/>
    <site name="top" pos="0 0 1"/>
    <body pos="0 0 0.3"><freejoint/><geom type="ellipsoid" size="0.1 0.08 0.05"/><site name="s"/></body>
  </worldbody>
  <tendon><spatial limited="true" range="0 1"><site site="top"/><site site="s"/></spatial></tendon>
</mujoco>"""


@needs_hostemu
def test_spatial_tendons_with_convex_pairs_refused():
    """no kernel carries both spatial tendons and the convex narrow phase: such a model is refused with a reason"""
    with tempfile.TemporaryDirectory() as tmp:
        xml, mjb = os.path.join(tmp, "m.xml"), os.path.join(tmp, "m.mjb")
        with open(xml, "w") as f:
            f.write(SPATIAL_CONVEX)
        Oracle(xml).save_mjb(mjb)
        m = mb.Model(mjb, library=hostemu_lib())
        with pytest.raises(mb.MjbError) as err:
            mb.Batch(m, 2)
    assert "spatial tendons" in str(err.value) and "convex" in str(err.value)


@needs_hostemu
def test_spatial_layout_of_other_models_unchanged():
    """models without spatial tendons allocate no path fields"""
    m = mb.Model(HUMANOID, library=hostemu_lib())
    b = mb.Batch(m, 2)
    for f in WRAP_INTS + ("wrap_xpos",):
        assert b.field_size(f) == 0, f


# ---- on the device ---------------------------------------------------------------------------------------------------
RTOL_TIGHT = 1e-9
GPU_CASES = [("tendon_paths", mb.SOLVER_PGS, True), ("tendon_paths", mb.SOLVER_NEWTON, True),
             ("tendon_paths", mb.SOLVER_CG, True), ("tendon_paths", mb.SOLVER_NEWTON, False),
             ("arm26", mb.SOLVER_PGS, True), ("arm26", mb.SOLVER_NEWTON, False),
             ("newton_cradle", mb.SOLVER_NEWTON, True), ("newton_cradle", mb.SOLVER_PGS, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("fixture,solver,warp_per_env", GPU_CASES)
def test_spatial_forward_gpu(fixture, solver, warp_per_env):
    """forward passes on the 32-lane and the lane-per-environment mappings: contacts, efc types / ids, solver_niter and
    the path ints exact, every field at 1e-9"""
    assert available()
    nenv, nstep = 8, 40
    m, b, o = make_pair(FIXTURES[fixture], solver, nenv=nenv, nconmax=48, njmax=200, warp_per_env=warp_per_env)
    s0 = states_for(o, nenv, seed=13)
    ctrl = controls_for(o, nenv, nstep, seed=13)
    ref, _, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1)
    for t in (0, 20, 39):
        compare_forward(b, o, ref[:, t, :], ctrl[:, t, :], rtol=RTOL_TIGHT, check_dual=(solver == mb.SOLVER_PGS))
        compare_wrap(b, o, ref[:, t, :], ctrl[:, t, :], exact=False, rtol=RTOL_TIGHT)


@pytest.mark.gpu
@pytest.mark.parametrize("fixture,solver,warp_per_env", [("tendon_paths", mb.SOLVER_PGS, True),
                                                         ("tendon_paths", mb.SOLVER_NEWTON, False),
                                                         ("arm26", mb.SOLVER_NEWTON, True)])
def test_spatial_stepwise_gpu(fixture, solver, warp_per_env):
    """each device step against the reference's mj_step started from the device's previous state and warm start"""
    nenv, nstep = 8, 60
    m, b, o = make_pair(FIXTURES[fixture], solver, nenv=nenv, nconmax=48, njmax=200, warp_per_env=warp_per_env)
    state = states_for(o, nenv, seed=17)
    ctrl = controls_for(o, nenv, nstep, seed=17)
    b.set_state(state)
    b.set_field("qacc_warmstart", 0.0)
    warm = np.zeros((nenv, o.size("nv")))
    for t in range(nstep):
        b.set_field("ctrl", ctrl[:, t])
        b.step(1)
        assert (b.warnings() == 0).all(), t
        got, gwarm, gnefc = b.get_state(), b.field("qacc_warmstart"), b.field("nefc")[:, 0]
        for e in range(nenv):
            o.reset()
            o.set_state(state[e])
            o.dfield("qacc_warmstart")[:] = warm[e]
            o.dfield("ctrl")[:] = ctrl[e, t]
            o.step()
            assert gnefc[e] == int(o.scalar("nefc")), (t, e)
            for a, r in ((got[e], o.get_state()), (gwarm[e], np.array(o.dfield("qacc_warmstart")))):
                assert np.abs(a - r).max() <= RTOL_TIGHT * max(1.0, np.abs(r).max()), (t, e)
        state, warm = got, gwarm


@pytest.mark.gpu
def test_spatial_rollout_sensordata_gpu():
    """mjb_rollout's sensordata (tendon, tendon-limit and actuator sensors) against the reference's rollout"""
    nenv, nstep = 16, 30
    m, b, o = make_pair(PATHS, mb.SOLVER_NEWTON, nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=19)
    ctrl = controls_for(o, nenv, nstep, seed=19)
    out, sens = b.rollout(s0, ctrl, return_sensordata=True)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1)
    assert stats[:, 3].sum() == 0 and (b.warnings() == 0).all()
    assert np.abs(out - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max())
    for e in (0, 7, 15):
        o.reset()
        o.set_state(s0[e])
        for t in range(nstep):
            o.dfield("ctrl")[:] = ctrl[e, t]
            o.step()
            r = np.array(o.dfield("sensordata"))
            assert np.abs(sens[e, t] - r).max() <= 1e-7 * max(1.0, np.abs(r).max()), (e, t)


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", ["tendon_paths", "arm26"])
def test_spatial_4096_envs_gpu(fixture):
    """4096 environments x 200 steps: no warning the reference does not raise itself on the same states, every
    state finite"""
    nenv, nstep = 4096, 200
    m, b, o = make_pair(FIXTURES[fixture], mb.SOLVER_NEWTON, nenv=nenv, nconmax=48, njmax=200)
    s0 = states_for(o, nenv, seed=23)
    ctrl = controls_for(o, nenv, nstep, seed=23)
    b.rollout(s0, ctrl, return_state=False)
    w = b.warnings()
    _, stats, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1, want_state=False)
    warned = set(np.nonzero(w.sum(axis=1))[0].tolist())
    assert warned <= set(np.nonzero(stats[:, 3])[0].tolist()), warned
    assert np.isfinite(b.get_state()).all()


@pytest.mark.gpu
def test_spatial_path_choice_gpu():
    """a spatial-tendon PGS batch steps with the fused kernel (no split step to profile); humanoid keeps the split
    step"""
    m = mb.Model(PATHS)
    m.set_option("solver", mb.SOLVER_PGS)
    b = mb.Batch(m, 64)
    with pytest.raises(mb.MjbError):
        b.step_profile()
    h = mb.Model(HUMANOID)
    h.set_option("solver", mb.SOLVER_PGS)
    hb = mb.Batch(h, 64)
    assert len(hb.step_profile()) == 4
