"""Convex narrow phase (native GJK / EPA, multiCCD, plane-ellipsoid) against the reference engine.

CPU tests: the kernel source compiled for the host (tests/hostemu) must reproduce the oracle bit for bit on
models/convex.xml.  GPU tests: libmjb200 on the device against the oracle, at the tolerances of the other parity
tests, and a 4096-environment run that exercises the polytope scratch at scale."""
import ctypes as C
import os

import numpy as np
import pytest

import mujoco_b200 as mb
from mjb_util import HOSTEMU, ROOT, compare_forward, hostemu_lib, make_pair
from oracle_util import available

CONVEX = os.path.join(ROOT, "tests", "golden", "convex.mjb")   # models/convex.xml, compiled by make_convex_fixture.py
NBODY = 8   # free bodies of models/convex.xml
PLANE, SPHERE, CAPSULE, ELLIPSOID, CYLINDER, BOX = 0, 2, 3, 4, 5, 6
# the nine pair types (lower geom type first) the convex narrow phase adds
NEW_PAIRS = {(PLANE, ELLIPSOID), (SPHERE, ELLIPSOID), (CAPSULE, ELLIPSOID), (ELLIPSOID, ELLIPSOID),
             (ELLIPSOID, CYLINDER), (ELLIPSOID, BOX), (CAPSULE, CYLINDER), (CYLINDER, CYLINDER), (CYLINDER, BOX)}
# pairs multiCCD may add points to (neither geom a sphere or an ellipsoid)
MULTI_PAIRS = {(CAPSULE, CYLINDER), (CYLINDER, CYLINDER), (CYLINDER, BOX)}

needs_hostemu = pytest.mark.skipif(not (available() and os.path.exists(HOSTEMU)), reason="oracle or hostemu not built")


def pile_states(o, nenv, seed):
    """the free bodies of the pile at random extra heights, orientations and velocities"""
    rng = np.random.default_rng(seed)
    o.reset()
    s0 = np.tile(o.get_state(), (nenv, 1))
    nq = o.size("nq")
    for e in range(nenv):
        for k in range(NBODY):
            s0[e, 1 + 7 * k:1 + 7 * k + 2] += rng.uniform(-0.03, 0.03, 2)
            s0[e, 1 + 7 * k + 2] += rng.uniform(-0.01, 0.15)
            s0[e, 1 + 7 * k + 3:1 + 7 * k + 7] = rng.normal(size=4)
        s0[e, 1 + nq:] = rng.normal(0, 1.0, o.size("nv"))
    return s0


def contact_types(b, o):
    """set of (geom_type1, geom_type2) in the batch's current contact lists, and the largest contact count of a pair"""
    g1, g2, nc = b.field("con_geom1"), b.field("con_geom2"), b.field("ncon")[:, 0]
    gt = o.mfield("geom_type")
    types, most = set(), 0
    for e in range(g1.shape[0]):
        per = {}
        for c in range(nc[e]):
            key = (int(g1[e, c]), int(g2[e, c]))
            per[key] = per.get(key, 0) + 1
            types.add((int(gt[key[0]]), int(gt[key[1]])))
        for (a, z), n in per.items():
            if (int(gt[a]), int(gt[z])) in MULTI_PAIRS:
                most = max(most, n)
    return types, most


def rollout_bit_exact(solver, nenv=12, nstep=150, seed=7, check_every=5, **opts):
    m, b, o = make_pair(CONVEX, solver, library=hostemu_lib(), nenv=nenv, nconmax=64, njmax=320, **opts)
    s0 = pile_states(o, nenv, seed)
    ctrl = np.zeros((nenv, nstep, 0))
    out = b.rollout(s0, ctrl)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=4)
    assert stats[:, 3].sum() == 0 and (b.warnings() == 0).all()
    assert np.array_equal(out, ref)
    types, most = set(), 0
    for t in range(2, nstep, check_every):
        compare_forward(b, o, ref[:, t, :], np.zeros((nenv, 0)), rtol=0, exact=True, check_dual=(solver == mb.SOLVER_PGS))
        tt, mm = contact_types(b, o)
        types |= tt
        most = max(most, mm)
    return types, most


@needs_hostemu
@pytest.mark.parametrize("solver", [mb.SOLVER_PGS, mb.SOLVER_NEWTON, mb.SOLVER_CG])
def test_convex_forward_bit_exact(solver):
    """every mjData field after mj_forward, bit for bit, on piles that put the new pair types in contact"""
    m, b, o = make_pair(CONVEX, solver, library=hostemu_lib(), nenv=12, nconmax=64, njmax=320)
    s0 = pile_states(o, 12, seed=2)
    ref, _, _ = o.rollout(s0, np.zeros((12, 60, 0)), nthread=4)
    for t in (0, 20, 40, 59):
        compare_forward(b, o, ref[:, t, :], np.zeros((12, 0)), rtol=0, exact=True, check_dual=(solver == mb.SOLVER_PGS))


@needs_hostemu
@pytest.mark.parametrize("solver", [mb.SOLVER_NEWTON, mb.SOLVER_PGS])
def test_convex_rollout_bit_exact_covers_all_pairs(solver):
    """150-step rollouts of perturbed piles bit for bit; over the rollout every one of the nine new pair types makes
    contact, and multiCCD finds more than one point for some pair"""
    types, most = rollout_bit_exact(solver)
    assert NEW_PAIRS <= types, NEW_PAIRS - types
    assert most > 1


@needs_hostemu
@pytest.mark.parametrize("variant", ["nomulticcd", "epa_cap", "rk4", "implicitfast", "noislands"])
def test_convex_variants_bit_exact(variant):
    """mjDSBL_MULTICCD; a small iteration cap with a loose tolerance (EPA stops at its cap); RK4; implicitfast;
    islands off (the model's eight free bodies otherwise solve as constraint islands)"""
    opts = {"nomulticcd": dict(disableflags=1 << 19), "epa_cap": dict(ccd_iterations=5, ccd_tolerance=1e-3),
            "rk4": dict(integrator=1), "implicitfast": dict(integrator=3), "noislands": dict(disableflags=1 << 18)}[variant]
    types, most = rollout_bit_exact(mb.SOLVER_NEWTON, nenv=8, nstep=100, seed=11, check_every=9, **opts)
    assert len(types & NEW_PAIRS) >= 6
    if variant == "nomulticcd":
        assert most <= 1


@needs_hostemu
def test_convex_mj_step_symbols_and_mjdata_bridge_bit_exact():
    """mj_step / mj_step1 + mj_step2 under the reference's names, and mjb_step_mjdata, on the reference's own mjData
    of the convex model: the reference's trajectory step for step"""
    from oracle_util import Oracle
    lib = C.CDLL(HOSTEMU)
    for name in ("mj_step", "mj_step1", "mj_step2"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p]
        getattr(lib, name).restype = None
    lib.mjb_forget_model.argtypes = [C.c_void_p]
    ref, ours = Oracle(CONVEX), Oracle(CONVEX)
    s0 = pile_states(ref, 1, seed=5)[0]
    for o in (ref, ours):
        o.reset()
        o.set_state(s0)
    for t in range(60):
        ref.step()
        if t % 2:
            lib.mj_step(ours.m, ours.d)
        else:
            lib.mj_step1(ours.m, ours.d)
            lib.mj_step2(ours.m, ours.d)
        assert np.array_equal(ref.get_state(), ours.get_state()), t
        assert np.array_equal(np.array(ref.dfield("qfrc_constraint")), np.array(ours.dfield("qfrc_constraint")))
    lib.mjb_forget_model(ours.m)

    nenv = 3
    ref = [Oracle(CONVEX) for _ in range(nenv)]
    ours = [Oracle(CONVEX) for _ in range(nenv)]
    m = mb.Model(CONVEX, library=hostemu_lib())
    b = mb.Batch(m, nenv, nconmax=64, njmax=320)
    states = pile_states(ref[0], nenv, seed=6)
    for e in range(nenv):
        for o in (ref[e], ours[e]):
            o.reset()
            o.set_state(states[e])
    for t in range(40):
        for e in range(nenv):
            ref[e].step()
        b.step_mjdata([o.d for o in ours])
        for e in range(nenv):
            assert np.array_equal(ref[e].get_state(), ours[e].get_state()), (t, e)
            for f in ("qacc", "qfrc_constraint", "geom_xpos"):
                assert np.array_equal(np.array(ref[e].dfield(f)), np.array(ours[e].dfield(f))), (t, e, f)


@needs_hostemu
def test_nativeccd_disabled_is_refused():
    """the libccd path (mjDSBL_NATIVECCD) is not built: a convex model with that flag is refused, naming it"""
    m = mb.Model(CONVEX, library=hostemu_lib())
    m.set_option("disableflags", 1 << 17)
    with pytest.raises(Exception) as err:
        mb.Batch(m, 2)
    assert "NATIVECCD" in str(err.value)


# ---- on the device ---------------------------------------------------------------------------------------------------
RTOL_TRAJ = 1e-6      # rollout bound over 120 steps
RTOL_TIGHT = 1e-9     # fields, and rollouts over the first 30 steps


@pytest.mark.gpu
@pytest.mark.parametrize("solver,warp_per_env", [(mb.SOLVER_PGS, True), (mb.SOLVER_NEWTON, True), (mb.SOLVER_CG, True),
                                                 (mb.SOLVER_NEWTON, False)])
def test_convex_colliders_gpu(solver, warp_per_env):
    """the convex pairs on the device (32 lanes per environment, and the lane-per-environment mapping): contact lists
    exact and fields at 1e-9 against the reference engine, rollouts at 1e-9 for 30 steps and 1e-6 over 120"""
    assert available()
    nenv, nstep = 16, 120
    m, b, o = make_pair(CONVEX, solver, nenv=nenv, nconmax=64, njmax=320, warp_per_env=warp_per_env)
    s0 = pile_states(o, nenv, seed=7)
    ctrl = np.zeros((nenv, nstep, 0))
    out = b.rollout(s0, ctrl)
    ref, stats, _ = o.rollout(s0, ctrl, nthread=os.cpu_count() or 1)
    assert stats[:, 3].sum() == 0 and (b.warnings() == 0).all()
    err = (np.abs(out - ref) / np.maximum(1.0, np.abs(ref).max(axis=(0, 1)))).max(axis=(0, 2))
    print("convex rollout rel err: step 30 %.3e, step %d %.3e" % (err[:30].max(), nstep, err.max()))
    assert err[:30].max() < RTOL_TIGHT and err.max() < RTOL_TRAJ
    types = set()
    for t in range(2, nstep, 6):
        compare_forward(b, o, ref[:, t, :], np.zeros((nenv, 0)), rtol=RTOL_TIGHT, check_dual=(solver == mb.SOLVER_PGS))
        types |= contact_types(b, o)[0]
    assert NEW_PAIRS <= types, NEW_PAIRS - types


@pytest.mark.gpu
def test_convex_4096_envs_gpu():
    """4096 piles x 200 steps: no contact / constraint overflow, no warning the reference engine does not raise on
    the same states itself (a few random piles start deep enough inside each other to blow up there too), every state
    finite (the polytope scratch and the stored pre-contacts at scale)"""
    nenv, nstep = 4096, 200
    m, b, o = make_pair(CONVEX, mb.SOLVER_NEWTON, nenv=nenv, nconmax=64, njmax=320)
    s0 = pile_states(o, nenv, seed=21)
    b.set_state(s0)
    b.step(nstep)
    w = b.warnings()
    assert (w[:, 1] == 0).all() and (w[:, 2] == 0).all()          # mjWARN_CONTACTFULL, mjWARN_CNSTRFULL
    _, stats, _ = o.rollout(s0, np.zeros((nenv, nstep, 0)), nthread=os.cpu_count() or 1, want_state=False)
    warned = set(np.nonzero(w.sum(axis=1))[0].tolist())
    assert warned <= set(np.nonzero(stats[:, 3])[0].tolist()), warned
    assert len(warned) < nenv // 100
    assert np.isfinite(b.get_state()).all()
    assert (b.field("ncon")[:, 0] > 0).mean() > 0.9
