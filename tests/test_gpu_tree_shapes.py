"""The cooperative tree passes and the primal solvers on generated kinematic trees, against the oracle.

Every cooperative loop of the step spreads the items of one level over the lanes that own an environment (MJB_PFOR)
and separates levels with MJB_PSYNC, in an order fixed by host-built schedules (mjb_model.cc): body levels and child
lists (kinematics, tree_accumulate, com_vel, rne in mjb_smooth.h), dof levels and per-dof descendant lists
(solve_LD), the L'DL factor program (factor_I), and the element-wise Hessian, Cholesky factor and rank-one updates of
the Newton / CG solver (mjb_newton.h).  How those loops wrap over 32, 16 or 8 lanes depends on the tree: its depth,
fan-out, dof count and descendant counts.  The models of the other tests are small and shallow (humanoid nv 27, ant
nv 14, trees of depth 1), so no list there is longer than one pass of the lanes.

The shapes here sit on both sides of every lane boundary: hinge chains on a free base (nv 7 .. 59), a 59-link chain
on a fixed base (depth 59, descendant lists of 58 dofs), a chain of mixed joints (hinge / slide / ball, two joints on
some bodies, a welded child, ref / armature / damping / stiffness / limits), stars of 15 .. 53 arms (one tree level
wider than a warp), a branched tree with self-collision, dense-Jacobian chains of nv 60, 70 and 100 (above the
nv < 60 of jacobian="auto"), forests of 21 and 29 two-dof trees (more islands than the 20 with solver statistics,
and the same forest solved as one island), and a chain and a star with a sensor (the non-lean kernels).  The MJCF is
written here and compiled by the reference's own compiler; a CPU test checks every shape's sizes, depth and
descendant counts, so a mistaken generator fails rather than quietly testing another shape.

Against the reference: contact lists, counts and solver_niter (per island) exact, everything else at 1e-9, on the
fused kernel (32 and 16 lanes, lean and non-lean), one lane per environment, the split step with its part-lane
variants and the persistent rollout.  Paths that run the same computation must agree bit for bit.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import mujoco_b200 as mb
from mjb_util import HOSTEMU, compare_forward, hostemu_lib, perturbed_states
from oracle_util import Oracle, available

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

RTOL_TIGHT = 1e-9
DSBL_ISLAND = 1 << 18
NISLAND = 20                 # mjNISLAND: islands with solver statistics
SOLVERS = {"pgs": mb.SOLVER_PGS, "cg": mb.SOLVER_CG, "newton": mb.SOLVER_NEWTON}

LINK = 0.1                   # link length of chains and arms
RADIUS = 0.02                # capsule radius
FLOOR = '    <geom name="floor" type="plane" size="0 0 1" contype="0" conaffinity="1"/>\n'
# capsules and spheres collide with the floor only (contype 1 against the floor's conaffinity 1), unless a shape
# enables self-collision
FLOOR_ONLY = 'contype="1" conaffinity="0"'


def mjcf(name, body, option="", sensor="", defaults=FLOOR_ONLY):
    return ('<mujoco model="%s">\n'
            '  <option timestep="0.001" %s/>\n'
            '  <default><geom %s condim="3"/><joint damping="0.05" armature="0.002"/></default>\n'
            '  <worldbody>\n%s%s  </worldbody>\n%s'
            '</mujoco>\n') % (name, option, defaults, FLOOR, body,
                              "  <sensor>%s</sensor>\n" % sensor if sensor else "")


def hinge_chain(n, indent, first="0 0 0", axis=lambda i: "0 1 0" if i % 2 == 0 else "0 0 1"):
    """n nested hinge links, each a capsule of LINK along x, the first at `first` in its parent"""
    out = []
    for i in range(n):
        pad = indent + "  " * i
        pos = first if i == 0 else "%r 0 0" % LINK
        out.append('%s<body name="l%d" pos="%s">\n%s  <joint name="j%d" type="hinge" axis="%s"/>\n'
                   '%s  <geom type="capsule" size="%r" fromto="0 0 0 %r 0 0" mass="0.1"/>\n'
                   % (pad, i, pos, pad, i, axis(i), pad, RADIUS, LINK))
    for i in reversed(range(n)):
        out.append("%s</body>\n" % (indent + "  " * i))
    return "".join(out)


def chain_xml(n, name, option="", sensor=""):
    """free base (a sphere) carrying a chain of n hinge links"""
    body = ('    <body name="base" pos="0 0 0.1">\n      <freejoint name="root"/>\n'
            '      <geom type="sphere" size="0.05" mass="1"/>\n%s    </body>\n') % hinge_chain(n, "      ", "0.05 0 0")
    return mjcf(name, body, option, sensor)


def fixed_chain_xml(n):
    """a chain of n hinge links attached to the world just above the floor"""
    body = '    <body name="mount" pos="0 0 0.025">\n%s    </body>\n' % hinge_chain(n, "      ")
    return mjcf("fixed%d" % n, body)


def mixed_chain_xml():
    """30 links on a free base: hinge / slide / ball in turn, a second (hinge) joint on links 4, 19 and 24, link 13 a
    welded child without a joint; non-zero ref, armature, damping, stiffness and limits (nv 58)"""
    out, pad = [], "      "
    for i in range(30):
        p = pad + "  " * i
        pos = "0.05 0 0" if i == 0 else "%r 0 0" % LINK
        joints = []
        if i != 13:
            kind = ("hinge", "slide", "ball")[i % 3]
            if kind == "hinge":
                joints.append('<joint name="j%d" type="hinge" axis="0 %d %d" ref="%r" range="-%r %r" limited="true" '
                              'armature="0.01" damping="0.05" stiffness="0.5"/>'
                              % (i, i % 2, 1 - i % 2, 0.1 * (i % 4), 40 + i, 50 + i))
            elif kind == "slide":
                joints.append('<joint name="j%d" type="slide" axis="1 0 0" ref="0.01" range="-0.02 0.02" limited="true" '
                              'armature="0.02" damping="0.5" stiffness="20"/>' % i)
            else:
                joints.append('<joint name="j%d" type="ball" range="0 %r" limited="true" armature="0.01" damping="0.02"/>'
                              % (i, 30 + i))
            if i in (4, 19, 24):
                joints.append('<joint name="k%d" type="hinge" axis="0 0 1" ref="-0.2" range="-60 60" limited="true" '
                              'damping="0.03" stiffness="0.2"/>' % i)
        out.append('%s<body name="l%d" pos="%s">\n%s%s  <geom type="capsule" size="%r" fromto="0 0 0 %r 0 0" mass="0.1"/>\n'
                   % (p, i, pos, "".join("%s  %s\n" % (p, j) for j in joints), p, RADIUS, LINK))
    for i in reversed(range(30)):
        out.append("%s</body>\n" % (pad + "  " * i))
    body = ('    <body name="base" pos="0 0 0.1">\n      <freejoint name="root"/>\n'
            '      <geom type="sphere" size="0.05" mass="1"/>\n%s    </body>\n') % "".join(out)
    return mjcf("mixed30", body)


def star_xml(k, name, sensor=""):
    """free base (a sphere) with k one-link hinge arms in the horizontal plane, flapping up and down"""
    arms = []
    for i in range(k):
        a = 2 * np.pi * i / k
        c, s = float(np.cos(a)), float(np.sin(a))
        arms.append('      <body name="a%d" pos="%r %r 0">\n        <joint name="j%d" type="hinge" axis="%r %r 0"/>\n'
                    '        <geom type="capsule" size="%r" fromto="0 0 0 %r %r 0" mass="0.05"/>\n      </body>\n'
                    % (i, 0.05 * c, 0.05 * s, i, -s, c, RADIUS, 3 * LINK * c, 3 * LINK * s))
    body = ('    <body name="base" pos="0 0 0.1">\n      <freejoint name="root"/>\n'
            '      <geom type="sphere" size="0.05" mass="1"/>\n%s    </body>\n') % "".join(arms)
    return mjcf(name, body, sensor=sensor)


def branched_xml():
    """free base -> 4 limbs -> 3 segments each -> 3 more below each segment of two of the limbs: 34 hinges, nv 40,
    depth 4; all geoms collide with each other (parent / child pairs excepted) and with the floor"""
    def limb(name, depth, indent, ang, r):
        c, s = float(np.cos(ang)), float(np.sin(ang))
        out = ('%s<body name="%s" pos="%r %r 0">\n%s  <joint name="%s" type="hinge" axis="%r %r 0"/>\n'
               '%s  <geom type="capsule" size="%r" fromto="0 0 0 %r %r -0.03" mass="0.05"/>\n'
               % (indent, name, r * c, r * s, indent, name, -s, c, indent, RADIUS, LINK * c, LINK * s))
        for j in range(3 if depth > 0 else 0):
            out += limb("%s_%d" % (name, j), depth - 1, indent + "  ", ang + 0.6 * (j - 1), LINK)
        return out + "%s</body>\n" % indent
    limbs = "".join(limb("b%d" % i, 2 if i < 2 else 1, "      ", np.pi / 2 * i, 0.06) for i in range(4))
    body = ('    <body name="base" pos="0 0 0.15">\n      <freejoint name="root"/>\n'
            '      <geom type="sphere" size="0.05" mass="1"/>\n%s    </body>\n') % limbs
    return mjcf("branched", body, defaults='contype="1" conaffinity="1"')


def forest_xml(n):
    """n separate trees, each a body with a vertical slide and a hinge carrying a horizontal capsule that rests on
    the floor (the trees never touch each other)"""
    trees = []
    for i in range(n):
        x, y = 0.3 * (i % 6), 0.3 * (i // 6)
        trees.append('    <body name="t%d" pos="%r %r %r">\n      <joint name="s%d" type="slide" axis="0 0 1"/>\n'
                     '      <joint name="h%d" type="hinge" axis="0 1 0"/>\n'
                     '      <geom type="capsule" size="%r" fromto="-0.08 0 0 0.08 0 0" mass="0.2"/>\n    </body>\n'
                     % (i, x, y, RADIUS, i, i, RADIUS))
    return mjcf("forest%d" % n, "".join(trees))


# name -> (MJCF, expected nv, nbody, body depth, largest descendant count of a dof, ntree)
# (nbody counts the world; depth is the depth of the deepest body, the world at depth 0)
def _chain(n):
    return (chain_xml(n, "chain%d" % n), 6 + n, n + 2, n + 1, n + 5, 1)


def _star(k):
    return (star_xml(k, "star%d" % k), 6 + k, k + 2, 2, k + 5, 1)


CHAINS = (1, 10, 11, 26, 27, 28, 41, 53)
STARS = (15, 16, 17, 33, 53)
SHAPES = {}
SHAPES.update({"chain%d" % n: _chain(n) for n in CHAINS})
SHAPES["fixed59"] = (fixed_chain_xml(59), 59, 61, 60, 58, 1)
SHAPES["mixed30"] = (mixed_chain_xml(), 58, 32, 31, 57, 1)
SHAPES.update({"star%d" % k: _star(k) for k in STARS})
SHAPES["branched"] = (branched_xml(), 40, 36, 4, 39, 1)
SHAPES.update({"dense%d" % nv: (chain_xml(nv - 6, "dense%d" % nv, option='jacobian="dense"'), nv, nv - 4, nv - 5, nv - 1, 1)
               for nv in (60, 70, 100)})
SHAPES.update({"forest%d" % n: (forest_xml(n), 2 * n, n + 1, 1, 1, n) for n in (21, 29)})
SHAPES["chain28_sensor"] = (chain_xml(28, "chain28_sensor", sensor='<jointpos joint="j27"/>'), 34, 30, 29, 33, 1)
SHAPES["star33_sensor"] = (star_xml(33, "star33_sensor", sensor='<jointpos joint="j32"/>'), 39, 35, 2, 38, 1)


_paths = {}


@pytest.fixture(scope="module")
def shape(tmp_path_factory):
    """name -> path of the compiled shape (.mjb written by the reference's compiler)"""
    if not available():
        pytest.skip("oracle not built")
    d = tmp_path_factory.mktemp("trees")

    def path(name):
        if name not in _paths or not os.path.exists(_paths[name]):
            xml = d / ("%s.xml" % name)
            xml.write_text(SHAPES[name][0])
            out = str(d / ("%s.mjb" % name))
            Oracle(str(xml)).save_mjb(out)
            _paths[name] = out
        return _paths[name]
    return path


def tree_stats(o):
    """(nv, nbody, deepest body depth, largest number of strict descendant dofs of a dof, ntree) read from the
    oracle's model"""
    bp = o.mfield("body_parentid")
    depth = [0] * len(bp)
    for i in range(1, len(bp)):
        depth[i] = depth[bp[i]] + 1
    dp = o.mfield("dof_parentid")
    ndesc = [0] * len(dp)
    for i in range(len(dp)):
        j = dp[i]
        while j >= 0:
            ndesc[j] += 1
            j = dp[j]
    return o.size("nv"), o.size("nbody"), max(depth), max(ndesc), o.size("ntree")


def shape_states(name, o, nenv, seed):
    """seeded states of a shape: small random joint angles and random velocities around qpos0, the chains, arms
    and limbs lying just above or in the floor, so that many links touch it without deep penetration; the forest's
    trees are each pushed 1..3 mm into the floor (every tree touches, one island per tree)"""
    if name.startswith("forest"):
        rng = np.random.default_rng(seed)
        o.reset()
        s = np.tile(o.get_state(), (nenv, 1))
        nq = o.size("nq")
        for e in range(nenv):
            s[e, 1:1 + nq:2] = -rng.uniform(0.001, 0.003, nq // 2)     # slides
            s[e, 2:1 + nq:2] = rng.normal(0, 0.05, nq // 2)            # hinges
            s[e, 1 + nq:] = rng.normal(0, 0.1, nq)
        return s
    if name.startswith("fixed"):
        return perturbed_states(o, nenv, seed, qvel_std=0.3, qpos_std=0.03)
    return perturbed_states(o, nenv, seed, height=[0.015, 0.02, 0.03, 0.06], qvel_std=0.3, qpos_std=0.03)


def oracle_counts(o, states):
    """(ncon, nefc, nisland) of the reference's mj_forward for every state"""
    out = []
    for s in states:
        o.reset()
        o.set_state(s)
        o.forward()
        out.append((int(o.scalar("ncon")), int(o.scalar("nefc")), int(o.scalar("nisland"))))
    return np.array(out)


# test cases: a shape, or a shape with options (the forests solved as one island)
CASES = {name: (name, {}) for name in SHAPES}
CASES.update({"forest%d_mono" % n: ("forest%d" % n, {"disableflags": DSBL_ISLAND}) for n in (21, 29)})


def caps_for(counts):
    """contact and row capacity of a batch whose environments reach these (ncon, nefc) counts"""
    return max(1, int(counts[:, 0].max())), max(1, int(counts[:, 1].max()))


def make_case(shape, case, solver, nenv, seed, library=None, warp_per_env=True, headroom=False, **extra):
    """(batch, oracle, states) with identical options; caps sized from the reference's counts on these states (with
    headroom for a rollout)"""
    name, opts = CASES[case]
    path = shape(name)
    opts = dict(opts, **extra)
    m = mb.Model(path, library=library)
    o = Oracle(path)
    m.set_option("solver", SOLVERS[solver])
    o.set_opt("solver", SOLVERS[solver])
    for k, v in opts.items():
        m.set_option(k, v)
        o.set_opt(k, v)
    s = shape_states(name, o, nenv, seed)
    nconmax, njmax = caps_for(oracle_counts(o, s))
    if headroom:
        nconmax, njmax = nconmax + nconmax // 2 + 8, njmax + njmax // 2 + 32
    b = mb.Batch(m, nenv, nconmax=nconmax, njmax=njmax, warp_per_env=warp_per_env)
    return b, o, s


def no_warnings(b, tag):
    w = b.warnings()
    assert not w.any(), tag + ("warnings (CONTACTFULL / CNSTRFULL ...) in environments", np.argwhere(w.any(axis=1))[:8, 0].tolist())


def forward_tagged(b, o, s, tag, solver, **kw):
    try:
        compare_forward(b, o, s, np.zeros((s.shape[0], 0)), check_dual=(solver == "pgs"), **kw)
    except AssertionError as ex:
        raise AssertionError("%s (the detail names the environment): %s" % (tag, ex)) from ex
    no_warnings(b, tag)


# ---- CPU: the generator and the host emulation -----------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shape_has_the_tree_it_was_built_for(shape, name):
    """nv, nbody, depth, largest descendant list and tree count from the reference's compiled model; the states
    reach contacts (the forests: every tree touches, more trees than NISLAND islands)"""
    o = Oracle(shape(name))
    assert tree_stats(o) == SHAPES[name][1:], (name, tree_stats(o), SHAPES[name][1:])
    assert int(o.opt("jacobian")) == (0 if name.startswith("dense") else 2)     # mjJAC_DENSE / mjJAC_AUTO
    assert (o.size("nsensor") > 0) == name.endswith("_sensor")
    counts = oracle_counts(o, shape_states(name, o, 8, seed=1))
    assert counts[:, 1].max() > 0, name
    if name.startswith("forest"):
        n = int(name[6:])
        assert (counts[:, 2] == n).all() and n > NISLAND, counts[:, 2]
    elif name != "chain1":
        assert counts[:, 1].max() > 32, (name, counts[:, 1])     # rows past one pass of the lanes


@pytest.mark.parametrize("solver", sorted(SOLVERS))
@pytest.mark.parametrize("case", sorted(CASES))
def test_forward_bit_exact_on_host_emulation(shape, case, solver):
    """the kernel source compiled for the host reproduces the reference bit for bit on every shape"""
    if not os.path.exists(HOSTEMU):
        pytest.skip("host emulation library not built")
    b, o, s = make_case(shape, case, solver, 4, seed=2, library=hostemu_lib())
    forward_tagged(b, o, s, (case, solver, "host emulation"), solver, rtol=0, exact=True)


@pytest.mark.parametrize("solver", sorted(SOLVERS))
@pytest.mark.parametrize("case", ["chain53", "fixed59", "dense70", "forest29"])
def test_rollout_bit_exact_on_host_emulation(shape, case, solver):
    """20 steps on the host emulation against the reference's rollout, bit for bit"""
    if not os.path.exists(HOSTEMU):
        pytest.skip("host emulation library not built")
    b, o, s = make_case(shape, case, solver, 4, seed=3, library=hostemu_lib(), headroom=True)
    out = b.rollout(s, None, nstep=20)
    ref, stats, _ = o.rollout(s, np.zeros((4, 20, 0)))
    assert stats[:, 3].sum() == 0
    no_warnings(b, (case, solver, "host emulation rollout"))
    bad = [e for e in range(4) if not np.array_equal(out[e], ref[e])]
    assert not bad, (case, solver, "host emulation rollout", "environments", bad)


def test_dense_jacobian_at_any_nv_and_the_site_transmission_limit(shape, tmp_path):
    """jacobian="dense" is accepted at any nv (the device paths are tested above on nv 60, 70 and 100); "auto" at
    nv >= 60 is sparse and refused; a site transmission is refused above nv 64 (fwd_velocity gathers its nonzero
    moments into a list of 64) and accepted at nv 64"""
    if not os.path.exists(HOSTEMU):
        pytest.skip("host emulation library not built")
    mb.Batch(mb.Model(shape("dense100"), library=hostemu_lib()), 1).close()
    m = mb.Model(shape("dense70"), library=hostemu_lib())
    m.set_option("jacobian", 2)                       # mjJAC_AUTO
    with pytest.raises(mb.MjbError, match="sparse"):
        mb.Batch(m, 1)
    for nv, ok in ((64, True), (65, False)):
        xml = chain_xml(nv - 6, "site%d" % nv, option='jacobian="dense"').replace(
            '<geom type="sphere" size="0.05" mass="1"/>',
            '<geom type="sphere" size="0.05" mass="1"/><site name="s0"/>').replace(
            "</mujoco>", '  <actuator><general site="s0" gear="0 0 1 0 0 0"/></actuator>\n</mujoco>')
        (tmp_path / "site.xml").write_text(xml)
        path = str(tmp_path / ("site%d.mjb" % nv))
        Oracle(str(tmp_path / "site.xml")).save_mjb(path)
        m = mb.Model(path, library=hostemu_lib())
        assert m.size("nv") == nv
        if ok:
            mb.Batch(m, 1).close()
        else:
            with pytest.raises(mb.MjbError, match="nv > 64"):
                mb.Batch(m, 1)


# ---- GPU ---------------------------------------------------------------------------------------------------------

MAPPINGS = {"lanes32": ("32", True), "lanes16": ("16", True), "lane_per_env": (None, False)}


def set_mapping(monkeypatch, mapping):
    """MJB_LANES is read when a batch is made; returns warp_per_env"""
    lanes, warp = MAPPINGS[mapping]
    if lanes:
        monkeypatch.setenv("MJB_LANES", lanes)
    else:
        monkeypatch.delenv("MJB_LANES", raising=False)
    return warp


STEP_FIELDS = ("ncon", "nefc", "efc_type", "efc_id", "solver_niter", "efc_force", "qacc", "qfrc_constraint")


def device_step(b):
    """one mj_step of the batch from its current state and warm start; what the step comparison reads"""
    b.step(1)
    out = {f: b.field(f) for f in STEP_FIELDS}
    out["state"] = b.get_state()
    out["qacc_warmstart"] = b.field("qacc_warmstart")
    return out


def compare_step(got, o, states, warm, tag, full=True):
    """the reference's mj_step from the same states and warm starts: counts, types, ids and solver_niter (every
    island) exact; forces, accelerations, the next state and warm start at 1e-9.  full=False (RK4): the next state
    and warm start only"""
    for e in range(states.shape[0]):
        o.reset()
        o.set_state(states[e])
        o.dfield("qacc_warmstart")[:] = warm[e]
        o.step()
        t = tag + ("env", e)
        refs = [("state", o.get_state()), ("qacc_warmstart", o.dfield("qacc_warmstart"))]
        if full:
            n = int(o.scalar("nefc"))
            assert got["nefc"][e, 0] == n and got["ncon"][e, 0] == int(o.scalar("ncon")), t + ("ncon / nefc", got["ncon"][e, 0], got["nefc"][e, 0], int(o.scalar("ncon")), n)
            assert np.array_equal(got["efc_type"][e, :n], o.dfield("efc_type")[:n]), t + ("efc_type",)
            assert np.array_equal(got["efc_id"][e, :n], o.dfield("efc_id")[:n]), t + ("efc_id",)
            nit = np.array(o.dfield("solver_niter"))
            assert np.array_equal(got["solver_niter"][e, :len(nit)], nit), t + ("solver_niter", got["solver_niter"][e], nit)
            refs += [("efc_force", o.dfield("efc_force")[:n]), ("qacc", o.dfield("qacc")),
                     ("qfrc_constraint", o.dfield("qfrc_constraint"))]
        for f, ref in refs:
            r = np.asarray(ref, dtype=np.float64)
            a = got[f][e, :r.size]
            err = np.abs(a - r).max() / max(1.0, np.abs(r).max()) if r.size else 0.0
            assert err <= RTOL_TIGHT, t + (f, err)


def stepwise_rollout(b, o, s0, nstep, tag, full=True):
    """nstep steps of the batch, each checked against the reference's mj_step started from the device's previous
    state and warm start (so that chaos can neither hide an error nor cause a false failure)"""
    b.set_state(s0)
    b.set_field("qacc_warmstart", 0.0)
    state, warm = s0, np.zeros((s0.shape[0], o.size("nv")))
    for t in range(nstep):
        got = device_step(b)
        no_warnings(b, tag + ("step", t))
        compare_step(got, o, state, warm, tag + ("step", t), full)
        state, warm = got["state"], got["qacc_warmstart"]
    return state


@pytest.mark.gpu
@pytest.mark.parametrize("solver", sorted(SOLVERS))
@pytest.mark.parametrize("case", sorted(CASES))
def test_forward_every_mapping(shape, case, solver, monkeypatch):
    """mjb_forward on the fused kernel with 32 lanes, with 16 lanes (the automatic choice for chain1 / chain10 and
    the primal solvers, forced elsewhere) and one lane per environment, each against the reference at 1e-9 (contact
    lists, counts and solver_niter exact); the PGS solve is bit-identical on the three"""
    first = None
    for mapping in MAPPINGS:
        warp = set_mapping(monkeypatch, mapping)
        b, o, s = make_case(shape, case, solver, 6, seed=4, warp_per_env=warp)
        forward_tagged(b, o, s, (case, solver, "forward", mapping), solver, rtol=RTOL_TIGHT)
        got = {f: b.field(f) for f in ("efc_force", "qacc", "qfrc_constraint", "solver_niter")}
        b.close()
        if solver != "pgs":
            continue
        if first is None:
            first = got
        for f in got:
            bad = np.argwhere((first[f] != got[f]).any(axis=1))[:8, 0].tolist()
            assert not bad, (case, solver, "forward", mapping, "differs from lanes32 in", f, "environments", bad)


LANE_PER_ENV_CASES = ["chain53", "fixed59", "mixed30", "star53", "branched", "dense100", "forest29", "forest29_mono",
                      "chain28_sensor"]
ROLLOUTS = ([(c, "default", 30) for c in sorted(CASES)] + [(c, "lanes16", 10) for c in sorted(CASES)] +
            [(c, "lane_per_env", 5) for c in LANE_PER_ENV_CASES])


@pytest.mark.gpu
@pytest.mark.parametrize("solver", sorted(SOLVERS))
@pytest.mark.parametrize("case,mapping,nstep", ROLLOUTS)
def test_stepwise_rollout(shape, case, mapping, nstep, solver, monkeypatch):
    """steps from seeded states on the step path of the batch: 30 on the default path (the split step for PGS on one
    tree, the fused kernel otherwise, 16 lanes where chosen automatically), 10 with 16 lanes forced, 5 with one
    lane per environment; each step against the reference from the device's previous state and warm start.  The
    first step starts from identical states."""
    if mapping == "default":
        monkeypatch.delenv("MJB_LANES", raising=False)
        warp = True
    else:
        warp = set_mapping(monkeypatch, mapping)
    b, o, s = make_case(shape, case, solver, 4, seed=5, warp_per_env=warp, headroom=True)
    stepwise_rollout(b, o, s, nstep, (case, solver, "rollout", mapping))


@pytest.mark.gpu
@pytest.mark.parametrize("integrator", ["rk4", "implicitfast"])
@pytest.mark.parametrize("solver", ["newton", "pgs"])
@pytest.mark.parametrize("case", ["mixed30", "chain27"])
def test_integrators(shape, case, solver, integrator):
    """RK4 (four forward passes per step and the Runge-Kutta combination) and implicitfast (the split step's
    non-lean halves for PGS), stepwise against the reference"""
    opt = mb.INT_RK4 if integrator == "rk4" else mb.INT_IMPLICITFAST
    b, o, s = make_case(shape, case, solver, 4, seed=6, headroom=True, integrator=opt)
    stepwise_rollout(b, o, s, 15, (case, solver, integrator), full=(integrator != "rk4"))


EDGES = {"ls_iterations1": {"ls_iterations": 1}, "ls_iterations3": {"ls_iterations": 3},
         "iterations1": {"iterations": 1}, "tolerance0": {"tolerance": 0.0}}


@pytest.mark.gpu
@pytest.mark.parametrize("edge", sorted(EDGES))
@pytest.mark.parametrize("solver", ["newton", "cg"])
@pytest.mark.parametrize("case", ["chain41", "dense70"])
def test_primal_solver_edges(shape, case, solver, edge, monkeypatch):
    """line-search caps of 1 and 3, a single iteration, and no tolerance (every solve runs to the cap): a forward
    pass on 32 and 16 lanes and five steps (one with a single iteration), against the reference"""
    for mapping in ("lanes32", "lanes16"):
        set_mapping(monkeypatch, mapping)
        b, o, s = make_case(shape, case, solver, 4, seed=7, headroom=True, **EDGES[edge])
        forward_tagged(b, o, s, (case, solver, edge, "forward", mapping), solver, rtol=RTOL_TIGHT)
        # (a single iteration leaves these stiff chains unstable within a few steps, in the reference as well)
        stepwise_rollout(b, o, s, 1 if edge == "iterations1" else 5, (case, solver, edge, "rollout", mapping))
        b.close()


PERSISTENT = ["chain11", "chain28", "star17", "star53"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PERSISTENT)
def test_persistent_rollout(shape, case):
    """k_rollout with every CTA but the last one full (32 environments each), bit-identical to the per-step split
    step launches; its first step against the reference"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nenv, nstep = 32 * sms - 5, 10
    b, o, s = make_case(shape, case, "pgs", nenv, seed=8, headroom=True)
    out, niter = {}, {}
    try:
        for mode in (1, 0):
            b.set_debug("persistent", mode)
            out[mode] = b.rollout(s, None, nstep=nstep)
            niter[mode] = b.field("solver_niter")
            no_warnings(b, (case, "pgs", "persistent" if mode else "split step"))
    finally:
        b.set_debug("persistent", 1)
    bad = np.argwhere((out[1] != out[0]).any(axis=(1, 2)))[:8, 0].tolist()
    assert not bad, (case, "pgs", "persistent rollout differs from the split step in environments", bad)
    assert np.array_equal(niter[1], niter[0]), (case, "pgs", "persistent solver_niter")
    pick = list(range(0, nenv, nenv // 12)) + [nenv - 1]
    for e in pick:
        o.reset()
        o.set_state(s[e])
        o.step()
        r = o.get_state()
        err = np.abs(out[1][e, 0] - r).max() / max(1.0, np.abs(r).max())
        assert err <= RTOL_TIGHT, (case, "pgs", "persistent first step", "env", e, err)


# ---- once-per-process switches -----------------------------------------------------------------------------------

SWITCH_CASES = ["chain28", "chain53", "star33", "mixed30", "chain28_sensor", "star33_sensor"]
SWITCHES = [("MJB_PART_LANES", "8"), ("MJB_PART_LANES", "32"), ("MJB_SPLIT", "0")]

SCRIPT = r'''
import json, sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(here)r)
import test_gpu_tree_shapes as T
paths, out = json.loads(sys.argv[1]), sys.argv[2]
res = {}
for case in T.SWITCH_CASES:
    b, o, s = T.make_case(paths.__getitem__, case, "pgs", 37, seed=9, headroom=True)
    b.set_state(s)
    b.set_field("qacc_warmstart", 0.0)
    for k, v in T.device_step(b).items():
        res["%%s_step_%%s" %% (case, k)] = v
    res[case + "_rollout"] = b.rollout(s, None, nstep=10)
    res[case + "_niter"] = b.field("solver_niter")
    res[case + "_warning"] = b.field("warning")
np.savez(out, **res)
'''


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_split_step_switches_bit_identical(shape, tmp_path):
    """the halves of the split step on 8 or 32 lanes instead of 16, and the fused step instead of the split step,
    give the same bits as the default (a split step and a 10-step rollout, the persistent kernel on the lean
    shapes), on long chains, a wide star, the mixed-joint chain and the non-lean twins (37 environments: a short
    last warp)"""
    import json
    paths = json.dumps({CASES[c][0]: shape(CASES[c][0]) for c in SWITCH_CASES})

    def run(tag, env):
        out = str(tmp_path / (tag + ".npz"))
        e = dict(os.environ)
        for k, _ in SWITCHES:
            e.pop(k, None)
        e.pop("MJB_LANES", None)
        e.update(env)
        subprocess.run([sys.executable, "-c", SCRIPT % {"root": ROOT, "here": HERE}, paths, out],
                       check=True, env=e, timeout=900)
        return np.load(out)

    base = run("default", {})
    for case in SWITCH_CASES:
        assert not base[case + "_warning"].any(), (case, "pgs", "default path warnings")
    for k, v in SWITCHES:
        got = run("%s_%s" % (k, v), {k: v})
        for f in base.files:
            bad = np.argwhere((base[f] != got[f]).reshape(base[f].shape[0], -1).any(axis=1))[:8, 0].tolist()
            assert not bad, ("%s=%s" % (k, v), f, "pgs", "environments", bad)
