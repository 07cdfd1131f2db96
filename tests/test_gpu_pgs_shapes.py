"""The PGS solve kernels at every row count, register class and shared-memory layout, against the oracle.

The device PGS code picks its path from the problem size: the split step's k_pgs4 (mjb_pgs4.h: eight environments
per warp, a register class of 4..16 chain elements per lane chosen by the largest problem of the warp, a tail of
nefc % 4 rows, packed records or the slot layout, generic sweeps above 67 rows or past the visiting-order table), the
persistent rollout's shared pool (mjb_krollout.cu: a second placement pass, or no room at all), and the fused
kernel's solve_pgs (mjb_constraint.h: AR on chip for nefc <= 24, a 4-slot row ring up to 64 rows, global memory
beyond and on the other mappings).  Models of the usual tests reach these paths by chance.

Here the test sets the row count.  The model is a "comb": one free body carrying NSPHERE small spheres over a plane,
sphere k hanging k * DELTA below sphere 0.  Held upright at height r + DELTA * (NSPHERE - K) - DELTA / 2, exactly the
K lowest spheres touch the plane, so with condim 1 an environment has nefc == K rows for any K from 0 to NSPHERE.
Variants add four pyramid rows per contact (condim 3), six dry-friction rows of the free joint (frictionloss) or six
equality rows of a weld to the world (which also makes the model non-lean).  The MJCF is written here and compiled
by the reference's own compiler; every batch checks that each environment has the row count it was built for.

Every sweep compares ncon / nefc / efc_type / efc_id and solver_niter exactly and forces, accelerations and the next
state at 1e-9 with the reference engine; device paths that run the same computation must agree bit for bit.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import mujoco_b200 as mb
from mjb_util import HOSTEMU, compare_forward, hostemu_lib
from oracle_util import Oracle, available

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

RTOL_TIGHT = 1e-9
NSPHERE = 130
RADIUS = 0.05
DELTA = 1e-3            # height step between consecutive spheres (the half step below is the margin of a row count)

VARIANTS = ("c1", "c3", "floss", "weld")
FUSED_VARIANTS = ("c1", "floss", "weld")
# every row count of the register classes 4..16 with every tail, the class-16 edge (67 / 68) and three above it
SWEEP = list(range(0, 71)) + [80, 100, 128]


def comb_xml(variant):
    condim = 3 if variant == "c3" else 1
    joint = '<joint name="root" type="free" frictionloss="0.05"/>' if variant == "floss" else '<freejoint name="root"/>'
    spheres = []
    for k in range(NSPHERE):
        x, y = 0.04 * (k % 13 - 6), 0.04 * (k // 13 - 4.5)
        spheres.append('      <geom type="sphere" size="%r" pos="%r %r %r"/>' % (RADIUS, x, y, -k * DELTA))
    weld = '  <equality><weld body1="comb"/></equality>\n' if variant == "weld" else ""
    return ('<mujoco model="comb_%s">\n'
            '  <option timestep="0.002"/>\n'
            '  <default><geom condim="%d" margin="0" gap="0"/></default>\n'
            '  <worldbody>\n'
            '    <geom name="floor" type="plane" size="0 0 1"/>\n'
            '    <body name="comb" pos="0 0 0.3">\n'
            '      %s\n%s\n'
            '    </body>\n'
            '  </worldbody>\n%s'
            '</mujoco>\n') % (variant, condim, joint, "\n".join(spheres), weld)


def contacts_for(variant, nefc):
    """number of touching spheres that gives `nefc` rows in this variant"""
    if variant == "c3":
        assert nefc % 4 == 0
        return nefc // 4
    extra = 6 if variant in ("floss", "weld") else 0
    assert nefc >= extra
    return nefc - extra


def targets(variant, values=SWEEP):
    """the row counts of `values` that this variant can produce"""
    if variant == "c3":
        return [n for n in values if n % 4 == 0]
    if variant in ("floss", "weld"):
        return [n for n in values if n >= 6]
    return list(values)


def mixed_warps(variant):
    """warps of mixed sizes: 0 next to 67 rows; one 68-row problem (generic sweeps for the whole warp) among small
    ones; a short last warp"""
    if variant == "c3":
        return [0, 64, 4, 8, 32, 12, 60, 20] + [4, 68, 0, 8, 12, 16, 20, 24] + [64, 4, 24, 0, 8]
    if variant in ("floss", "weld"):
        return [6, 67, 7, 8, 33, 9, 64, 11] + [9, 68, 6, 7, 12, 13, 14, 10] + [66, 6, 25, 7, 9]
    return [0, 67, 1, 2, 33, 3, 64, 5] + [3, 68, 1, 0, 2, 7, 11, 4] + [66, 1, 25, 0, 9]


def split_step_warps(variant):
    """the environments of the split-step sweep, warp by warp: (a) eight of the same row count; (a') one row count
    next to seven empty environments, so that every register class 4..16 with every tail fits the packed layout;
    (b) mixed warps and a short last warp"""
    uniform = [n for n in targets(variant) for _ in range(8)]
    empty = 6 if variant in ("floss", "weld") else 0
    single = [x for n in targets(variant, range(1, 68)) if n > empty for x in [n] + [empty] * 7]
    return uniform, single, mixed_warps(variant)


def pgs4_path(warp, budget=56 * 1024, own_beta=8 * 128, slack=0):
    """the path pgs4_warp takes for a warp of these row counts (the arithmetic of mjb_pgs4.h, restated): ("none",),
    ("generic",), ("packed", register class) or ("slot", template class); `budget` = bytes of the region"""
    top = max(warp)
    if top == 0:
        return ("none",)
    if top > 67:
        return ("generic",)
    nqt = (top & ~3) >> 2
    cls = 4 if nqt <= 4 else nqt
    total = 0
    for n in warp:
        nqp = (((n & ~3) >> 2) + 1) & ~1
        total += (n * (4 * nqp + 6) + 16 if n else 0) + 6 * (n + (n & 1))
    if total * 8 + slack <= budget - own_beta:
        return ("packed", cls)
    if budget < 8 * 1384 * 4 + own_beta:
        return ("generic",)
    return ("slot", 4 if cls == 4 else 8 if cls <= 8 else 16)


def pool_passes(cta, pool_bytes=99 * 1024 - 128 - 8 * 128, slack=1024):
    """placement passes of the persistent kernel's PGS pool for the four warps of a CTA (RolloutPool.place restated):
    per warp the pass that places it, or None when its records can never fit"""
    need = []
    for w in range(4):
        warp = cta[8 * w:8 * w + 8]
        total = sum((n * (4 * ((((n & ~3) >> 2) + 1) & ~1) + 6) + 16 if n else 0) + 6 * (n + (n & 1)) for n in warp)
        need.append(0 if max(warp) == 0 or max(warp) > 67 else total * 8 + slack)
    out, done, p = [None] * 4, [False] * 4, 0
    while not all(done):
        p += 1
        off = 0
        for w in range(4):
            if done[w]:
                continue
            if need[w] == 0 or need[w] > pool_bytes:
                out[w] = (p if need[w] == 0 else None)
                done[w] = True
            elif off + need[w] <= pool_bytes:
                off += need[w]
                out[w] = p
                done[w] = True
    return out


_paths = {}


@pytest.fixture(scope="module")
def comb(tmp_path_factory):
    """variant -> path of the compiled comb (.mjb written by the reference's compiler)"""
    if not available():
        pytest.skip("oracle not built")
    d = tmp_path_factory.mktemp("comb")

    def path(variant):
        if variant not in _paths or not os.path.exists(_paths[variant]):
            xml = d / ("comb_%s.xml" % variant)
            xml.write_text(comb_xml(variant))
            out = str(d / ("comb_%s.mjb" % variant))
            Oracle(str(xml)).save_mjb(out)
            _paths[variant] = out
        return _paths[variant]
    return path


def comb_states(o, variant, nefcs, seed=0, qvel_std=0.1):
    """upright comb at the height that gives each environment its row count, with small seeded velocities"""
    rng = np.random.default_rng(seed)
    o.reset()
    base = o.get_state()
    nq = o.size("nq")
    out = np.tile(base, (len(nefcs), 1))
    for e, n in enumerate(nefcs):
        K = contacts_for(variant, n)
        out[e, 1:4] = (0.0, 0.0, RADIUS + DELTA * (NSPHERE - K) - DELTA / 2)
        out[e, 4:8] = (1.0, 0.0, 0.0, 0.0)
        out[e, 1 + nq:1 + nq + 6] = rng.normal(0, qvel_std, 6)
    return out


def caps(variant, nefcs):
    """contact and row capacity of a batch that holds these problems"""
    top = max(nefcs)
    return max(1, max(contacts_for(variant, n) for n in nefcs)), max(1, top)


def make_comb(path, variant, nefcs, seed=0, library=None, njmax=None, **opts):
    """(model, batch, oracle, states) with identical options; the batch has checked that every environment has the
    row count it was built for (a wrong height must fail here, not quietly test another size)"""
    m = mb.Model(path, library=library)
    o = Oracle(path)
    m.set_option("solver", mb.SOLVER_PGS)
    o.set_opt("solver", 0)
    for k, v in opts.items():
        m.set_option(k, v)
        o.set_opt(k, v)
    nconmax, nj = caps(variant, nefcs)
    b = mb.Batch(m, len(nefcs), nconmax=nconmax, njmax=njmax or nj)
    s = comb_states(o, variant, nefcs, seed)
    b.set_state(s)
    b.set_field("qacc_warmstart", 0.0)
    b.forward()
    got = b.field("nefc")[:, 0]
    assert np.array_equal(got, np.asarray(nefcs)), [(e, n, g) for e, (n, g) in enumerate(zip(nefcs, got)) if n != g][:8]
    return m, b, o, s


def step_fields(b):
    """one split step from the current batch state; what the tests compare"""
    b.set_field("qacc_warmstart", 0.0)
    b.step(1)
    out = {f: b.field(f) for f in ("ncon", "nefc", "efc_type", "efc_id", "solver_niter", "efc_force", "qacc",
                                   "qfrc_constraint", "warning")}
    out["state"] = b.get_state()
    return out


def assert_same(a, b_, what, nefcs=None):
    """bit-identical fields; a failure names the first differing environments and their row counts"""
    for k in a:
        if not np.array_equal(a[k], b_[k], equal_nan=True):
            envs = sorted(set(np.argwhere(a[k] != b_[k])[:, 0].tolist()))[:8]
            raise AssertionError((what, k, "environments", envs, "rows", [nefcs[e] for e in envs] if nefcs else None))


def compare_step(got, o, states, nefcs, case):
    """the oracle's mj_step from the same states; counts and types exact, forces / state at 1e-9"""
    for e in range(states.shape[0]):
        o.reset()
        o.set_state(states[e])
        o.step()
        n = int(o.scalar("nefc"))
        tag = (case, "env", e, "nefc", nefcs[e])
        assert n == nefcs[e] and got["nefc"][e, 0] == n, tag
        assert got["ncon"][e, 0] == int(o.scalar("ncon")), tag
        assert np.array_equal(got["efc_type"][e, :n], o.dfield("efc_type")[:n]), tag
        assert np.array_equal(got["efc_id"][e, :n], o.dfield("efc_id")[:n]), tag
        nit = np.array(o.dfield("solver_niter"))
        assert np.array_equal(got["solver_niter"][e, :len(nit)], nit), tag + ("solver_niter", got["solver_niter"][e, :2], nit[:2])
        for f, ref in (("efc_force", o.dfield("efc_force")[:n]), ("qacc", o.dfield("qacc")),
                       ("qfrc_constraint", o.dfield("qfrc_constraint")), ("state", o.get_state())):
            r = np.asarray(ref, dtype=np.float64)
            a = got[f][e, :r.size]
            err = np.abs(a - r).max() / max(1.0, np.abs(r).max()) if r.size else 0.0
            assert err <= RTOL_TIGHT, tag + (f, err)
        assert not got["warning"][e].any(), tag + ("warning", got["warning"][e])


# ---- CPU: the fixture's arithmetic -----------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
def test_comb_row_counts_on_the_oracle(comb, variant):
    """the reference engine itself gives every target row count (all targets of the sweeps, all variants)"""
    o = Oracle(comb(variant))
    nt = targets(variant) + targets(variant, [NSPHERE]) if variant == "c1" else targets(variant)
    s = comb_states(o, variant, nt)
    for e, n in enumerate(nt):
        o.reset()
        o.set_state(s[e])
        o.forward()
        assert int(o.scalar("nefc")) == n, (variant, n, int(o.scalar("nefc")))
        assert int(o.scalar("ncon")) == contacts_for(variant, n)
        assert int(o.scalar("ne")) == (6 if variant == "weld" else 0) and int(o.scalar("nf")) == (6 if variant == "floss" else 0)


@pytest.mark.parametrize("variant", VARIANTS)
def test_comb_forward_bit_exact_on_host_emulation(comb, variant):
    """the kernel source compiled for the host reproduces the reference bit for bit on a few row counts"""
    if not os.path.exists(HOSTEMU):
        pytest.skip("host emulation library not built")
    nefcs = targets(variant, [0, 3, 6, 7, 24, 25, 33, 64, 68])
    m, b, o, s = make_comb(comb(variant), variant, nefcs, seed=1, library=hostemu_lib())
    compare_forward(b, o, s, np.zeros((len(nefcs), 0)), rtol=0, exact=True)


@pytest.mark.parametrize("variant", VARIANTS)
def test_sweeps_reach_every_class_tail_and_layout(variant):
    """which k_pgs4 paths the split-step sweep takes (the kernel's size arithmetic restated): every register class
    4..16 with every tail in the packed layout for the row-count variants (multiples of four for condim 3), the slot
    layout in its 8- and 16-element templates, and the generic sweeps; and the persistent kernel's pool in one pass,
    in four passes and never"""
    uniform, single, mixed = split_step_warps(variant)
    envs = uniform + single + mixed
    reached = set()
    for w in range(0, len(envs), 8):
        warp = envs[w:w + 8]
        path = pgs4_path(warp)
        reached.add(path + ((max(warp) % 4,) if path[0] == "packed" else ()))
    tails = (0,) if variant == "c3" else (0, 1, 2, 3)
    for cls in range(4, 17):
        for t in tails:
            assert ("packed", cls, t) in reached, (variant, cls, t)
    assert {("slot", 8), ("slot", 16), ("generic",)} <= reached, reached
    if variant == "c1":
        assert ("none",) in reached
        passes = [tuple(pool_passes(c)) for c in (rollout_pattern(96)[i:i + 32] for i in range(0, 96, 32))]
        assert passes[0] == (1, 1, 1, 1) and passes[1] == (1, 2, 3, 4) and passes[2][0] is None, passes


# ---- GPU sweeps ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("variant", FUSED_VARIANTS)
def test_fused_solve_every_row_count(comb, variant, monkeypatch):
    """solve_pgs of the fused kernels through mjb_forward, one environment per row count, on three mappings: 32 lanes
    per environment (MODE 2, AR on chip, up to 24 rows; MODE 1, the row ring with a second half-warp above 32 rows,
    up to 64; MODE 0 beyond), k_step_any16 (MJB_LANES=16) and one lane per environment (both always MODE 0).  Each
    matches the oracle, and the three agree bit for bit"""
    nefcs = targets(variant)
    o = Oracle(comb(variant))
    o.set_opt("solver", 0)
    s = comb_states(o, variant, nefcs, seed=2)
    nconmax, njmax = caps(variant, nefcs)
    first = None
    for mapping in ("warp32", "lanes16", "lane_per_env"):
        if mapping == "lanes16":
            monkeypatch.setenv("MJB_LANES", "16")    # read when the batch is made
        else:
            monkeypatch.delenv("MJB_LANES", raising=False)
        m = mb.Model(comb(variant))
        m.set_option("solver", mb.SOLVER_PGS)
        b = mb.Batch(m, len(nefcs), nconmax=nconmax, njmax=njmax, warp_per_env=(mapping != "lane_per_env"))
        try:
            compare_forward(b, o, s, np.zeros((len(nefcs), 0)), rtol=RTOL_TIGHT)
        except AssertionError as ex:
            raise AssertionError("fused %s %s (row counts by environment: %s): %s" % (variant, mapping, nefcs, ex)) from ex
        assert np.array_equal(b.field("nefc")[:, 0], nefcs)
        got = {f: b.field(f) for f in ("efc_force", "qacc", "qfrc_constraint", "solver_niter")}
        if first is None:
            first = got
        else:
            assert_same(first, got, ("fused", variant, mapping), nefcs)
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_split_step_pgs4_every_class_tail_and_layout(comb, variant):
    """k_pgs4 through one split step.  (a) eight environments of the same row count per warp, every count of
    SWEEP: packed records up to 24 rows, the slot layout from 25 (56 KB per warp), generic sweeps above 67; (a') one
    environment of 1..67 rows among seven empty ones: the packed layout in every register class with every tail;
    (b) mixed warps and a short last warp; (c) the slot layout forced, bit-identical.  (Which warp takes which path
    is test_sweeps_reach_every_class_tail_and_layout.)"""
    uniform, single, mixed = split_step_warps(variant)
    nefcs = uniform + single + mixed
    m, b, o, s = make_comb(comb(variant), variant, nefcs, seed=3)
    b.set_state(s)
    packed = step_fields(b)
    b.set_debug("pgs4_slots", 1)
    try:
        b.set_state(s)
        slots = step_fields(b)
    finally:
        b.set_debug("pgs4_slots", 0)
    assert_same(packed, slots, ("split", variant, "pgs4_slots"), nefcs)
    # against the oracle: one environment per warp of (a), the loaded environment of every warp of (a'), and every
    # environment of (b)
    n0 = len(uniform) + len(single)
    pick = list(range(0, n0, 8)) + list(range(n0, len(nefcs)))
    sub = {k: v[pick] for k, v in packed.items()}
    compare_step(sub, o, s[pick], [nefcs[i] for i in pick], ("split", variant))
    # and the eight environments of a uniform warp carry different velocities: check them all on a few counts
    for n in targets(variant, [3, 24, 25, 47, 67]):
        i = uniform.index(n)
        rows = list(range(i, i + 8))
        compare_step({k: v[rows] for k, v in packed.items()}, o, s[rows], [n] * 8, ("split-warp", variant, n))


@pytest.mark.gpu
def test_iteration_caps_grow_and_reuse_the_order_table(comb):
    """opt.iterations 50, 150 (the visiting-order table grows), 50 (the larger table is reused), 5000 (beyond the
    table: generic sweeps), each checked against the oracle; then 300 sweeps without tolerance, long enough for
    non-restarting runs to pass the 128 entries of the momentum table"""
    variant = "c1"
    nefcs = [n for n in (1, 3, 5, 12, 24, 25, 31, 40, 47, 55, 63, 67) for _ in range(8)]
    pick = list(range(0, len(nefcs), 8))
    for iters, tol in ((50, None), (150, None), (50, None), (5000, None), (300, 0.0)):
        opts = {"iterations": iters} if tol is None else {"iterations": iters, "tolerance": tol}
        m, b, o, s = make_comb(comb(variant), variant, nefcs, seed=4, **opts)
        b.set_state(s)
        got = step_fields(b)
        compare_step({k: v[pick] for k, v in got.items()}, o, s[pick], [nefcs[i] for i in pick], ("iterations", iters, tol))
        b.close()


def rollout_pattern(nenv):
    """per-CTA row counts for the persistent kernel (32 environments = four PGS warps per CTA): CTAs that place all
    four warps in one pass, CTAs of four 8 x 31-row warps (about 90 KB each against the 99 KB pool: one warp per
    pass), and CTAs with an 8 x 40-row warp (about 134 KB: never fits, generic sweeps) next to fitting ones"""
    small = [0, 1, 2, 3, 4, 7, 9, 12, 5, 13, 17, 21, 24, 6, 11, 19, 2, 8, 15, 22, 10, 14, 16, 18, 20, 23, 3, 1, 0, 5, 9, 4]
    second = [31] * 32
    never = [40] * 8 + [31] * 8 + small[:16]
    out = []
    for c in range(nenv // 32):
        out += (small, second, never)[c % 3]
    return out


def rollout_case(path, nenv, nstep):
    m = mb.Model(path)
    m.set_option("solver", mb.SOLVER_PGS)
    m.set_option("timestep", 2e-4)   # short steps: the designed row counts hold for most of the rollout
    o = Oracle(path)
    o.set_opt("solver", 0)
    o.set_opt("timestep", 2e-4)
    nefcs = rollout_pattern(nenv)
    s0 = comb_states(o, "c1", nefcs, seed=5)
    b = mb.Batch(m, nenv, nconmax=48, njmax=48)
    return m, b, o, s0, nefcs


@pytest.mark.gpu
def test_rollout_of_a_model_without_actuators(comb):
    """mjb_rollout first zeroes the controls, an empty field when nu == 0: that must launch nothing (a grid of zero
    blocks is a launch error, which stayed pending and failed the state upload of the same call)"""
    nefcs = [0, 5, 24, 40]
    m, b, o, s = make_comb(comb("c1"), "c1", nefcs, seed=7)
    ref, stats, _ = o.rollout(s, np.zeros((len(nefcs), 3, 0)))
    for _ in range(2):
        out = b.rollout(s, None, nstep=3)
        assert not b.warnings().any() and stats[:, 3].sum() == 0
        assert (np.abs(out - ref) / np.maximum(1.0, np.abs(ref).max(axis=(0, 1)))).max() < RTOL_TIGHT


@pytest.mark.gpu
def test_persistent_rollout_pool_passes(comb):
    """k_rollout with every CTA full: pool placement in one pass, in several passes, and a warp that can never fit
    (generic sweeps), bit-identical to the per-step launches and within 1e-9 of the reference"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nenv, nstep = 32 * sms, 10
    m, b, o, s0, nefcs = rollout_case(comb("c1"), nenv, nstep)
    b.set_state(s0)
    b.forward()
    assert np.array_equal(b.field("nefc")[:, 0], nefcs)
    out, niter, warn = {}, {}, {}
    try:
        for mode in (1, 0):
            b.set_debug("persistent", mode)
            out[mode] = b.rollout(s0, None, nstep=nstep)
            niter[mode] = b.field("solver_niter").copy()
            warn[mode] = b.field("warning").copy()
    finally:
        b.set_debug("persistent", 1)
    assert np.array_equal(out[1], out[0])
    assert np.array_equal(niter[1], niter[0]) and np.array_equal(warn[1], warn[0])
    assert not warn[1].any()
    ref, stats, _ = o.rollout(s0, np.zeros((nenv, nstep, 0)), nthread=os.cpu_count() or 1)
    assert stats[:, 3].sum() == 0
    rel = (np.abs(out[1] - ref) / np.maximum(1.0, np.abs(ref).max(axis=(0, 1)))).max()
    assert rel < RTOL_TIGHT, rel
    # (the short steps keep the designed sizes: at the last step nearly every environment is within one row of them)
    assert (np.abs(b.field("nefc")[:, 0] - np.asarray(nefcs)) <= 1).mean() > 0.95


# ---- once-per-process switches -----------------------------------------------------------------------------------

SWITCHES = [("MJB_PART_LANES", "8"), ("MJB_PART_LANES", "32"), ("MJB_ROLLOUT_POOL_KB", "8"),
            ("MJB_ROLLOUT_POOL_KB", "24"), ("MJB_PGS4_SLOTS", "1"), ("MJB_SPLIT", "0")]

SCRIPT = r'''
import sys, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(here)r)
import mujoco_b200 as mb
import test_gpu_pgs_shapes as T
from mjb_util import HUMANOID, perturbed_states
from oracle_util import Oracle
comb, out, sms = sys.argv[1], sys.argv[2], int(sys.argv[3])
res = {}
nefcs = [n for n in T.targets("c1") for _ in range(8)] + T.mixed_warps("c1")
m, b, o, s = T.make_comb(comb, "c1", nefcs, seed=3)
b.set_state(s)
for k, v in T.step_fields(b).items():
    res["split_" + k] = v
m, b, o, s0, _ = T.rollout_case(comb, 32 * sms, 10)
res["roll_comb"] = b.rollout(s0, None, nstep=10)
res["roll_comb_niter"] = b.field("solver_niter")
res["roll_comb_warning"] = b.field("warning")
nenv, nstep = 64, 20
m = mb.Model(HUMANOID); m.set_option("solver", mb.SOLVER_PGS)
o = Oracle(HUMANOID); o.set_opt("solver", 0)
b = mb.Batch(m, nenv, nconmax=48, njmax=128)
s0 = perturbed_states(o, nenv, seed=11, height=[0.2, 0.3, 0.5, 0.8], qvel_std=0.5, qpos_std=0.2)
ctrl = np.random.default_rng(12).uniform(-1, 1, (nenv, nstep, o.size("nu")))
res["roll_humanoid"] = b.rollout(s0, ctrl)
res["roll_humanoid_niter"] = b.field("solver_niter")
res["roll_humanoid_warning"] = b.field("warning")
np.savez(out, **res)
'''


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_process_switches_bit_identical(comb, tmp_path):
    """the switches read once per process (halves of the split step on 8 / 32 lanes, the persistent kernel's pool
    size, the slot layout, the fused step instead of the split step) change the path, never the result: the comb's
    split step and persistent-size rollout and a 20-step contact-rich humanoid rollout, bit for bit"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    path = comb("c1")

    def run(name, env):
        out = str(tmp_path / (name + ".npz"))
        e = dict(os.environ)
        for k, _ in SWITCHES:
            e.pop(k, None)
        e.update(env)
        subprocess.run([sys.executable, "-c", SCRIPT % {"root": ROOT, "here": HERE}, path, out, str(sms)],
                       check=True, env=e, timeout=600)
        return np.load(out)

    base = run("default", {})
    for k, v in SWITCHES:
        got = run("%s_%s" % (k, v), {k: v})
        for f in base.files:
            assert np.array_equal(base[f], got[f], equal_nan=True), ("%s=%s" % (k, v), f, np.argwhere(base[f] != got[f])[:4])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["c1", "weld"])
def test_row_cap_edge(comb, variant):
    """njmax equal to the row count: the rows fill the arena exactly, no mjWARN_CNSTRFULL, and the reference's
    results (forward and one split step)"""
    for n in targets(variant, [1, 3, 24, 25, 33, 64, 67, 68, 100, 128]):
        nefcs = [n] * 8
        m, b, o, s = make_comb(comb(variant), variant, nefcs, seed=6, njmax=n)
        assert not b.warnings().any(), (variant, n, b.warnings()[0])
        compare_forward(b, o, s, np.zeros((8, 0)), rtol=RTOL_TIGHT)
        b.set_state(s)
        compare_step(step_fields(b), o, s, nefcs, ("cap", variant, n))
