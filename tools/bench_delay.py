"""Cost of history buffers: tests/golden/ant_delay.mjb (models/ant_delay.xml: delayed actuators and delayed / sampled
sensors) x N environments on the device, Newton and PGS, next to the same model with every history attribute removed
(compiled from the XML at run time), which runs the kernels of a model without buffers.  The states start from the
same seeded perturbations with the controls held; CUDA events around the timed rollout after a warm-up that runs the
same call.  Records the card name and power limit beside the numbers.  Prints one JSON line.

usage: python tools/bench_delay.py [--nenv 4096] [--steps 200] [--warmup 50]"""
import argparse
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

import mujoco_b200 as mb  # noqa: E402
from bench_convex import card  # noqa: E402
from mjb_util import perturbed_states  # noqa: E402
from oracle_util import Oracle  # noqa: E402

DELAY = os.path.join(ROOT, "tests", "golden", "ant_delay.mjb")
XML = os.path.join(ROOT, "models", "ant_delay.xml")


def device_rate(path, solver, nenv, nstep, warmup, s0, ctrl):
    m = mb.Model(path)
    m.set_option("solver", solver)
    b = mb.Batch(m, nenv, nconmax=48, njmax=200)
    stream = torch.cuda.ExternalStream(b.stream())
    b.set_state(s0)
    b.set_field("ctrl", ctrl)
    b.rollout_device(warmup, 0, 0)         # the same call as the timed window: every kernel loaded before the clock
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    b.rollout_device(nstep, 0, 0)
    e1.record(stream)
    stream.synchronize()
    ms = e0.elapsed_time(e1)
    return {"env_steps_per_s": nenv * nstep / ms * 1e3, "ms_per_step": ms / nstep, "warnings": int(b.warnings().sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nenv", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    res = {"nenv": a.nenv, "steps": a.steps, **card()}
    with tempfile.TemporaryDirectory() as tmp:
        stripped = os.path.join(tmp, "ant_nodelay.mjb")
        xml = os.path.join(tmp, "ant_nodelay.xml")
        with open(XML) as f:
            text = re.sub(r'\s(delay|nsample|interp|interval)="[^"]*"', "", f.read())
        with open(xml, "w") as f:
            f.write(text)
        Oracle(xml).save_mjb(stripped)
        o = Oracle(DELAY)
        s0 = perturbed_states(o, a.nenv, seed=31, qvel_std=0.5, qpos_std=0.05)
        rng = np.random.default_rng(31)
        lo, hi = o.mfield("actuator_ctrlrange").reshape(-1, 2).T
        ctrl = rng.uniform(lo, hi, (a.nenv, o.size("nu")))
        nh = 1 + o.size("nq") + o.size("nv") + o.size("na")
        for name, solver in (("newton", mb.SOLVER_NEWTON), ("pgs", mb.SOLVER_PGS)):
            res["ant_delay_" + name] = device_rate(DELAY, solver, a.nenv, a.steps, a.warmup, s0, ctrl)
            res["ant_nodelay_" + name] = device_rate(stripped, solver, a.nenv, a.steps, a.warmup, s0[:, :nh], ctrl)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
