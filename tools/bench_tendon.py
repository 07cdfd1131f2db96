"""Throughput of spatial tendons: tests/golden/arm26.mjb (the reference's 2-link arm with six muscles on
cylinder-wrapped tendons) and tests/golden/tendon_paths.mjb (models/tendon_paths.xml) x N environments on the device,
Newton and PGS, next to the reference engine's threaded CPU rollout of the same states and controls.  Times the device
with CUDA events after a warm-up that runs the same calls, and records the card name and power limit beside the
numbers.  Prints one JSON line.

usage: python tools/bench_tendon.py [--nenv 4096] [--steps 200] [--warmup 50] [--cpu-envs 256]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import mujoco_b200 as mb  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_convex import card  # noqa: E402
from test_spatial_tendons import ARM26, PATHS, controls_for, states_for  # noqa: E402


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


def cpu_rate(path, solver, nenv, nstep, s0, ctrl):
    from oracle_util import Oracle
    o = Oracle(path)
    o.set_opt("solver", solver)
    nthread = os.cpu_count() or 1
    c = np.repeat(ctrl[:nenv, None, :], nstep, axis=1)
    _, _, sec = o.rollout(s0[:nenv], c, nthread=nthread, want_state=False)
    return {"env_steps_per_s": nenv * nstep / sec, "threads": nthread, "nenv": nenv}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nenv", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--cpu-envs", type=int, default=256)
    a = ap.parse_args()
    from oracle_util import Oracle
    res = {"nenv": a.nenv, "steps": a.steps, **card()}
    for model, path in (("arm26", ARM26), ("tendon_paths", PATHS)):
        o = Oracle(path)
        s0 = states_for(o, a.nenv, seed=31)
        ctrl = controls_for(o, a.nenv, 1, seed=31)[:, 0]   # held constant over the window
        for name, solver in (("newton", mb.SOLVER_NEWTON), ("pgs", mb.SOLVER_PGS)):
            key = model + "_" + name
            res[key] = device_rate(path, solver, a.nenv, a.steps, a.warmup, s0, ctrl)
            try:
                res[key + "_cpu_reference"] = cpu_rate(path, solver, a.cpu_envs, a.steps, s0, ctrl)
            except Exception as err:   # the oracle library is optional on the device machine
                res[key + "_cpu_reference"] = {"error": str(err)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
