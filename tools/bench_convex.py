"""Throughput of the convex narrow phase: models/convex.xml (eight free ellipsoids, cylinders, a box, a sphere and a
capsule piled on a plane) x N environments on the device, Newton and PGS, next to the reference engine's threaded CPU
rollout of the same states.  Times the device with CUDA events after a warm-up that runs the same calls, and records
the card name and power limit beside the numbers.  Prints one JSON line.

usage: python tools/bench_convex.py [--nenv 4096] [--steps 200] [--warmup 50] [--cpu-envs 256]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import mujoco_b200 as mb  # noqa: E402
from test_convex import CONVEX, pile_states  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def device_rate(solver, nenv, nstep, warmup, s0):
    m = mb.Model(CONVEX)
    m.set_option("solver", solver)
    b = mb.Batch(m, nenv, nconmax=64, njmax=320)
    stream = torch.cuda.ExternalStream(b.stream())
    b.set_state(s0)
    b.rollout_device(warmup, 0, 0)         # the same call as the timed window: every kernel loaded before the clock
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    b.rollout_device(nstep, 0, 0)
    e1.record(stream)
    stream.synchronize()
    ms = e0.elapsed_time(e1)
    nc = b.field("ncon")[:, 0]
    return {"env_steps_per_s": nenv * nstep / ms * 1e3, "ms_per_step": ms / nstep, "ncon_mean": float(nc.mean()),
            "warnings": int(b.warnings().sum())}


def cpu_rate(solver, nenv, nstep, s0):
    from oracle_util import Oracle
    o = Oracle(CONVEX)
    o.set_opt("solver", solver)
    nthread = os.cpu_count() or 1
    _, _, sec = o.rollout(s0[:nenv], np.zeros((nenv, nstep, 0)), nthread=nthread, want_state=False)
    return {"env_steps_per_s": nenv * nstep / sec, "threads": nthread, "nenv": nenv}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nenv", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--cpu-envs", type=int, default=256)
    a = ap.parse_args()
    from oracle_util import Oracle
    s0 = pile_states(Oracle(CONVEX), a.nenv, seed=21)
    res = {"model": "convex.xml", "nenv": a.nenv, "steps": a.steps, **card()}
    for name, solver in (("newton", mb.SOLVER_NEWTON), ("pgs", mb.SOLVER_PGS)):
        res[name] = device_rate(solver, a.nenv, a.steps, a.warmup, s0)
        try:
            res[name + "_cpu_reference"] = cpu_rate(solver, a.cpu_envs, a.steps, s0)
        except Exception as err:   # the oracle library is optional on the device machine
            res[name + "_cpu_reference"] = {"error": str(err)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
