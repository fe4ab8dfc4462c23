"""Cost of Ant / Humanoid domain randomisation (task.randomize with the built-in randomization_params blocks):
  * the whole env.step() with randomisation off and on -- Humanoid at 8192 envs, Ant at 16384;
  * the bare Humanoid step launch (Sim.task_step) with a gravity vector bound (the gravity-reading instantiation) and
    without (the plain kernel), on the same sim.
Each pair is timed with CUDA events, alternately, several rounds each, under random actions.  Prints one JSON line with the
GPU's name and power limit read in the same run.

    python tools/dr_cost.py [--steps 200] [--rounds 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"Humanoid": 8192, "Ant": 16384}


def make(task, n, randomize):
    import isaacgymenvs_b200
    from isaacgymenvs_b200 import config
    cfg = config.builtin_cfg(task, {"sim_device": "cuda:0", "rl_device": "cuda:0"})
    cfg["task"]["task"]["randomize"] = randomize
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return isaacgymenvs_b200.make(seed=42, task=task, num_envs=n, sim_device="cuda:0", rl_device="cuda:0", headless=True, cfg=cfg)


def alternate(fns, acts, steps, rounds, setup=None):
    """per-step ms of each callable, timed alternately over `rounds` rounds of `steps` calls; setup[key]() runs before each"""
    setup = setup or {}
    for key, fn in fns.items():                                     # warm-up: module load, first-step resets
        setup.get(key, lambda: None)()
        for k in range(20):
            fn(acts[k])
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for key, fn in fns.items():
            setup.get(key, lambda: None)()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for k in range(steps):
                fn(acts[k])
            t1.record(); torch.cuda.synchronize()
            ms[key].append(t0.elapsed_time(t1) / steps)
    return ms


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dr_cost.py: no CUDA device")
    from isaacgymenvs_b200 import engine
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "steps_per_round": a.steps, "rounds": a.rounds}
    g = torch.Generator(device="cuda:0"); g.manual_seed(0)
    for task, n in SIZES.items():
        envs = {on: make(task, n, on) for on in (False, True)}
        acts = torch.rand((a.steps, n, envs[False].num_acts), device="cuda:0", generator=g) * 2 - 1
        ms = alternate({on: envs[on].step for on in (False, True)}, acts, a.steps, a.rounds)
        res[task] = {"envs": n, "env_step_ms_off": ms[False], "env_step_ms_on": ms[True],
                     "median_off": median(ms[False]), "median_on": median(ms[True])}
        if task == "Humanoid":
            sim = envs[False].sim
            grav = torch.tensor([0.0, 0.0, -9.81], device="cuda:0")
            unbind = lambda: engine._check(engine.lib().b2g_bind(sim._h, ctypes.c_int32(engine.T_GRAVITY), None, ctypes.c_size_t(0)), "unbind")
            ms = alternate({"unbound": sim.task_step, "bound": sim.task_step}, acts, a.steps, a.rounds,
                           setup={"unbound": unbind, "bound": lambda: sim._bind(engine.T_GRAVITY, grav)})
            res[task].update({"launch_ms_gravity_unbound": ms["unbound"], "launch_ms_gravity_bound": ms["bound"],
                              "median_launch_unbound": median(ms["unbound"]), "median_launch_bound": median(ms["bound"])})
        del envs
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
