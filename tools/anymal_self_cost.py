"""Cost of AnymalTerrain's link-link contact (env.selfCollision): the whole env.step() at 4096 envs on the curriculum height
field, with the flag off and on, timed with CUDA events; the two envs are timed alternately, several rounds each.  Prints one
JSON line with the GPU's name and power limit read in the same run.

    python tools/anymal_self_cost.py [--envs 4096] [--steps 200] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make(n, on):
    import isaacgymenvs_b200
    from isaacgymenvs_b200 import config
    cfg = config.builtin_cfg("AnymalTerrain", {"sim_device": "cuda:0", "rl_device": "cuda:0"})
    cfg["task"]["env"]["selfCollision"] = on
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return isaacgymenvs_b200.make(seed=42, task="AnymalTerrain", num_envs=n, sim_device="cuda:0", rl_device="cuda:0",
                                      headless=True, cfg=cfg)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("anymal_self_cost.py: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    envs = {on: make(a.envs, on) for on in (False, True)}
    assert envs[True].sim.quad_ns() == 3 and envs[False].sim.quad_ns() == 3
    g = torch.Generator(device="cuda:0"); g.manual_seed(0)
    acts = torch.rand((a.steps, a.envs, 12), device="cuda:0", generator=g) * 2 - 1
    for env in envs.values():                                   # warm-up: module load, first-step resets
        for k in range(20):
            env.step(acts[k])
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    for _ in range(a.rounds):
        for on in (False, True):
            env = envs[on]
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for k in range(a.steps):
                env.step(acts[k])
            t1.record(); torch.cuda.synchronize()
            ms[on].append(t0.elapsed_time(t1) / a.steps)
    res = {"gpu": gpu, "envs": a.envs, "steps_per_round": a.steps, "rounds": a.rounds,
           "step_ms_off": ms[False], "step_ms_on": ms[True],
           "median_off": sorted(ms[False])[len(ms[False]) // 2], "median_on": sorted(ms[True])[len(ms[True]) // 2]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
