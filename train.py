#!/usr/bin/env python
"""train.py -- the reference's launcher surface (`python train.py task=Ant headless=True`, isaacgymenvs/train.py:71-215)
over this repo's environments.  The reference hands the env to rl_games (not installable here: no network); this launcher
reads the same `key=value` overrides, takes the PPO hyper-parameters of the reference's cfg/train/<Task>PPO.yaml
(a2c_continuous: network units, learning rate, horizon, minibatch, mini-epochs, critic coefficient, KL threshold, reward scale,
bounds loss) and runs the compact learner of tools/train_ppo.py, which drives the env through the RLGPUEnv contract
(utils/rlgames_utils.py:242-295: reset() / step() with dict observations, `time_outs` for the value bootstrap).

    python train.py task=Ant headless=True                       # 4096 envs, 500 epochs (AntPPO.yaml)
    python train.py task=ShadowHand num_envs=8192 max_iterations=300 task.env.objectType=pen task.env.forceScale=1.0
    python train.py task=Humanoid seed=7 sim_device=cuda:0 rl_device=cuda:0 task.env.selfCollision=True
    python train.py task=Humanoid task.task.randomize=True       # the randomization_params block of Humanoid.yaml

Demonstration tooling (DESIGN.md section 6e), not part of the measured hot path.
"""
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# cfg/train/<Task>PPO.yaml of the reference: params.network.mlp.units; params.config.{learning_rate, horizon_length, minibatch_size,
# mini_epochs, critic_coef, kl_threshold, reward_shaper.scale_value, bounds_loss_coef, max_epochs}; cfg/task/<Task>.yaml env.numEnvs
PPO = {
    "Ant":           dict(units=[256, 128, 64], lr=3e-4, horizon=16, minibatch=32768, mini_epochs=4, critic_coef=2, kl=0.008, rew_scale=0.01, bounds=1e-4, epochs=500, num_envs=4096),
    "Humanoid":      dict(units=[400, 200, 100], lr=5e-4, horizon=32, minibatch=32768, mini_epochs=5, critic_coef=4, kl=0.008, rew_scale=0.01, bounds=1e-4, epochs=1000, num_envs=4096),
    "Cartpole":      dict(units=[32, 32], lr=3e-4, horizon=16, minibatch=8192, mini_epochs=8, critic_coef=4, kl=0.008, rew_scale=0.1, bounds=1e-4, epochs=100, num_envs=512),
    "AnymalTerrain": dict(units=[512, 256, 128], lr=3e-4, horizon=24, minibatch=16384, mini_epochs=5, critic_coef=2, kl=0.008, rew_scale=1.0, bounds=0.0, epochs=1500, num_envs=4096),
    "ShadowHand":    dict(units=[512, 512, 256, 128], lr=5e-4, horizon=8, minibatch=32768, mini_epochs=5, critic_coef=4, kl=0.016, rew_scale=0.01, bounds=1e-4, epochs=5000, num_envs=16384),
}


def parse_overrides(argv):
    """hydra-style `key=value` words -> dict (cfg/config.yaml:1-60 of the reference names the top-level keys)."""
    out = {}
    for w in argv:
        if "=" not in w:
            raise SystemExit(f"train.py: expected key=value, got {w!r}")
        k, v = w.split("=", 1)
        out[k] = v
    return out


def to_ppo_argv(ov):
    """the argument list of tools/train_ppo.py for a set of reference-style overrides"""
    task = ov.get("task", "Ant")
    if task not in PPO:
        raise SystemExit(f"train.py: task {task!r} is not one of {sorted(PPO)}")
    hp = PPO[task]
    known = {"task", "num_envs", "seed", "max_iterations", "sim_device", "rl_device", "headless", "pipeline", "graphics_device_id",
             "experiment", "wandb_activate", "capture_video", "force_render", "test", "checkpoint", "multi_gpu"}
    bad = [k for k in ov if k not in known and not k.startswith("task.env.") and k != "task.task.randomize"]
    if bad:
        raise SystemExit(f"train.py: overrides {bad} are not provided here (top-level keys of cfg/config.yaml, task.env.* and "
                         "task.task.randomize are)")
    randomize = ov.get("task.task.randomize", "False")
    if randomize not in ("True", "true", "False", "false"):
        raise SystemExit(f"train.py: task.task.randomize={randomize!r}: True or False")
    for k in ("test", "checkpoint", "multi_gpu", "capture_video"):
        if ov.get(k, "False") not in ("False", "false", "", "0"):
            raise SystemExit(f"train.py: {k} is not provided by the demonstration learner")
    if ov.get("sim_device", "cuda:0") != ov.get("rl_device", ov.get("sim_device", "cuda:0")):
        raise SystemExit("train.py: the learner runs on the simulation device (sim_device == rl_device)")
    env = dict((k[len("task.env."):], v) for k, v in ov.items() if k.startswith("task.env."))
    selfc = env.pop("selfCollision", "False") in ("True", "true", "1")
    argv = ["--task", task, "--num-envs", str(int(ov.get("num_envs") or hp["num_envs"])), "--epochs", str(int(ov.get("max_iterations") or hp["epochs"])),
            "--horizon", str(hp["horizon"]), "--minibatch", str(hp["minibatch"]), "--seed", str(int(ov.get("seed", 42))),
            "--device", ov.get("sim_device", "cuda:0"), "--units", ",".join(str(u) for u in hp["units"]), "--lr", repr(hp["lr"]),
            "--mini-epochs", str(hp["mini_epochs"]), "--critic-coef", repr(float(hp["critic_coef"])), "--kl-threshold", repr(hp["kl"]),
            "--reward-scale", repr(hp["rew_scale"]), "--bounds-coef", repr(hp["bounds"])]
    if selfc:
        argv.append("--self-collision")
    if randomize in ("True", "true"):
        argv.append("--randomize")
    if env:
        argv += ["--env", ",".join(f"{k}={v}" for k, v in env.items())]
    if ov.get("experiment"):
        argv += ["--out", os.path.join("runs", ov["experiment"] + ".json")]
    return argv


def main(argv=None):
    ov = parse_overrides(sys.argv[1:] if argv is None else argv)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train_ppo
    train_ppo.main(to_ppo_argv(ov))


if __name__ == "__main__":
    main()
