"""CUDA-native (H100) vectorised environment stepper behind the IsaacGymEnvs surface.

    import isaacgymenvs_b200 as isaacgymenvs
    envs = isaacgymenvs.make(seed=0, task="Ant", num_envs=16384, sim_device="cuda:0", rl_device="cuda:0")
    obs = envs.reset(); obs, rew, done, info = envs.step(actions)

`make` keeps the reference's signature and return type (`isaacgymenvs/__init__.py:14-55`).
"""
import os


def make(seed: int, task: str, num_envs: int, sim_device: str, rl_device: str, graphics_device_id: int = -1,
         headless: bool = False, multi_gpu: bool = False, virtual_screen_capture: bool = False,
         force_render: bool = True, cfg=None, cfg_dir: str = None):
    """cfg: an already composed config dict (root keys + cfg['task']); cfg_dir: a reference-format
    `cfg/` directory to compose from (unmodified YAML); neither: the built-in restatement."""
    from . import config as _config
    from .tasks import isaacgym_task_map
    overrides = {"seed": seed, "sim_device": sim_device, "rl_device": rl_device,
                 "graphics_device_id": graphics_device_id, "headless": headless, "multi_gpu": multi_gpu}
    if cfg is None:
        cfg = (_config.load_reference_cfg(cfg_dir, task, overrides) if cfg_dir
               else _config.builtin_cfg(task, overrides))
    task_cfg = cfg["task"]
    task_cfg["env"]["numEnvs"] = num_envs                     # isaacgymenvs/__init__.py:35-38
    task_cfg["seed"] = seed
    if multi_gpu:                                             # utils/rlgames_utils.py:89-107
        local_rank = int(os.getenv("LOCAL_RANK", "0"))
        global_rank = int(os.getenv("RANK", "0"))
        sim_device = rl_device = f"cuda:{local_rank}"
        task_cfg["env_id_offset"] = global_rank * num_envs
        task_cfg["rank"] = global_rank
    name = task_cfg.get("name", task)
    if name not in isaacgym_task_map:
        raise KeyError(f"task {name!r} has no fused CUDA kernel (supported: {sorted(isaacgym_task_map)})")
    return isaacgym_task_map[name](cfg=task_cfg, rl_device=rl_device, sim_device=sim_device,
                                   graphics_device_id=graphics_device_id, headless=headless,
                                   virtual_screen_capture=virtual_screen_capture, force_render=force_render)
