"""Golden vectors for the observation / action noise of domain randomisation, from the REFERENCE's own
`VecTask.apply_randomizations` (tasks/base/vec_task.py:610-718), build container only:
    python tests/golden/make_golden_dr.py
The reference module is loaded by path (numpy 2: `np.Inf` aliased; `gym` stubbed; `isaacgym` = this repo's shim, for the
type names in annotations only) and the method is called on a bare instance whose `gym.get_frame_count` is scripted.
The noise lambdas it installs are then applied to fixed tensors under torch.manual_seed.  Output: tests/golden/dr_noise.npz."""
import importlib.util
import os
import sys
import types
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF_ROOT = os.environ.get("ISAACGYMENVS_ROOT", ".")     # an IsaacGymEnvs checkout
OUT = os.path.dirname(os.path.abspath(__file__))

CASES = {
    "gauss_add_linear": dict(frequency=1, observations=dict(range=[0.0, 0.002], range_correlated=[0.0, 0.001], operation="additive",
                                                            distribution="gaussian", schedule="linear", schedule_steps=40000),
                             actions=dict(range=[0.0, 0.05], range_correlated=[0.0, 0.015], operation="additive", distribution="gaussian")),
    "gauss_scale_const": dict(frequency=1, observations=dict(range=[1.0, 0.1], range_correlated=[1.0, 0.05], operation="scaling",
                                                             distribution="gaussian", schedule="constant", schedule_steps=100)),
    "uniform_add": dict(frequency=1, actions=dict(range=[-0.1, 0.2], range_correlated=[-0.01, 0.03], operation="additive",
                                                  distribution="uniform", schedule="linear", schedule_steps=1000)),
    "uniform_scale": dict(frequency=1, observations=dict(range=[0.9, 1.2], operation="scaling", distribution="uniform",
                                                         schedule="linear", schedule_steps=500)),
}
FRAMES = [0, 50, 250, 20000, 60000]


def load_reference_vec_task():
    np.Inf = np.inf
    from isaacgymenvs_b200 import compat
    compat.install(reference_root=REF_ROOT)
    gym = types.ModuleType("gym"); gym.spaces = types.ModuleType("gym.spaces"); gym.spaces.Box = lambda *a, **k: None; gym.Space = object
    sys.modules["gym"] = gym; sys.modules["gym.spaces"] = gym.spaces

    def ld(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REF_ROOT, "isaacgymenvs", rel))
        mod = importlib.util.module_from_spec(spec); sys.modules[modname] = mod; spec.loader.exec_module(mod)
        return mod
    ld("isaacgymenvs.utils.torch_jit_utils", "utils/torch_jit_utils.py")
    ld("isaacgymenvs.utils.dr_utils", "utils/dr_utils.py")
    ld("isaacgymenvs.utils.utils", "utils/utils.py")
    return ld("isaacgymenvs.tasks.base.vec_task", "tasks/base/vec_task.py")


def main():
    vt = load_reference_vec_task()
    blob = {"frames": np.array(FRAMES)}
    g = torch.Generator().manual_seed(5)
    x_obs = torch.randn(64, 60, generator=g); x_act = torch.rand(64, 8, generator=g) * 2 - 1
    blob["x_observations"] = x_obs.numpy(); blob["x_actions"] = x_act.numpy()
    for cname, params in CASES.items():
        for frame in FRAMES:
            Bare = type("Bare", (vt.VecTask,), {"pre_physics_step": lambda self, a: None, "post_physics_step": lambda self: None})
            t = object.__new__(Bare)
            t.num_environments, t.first_randomization, t.dr_randomizations, t.envs, t.sim = 64, True, {}, [], None
            t.randomize_buf = torch.zeros(64, dtype=torch.long); t.reset_buf = torch.ones(64, dtype=torch.long)
            class Gym:                                             # any gym.* attribute exists; only the frame count matters
                def __getattr__(self, name):
                    return (lambda sim, f=frame: f) if name == "get_frame_count" else (lambda *a, **k: None)
            t.gym = Gym()
            vt.check_buckets = lambda *a, **k: None
            t.actor_params_generator, t.extern_actor_params = None, {}
            t.apply_randomizations(dict(params, actor_params={}))       # the method indexes ["actor_params"] unconditionally
            for key, x in (("observations", x_obs), ("actions", x_act)):
                if key not in params:
                    continue
                torch.manual_seed(1000 + frame)
                lam = t.dr_randomizations[key]["noise_lambda"]
                y1 = lam(x.clone()); y2 = lam(x.clone())           # second call re-uses the correlated sample
                blob[f"{cname}_{frame}_{key}_1"] = y1.numpy(); blob[f"{cname}_{frame}_{key}_2"] = y2.numpy()
    np.savez_compressed(os.path.join(OUT, "dr_noise.npz"), **blob)
    print("wrote dr_noise.npz with", len(blob), "arrays")


if __name__ == "__main__":
    main()
