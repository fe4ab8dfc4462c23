"""Compatibility path: run UNMODIFIED reference task files (which `import isaacgym` and subclass
`isaacgymenvs.tasks.base.vec_task.VecTask`) on the CUDA engine through the generic `gym.*` tensor
API -- Python hooks run as they are, `gym.simulate` is the CUDA physics kernel (SURVEY.md 8f rank 2).

    from isaacgymenvs_b200 import compat
    compat.install()                      # puts `isaacgym` and the hook-style VecTask in sys.modules
    from isaacgymenvs.tasks.ant import Ant   # the reference's own file

The reference's own `tasks/base/vec_task.py` cannot be imported under NumPy 2 (`np.Inf`,
SURVEY.md 3.3), so `install()` also provides that module; everything else of `isaacgymenvs`
(task files, `utils/torch_jit_utils.py`) is the user's unmodified checkout.
"""
import sys
import types


def install(reference_root=None):
    from . import gymapi, gymtorch, vec_task_hooks
    pkg = types.ModuleType("isaacgym")
    pkg.gymapi, pkg.gymtorch = gymapi, gymtorch
    pkg.gymutil = types.ModuleType("isaacgym.gymutil")
    pkg.terrain_utils = types.ModuleType("isaacgym.terrain_utils")
    from .. import terrain as _t
    for n in ("SubTerrain", "random_uniform_terrain", "pyramid_sloped_terrain", "pyramid_stairs_terrain",
              "discrete_obstacles_terrain", "stepping_stones_terrain", "convert_heightfield_to_trimesh"):
        setattr(pkg.terrain_utils, n, getattr(_t, n))
    sys.modules["isaacgym"] = pkg
    sys.modules["isaacgym.gymapi"] = gymapi
    sys.modules["isaacgym.gymtorch"] = gymtorch
    sys.modules["isaacgym.gymutil"] = pkg.gymutil
    sys.modules["isaacgym.terrain_utils"] = pkg.terrain_utils
    if reference_root is not None:
        # make `isaacgymenvs.*` importable from a checkout WITHOUT running its package __init__ (hydra)
        import os
        for name, rel in (("isaacgymenvs", ""), ("isaacgymenvs.utils", "utils"), ("isaacgymenvs.tasks", "tasks"),
                          ("isaacgymenvs.tasks.base", "tasks/base")):
            if name not in sys.modules:
                m = types.ModuleType(name)
                m.__path__ = [os.path.join(reference_root, "isaacgymenvs", rel)]
                sys.modules[name] = m
    sys.modules["isaacgymenvs.tasks.base.vec_task"] = vec_task_hooks
    return pkg
