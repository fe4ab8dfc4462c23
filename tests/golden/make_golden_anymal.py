"""Golden vectors for AnymalTerrain from the REFERENCE's own code (build container only):
    python tests/golden/make_golden_anymal.py
`tasks/anymal_terrain.py` is loaded by path with isaacgym stubbed; its METHODS check_termination
(:294-300), compute_reward (:315-382), compute_observations (:302-313), get_heights (:515-538) and
the jit helpers quat_apply_yaw / wrap_to_pi (:676-687) are called on a namespace `self`; the
"prepare quantities" lines of post_physics_step (:464-471), which are inline in the reference, are
replayed with the reference's jit functions.  Output: tests/golden/anymal_terrain.npz."""
import importlib.util
import os
import sys
import types
import numpy as np
import torch

REF = os.path.join(os.environ.get("ISAACGYMENVS_ROOT", "."), "isaacgymenvs")     # an IsaacGymEnvs checkout
OUT = os.path.dirname(os.path.abspath(__file__))


def load():
    for name in ("isaacgym", "isaacgym.gymtorch", "isaacgym.gymapi", "isaacgym.gymutil", "isaacgym.terrain_utils"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["isaacgym"].gymtorch = sys.modules["isaacgym.gymtorch"]
    sys.modules["isaacgym"].gymapi = sys.modules["isaacgym.gymapi"]
    sys.modules["isaacgym"].gymutil = sys.modules["isaacgym.gymutil"]
    for name in ("isaacgymenvs", "isaacgymenvs.utils", "isaacgymenvs.tasks", "isaacgymenvs.tasks.base"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["isaacgymenvs.tasks"].__path__ = []
    vt = types.ModuleType("isaacgymenvs.tasks.base.vec_task"); vt.VecTask = type("VecTask", (), {})
    sys.modules["isaacgymenvs.tasks.base.vec_task"] = vt

    def ld(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec); sys.modules[modname] = mod; spec.loader.exec_module(mod)
        return mod
    tju = ld("isaacgymenvs.utils.torch_jit_utils", "utils/torch_jit_utils.py")
    at = ld("isaacgymenvs.tasks.anymal_terrain", "tasks/anymal_terrain.py")
    return tju, at


def main():
    tju, at = load()
    g = torch.Generator().manual_seed(4321)
    n = 384
    dt = 4 * 0.005
    rows, cols = 1200, 2000                      # tot_rows/tot_cols of the default 10x20 x 8 m map + 20 m border
    hs = (torch.randn(rows // 8, cols // 8, generator=g) * 30).round().to(torch.int16)
    hs = hs.repeat_interleave(8, 0).repeat_interleave(8, 1).contiguous()      # blocky terrain, +-0.15 m steps

    s = types.SimpleNamespace()
    s.num_envs, s.num_dof, s.num_actions, s.device = n, 12, 12, "cpu"
    s.cfg = {"env": {"terrain": {"terrainType": "trimesh"}}}
    s.terrain = types.SimpleNamespace(border_size=20, horizontal_scale=0.1, vertical_scale=0.005)
    s.height_samples = hs
    s.base_index = 0
    s.knee_indices = torch.tensor([2, 5, 8, 11]); s.feet_indices = torch.tensor([3, 6, 9, 12])
    s.allow_knee_contacts = True
    s.max_episode_length = int(20 / dt + 0.5); s.max_episode_length_s = 20
    s.dt = dt
    scales = dict(termination=0.0, lin_vel_xy=1.0, lin_vel_z=-4.0, ang_vel_z=0.5, ang_vel_xy=-0.05, orient=-0.0, torque=-0.00002,
                  joint_acc=-0.0005, base_height=-0.0, air_time=1.0, collision=-0.25, stumble=-0.0, action_rate=-0.01, hip=-0.0)
    s.rew_scales = {k: v * dt for k, v in scales.items()}
    s.lin_vel_scale, s.ang_vel_scale, s.dof_pos_scale, s.dof_vel_scale, s.height_meas_scale = 2.0, 0.25, 1.0, 0.05, 5.0
    s.commands_scale = torch.tensor([2.0, 2.0, 0.25])
    # ---- state
    root = torch.zeros(n, 13)
    root[:, 0] = torch.rand(n, generator=g) * 70 + 2; root[:, 1] = torch.rand(n, generator=g) * 150 + 2
    root[:, 2] = torch.rand(n, generator=g) * 0.6 + 0.3
    q = torch.randn(n, 4, generator=g) * torch.tensor([0.2, 0.2, 1.0, 0.0]) + torch.tensor([0, 0, 0, 1.0])
    root[:, 3:7] = q / q.norm(dim=-1, keepdim=True)
    root[:, 7:13] = torch.randn(n, 6, generator=g)
    s.root_states = root
    default = torch.tensor([0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, 0.4, -0.8, -0.03, -0.4, 0.8]).repeat(n, 1)   # LF, LH, RF, RH
    s.default_dof_pos = default
    s.dof_pos = default + torch.randn(n, 12, generator=g) * 0.3
    s.dof_vel = torch.randn(n, 12, generator=g) * 4
    cf = torch.randn(n, 13, 3, generator=g) * 20
    cf = cf * (torch.rand(n, 13, 1, generator=g) < 0.4)                        # most bodies out of contact
    s.contact_forces = cf
    s.commands = torch.zeros(n, 4)
    s.commands[:, 0:2] = torch.rand(n, 2, generator=g) * 2 - 1
    s.commands[:, 3] = torch.rand(n, generator=g) * 6.28 - 3.14
    s.commands[: n // 8] *= 0.05                                                # some near-zero commands
    s.actions = torch.rand(n, 12, generator=g) * 2 - 1
    s.last_actions = torch.rand(n, 12, generator=g) * 2 - 1
    s.last_dof_vel = s.dof_vel + torch.randn(n, 12, generator=g)
    s.torques = torch.randn(n, 12, generator=g) * 40
    s.feet_air_time = torch.rand(n, 4, generator=g) * (torch.rand(n, 4, generator=g) < 0.6)
    s.progress_buf = torch.randint(0, s.max_episode_length + 1, (n,), generator=g)
    s.timeout_buf = torch.zeros(n, dtype=torch.bool)
    s.reset_buf = torch.ones(n, dtype=torch.long)
    s.gravity_vec = torch.tensor([0.0, 0.0, -1.0]).repeat(n, 1); s.forward_vec = torch.tensor([1.0, 0, 0]).repeat(n, 1)
    s.episode_sums = {k: torch.zeros(n) for k in ("lin_vel_xy", "lin_vel_z", "ang_vel_z", "ang_vel_xy", "orient", "torques", "joint_acc",
                                                  "base_height", "air_time", "collision", "stumble", "action_rate", "hip")}
    inp = dict(root=root.numpy().copy(), dof_pos=s.dof_pos.numpy().copy(), dof_vel=s.dof_vel.numpy().copy(),
               contact_forces=cf.numpy().copy(), commands_in=s.commands.numpy().copy(), actions=s.actions.numpy().copy(),
               last_actions=s.last_actions.numpy().copy(), last_dof_vel=s.last_dof_vel.numpy().copy(), torques=s.torques.numpy().copy(),
               feet_air_time_in=s.feet_air_time.numpy().copy(), progress=s.progress_buf.numpy().copy(),
               height_samples=hs.numpy()[::8, ::8].copy(), default_dof_pos=default[0].numpy().copy())
    # ---- post_physics_step :464-471 ("prepare quantities"), replayed with the reference's jit functions
    s.base_quat = s.root_states[:, 3:7]
    s.base_lin_vel = tju.quat_rotate_inverse(s.base_quat, s.root_states[:, 7:10])
    s.base_ang_vel = tju.quat_rotate_inverse(s.base_quat, s.root_states[:, 10:13])
    s.projected_gravity = tju.quat_rotate_inverse(s.base_quat, s.gravity_vec)
    forward = tju.quat_apply(s.base_quat, s.forward_vec)
    heading = torch.atan2(forward[:, 1], forward[:, 0])
    s.commands[:, 2] = torch.clip(0.5 * at.wrap_to_pi(s.commands[:, 3] - heading), -1., 1.)
    # ---- the reference's own methods
    s.height_points = at.AnymalTerrain.init_height_points(s)
    s.get_heights = lambda env_ids=None: at.AnymalTerrain.get_heights(s, env_ids)
    at.AnymalTerrain.check_termination(s)
    reset = s.reset_buf.clone()
    at.AnymalTerrain.compute_reward(s)
    at.AnymalTerrain.compute_observations(s)
    out = dict(base_lin_vel=s.base_lin_vel.numpy(), base_ang_vel=s.base_ang_vel.numpy(), projected_gravity=s.projected_gravity.numpy(),
               commands=s.commands.numpy(), heading=heading.numpy(), reset=reset.numpy().astype(np.int64), rew=s.rew_buf.numpy(),
               feet_air_time=s.feet_air_time.numpy(), obs=s.obs_buf.numpy(), measured_heights=s.measured_heights.numpy(),
               episode_sums=np.stack([s.episode_sums[k].numpy() for k in s.episode_sums]),
               wrap_to_pi_in=np.linspace(-7, 7, 57).astype(np.float32),
               wrap_to_pi_out=at.wrap_to_pi(torch.linspace(-7, 7, 57)).numpy())
    np.savez_compressed(os.path.join(OUT, "anymal_terrain.npz"), **inp, **out)
    print("wrote anymal_terrain.npz", {k: v.shape for k, v in out.items() if hasattr(v, "shape")})


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    main()
