"""Generate golden input/output vectors from the REFERENCE's own @torch.jit.script functions.

Run in the build container only (needs an IsaacGymEnvs checkout named by ISAACGYMENVS_ROOT):
    python tests/golden/make_golden.py
The reference task modules are loaded BY PATH from that checkout with `isaacgym` and the VecTask
base stubbed out (SURVEY.md 8c) -- nothing is copied.  Outputs: tests/golden/*.npz (committed).
Pins: compute_ant_observations / compute_ant_reward (tasks/ant.py:325-408),
compute_humanoid_observations / compute_humanoid_reward (tasks/humanoid.py:323-413),
compute_cartpole_reward (tasks/cartpole.py:180-196) and the quaternion helpers they call
(utils/torch_jit_utils.py).
"""
import importlib.util
import os
import sys
import types
import numpy as np
import torch

REF = os.path.join(os.environ.get("ISAACGYMENVS_ROOT", "."), "isaacgymenvs")     # an IsaacGymEnvs checkout
OUT = os.path.dirname(os.path.abspath(__file__))


def load_reference_modules():
    for name in ("isaacgym", "isaacgym.gymtorch", "isaacgym.gymapi", "isaacgym.gymutil", "isaacgym.terrain_utils"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["isaacgym"].gymtorch = sys.modules["isaacgym.gymtorch"]
    sys.modules["isaacgym"].gymapi = sys.modules["isaacgym.gymapi"]
    for name in ("isaacgymenvs", "isaacgymenvs.utils", "isaacgymenvs.tasks", "isaacgymenvs.tasks.base"):
        sys.modules.setdefault(name, types.ModuleType(name))
    vt = types.ModuleType("isaacgymenvs.tasks.base.vec_task")
    vt.VecTask = type("VecTask", (), {})
    sys.modules["isaacgymenvs.tasks.base.vec_task"] = vt

    def load(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod
    tju = load("isaacgymenvs.utils.torch_jit_utils", "utils/torch_jit_utils.py")
    ant = load("ref_ant", "tasks/ant.py")
    hum = load("ref_humanoid", "tasks/humanoid.py")
    sys.modules["isaacgymenvs.tasks"].__path__ = []
    cart = load("isaacgymenvs.tasks.cartpole", "tasks/cartpole.py")
    return tju, ant, hum, cart


def rand_quat(g, n):
    q = torch.randn(n, 4, generator=g)
    return q / q.norm(dim=-1, keepdim=True)


def locomotion_inputs(g, n, nd, nsens, lo, hi, dt):
    root = torch.zeros(n, 13)
    root[:, 0:2] = torch.randn(n, 2, generator=g) * 20.0
    root[:, 2] = torch.rand(n, generator=g) * 1.2 + 0.1
    root[:, 3:7] = rand_quat(g, n)
    # a quarter of the envs nearly upright and facing +x, so the thresholds in the reward trigger
    k = n // 4
    small = torch.randn(k, 3, generator=g) * 0.1
    root[:k, 3:6] = small
    root[:k, 6] = 1.0
    root[:k, 3:7] /= root[:k, 3:7].norm(dim=-1, keepdim=True)
    root[:, 7:13] = torch.randn(n, 6, generator=g)
    lo_t, hi_t = torch.tensor(lo, dtype=torch.float), torch.tensor(hi, dtype=torch.float)
    u = torch.rand(n, nd, generator=g) * 1.1 - 0.05          # a few beyond the limits
    dof_pos = lo_t + (hi_t - lo_t) * u
    dof_vel = torch.randn(n, nd, generator=g) * 3.0
    sensors = torch.randn(n, nsens * 6, generator=g) * 5.0
    actions = torch.rand(n, nd, generator=g) * 2 - 1
    targets = torch.tensor([1000.0, 0, 0]).repeat(n, 1)
    potentials = -(1000.0 + torch.randn(n, generator=g) * 30) / dt
    return root, dof_pos, dof_vel, sensors, actions, targets, potentials, lo_t, hi_t


def main():
    tju, ant, hum, cart = load_reference_modules()
    g = torch.Generator().manual_seed(1234)
    n = 512
    dt = 0.0166
    inv_start_rot = torch.tensor([0.0, 0, 0, 1]).repeat(n, 1)
    b0 = torch.tensor([1.0, 0, 0]).repeat(n, 1)
    b1 = torch.tensor([0.0, 0, 1]).repeat(n, 1)

    # ---------------- Ant (cfg/task/Ant.yaml values)
    lo = np.radians([-40, 30, -40, -100, -40, -100, -40, 30]).astype(np.float32)
    hi = np.radians([40, 100, 40, -30, 40, -30, 40, 100]).astype(np.float32)
    root, dof_pos, dof_vel, sensors, actions, targets, potentials, lo_t, hi_t = locomotion_inputs(g, n, 8, 4, lo, hi, dt)
    obs, pot, prev_pot, up_vec, heading_vec = ant.compute_ant_observations(
        torch.zeros(n, 60), root.clone(), targets, potentials.clone(), inv_start_rot, dof_pos, dof_vel,
        lo_t, hi_t, 0.2, sensors, actions, dt, 0.1, b0, b1, 2)
    progress = torch.randint(0, 1002, (n,), generator=g)
    reset_in = torch.zeros(n, dtype=torch.long)
    rew, reset = ant.compute_ant_reward(obs, reset_in, progress, actions, 0.1, 0.5, pot, prev_pot,
                                        0.005, 0.05, 0.1, 0.31, -2.0, 1000.0)
    np.savez_compressed(os.path.join(OUT, "ant_obs_reward.npz"),
                        root=root.numpy(), dof_pos=dof_pos.numpy(), dof_vel=dof_vel.numpy(), sensors=sensors.numpy(),
                        actions=actions.numpy(), potentials_in=potentials.numpy(), lower=lo, upper=hi,
                        progress=progress.numpy(), obs=obs.numpy(), potentials=pot.numpy(), prev_potentials=prev_pot.numpy(),
                        up_vec=up_vec.numpy(), heading_vec=heading_vec.numpy(), rew=rew.numpy(), reset=reset.numpy(),
                        dt=np.float64(dt))

    # ---------------- Humanoid (cfg/task/Humanoid.yaml values)
    from isaacgymenvs_b200.assets import load_compiled
    hm = load_compiled("humanoid")
    lo = np.minimum(hm.lower[1:], hm.upper[1:]).astype(np.float32)
    hi = np.maximum(hm.lower[1:], hm.upper[1:]).astype(np.float32)
    root, dof_pos, dof_vel, sensors, actions, targets, potentials, lo_t, hi_t = locomotion_inputs(g, n, 21, 2, lo, hi, dt)
    root[:, 2] = torch.rand(n, generator=g) * 1.5 + 0.3
    dof_force = torch.randn(n, 21, generator=g) * 40
    motor_efforts = torch.tensor(hm.actuator_gear, dtype=torch.float)
    obs, pot, prev_pot, up_vec, heading_vec = hum.compute_humanoid_observations(
        torch.zeros(n, 108), root.clone(), targets, potentials.clone(), inv_start_rot, dof_pos, dof_vel, dof_force,
        lo_t, hi_t, 0.1, sensors, actions, dt, 0.01, 0.25, b0, b1)
    progress = torch.randint(0, 1002, (n,), generator=g)
    rew, reset = hum.compute_humanoid_reward(obs, torch.zeros(n, dtype=torch.long), progress, actions, 0.1, 0.5, pot,
                                             prev_pot, 0.01, 0.05, 0.25, float(motor_efforts.max()), motor_efforts,
                                             0.8, -1.0, 1000.0)
    np.savez_compressed(os.path.join(OUT, "humanoid_obs_reward.npz"),
                        root=root.numpy(), dof_pos=dof_pos.numpy(), dof_vel=dof_vel.numpy(), dof_force=dof_force.numpy(),
                        sensors=sensors.numpy(), actions=actions.numpy(), potentials_in=potentials.numpy(), lower=lo, upper=hi,
                        motor_efforts=motor_efforts.numpy(), progress=progress.numpy(), obs=obs.numpy(),
                        potentials=pot.numpy(), prev_potentials=prev_pot.numpy(), up_vec=up_vec.numpy(),
                        heading_vec=heading_vec.numpy(), rew=rew.numpy(), reset=reset.numpy(), dt=np.float64(dt))

    # ---------------- Cartpole
    pole_angle = torch.randn(n, generator=g) * 1.0
    pole_vel = torch.randn(n, generator=g) * 3
    cart_vel = torch.randn(n, generator=g) * 2
    cart_pos = torch.randn(n, generator=g) * 2
    progress = torch.randint(0, 502, (n,), generator=g)
    rew, reset = cart.compute_cartpole_reward(pole_angle, pole_vel, cart_vel, cart_pos, 3.0,
                                              torch.zeros(n, dtype=torch.long), progress, 500.0)
    np.savez_compressed(os.path.join(OUT, "cartpole_reward.npz"), pole_angle=pole_angle.numpy(), pole_vel=pole_vel.numpy(),
                        cart_vel=cart_vel.numpy(), cart_pos=cart_pos.numpy(), progress=progress.numpy(),
                        rew=rew.numpy(), reset=reset.numpy())

    # ---------------- quaternion helpers (known-answer vectors for the device math)
    qa, qb = rand_quat(g, n), rand_quat(g, n)
    v = torch.randn(n, 3, generator=g)
    r, p, y = tju.get_euler_xyz(qa)
    np.savez_compressed(os.path.join(OUT, "quat_ops.npz"), qa=qa.numpy(), qb=qb.numpy(), v=v.numpy(),
                        quat_mul=tju.quat_mul(qa, qb).numpy(), quat_rotate=tju.quat_rotate(qa, v).numpy(),
                        quat_rotate_inverse=tju.quat_rotate_inverse(qa, v).numpy(), quat_apply=tju.quat_apply(qa, v).numpy(),
                        roll=r.numpy(), pitch=p.numpy(), yaw=y.numpy(),
                        normalize_angle=tju.normalize_angle(v[:, 0] * 3).numpy())
    print("golden vectors written to", OUT)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    main()
