"""Ant and Humanoid domain randomisation on the device: the Humanoid step kernels' gravity-reading instantiations, the refusal of
a bound gravity vector by every kernel that would not read it, and the built-in randomisation blocks under random actions."""
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

GRAVITY = (0.3, -0.2, -9.5)


def _env(task, n, env=None, sim=None, randomize=False):
    from isaacgymenvs_b200 import config
    from isaacgymenvs_b200.tasks import isaacgym_task_map
    cfg = config.builtin_cfg(task, {"sim_device": "cuda:0", "rl_device": "cuda:0"})
    cfg["task"]["env"]["numEnvs"] = n; cfg["task"]["seed"] = 42
    cfg["task"]["env"].update(env or {})
    cfg["task"]["sim"].update(sim or {})
    cfg["task"]["task"]["randomize"] = randomize
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return isaacgym_task_map[task](cfg=cfg["task"], rl_device="cuda:0", sim_device="cuda:0", graphics_device_id=-1, headless=True)


def _run(env, steps=20):
    n = env.num_envs
    g = torch.Generator(device="cuda:0").manual_seed(0)
    resets = 0
    for _ in range(steps):
        resets += int(env.reset_buf.sum())
        obs, rew, reset, _ = env.step(2 * torch.rand((n, env.num_acts), device="cuda:0", generator=g) - 1)
    torch.cuda.synchronize()
    return resets, [obs["obs"].clone(), rew.clone(), reset.clone(), env.root_states.clone(), env.dof_state.clone(),
                    env.vec_sensor_tensor.clone(), env.dof_force_tensor.clone()]


@pytest.mark.parametrize("self_collision", [False, True])
@pytest.mark.parametrize("n", [512, 500])          # whole 16-env tiles (bulk-copy I/O), and not
def test_bound_configured_gravity_equals_the_plain_kernel(self_collision, n):
    """20 fused Humanoid steps (every env resets on the first) with the configured gravity bound: bit-identical to the plain
    kernel that reads the model's gravity."""
    from isaacgymenvs_b200 import engine
    out = []
    for bound in (False, True):
        env = _env("Humanoid", n, env={"selfCollision": self_collision})
        if bound:
            env.sim._bind(engine.T_GRAVITY, torch.tensor([0.0, 0.0, -9.81], device="cuda:0"))
        resets, res = _run(env)
        assert resets >= n
        out.append(res)
        env.sim.close()
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize("self_collision", [False, True])
def test_bound_gravity_equals_a_sim_created_with_it(self_collision):
    """A Humanoid with GRAVITY bound to (0.3, -0.2, -9.5) steps bit-identically to one created with that sim.gravity."""
    from isaacgymenvs_b200 import engine
    n = 512
    out = []
    for how in ("created", "bound", "default"):
        env = _env("Humanoid", n, env={"selfCollision": self_collision}, sim={"gravity": list(GRAVITY)} if how == "created" else None)
        if how == "bound":
            env.sim._bind(engine.T_GRAVITY, torch.tensor(GRAVITY, device="cuda:0"))
        out.append(_run(env)[1])
        env.sim.close()
    created, bound, default = out
    for x, y in zip(created, bound):
        assert torch.equal(x, y)
    assert not torch.equal(bound[3], default[3])                  # the bound vector is what the physics reads


def test_bound_gravity_refused_where_no_kernel_reads_it(monkeypatch):
    """Ant (four-chain step and simulate), Cartpole and a one-lane Humanoid (no gravity instantiation) refuse a bound gravity
    at the physics launch; the reset launch involves no gravity and runs."""
    from isaacgymenvs_b200 import engine
    grav = torch.tensor(GRAVITY, device="cuda:0")
    for task, nact in (("Ant", 8), ("Cartpole", 1)):
        env = _env(task, 64)
        env.sim._bind(engine.T_GRAVITY, grav)
        with pytest.raises(engine.EngineError, match="GRAVITY"):
            env.step(torch.zeros((64, nact), device="cuda:0"))
        with pytest.raises(engine.EngineError, match="GRAVITY"):
            env.sim.simulate()
        env.reset_buf[:] = 1
        env.reset_done()
        torch.cuda.synchronize()
        env.sim.close()
    monkeypatch.setenv("B2G_SINGLE_LANE", "1")
    env = _env("Humanoid", 64)
    env.sim._bind(engine.T_GRAVITY, grav)
    with pytest.raises(engine.EngineError, match="gravity bound 1"):
        env.step(torch.zeros((64, 21), device="cuda:0"))
    env.sim.close()


@pytest.mark.parametrize("task,n", [("Humanoid", 8192), ("Ant", 16384)])
def test_builtin_blocks_stay_finite(task, n):
    """env.step() with the built-in randomisation block for 1000 steps under random actions: every observation, reward and
    state stays finite."""
    torch.manual_seed(0)
    env = _env(task, n, randomize=True)
    assert env.physical_randomizer is not None
    g = torch.Generator(device="cuda:0").manual_seed(1)
    ok = torch.ones((), dtype=torch.bool, device="cuda:0")
    for _ in range(1000):
        obs, rew, reset, _ = env.step(2 * torch.rand((n, env.num_acts), device="cuda:0", generator=g) - 1)
        ok &= torch.isfinite(obs["obs"]).all() & torch.isfinite(rew).all()
    torch.cuda.synchronize()
    assert bool(ok)
    for t in (env.root_states, env.dof_state, env.potentials, env.prev_potentials, env.physical_randomizer.dof_props,
              env.physical_randomizer.friction):
        assert torch.isfinite(t).all()
    if task == "Humanoid":
        assert torch.isfinite(env.randomizer.gravity).all()
    env.sim.close()
