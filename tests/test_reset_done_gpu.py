"""GPU: VecTask.reset_done() (b2g_reset_flagged) leaves a flagged env in exactly the state the fused step's reset_idx gives it,
and leaves every other env alone.  With controlFrequencyInv = 0 the step runs no simulate, so its reset_idx is the only
writer of the reset envs' DOF, root and goal state: both paths run from the same snapshot and must agree bit for bit."""
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _flag_half(env, n):
    """reset_buf on about half the envs, reset counts spread over [0, 1000); returns the mask of flagged envs"""
    rng = np.random.default_rng(3)
    flag = rng.random(n) < 0.5
    env.reset_buf.copy_(torch.tensor(flag, dtype=torch.long, device=env.device))
    env.reset_count.copy_(torch.tensor(rng.integers(0, 1000, n), dtype=torch.int32, device=env.device))
    assert 0 < flag.sum() < n
    return flag


def _reset_done_vs_step(env, n, state, actions):
    """state: name -> tensor written by reset_done.  Returns (after reset_done, after step) as per-env numpy rows; asserts that
    reset_done changed no unflagged env"""
    flag = _flag_half(env, n)
    snap = {k: v.clone() for k, v in state.items()}
    rows = lambda: {k: v.detach().reshape(n, -1).cpu().numpy().copy() for k, v in state.items()}
    before = rows()
    env.reset_done()
    torch.cuda.synchronize()
    done = rows()
    for k in state:
        assert np.array_equal(done[k][~flag], before[k][~flag]), k
    for k, v in state.items():
        v.copy_(snap[k])
    env.step(actions)
    torch.cuda.synchronize()
    return flag, done, rows()


@pytest.mark.parametrize("variant", ["cube", "pen", "force"])
def test_hand_reset_done_matches_the_step_reset(variant):
    from tests.test_gpu_parity import _hand_env
    gold = np.load(os.path.join(GOLD, "shadow_hand.npz"))
    gi = lambda k: gold[f"a_in_{k}"]
    n = gi("reset").shape[0]
    more = {"pen": {"objectType": "pen"}, "force": {"forceScale": 2.0}}.get(variant, {})
    env = _hand_env(n, "a", "full_state", **more)
    dev = env.device
    t = lambda a, dt=torch.float32: torch.tensor(np.asarray(a), dtype=dt, device=dev)
    env.root_state_tensor.copy_(t(gi("root")))
    env.initial_root_states.view(n, 3, 13)[:, 1].copy_(t(gi("object_init")))
    env.initial_root_states.view(n, 3, 13)[:, 2].copy_(t(gi("goal_init")))
    env.dof_state.copy_(t(gi("dof_state")))
    env.prev_targets.copy_(t(gi("prev_targets"))); env.cur_targets.copy_(t(gi("cur_targets")))
    env.goal_states.copy_(t(gi("goal_states")))
    env.vec_sensor_tensor.copy_(t(gi("sensors"))); env.dof_force_tensor.copy_(t(gi("dof_force")))
    env.reset_goal_buf.copy_(t(gi("reset_goal"), torch.long))
    env.progress_buf.copy_(t(gi("progress"), torch.long)); env.successes.copy_(t(gi("successes")))
    env.goal_reset_count.copy_(t(gi("goal_reset_count"), torch.int32))
    state = {"root": env.root_state_tensor, "dof": env.dof_state, "goal": env.goal_states, "cur": env.cur_targets,
             "prev": env.prev_targets, "reset": env.reset_buf, "reset_goal": env.reset_goal_buf, "progress": env.progress_buf,
             "successes": env.successes, "count": env.reset_count, "goal_count": env.goal_reset_count}
    if variant == "force":
        assert env.sim.task.force_scale > 0
        env.object_rb_forces.normal_()
        state.update(force=env.object_rb_forces, force_prob=env.random_force_prob)
    flag, done, stepped = _reset_done_vs_step(env, n, state, t(gi("actions")))
    free = np.setdiff1d(np.arange(env.num_dofs), env.actuated_dof_indices_np)      # DOFs no action drives
    assert len(free) > 0
    checks = {"dof": slice(None), "root": slice(13, 39), "goal": slice(None), "count": slice(None), "cur": free, "prev": free}
    if variant == "force":
        checks["force_prob"] = slice(None)
        assert np.all(done["force"][flag] == 0.0)
    for k, cols in checks.items():
        assert np.array_equal(done[k][flag][:, cols], stepped[k][flag][:, cols]), k
    env.sim.close()


@pytest.mark.parametrize("task", ["Cartpole", "Ant", "Humanoid"])
def test_reset_done_matches_the_step_reset(task):
    from tests.test_gpu_parity import _make
    n = 256
    env = _make(task, n, controlFrequencyInv=0)
    state = {"dof": env.dof_state, "reset": env.reset_buf, "progress": env.progress_buf, "count": env.reset_count}
    if task != "Cartpole":
        state.update(root=env.root_states, pot=env.potentials, ppot=env.prev_potentials)
    g = torch.Generator(device=env.device).manual_seed(0)
    actions = 2 * torch.rand((n, env.num_actions), device=env.device, generator=g) - 1
    flag, done, stepped = _reset_done_vs_step(env, n, state, actions)
    for k in [k for k in state if k not in ("reset", "progress")]:
        assert np.array_equal(done[k][flag], stepped[k][flag]), k
    env.sim.close()
