"""Ant and Humanoid physical domain randomisation on the CPU: the built-in randomization_params blocks (restated from the
reference's Ant.yaml / Humanoid.yaml, checked against them by tests/test_host_side.py) on the fused tasks with the engine
replaced by the stand-in of tests/test_fused_host_path.py.  The Humanoid kernels that read the bound gravity are covered by
tests/test_locomotion_domain_randomisation_gpu.py."""
import copy
import importlib.util
import os

import pytest
import torch

from tests.test_fused_host_path import _make, fused_cpu  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = torch.tensor([0.0, 0.0, -9.81])


def _humanoid(n, dr=None):
    sec = {"randomize": True}
    if dr is not None:
        sec["randomization_params"] = dr
    return _make("Humanoid", n, task_section=sec)


def test_builtin_humanoid_binds_mass_dof_friction_and_gravity(fused_cpu):
    n = 32
    env = _humanoid(n)
    E, b = env.sim.E, env.sim.bound
    nl, nd = env.model.nl, env.model.ndof
    assert b[E.T_ENV_MASS_SCALE].shape == (n, nl) and b[E.T_ENV_DOF_PROPS].shape == (n, nd, 4)
    assert b[E.T_ENV_FRICTION].shape == (n,) and b[E.T_GRAVITY].shape == (3,)
    assert E.T_ENV_OBJ_PROPS not in b and E.T_ENV_TENDON_DAMPING not in b


def test_humanoid_frame_zero_draws_are_the_identity(fused_cpu):
    """The linear schedule at frame 0 (apply_random_samples at step 0 in the reference): every scaling factor is exactly 1,
    every additive sample exactly 0, so the first step runs the configured model under the configured gravity."""
    n = 256
    torch.manual_seed(0)
    env = _humanoid(n)
    E, b, pr = env.sim.E, env.sim.bound, env.physical_randomizer
    env.step(torch.zeros(n, 21))                                  # frame 0, every env resets: the first gravity draw
    assert (b[E.T_ENV_MASS_SCALE] == 1.0).all()
    assert torch.equal(b[E.T_ENV_DOF_PROPS], pr.og_dof.unsqueeze(0).expand(n, -1, -1))
    assert (b[E.T_ENV_FRICTION] == pr.og_friction).all()
    assert torch.equal(b[E.T_GRAVITY], G)


def test_humanoid_redraw_on_reset_steps_with_the_schedule_spread(fused_cpu):
    """Past the frequency (600 frames), a step with resets redraws the flagged envs whose counters passed it, with the spread
    the linear schedule gives at that frame (frame / 3000), and redraws gravity; a step without resets changes nothing."""
    n = 4096
    q = n // 4
    torch.manual_seed(1)
    env = _humanoid(n)
    E, b, pr = env.sim.E, env.sim.bound, env.physical_randomizer
    ms, dp, fr, g = (b[s] for s in (E.T_ENV_MASS_SCALE, E.T_ENV_DOF_PROPS, E.T_ENV_FRICTION, E.T_GRAVITY))
    a = torch.zeros(n, 21)
    env.step(a)                                                   # frame 0
    s0 = [t.clone() for t in (ms, dp, fr, g)]
    frame = 1500
    s = frame / 3000
    env.control_steps = frame
    env.randomize_buf[: 2 * q] = 700                              # counters past the frequency ...
    env.randomize_buf[2 * q:] = 10
    env.reset_buf[:q] = 1                                         # ... flagged: envs [0, q) are redrawn
    env.reset_buf[2 * q: 3 * q] = 1                               # flagged, counter below the frequency: kept
    env.step(a)
    changed = (dp != s0[1]).any(-1).any(-1)
    assert changed[:q].all() and not changed[q:].any()
    assert not (fr[q:] != s0[2][q:]).any() and (fr[:q] != s0[2][:q]).float().mean() > 0.99
    assert torch.equal(ms, s0[0])                                 # setup_only
    og = pr.og_dof
    damp = dp[:q, :, 0] / og[:, 0]                                # uniform on [1 - 0.5 s, 1 + 0.5 s]
    assert damp.min() >= 1 - 0.5 * s - 1e-6 and damp.max() <= 1 + 0.5 * s + 1e-6
    assert abs(float(damp.std()) - s / 12 ** 0.5) < 0.05 * s / 12 ** 0.5
    f = fr[:q] / pr.og_friction                                   # uniform on [1 - 0.3 s, 1 + 0.3 s], no buckets
    assert f.min() >= 1 - 0.3 * s - 1e-6 and f.max() <= 1 + 0.3 * s + 1e-6 and f.unique().numel() > q // 2
    lim = pr.limited
    dl = dp[:q, lim, 2] - og[lim, 2]                              # N(0, 0.01 s)
    assert abs(float(dl.std()) - 0.01 * s) < 0.05 * 0.01 * s
    assert not torch.equal(g, s0[3]) and (g - G).abs().max() < 6 * 0.4 * s   # gravity: G + N(0, 0.4 s) per component
    s1 = [t.clone() for t in (ms, dp, fr, g)]
    env.control_steps = frame + 1000                              # the frequency elapsed again, but no env resets
    env.randomize_buf[:] = 700
    env.step(a)
    assert all(torch.equal(x, y) for x, y in zip(s1, (ms, dp, fr, g)))


def test_restitution_scaling_only(fused_cpu):
    from isaacgymenvs_b200 import config
    dr = copy.deepcopy(config.builtin_cfg("Humanoid")["task"]["task"]["randomization_params"])
    torch.manual_seed(2)
    env = _humanoid(8, dr)                                        # scaling: drawn, nothing bound for it
    assert "restitution" in env.physical_randomizer.props["rigid_shape_properties"]
    dr["actor_params"]["humanoid"]["rigid_shape_properties"]["restitution"]["operation"] = "additive"
    with pytest.raises(NotImplementedError):
        _humanoid(8, dr)


def test_builtin_ant_binds_mass_and_dof_only(fused_cpu):
    n = 32
    env = _make("Ant", n, task_section={"randomize": True})
    E, b = env.sim.E, env.sim.bound
    assert b[E.T_ENV_MASS_SCALE].shape == (n, env.model.nl) and b[E.T_ENV_DOF_PROPS].shape == (n, env.model.ndof, 4)
    assert E.T_ENV_FRICTION not in b and E.T_GRAVITY not in b
    assert env.randomizer.gravity is None


def test_train_launcher_maps_randomize(monkeypatch):
    spec = importlib.util.spec_from_file_location("b2g_train", os.path.join(ROOT, "train.py"))
    tr = importlib.util.module_from_spec(spec); spec.loader.exec_module(tr)
    on = tr.to_ppo_argv(tr.parse_overrides(["task=Humanoid", "task.task.randomize=True"]))
    off = tr.to_ppo_argv(tr.parse_overrides(["task=Humanoid", "task.task.randomize=False"]))
    assert "--randomize" in on and "--randomize" not in off and "--env" not in on
    with pytest.raises(SystemExit):
        tr.to_ppo_argv(tr.parse_overrides(["task=Humanoid", "task.task.randomize=maybe"]))
    # tools/train_ppo.py puts it into the task config it hands to make()
    import sys
    import isaacgymenvs_b200
    monkeypatch.syspath_prepend(os.path.join(ROOT, "tools"))
    sys.modules.pop("train_ppo", None)
    import train_ppo
    seen = {}

    class _Stop(Exception):
        pass

    def make(**kw):
        seen.update(kw)
        raise _Stop

    monkeypatch.setattr(isaacgymenvs_b200, "make", make)
    with pytest.raises(_Stop):
        train_ppo.main(on)
    assert seen["cfg"]["task"]["task"]["randomize"] is True and seen["task"] == "Humanoid"
