"""ShadowHand physical domain randomisation on the CPU: the reference's ShadowHand.yaml randomization_params block (two actor
types, tendon_properties, the object's scale, bucketed friction, sim_params.gravity) on the fused task with the engine
replaced by the stand-in of tests/test_fused_host_path.py.  The kernels that read the bound tensors are covered by
tests/test_hand_domain_randomisation_gpu.py."""
import os

import numpy as np
import pytest
import torch

from tests.test_fused_host_path import _make, fused_cpu  # noqa: F401  (fixture)


@pytest.fixture
def dr_block():
    """randomization_params of the reference's ShadowHand.yaml (unpacked from tests/golden/reference_data.tar.xz)"""
    import yaml
    from tests.conftest import REFERENCE
    with open(os.path.join(REFERENCE, "isaacgymenvs", "cfg", "task", "ShadowHand.yaml")) as f:
        return yaml.safe_load(f)["task"]["randomization_params"]


def _hand(n, dr):
    return _make("ShadowHand", n, task_section={"randomize": True, "randomization_params": dr})


def _on_grid(v, lo, hi, nb):
    k = (v - lo) / ((hi - lo) / nb)
    return torch.allclose(k, torch.round(k), atol=1e-3)


def test_construction_binds_every_slot(fused_cpu, dr_block):
    n = 64
    torch.manual_seed(0)
    env = _hand(n, dr_block)
    E, b = env.sim.E, env.sim.bound
    nl, nd = env.model.nl, env.model.ndof
    assert b[E.T_ENV_MASS_SCALE].shape == (n, nl) and b[E.T_ENV_DOF_PROPS].shape == (n, nd, 4)
    assert b[E.T_ENV_FRICTION].shape == (n,) and b[E.T_ENV_OBJ_PROPS].shape == (n, 4)
    assert b[E.T_ENV_TENDON_DAMPING].shape == (n, 4) and b[E.T_GRAVITY].shape == (3,)


def test_samples_in_range_loguniform_and_buckets(fused_cpu, dr_block):
    n = 4096
    torch.manual_seed(1)
    env = _hand(n, dr_block)
    pr, E, b = env.physical_randomizer, env.sim.E, env.sim.bound
    og = pr.og_dof
    pos = torch.tensor(np.asarray(env.model.drive_mode[1:]) == 1)
    assert pos.sum() == 20                          # the actuated DOFs: og damping = joint damping + kd, og stiffness = kp
    t = lambda a: torch.tensor(np.asarray(a)[1:], dtype=torch.float32)
    assert torch.allclose(og[:, 0], torch.where(pos, t(env.model.damping) + t(env.model.kd), t(env.model.damping)))
    assert torch.allclose(og[:, 1], torch.where(pos, t(env.model.kp), t(env.model.stiffness)))
    dp = b[E.T_ENV_DOF_PROPS][:, pos]
    og = og[pos]
    f = dp[..., 0] / og[:, 0]
    assert (f >= 0.3 - 1e-5).all() and (f <= 3.0 + 1e-5).all()
    lf = torch.log(f[:, 0])                                                # loguniform: log of the factor is uniform
    assert abs(float(lf.mean()) - 0.5 * (np.log(0.3) + np.log(3.0))) < 0.05 and float((f[:, 0] < 1.0).float().mean()) > 0.45
    k = dp[..., 1] / og[:, 1]
    assert (k >= 0.75 - 1e-5).all() and (k <= 1.5 + 1e-5).all()
    lim = pr.limited[pos]
    assert (dp[:, lim, 2] - og[lim, 2]).abs().max() < 0.06 and (dp[:, lim, 2] - og[lim, 2]).abs().max() > 1e-3
    td = b[E.T_ENV_TENDON_DAMPING] / 0.1
    assert (td >= 0.3 - 1e-5).all() and (td <= 3.0 + 1e-5).all() and td.std() > 0.3      # per tendon
    assert not torch.equal(td[:, 0], td[:, 1])
    ms = b[E.T_ENV_MASS_SCALE]
    assert (ms >= 0.5).all() and (ms <= 1.5).all()
    fr = b[E.T_ENV_FRICTION]
    assert (fr >= 0.7 - 1e-6).all() and (fr < 1.3).all() and _on_grid(fr, 0.7, 1.3, 250) and fr.unique().numel() > 100
    op = b[E.T_ENV_OBJ_PROPS]
    assert (op[:, 0] >= 0.95).all() and (op[:, 0] <= 1.05).all() and op[:, 0].std() > 0.02      # scale
    assert (op[:, 1] >= 0.5).all() and (op[:, 1] <= 1.5).all()                                     # mass factor
    assert (op[:, 2] >= 0.7 - 1e-6).all() and (op[:, 2] < 1.3).all() and _on_grid(op[:, 2], 0.7, 1.3, 250)
    assert (op[:, 3] == 0).all()


def test_setup_only_once_and_redraw_rule(fused_cpu, dr_block):
    n = 64
    dr = dict(dr_block, frequency=3)
    torch.manual_seed(2)
    env = _hand(n, dr)
    E, b = env.sim.E, env.sim.bound
    ms, dp, op, fr, td, g = (b[s] for s in (E.T_ENV_MASS_SCALE, E.T_ENV_DOF_PROPS, E.T_ENV_OBJ_PROPS, E.T_ENV_FRICTION,
                                           E.T_ENV_TENDON_DAMPING, E.T_GRAVITY))
    snap = lambda: [t.clone() for t in (ms, dp, op, fr, td)]
    s0 = snap()
    a = torch.zeros(n, 20)
    env.step(a)                                        # all envs reset (first step), counters 0 < 3: nothing per-env changes
    assert all(torch.equal(x, y) for x, y in zip(s0, snap()))
    for _ in range(3):
        env.step(a)                                    # the stand-in clears reset_buf: no reset, no randomisation
    assert all(torch.equal(x, y) for x, y in zip(s0, snap()))
    env.reset_buf[: n // 2] = 1
    env.step(a)
    changed = (dp != s0[1]).any(-1).any(-1)
    assert changed[: n // 2].all() and not changed[n // 2:].any()
    tch = (td != s0[4]).any(-1)
    assert tch[: n // 2].all() and not tch[n // 2:].any()
    fch = fr != s0[3]
    assert not fch[n // 2:].any() and fch[: n // 2].float().mean() > 0.8
    assert torch.equal(ms, s0[0])                                         # setup_only: hand mass
    assert torch.equal(op[:, :2], s0[2][:, :2])                          # setup_only: object scale and mass
    och = op[:, 2] != s0[2][:, 2]
    assert not och[n // 2:].any() and och[: n // 2].float().mean() > 0.8   # object friction is redrawn
    assert (env.randomize_buf[: n // 2] <= 1).all() and (env.randomize_buf[n // 2:] >= 4).all()


def test_gravity_redrawn_every_frequency_frames_on_reset_steps(fused_cpu, dr_block):
    n = 16
    dr = dict(dr_block, frequency=4)
    torch.manual_seed(3)
    env = _hand(n, dr)
    g = env.sim.bound[env.sim.E.T_GRAVITY]
    g_og = torch.tensor([0.0, 0.0, -9.81])
    assert torch.equal(g, g_og)                                    # drawn with the first randomising step
    a = torch.zeros(n, 20)
    env.step(a)                                                    # frame 0, every env resets: first draw
    g1 = g.clone()
    assert not torch.equal(g1, g_og) and (g1 - g_og).abs().max() < 0.4 * 6
    for _ in range(5):
        env.step(a)                                                # frames 1..5: no reset, no draw even past the frequency
    assert torch.equal(g, g1)
    env.reset_buf[0] = 1
    env.step(a)                                                    # frame 6 >= 0 + 4 with a reset: redraw
    g2 = g.clone()
    assert not torch.equal(g2, g1)
    env.reset_buf[0] = 1
    env.step(a)                                                    # frame 7: 7 - 6 < 4
    assert torch.equal(g, g2)


def test_random_force_mass_stays_unrandomised(fused_cpu, dr_block):
    n = 32
    torch.manual_seed(4)
    env = _make("ShadowHand", n, env={"forceScale": 2.0}, task_section={"randomize": True, "randomization_params": dr_block})
    op = env.sim.bound[env.sim.E.T_ENV_OBJ_PROPS]
    assert op[:, 1].std() > 0.05
    assert env.object_rb_masses.shape == (1,) and abs(float(env.object_rb_masses[0]) - env._obj["mass"]) < 1e-7
    assert abs(float(env.sim.ext.obj_mass) - env._obj["mass"]) < 1e-6          # the model's object mass (force scale) is unchanged


def test_refused_where_not_provided(fused_cpu, dr_block):
    n = 8
    with pytest.raises(NotImplementedError):              # gravity is only read by the free-object kernels
        _make("Ant", n, task_section={"randomize": True, "randomization_params": {"frequency": 1, "sim_params": {"gravity": dr_block["sim_params"]["gravity"]}}})
    with pytest.raises(NotImplementedError):
        _hand(n, dict(dr_block, sim_params={"rest_offset": {"range": [0, 1], "operation": "additive", "distribution": "uniform"}}))
    with pytest.raises(NotImplementedError):
        _hand(n, dict(dr_block, actor_params={"goal": {"scale": dr_block["actor_params"]["object"]["scale"]}}))
    env = _hand(n, dr_block)
    from isaacgymenvs_b200 import engine
    with pytest.raises(engine.EngineError):
        env.rollout(torch.zeros(2, n, 20))
