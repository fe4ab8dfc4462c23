"""ShadowHand physical domain randomisation on the device: the randomised instantiations of the free-object simulate and the
fused ShadowHand step read per-env object size / mass / friction, hand masses / drive gains / limits / friction, tendon damping
and a bound gravity vector."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GRAVITY = (0.3, -0.2, -9.5)


def _identity_tensors(sim, m, obj, nten, dev):
    """the DR tensors holding the model's own values"""
    from isaacgymenvs_b200 import engine as E
    n = sim.num_envs
    pos = np.asarray(m.drive_mode[1:]) == 1
    damp = np.where(pos, np.asarray(m.damping[1:]) + np.asarray(m.kd[1:]), m.damping[1:])
    stiff = np.where(pos, m.kp[1:], m.stiffness[1:])
    lim = np.asarray(m.limited[1:]) > 0
    dp = np.stack([damp, stiff, np.where(lim, m.lower[1:], -3e38), np.where(lim, m.upper[1:], 3e38)], -1).astype(np.float32)
    return {E.T_ENV_MASS_SCALE: torch.ones(n, m.nl, device=dev),
            E.T_ENV_DOF_PROPS: torch.tensor(dp, device=dev).unsqueeze(0).repeat(n, 1, 1).contiguous(),
            E.T_ENV_FRICTION: torch.full((n,), float(np.asarray(m.cp_mu)[0]), device=dev),
            E.T_ENV_OBJ_PROPS: torch.tensor([1.0, 1.0, obj["mu"], 0.0], device=dev).repeat(n, 1).contiguous(),
            E.T_ENV_TENDON_DAMPING: torch.full((n, nten), 0.1, device=dev),
            E.T_GRAVITY: torch.tensor([0.0, 0.0, -9.81], device=dev)}


def test_randomised_groups_match_oracle():
    """Groups of envs, each with its own object scale / mass / friction, hand link masses, drive gains (damping, kp), limits,
    hand friction and tendon damping, all under a non-default gravity: one simulate from contact-rich states equals the fp64
    oracle run per group with those values baked in, to the tolerances of test_hand_baseline_size_simulate_matches_oracle.
    The oracle has one object friction for the hand-object and the object-ground contacts, so groups 0-3 keep the hand's
    friction at the ground's (1.0: both combined values are equal) and are compared in every env; groups 4-7 also vary the
    hand's friction and are compared where the object is clear of the ground.  The oracle has one damping for all tendons:
    a group's four tendons share theirs."""
    from isaacgymenvs_b200 import engine
    from oracle.oracle import OracleSim
    from tests.hand_common import DT, SUBSTEPS, settled_states
    from tests.test_gpu_parity import _hand_sim, _hand_load
    n, ng = 1024, 8
    base, obj, tendons, _, root, dof, o, tgt = settled_states(n, 25, 5, threads=8)
    sim = _hand_sim(n, base, obj, tendons)
    _hand_load(sim, root, dof, o, tgt)
    dev = sim.device
    t = {k: sim._bind(k, v) for k, v in _identity_tensors(sim, base, obj, len(tendons), dev).items()}
    t[engine.T_GRAVITY].copy_(torch.tensor(GRAVITY))
    rs = sim.root_state.cpu().numpy().astype(np.float64).reshape(n, 3, 13)
    r64 = np.ascontiguousarray(rs[:, 0]); o64 = np.ascontiguousarray(rs[:, 1])
    d64 = sim.dof_state.cpu().numpy().astype(np.float64).reshape(n, base.ndof, 2)
    t64 = sim.dof_target.cpu().numpy().astype(np.float64)
    airborne = o64[:, 2] > 0.1
    rng = np.random.default_rng(7)
    nl, nd = base.nl, base.ndof
    pos = np.asarray(base.drive_mode[1:]) == 1
    lim = np.asarray(base.limited[1:]) > 0
    dp0 = t[engine.T_ENV_DOF_PROPS][0].cpu().numpy().astype(np.float64)
    keep = np.zeros(n, bool)
    for g in range(ng):
        sl = slice(g * n // ng, (g + 1) * n // ng)
        ms = rng.uniform(0.5, 1.5, size=nl).astype(np.float32)
        damp = (dp0[:, 0] * np.exp(rng.uniform(np.log(0.3), np.log(3.0), size=nd))).astype(np.float32)
        kp = (dp0[:, 1] * np.exp(rng.uniform(np.log(0.75), np.log(1.5), size=nd))).astype(np.float32)
        lo = np.where(lim, dp0[:, 2] + rng.normal(0, 0.01, size=nd), -3e38).astype(np.float32)
        hi = np.where(lim, dp0[:, 3] + rng.normal(0, 0.01, size=nd), 3e38).astype(np.float32)
        mu_h = np.float32(1.0 if g < 4 else rng.uniform(0.7, 1.3))
        s, mf, mu_o = (np.float32(v) for v in (rng.uniform(0.95, 1.05), rng.uniform(0.5, 1.5), rng.uniform(0.7, 1.3)))
        td = np.float32(0.1 * np.exp(rng.uniform(np.log(0.3), np.log(3.0))))
        t[engine.T_ENV_MASS_SCALE][sl] = torch.tensor(ms, device=dev)
        t[engine.T_ENV_DOF_PROPS][sl] = torch.tensor(np.stack([damp, kp, lo, hi], -1), device=dev)
        t[engine.T_ENV_FRICTION][sl] = float(mu_h)
        t[engine.T_ENV_OBJ_PROPS][sl] = torch.tensor([s, mf, mu_o, 0.0], device=dev)
        t[engine.T_ENV_TENDON_DAMPING][sl] = float(td)
        m = copy.deepcopy(base)
        m.mass = np.asarray(m.mass, float) * ms.astype(np.float64)
        m.inertia = np.asarray(m.inertia, float) * ms.astype(np.float64)[:, None]
        m.damping = np.concatenate([[0.0], damp.astype(np.float64)])
        m.kd = np.zeros(nl)                                                   # a position drive's damping is the joint damping
        m.kp = np.concatenate([[0.0], np.where(pos, kp.astype(np.float64), base.kp[1:])])
        m.stiffness = np.concatenate([[0.0], np.where(pos, base.stiffness[1:], kp.astype(np.float64))])
        m.lower = np.concatenate([[0.0], np.where(lim, lo.astype(np.float64), base.lower[1:])])
        m.upper = np.concatenate([[0.0], np.where(lim, hi.astype(np.float64), base.upper[1:])])
        m.cp_mu = np.full_like(np.asarray(m.cp_mu, float), float(mu_h))
        s64, mf64 = float(s), float(mf)
        ob = dict(obj, mass=obj["mass"] * mf64, inertia=[v * mf64 * s64 * s64 for v in obj["inertia"]],
                  half=[v * s64 for v in obj["half"]], round=obj.get("round", 0.0) * s64,
                  mu=0.5 * (float(mu_h) + float(mu_o)))
        orc = OracleSim(m, DT, SUBSTEPS, GRAVITY, ground_mu=1.0, obj=ob, tendons=tendons, tendon_k=30.0, tendon_d=float(td), threads=8)
        r = np.ascontiguousarray(r64[sl]); d = np.ascontiguousarray(d64[sl]); oo = np.ascontiguousarray(o64[sl])
        orc.simulate(r, d, target=np.ascontiguousarray(t64[sl]), obj=oo)
        r64[sl] = r; d64[sl] = d; o64[sl] = oo
        keep[sl] = True if g < 4 else airborne[sl]
    sim.simulate(); torch.cuda.synchronize()
    rg = sim.root_state.cpu().numpy().astype(np.float64).reshape(n, 3, 13)[keep]
    dg = sim.dof_state.cpu().numpy().astype(np.float64).reshape(n, nd, 2)[keep]
    assert keep.sum() > 0.75 * n
    assert np.abs(rg[:, 1, :3] - o64[keep, :3]).max() < 5e-5
    assert np.abs(dg[..., 0] - d64[keep, :, 0]).max() < 1e-4
    qerr = np.abs(dg[..., 1] - d64[keep, :, 1]) / np.maximum(1.0, np.abs(d64[keep, :, 1]))
    assert qerr.max() < 5e-3, qerr.max()
    sim.close()


def test_identity_parameters_equal_the_plain_kernels():
    """The randomised instantiations with every DR tensor holding the model's own values give bit-identical results to the
    plain kernels: simulate from contact-rich states, and 20 fused ShadowHand steps (resets included)."""
    from isaacgymenvs_b200 import config, engine
    from isaacgymenvs_b200.tasks import isaacgym_task_map
    from tests.hand_common import settled_states
    from tests.test_gpu_parity import _hand_sim, _hand_load
    n = 512
    base, obj, tendons, _, root, dof, o, tgt = settled_states(n, 25, 5, threads=8)
    outs = []
    for dr in (False, True):
        sim = _hand_sim(n, base, obj, tendons)
        _hand_load(sim, root, dof, o, tgt)
        if dr:
            for k, v in _identity_tensors(sim, base, obj, len(tendons), sim.device).items():
                sim._bind(k, v)
        sim.simulate(); torch.cuda.synchronize()
        outs.append([sim.root_state.cpu(), sim.dof_state.cpu(), sim.tensors[engine.T_FORCE_SENSOR].cpu()])
        sim.close()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    res = []
    for dr in (False, True):
        cfg = config.builtin_cfg("ShadowHand", {"sim_device": "cuda:0", "rl_device": "cuda:0"})
        cfg["task"]["env"]["numEnvs"] = n; cfg["task"]["seed"] = 42
        env = isaacgym_task_map["ShadowHand"](cfg=cfg["task"], rl_device="cuda:0", sim_device="cuda:0", graphics_device_id=-1, headless=True)
        if dr:
            for k, v in _identity_tensors(env.sim, env.model, env._obj, len(env._tendons), env.sim.device).items():
                env.sim._bind(k, v)
        g = torch.Generator(device="cuda:0").manual_seed(0)
        for _ in range(20):
            obs, rew, reset, _ = env.step(2 * torch.rand((n, 20), device="cuda:0", generator=g) - 1)
        torch.cuda.synchronize()
        res.append([obs["obs"].clone(), rew.clone(), reset.clone(), env.root_state_tensor.clone()])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_openai_ff_randomisation_stays_finite_at_16384_envs():
    """env.step() with the reference's full randomisation block (ShadowHand.yaml = ShadowHandOpenAI_FF.yaml) at 16384 envs for
    500 steps under random actions: every observation and reward stays finite."""
    from isaacgymenvs_b200 import config
    from isaacgymenvs_b200.tasks import isaacgym_task_map
    n = 16384
    cfg = config.builtin_cfg("ShadowHand", {"sim_device": "cuda:0", "rl_device": "cuda:0"})
    cfg["task"]["env"]["numEnvs"] = n; cfg["task"]["seed"] = 42
    cfg["task"]["task"]["randomize"] = True
    torch.manual_seed(0)
    env = isaacgym_task_map["ShadowHand"](cfg=cfg["task"], rl_device="cuda:0", sim_device="cuda:0", graphics_device_id=-1, headless=True)
    g = torch.Generator(device="cuda:0").manual_seed(1)
    ok = torch.ones((), dtype=torch.bool, device="cuda:0")
    for _ in range(500):
        obs, rew, reset, _ = env.step(2 * torch.rand((n, 20), device="cuda:0", generator=g) - 1)
        ok &= torch.isfinite(obs["obs"]).all() & torch.isfinite(rew).all()
    torch.cuda.synchronize()
    assert bool(ok)
    assert torch.isfinite(env.root_state_tensor).all() and torch.isfinite(env.dof_state).all()
