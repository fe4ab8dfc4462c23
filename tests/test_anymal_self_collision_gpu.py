"""Link-link contact of ANYmal on the four-chain (quad) kernels, on the GPU: b2g_simulate against the fp64 oracle on the plane
and a height field, against the generic sub-step (B2G_NO_QUAD=1), and AnymalTerrain with env.selfCollision=True."""
import copy
import os
import subprocess
import sys
import warnings
import numpy as np
import pytest
import torch

from tests.anymal_self_common import G, anymal_self, crossed_states, sphere_overlap, compare_layered, per_link_contact
from tests.test_gpu_parity2 import _make_anymal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT, SUB = 0.005, 1


def _sim(m, n, hfk=None):
    from isaacgymenvs_b200 import engine
    kw = {}
    if hfk is not None:
        kw = dict(hfield=hfk["hfield"], hf_horizontal_scale=hfk["hf_scale"], hf_vertical_scale=hfk["hf_vscale"], hf_origin=hfk["hf_origin"])
    return engine.Sim(m, n, DT, SUB, G, **kw)


def _run(sim, root, dof, tau):
    from isaacgymenvs_b200 import engine
    nc = sim.acquire(engine.T_NET_CONTACT)
    sim.root_state.copy_(torch.tensor(root, dtype=torch.float32)); sim.dof_state.copy_(torch.tensor(dof.reshape(-1, 2), dtype=torch.float32))
    sim.dof_actuation.copy_(torch.tensor(tau, dtype=torch.float32))
    sim.simulate(); torch.cuda.synchronize()
    n = root.shape[0]
    return (sim.root_state.cpu().numpy().astype(np.float64), sim.dof_state.cpu().numpy().astype(np.float64).reshape(n, -1, 2),
            nc.cpu().numpy().reshape(n, -1, 3))


@pytest.mark.parametrize("terrain", ["plane", "heightfield"])
def test_quad_self_simulate_matches_oracle(terrain):
    """4096 crossed-leg states, some on the ground: the quad kernel with link-link contact vs the oracle, states and the
    net contact tensor (summed per link on the oracle's side)"""
    from oracle.oracle import OracleSim
    m = anymal_self()
    n = 4096
    rng = np.random.default_rng(23)
    hfk = None
    if terrain == "heightfield":
        hfk = dict(hfield=rng.uniform(0, 40, size=(64, 64)).astype(np.int16), hf_scale=0.25, hf_vscale=0.005, hf_origin=(-8.0, -8.0))
    root, dof = crossed_states(m, n, rng)
    if hfk is not None:
        root[:, 0:2] = rng.uniform(-5, 5, size=(n, 2))
    tau = rng.uniform(-1, 1, size=(n, m.ndof)) * 40.0
    sim = _sim(m, n, hfk)
    assert sim.quad_ns() == 3
    r32 = root.astype(np.float32).astype(np.float64); d32 = dof.astype(np.float32).astype(np.float64); t32 = tau.astype(np.float32).astype(np.float64)
    okw = {} if hfk is None else dict(hfield=hfk["hfield"].astype(np.float64) * hfk["hf_vscale"], hf_scale=hfk["hf_scale"], hf_origin=hfk["hf_origin"])
    orc = OracleSim(m, DT, SUB, G, ground_mu=1.0, threads=16, **okw)
    dep = sphere_overlap(m, orc, r32, d32)
    assert (dep > 0).mean() > 0.15, (dep > 0).mean()
    rg, dg, nc = _run(sim, root, dof, tau)
    r64, d64 = r32.copy(), d32.copy()
    out = orc.simulate(r64, d64, t32)
    compare_layered(m, rg, dg, r64, d64, nc, out["contact_force"])
    sim.close()


def test_quad_self_matches_generic_sub_step():
    """the same self-colliding sim on the generic Stepper (B2G_NO_QUAD=1, in a subprocess): the two engine formulations of
    the same contact, on the plane"""
    m = anymal_self()
    n = 4096
    rng = np.random.default_rng(29)
    root, dof = crossed_states(m, n, rng)
    tau = rng.uniform(-1, 1, size=(n, m.ndof)) * 40.0
    sim = _sim(m, n)
    assert sim.quad_ns() == 3
    rq, dq, ncq = _run(sim, root, dof, tau)
    sim.close()
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        np.savez(os.path.join(td, "in.npz"), root=root, dof=dof, tau=tau)
        code = ("import numpy as np, sys; sys.path.insert(0, %r)\n"
                "from tests.test_anymal_self_collision_gpu import _sim, _run\n"
                "from tests.anymal_self_common import anymal_self\n"
                "z = np.load(%r); m = anymal_self(); s = _sim(m, len(z['root'])); assert s.quad_ns() == 0\n"
                "r, d, c = _run(s, z['root'], z['dof'], z['tau']); np.savez(%r, r=r, d=d, c=c)\n") % (ROOT, os.path.join(td, "in.npz"), os.path.join(td, "out.npz"))
        env = dict(os.environ, B2G_NO_QUAD="1")
        subprocess.check_call([sys.executable, "-c", code], cwd=ROOT, env=env)
        g = np.load(os.path.join(td, "out.npz"))
        compare_layered(m, rq, dq, g["r"], g["d"], ncq, g["c"])


def _set_state(env, root, dof):
    env.root_states.copy_(torch.tensor(root, dtype=torch.float32, device=env.device))
    env.dof_state.copy_(torch.tensor(dof.reshape(-1, 2), dtype=torch.float32, device=env.device))


def test_anymal_terrain_self_collision_task():
    """env.selfCollision=True: no warning, the quad kernels, one step from crossed-leg states equals the oracle's PD loop
    (the tolerances of the AnymalTerrain parity tests); without the flag: the warning and the plain model"""
    from oracle.oracle import OracleSim
    from isaacgymenvs_b200 import engine
    n, nd = 1024, 12
    envs = {}
    for on in (False, True):
        engine._warned.discard("AnymalTerrain")
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            envs[on] = _make_anymal(n, terrain={"terrainType": "plane"}, addNoise=False, pushRobots=False, selfCollision=on)
        warned = any(issubclass(w.category, engine.UnmodelledPhysicsWarning) for w in rec)
        assert warned == (not on)
        assert bool(getattr(envs[on].model, "self_collide", False)) == on
        assert envs[on].sim.quad_ns() == 3
    env = envs[True]
    env.step(torch.zeros(n, nd, device=env.device))                # the first step resets every env
    rng = np.random.default_rng(31)
    m = env.model
    root, dof = crossed_states(m, n, rng, 0.45, 0.7)
    root[:, 0:2] = env.root_states[:, 0:2].cpu().numpy()
    dof[..., 1] *= 0.2
    _set_state(env, root, dof)
    orc = OracleSim(m, env.cfg["sim"]["dt"], env.cfg["sim"]["substeps"], G, ground_mu=env.cfg["env"]["terrain"]["dynamicFriction"], threads=16)
    env.env_friction[:] = float(np.asarray(m.cp_mu)[0])
    r64 = env.root_states.cpu().numpy().astype(np.float64); d64 = env.dof_state.cpu().numpy().astype(np.float64).reshape(n, nd, 2)
    assert (sphere_overlap(m, orc, r64, d64) > 0).mean() > 0.15
    q0 = env.default_dof_pos[0].cpu().numpy().astype(np.float64)
    Kp, Kd, sc = float(env.Kp), float(env.Kd), float(env.action_scale)
    a = rng.uniform(-1, 1, size=(n, nd)).astype(np.float32)
    ac = np.clip(a, -float(env.clip_actions), float(env.clip_actions)).astype(np.float64)
    for _ in range(env.decimation):
        tau = np.clip(Kp * (sc * ac + q0[None] - d64[..., 0]) - Kd * d64[..., 1], -80.0, 80.0)
        out = orc.simulate(r64, d64, tau)
    for _ in range(int(env.control_freq_inv)):
        out = orc.simulate(r64, d64, tau)
    obs, rew, reset, _ = env.step(torch.tensor(a, device=env.device))
    torch.cuda.synchronize()
    keep = reset.cpu().numpy() == 0
    assert keep.mean() > 0.5
    rg = env.root_states.cpu().numpy()[keep]; dg = env.dof_state.cpu().numpy().reshape(n, nd, 2)[keep]
    assert np.isfinite(rg).all() and np.isfinite(dg).all() and torch.isfinite(obs["obs"]).all()
    assert np.abs(rg[:, :7] - r64[keep][:, :7]).max() < 3e-4, np.abs(rg[:, :7] - r64[keep][:, :7]).max()
    assert (np.abs(rg[:, 7:] - r64[keep][:, 7:]) / np.maximum(1, np.abs(r64[keep][:, 7:]))).max() < 1e-2
    assert np.abs(dg[..., 0] - d64[keep][..., 0]).max() < 3e-4
    cg = env.contact_forces.cpu().numpy()[keep]
    co = per_link_contact(m, out["contact_force"])[keep]
    assert np.abs(cg - co).max() < 1e-2 * max(1.0, np.abs(co).max())


def test_knee_collision_term_from_self_contact():
    """Airborne ANYmals with crossed legs: the only contact a thigh ("knee", anymal_terrain.py:213) can have is with another
    leg.  With selfCollision the net contact tensor carries it and the knee-collision reward counts it, as the reference's
    contact tensor would; without, the tensor is zero."""
    n, nd = 1024, 12
    scales = {k: 0.0 for k in ("terminalReward", "linearVelocityXYRewardScale", "linearVelocityZRewardScale", "angularVelocityXYRewardScale",
                               "angularVelocityZRewardScale", "orientationRewardScale", "torqueRewardScale", "jointAccRewardScale",
                               "baseHeightRewardScale", "feetAirTimeRewardScale", "feetStumbleRewardScale", "actionRateRewardScale", "hipRewardScale")}
    scales["kneeCollisionRewardScale"] = 1.0                   # positive: the reward is clipped at zero from below
    counted = {}
    for on in (True, False):
        env = _make_anymal(n, terrain={"terrainType": "plane"}, addNoise=False, pushRobots=False, selfCollision=on, **scales)
        env.step(torch.zeros(n, nd, device=env.device))
        rng = np.random.default_rng(37)
        root, dof = crossed_states(env.model, n, rng, 3.0, 3.0)
        root[:, 7:13] = 0.0; dof[..., 1] = 0.0
        _set_state(env, root, dof)
        _, rew, _, _ = env.step(torch.zeros(n, nd, device=env.device))
        torch.cuda.synchronize()
        cf = env.contact_forces.cpu().numpy()
        knees = np.linalg.norm(cf[:, env._knees], axis=-1) > 1.0
        assert np.allclose(rew.cpu().numpy(), knees.sum(1) * env.dt, rtol=1e-5, atol=1e-7)
        if not on:
            assert np.abs(cf).max() == 0.0
        counted[on] = int(knees.any(1).sum())
    print(f"airborne crossed-leg states with a knee in contact: {counted[True]} of {n} (selfCollision on), {counted[False]} (off)")
    assert counted[True] > 0.02 * n and counted[False] == 0


def test_anymal_legs_interpenetrate_less():
    """Random-action rollouts of 1024 AnymalTerrain envs on the plane, with and without selfCollision: the share of sampled
    env-states with a candidate pair overlapping by more than 1 cm, and the deepest overlap.  Measured on an H100: the
    task's PD targets around the default pose rarely cross the legs (1 of 20480 sampled states above 1 cm without the
    contact, none with it), so the bound is on the deepest overlap (2.2 cm without, 0.7 cm with)."""
    from oracle.oracle import OracleSim
    from isaacgymenvs_b200 import engine
    share, deepest = {}, {}
    for on in (True, False):
        env = _make_anymal(1024, terrain={"terrainType": "plane"}, selfCollision=on)
        m = copy.deepcopy(env.model)
        if not on:
            from isaacgymenvs_b200.importer.model import enable_self_collision
            enable_self_collision(m); m.self_collide = False          # pair table for the measurement only
        orc = OracleSim(m, DT, SUB, G)
        g = torch.Generator(device="cuda:0"); g.manual_seed(3)
        hits = samples = 0; worst = 0.0
        for k in range(200):
            env.step(torch.rand((1024, 12), device="cuda:0", generator=g) * 2 - 1)
            if k % 10 != 9:
                continue
            torch.cuda.synchronize()
            dep = sphere_overlap(m, orc, env.root_states.cpu().numpy().astype(np.float64), env.dof_state.cpu().numpy().astype(np.float64).reshape(1024, -1, 2))
            hits += int((dep > 0.01).sum()); samples += 1024; worst = max(worst, float(dep.max()))
        assert torch.isfinite(env.root_states).all() and torch.isfinite(env.dof_state).all()
        share[on] = hits / samples; deepest[on] = worst
        print(f"AnymalTerrain, random actions, self-collision {'on' if on else 'off'}: {hits}/{samples} sampled env-states overlap > 1 cm "
              f"({100.0 * hits / samples:.2f} %), deepest {worst * 100:.1f} cm")
    assert share[True] <= share[False] and deepest[True] < 0.5 * deepest[False], (share, deepest)
