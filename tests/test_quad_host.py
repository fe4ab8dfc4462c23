"""CPU test of the quad sub-step (isaacgymenvs_b200/csrc/b2g_quad.cuh): the header is __host__ __device__, so
tests/quad_host.cu compiles it for the HOST and runs the arithmetic the CUDA kernels execute, lane by lane, against the
fp64 oracle -- same states, same tolerances as tests/test_gpu_parity.py::test_simulate_matches_oracle.  No GPU needed:
a wrong term in the specialised Ant / ANYmal step shows up here, before any GPU time is spent."""
import copy
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

from isaacgymenvs_b200 import engine
from isaacgymenvs_b200.assets import load_compiled
from oracle.oracle import OracleSim

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "quad_host.cu")
LIB = os.path.join(HERE, "libquadhost.so")
DEPS = [SRC] + [os.path.join(ROOT, "isaacgymenvs_b200", "csrc", f) for f in ("b2g_quad.cuh", "b2g_quad_host.h", "b2g_device.cuh")]
G = (0.0, 0.0, -9.81)


def _lib():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-shared",
                               "-Xcompiler", "-fPIC", "-o", LIB, SRC])
    lib = C.CDLL(LIB)
    lib.quad_host_simulate.restype = C.c_int
    return lib


def _model(name):
    m = copy.deepcopy(load_compiled(name))
    if name == "ant":
        m.sensor_body = np.array([2, 4, 6, 8], dtype=np.int32)
    else:
        m.sensor_body = np.zeros(0, dtype=np.int32)
    m.sensor_pos = np.zeros((len(m.sensor_body), 3)); m.sensor_quat = np.tile([0, 0, 0, 1.0], (len(m.sensor_body), 1))
    return m


def _random_states(m, n, rng, zlo, zhi):
    root = np.zeros((n, 13))
    root[:, 0:2] = rng.normal(size=(n, 2))
    root[:, 2] = rng.uniform(zlo, zhi, size=n)
    q = rng.normal(size=(n, 4)) * np.array([0.3, 0.3, 0.3, 0.0]) + np.array([0, 0, 0, 1.0])
    root[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    root[:, 7:13] = rng.normal(size=(n, 6)) * 0.5
    lo = np.where(m.limited[1:] > 0, m.lower[1:], -1.0); hi = np.where(m.limited[1:] > 0, m.upper[1:], 1.0)
    qpos = lo + (hi - lo) * rng.uniform(-0.05, 1.05, size=(n, m.ndof))
    qvel = rng.normal(size=(n, m.ndof))
    return root, np.stack([qpos, qvel], -1)


def _host_simulate(lib, m, dt, sub, root32, dof32, tau32, hfield=None, hf_scale=1.0, hf_vscale=1.0, hf_origin=(0.0, 0.0), ground_mu=1.0, want_spec=3,
                   spec_out=None, mass_scale=None, dof_props=None, env_friction=None):
    cm, keep = engine.pack_model(m)
    sp = engine.CSimParams()
    sp.dt, sp.substeps = dt, sub
    sp.gravity = (C.c_float * 3)(*G)
    sp.ground_friction = ground_mu
    if hfield is not None:
        hf = np.ascontiguousarray(hfield, dtype=np.int16)
        keep["hf"] = hf
        sp.hf_samples = hf.ctypes.data
        sp.hf_nx, sp.hf_ny = hf.shape
        sp.hf_horizontal_scale, sp.hf_vertical_scale = hf_scale, hf_vscale
        sp.hf_origin_x, sp.hf_origin_y = hf_origin
    n = root32.shape[0]
    sensor = np.zeros((n, max(len(m.sensor_body), 1), 6), np.float32)
    dfrc = np.zeros((n, m.ndof), np.float32)
    nc = np.zeros((n, m.nb, 3), np.float32)
    p = lambda a: C.c_void_p(a.ctypes.data)
    spec = C.c_int(-1)
    ns = lib.quad_host_simulate(C.byref(cm), C.byref(sp), C.c_int(n), p(root32), p(dof32), p(tau32), p(sensor), p(dfrc), p(nc), C.c_int(want_spec), C.byref(spec),
                                p(mass_scale) if mass_scale is not None else None, p(dof_props) if dof_props is not None else None,
                                p(env_friction) if env_friction is not None else None)
    if spec_out is not None:
        spec_out.append(spec.value)
    return ns, sensor[:, :len(m.sensor_body)], dfrc, nc


def _compare(m, rg, dg, out_g, r64, d64, out, qtol=5e-5):
    assert np.abs(rg[:, :7] - r64[:, :7]).max() < 2e-5
    verr = np.abs(rg[:, 7:] - r64[:, 7:]) / np.maximum(1.0, np.abs(r64[:, 7:]))
    assert verr.max() < 2e-3, verr.max()
    dq = np.abs(dg[..., 0] - d64[..., 0])
    assert dq.max() < qtol and np.quantile(dq, 0.999) < 3e-5, (dq.max(), np.quantile(dq, 0.999))
    qerr = np.abs(dg[..., 1] - d64[..., 1]) / np.maximum(1.0, np.abs(d64[..., 1]))
    # fp32 vs fp64 through a stiff contact: a handful of DOFs (feet pressed into the ground at > 30 rad/s) sit at ~2e-3,
    # the bulk two orders of magnitude lower
    assert qerr.max() < 4e-3 and np.quantile(qerr, 0.999) < 1e-3 and np.quantile(qerr, 0.99) < 2e-4, (qerr.max(), np.quantile(qerr, 0.999), np.quantile(qerr, 0.99))
    sensor, dfrc, nc = out_g
    if len(m.sensor_body):
        scale = max(1.0, np.abs(out["sensor"]).max())
        assert np.abs(sensor - out["sensor"]).max() < 2e-3 * scale
    assert np.abs(dfrc - out["dof_force"]).max() < 2e-3 * max(1.0, np.abs(out["dof_force"]).max())
    assert np.abs(nc - out["contact_force"]).max() < 2e-3 * max(1.0, np.abs(out["contact_force"]).max())


@pytest.mark.parametrize("name,zlo,zhi,tscale,dt,sub,damp,want,got", [
    ("ant", 0.15, 0.8, 15.0, 0.0166, 2, None, 3, 3),          # Ant: capsule links + symmetric torso -> the axisymmetric specialisation
    ("ant", 0.15, 0.8, 15.0, 0.0166, 2, None, 0, 0),          # ... and the general layout on the same model
    ("anymal", 0.3, 0.9, 40.0, 0.005, 1, None, 3, 0),         # ANYmal: general inertias -> the builder falls back by itself
    ("ant", 0.15, 0.8, 15.0, 0.0166, 2, (0.8, 0.5, 3.0), 3, 3),
    ("ant", 0.15, 0.8, 15.0, 0.0166, 2, (0.8, 0.5, 3.0), 0, 0)])
def test_quad_substep_matches_oracle(name, zlo, zhi, tscale, dt, sub, damp, want, got):
    lib = _lib()
    m = _model(name)
    if damp:          # AssetOptions.angular_damping / linear_damping / max_angular_velocity, exaggerated so that they matter in one step
        m.angular_damping, m.linear_damping, m.max_angular_velocity = damp
    n = 512
    rng = np.random.default_rng(7)
    root, dof = _random_states(m, n, rng, zlo, zhi)
    tau = rng.uniform(-1, 1, size=(n, m.ndof)) * tscale
    root32 = np.ascontiguousarray(root, np.float32); dof32 = np.ascontiguousarray(dof, np.float32); tau32 = np.ascontiguousarray(tau, np.float32)
    r64 = root32.astype(np.float64); d64 = dof32.astype(np.float64); t64 = tau32.astype(np.float64)
    orc = OracleSim(m, dt, sub, G, ground_mu=1.0, threads=8)
    out = orc.simulate(r64, d64, t64)
    used = []
    ns, sensor, dfrc, nc = _host_simulate(lib, m, dt, sub, root32, dof32, tau32, want_spec=want, spec_out=used)
    assert ns == (2 if name == "ant" else 3) and used == [got]
    _compare(m, root32.astype(np.float64), dof32.astype(np.float64), (sensor, dfrc, nc), r64, d64, out)
    # contacts were exercised
    assert (np.abs(out["contact_force"]).max(-1) > 0).mean() > 0.05


def test_quad_rollout_tracks_oracle():
    """30 control steps from rest on the ground: fp32 quad arithmetic vs the fp64 oracle (medians, as the GPU test)."""
    lib = _lib()
    m = _model("ant")
    n = 64
    rng = np.random.default_rng(3)
    root = np.zeros((n, 13)); root[:, 6] = 1; root[:, 2] = 0.5
    q0 = np.where(m.lower[1:] > 0, m.lower[1:], np.where(m.upper[1:] < 0, m.upper[1:], 0.0))
    dof = np.zeros((n, m.ndof, 2)); dof[..., 0] = q0
    root32 = np.ascontiguousarray(root, np.float32); dof32 = np.ascontiguousarray(dof, np.float32)
    r64 = root32.astype(np.float64); d64 = dof32.astype(np.float64)
    orc = OracleSim(m, 0.0166, 2, G, threads=8)
    amp = rng.uniform(-1, 1, size=(n, m.ndof)) * 15.0 * 0.3
    for k in range(30):
        tau32 = np.ascontiguousarray(amp * np.sin(0.3 * k), np.float32)
        _host_simulate(lib, m, 0.0166, 2, root32, dof32, tau32)
        orc.simulate(r64, d64, tau32.astype(np.float64))
    assert np.isfinite(root32).all() and np.isfinite(dof32).all()
    assert np.median(np.abs(root32[:, :3] - r64[:, :3]).max(1)) < 2e-3
    assert np.median(np.abs(dof32[..., 0] - d64[..., 0]).max(1)) < 5e-3


def test_quad_heightfield_matches_oracle():
    """ANYmal on a rough height field: the HF contact path of the quad sub-step vs the oracle."""
    lib = _lib()
    m = _model("anymal")
    n = 256
    rng = np.random.default_rng(11)
    nx, ny, hs, vs = 64, 64, 0.25, 0.005
    hf = (rng.uniform(0, 40, size=(nx, ny))).astype(np.int16)
    ox, oy = -8.0, -8.0
    root, dof = _random_states(m, n, rng, 0.35, 0.8)
    root[:, 0:2] = rng.uniform(-5, 5, size=(n, 2))
    tau = rng.uniform(-1, 1, size=(n, m.ndof)) * 40.0
    root32 = np.ascontiguousarray(root, np.float32); dof32 = np.ascontiguousarray(dof, np.float32); tau32 = np.ascontiguousarray(tau, np.float32)
    r64 = root32.astype(np.float64); d64 = dof32.astype(np.float64); t64 = tau32.astype(np.float64)
    orc = OracleSim(m, 0.005, 1, G, ground_mu=1.0, hfield=hf.astype(np.float64) * vs, hf_scale=hs, hf_origin=(ox, oy), threads=8)
    out = orc.simulate(r64, d64, t64)
    ns, sensor, dfrc, nc = _host_simulate(lib, m, 0.005, 1, root32, dof32, tau32, hfield=hf, hf_scale=hs, hf_vscale=vs, hf_origin=(ox, oy))
    assert ns == 3
    _compare(m, root32.astype(np.float64), dof32.astype(np.float64), (sensor, dfrc, nc), r64, d64, out)
    assert (np.abs(out["contact_force"]).max(-1) > 0).mean() > 0.05


def test_quad_path_rejects_other_topologies():
    lib = _lib()
    for name in ("humanoid", "cartpole"):
        m = copy.deepcopy(load_compiled(name))
        m.sensor_body = np.zeros(0, dtype=np.int32); m.sensor_pos = np.zeros((0, 3)); m.sensor_quat = np.zeros((0, 4))
        n = 2
        root32 = np.zeros((n, 13), np.float32); root32[:, 6] = 1
        dof32 = np.zeros((n, m.ndof, 2), np.float32); tau32 = np.zeros((n, m.ndof), np.float32)
        ns, *_ = _host_simulate(lib, m, 0.0166, 2, root32, dof32, tau32)
        assert ns == 0


@pytest.mark.parametrize("name,zlo,zhi,tscale,dt,sub", [("ant", 0.15, 0.8, 15.0, 0.0166, 2), ("anymal", 0.3, 0.9, 40.0, 0.005, 1)])
def test_quad_per_env_physical_parameters_match_oracle(name, zlo, zhi, tscale, dt, sub):
    """Physical domain randomisation (vec_task.py:720-828): per-env link-mass factors, joint damping / stiffness / limits and
    friction, read by the quad sub-step as parameter arrays.  Four groups of envs with different parameter sets; each group
    must equal the oracle run on a MODEL with those parameters baked in."""
    lib = _lib()
    base = _model(name)
    n, ng = 256, 4
    rng = np.random.default_rng(21)
    root, dof = _random_states(base, n, rng, zlo, zhi)
    tau = rng.uniform(-1, 1, size=(n, base.ndof)) * tscale
    root32 = np.ascontiguousarray(root, np.float32); dof32 = np.ascontiguousarray(dof, np.float32); tau32 = np.ascontiguousarray(tau, np.float32)
    nl, nd = base.nl, base.ndof
    mass_scale = np.ones((n, nl), np.float32); dof_props = np.zeros((n, nd, 4), np.float32); fric = np.zeros(n, np.float32)
    groups = []
    for g in range(ng):
        ms = rng.uniform(0.5, 2.0, size=nl).astype(np.float32) if g else np.full(nl, 2.0, np.float32)     # group 0: every mass doubled
        dmp = (base.damping[1:] * rng.uniform(0.5, 1.5, size=nd) + 0.05 * g).astype(np.float32)
        stf = (base.stiffness[1:] * rng.uniform(0.5, 1.5, size=nd) + 0.5 * g).astype(np.float32)
        lo = (np.where(base.limited[1:] > 0, base.lower[1:], -3e38) + np.where(base.limited[1:] > 0, rng.normal(0, 0.02, size=nd), 0)).astype(np.float32)
        hi = (np.where(base.limited[1:] > 0, base.upper[1:], 3e38) + np.where(base.limited[1:] > 0, rng.normal(0, 0.02, size=nd), 0)).astype(np.float32)
        mu = np.float32(0.4 + 0.3 * g)
        sl = slice(g * n // ng, (g + 1) * n // ng)
        mass_scale[sl] = ms; dof_props[sl, :, 0] = dmp; dof_props[sl, :, 1] = stf; dof_props[sl, :, 2] = lo; dof_props[sl, :, 3] = hi; fric[sl] = mu
        groups.append((sl, ms, dmp, stf, lo, hi, mu))
    r64 = root32.astype(np.float64); d64 = dof32.astype(np.float64); t64 = tau32.astype(np.float64)
    outs = []
    for sl, ms, dmp, stf, lo, hi, mu in groups:
        m = copy.deepcopy(base)
        m.mass = m.mass * ms.astype(np.float64)
        m.inertia = np.asarray(m.inertia, float) * ms.astype(np.float64)[:, None]      # recomputeInertia=True (vec_task.py:773): the inertia follows the mass
        m.damping = np.concatenate([[0.0], dmp.astype(np.float64)]); m.stiffness = np.concatenate([[0.0], stf.astype(np.float64)])
        lim = base.limited[1:] > 0
        m.lower = np.concatenate([[0.0], np.where(lim, lo.astype(np.float64), base.lower[1:])])
        m.upper = np.concatenate([[0.0], np.where(lim, hi.astype(np.float64), base.upper[1:])])
        m.cp_mu = np.full_like(np.asarray(m.cp_mu, float), float(mu))          # friction of every shape of the env
        orc = OracleSim(m, dt, sub, G, ground_mu=1.0, threads=8)
        r = np.ascontiguousarray(r64[sl]); d = np.ascontiguousarray(d64[sl])
        out = orc.simulate(r, d, np.ascontiguousarray(t64[sl]))
        r64[sl] = r; d64[sl] = d; outs.append(out)
    ns, sensor, dfrc, nc = _host_simulate(lib, base, dt, sub, root32, dof32, tau32, mass_scale=mass_scale, dof_props=dof_props, env_friction=fric)
    assert ns in (2, 3)
    out = {k: np.concatenate([o[k] for o in outs], 0) for k in ("sensor", "dof_force", "contact_force")}
    # ANYmal's 0.5 kg shanks under 40 N m reach |qd| > 30 rad/s in contact: fp32 round-off of a few 1e-5 rad in single DOFs
    _compare(base, root32.astype(np.float64), dof32.astype(np.float64), (sensor, dfrc, nc), r64, d64, out, qtol=2e-4 if name == "anymal" else 5e-5)
    # the parameters matter: the same states with the model's own parameters end up elsewhere
    rootb = np.ascontiguousarray(root, np.float32); dofb = np.ascontiguousarray(dof, np.float32)
    _host_simulate(lib, base, dt, sub, rootb, dofb, tau32)
    assert np.abs(dofb[..., 1] - dof32[..., 1]).max() > 1e-2
