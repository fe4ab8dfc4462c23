"""CPU test of the quad sub-step's link-link contact (QLane<.., SELF = true>, isaacgymenvs_b200/csrc/b2g_quad.cuh): the
header is __host__ __device__, so tests/quad_self_host.cu runs the arithmetic the CUDA kernels execute, lane by lane, against
the fp64 oracle with a self-colliding ANYmal (collision filter 0, anymal_terrain.py:282)."""
import copy
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

from isaacgymenvs_b200 import engine
from oracle.oracle import OracleSim
from tests.anymal_self_common import G, anymal_self, crossed_states, sphere_overlap, compare_layered
from tests.test_quad_host import _lib as _plain_lib, _host_simulate

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "quad_self_host.cu")
LIB = os.path.join(HERE, "libquadselfhost.so")
DEPS = [SRC] + [os.path.join(ROOT, "isaacgymenvs_b200", "csrc", f) for f in ("b2g_quad.cuh", "b2g_quad_host.h", "b2g_device.cuh")]
DT, SUB = 0.005, 1           # AnymalTerrain: sim dt 5 ms, one sub-step


def _lib():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-shared",
                               "-Xcompiler", "-fPIC", "-o", LIB, SRC])
    lib = C.CDLL(LIB)
    lib.quad_self_host_simulate.restype = C.c_int
    return lib


def _self_simulate(lib, m, root32, dof32, tau32, hfield=None, hf_scale=1.0, hf_vscale=1.0, hf_origin=(0.0, 0.0),
                   mass_scale=None, dof_props=None, env_friction=None):
    cm, keep = engine.pack_model(m)
    sp = engine.CSimParams()
    sp.dt, sp.substeps = DT, SUB
    sp.gravity = (C.c_float * 3)(*G)
    sp.ground_friction = 1.0
    if hfield is not None:
        hf = np.ascontiguousarray(hfield, dtype=np.int16)
        keep["hf"] = hf
        sp.hf_samples = hf.ctypes.data
        sp.hf_nx, sp.hf_ny = hf.shape
        sp.hf_horizontal_scale, sp.hf_vertical_scale = hf_scale, hf_vscale
        sp.hf_origin_x, sp.hf_origin_y = hf_origin
    n = root32.shape[0]
    dfrc = np.zeros((n, m.ndof), np.float32)
    nc = np.zeros((n, m.nb, 3), np.float32)
    p = lambda a: C.c_void_p(a.ctypes.data) if a is not None else None
    ns = lib.quad_self_host_simulate(C.byref(cm), C.byref(sp), C.c_int(n), p(root32), p(dof32), p(tau32), p(dfrc), p(nc),
                                     p(mass_scale), p(dof_props), p(env_friction))
    return ns, dfrc, nc


def _hfield(rng):
    nx, ny, hs, vs = 64, 64, 0.25, 0.005
    return dict(hfield=(rng.uniform(0, 40, size=(nx, ny))).astype(np.int16), hf_scale=hs, hf_vscale=vs, hf_origin=(-8.0, -8.0))


def _oracle(m, hfk):
    if hfk is None:
        return OracleSim(m, DT, SUB, G, ground_mu=1.0, threads=8)
    return OracleSim(m, DT, SUB, G, ground_mu=1.0, hfield=hfk["hfield"].astype(np.float64) * hfk["hf_vscale"], hf_scale=hfk["hf_scale"],
                     hf_origin=hfk["hf_origin"], threads=8)


@pytest.mark.parametrize("terrain", ["plane", "heightfield"])
@pytest.mark.parametrize("per_env", [False, True])
def test_quad_self_substep_matches_oracle(terrain, per_env):
    """Crossed-leg states, some on the ground: the SELF twin against the oracle (which bakes any per-env link masses and
    joint properties into its model), the contact is really applied, and where no pair overlaps the SELF twin is the plain
    quad sub-step."""
    lib = _lib()
    m = anymal_self()
    n, ng = 512, 4
    rng = np.random.default_rng(17 if terrain == "plane" else 19)
    hfk = _hfield(rng) if terrain == "heightfield" else None
    root, dof = crossed_states(m, n, rng)
    if hfk is not None:
        root[:, 0:2] = rng.uniform(-5, 5, size=(n, 2))
    tau = rng.uniform(-1, 1, size=(n, m.ndof)) * 40.0
    root32 = np.ascontiguousarray(root, np.float32); dof32 = np.ascontiguousarray(dof, np.float32); tau32 = np.ascontiguousarray(tau, np.float32)
    r64 = root32.astype(np.float64); d64 = dof32.astype(np.float64); t64 = tau32.astype(np.float64)
    dep = sphere_overlap(m, _oracle(m, hfk), r64, d64)
    assert (dep > 0).mean() > 0.15, (dep > 0).mean()                     # the sample really exercises link-link contact
    kw = dict(hfk or {})
    if per_env:
        nl, nd = m.nl, m.ndof
        mass_scale = np.ones((n, nl), np.float32); dof_props = np.zeros((n, nd, 4), np.float32)
        models = []
        for g in range(ng):
            ms = rng.uniform(0.5, 2.0, size=nl).astype(np.float32)
            dmp = (m.damping[1:] + 0.05 * (g + 1)).astype(np.float32); stf = (m.stiffness[1:] + 0.5 * g).astype(np.float32)
            sl = slice(g * n // ng, (g + 1) * n // ng)
            mass_scale[sl] = ms; dof_props[sl, :, 0] = dmp; dof_props[sl, :, 1] = stf; dof_props[sl, :, 2] = -3e38; dof_props[sl, :, 3] = 3e38
            mg = copy.deepcopy(m)
            mg.mass = m.mass * ms.astype(np.float64)
            mg.inertia = np.asarray(m.inertia, float) * ms.astype(np.float64)[:, None]
            mg.damping = np.concatenate([[0.0], dmp.astype(np.float64)]); mg.stiffness = np.concatenate([[0.0], stf.astype(np.float64)])
            models.append((sl, mg))
        kw.update(mass_scale=mass_scale, dof_props=dof_props)
    else:
        models = [(slice(0, n), m)]
    out = {"contact_force": np.zeros((n, m.nb, 3)), "dof_force": np.zeros((n, m.ndof))}
    for sl, mg in models:
        r = np.ascontiguousarray(r64[sl]); d = np.ascontiguousarray(d64[sl])
        o = _oracle(mg, hfk).simulate(r, d, np.ascontiguousarray(t64[sl]))
        r64[sl] = r; d64[sl] = d
        for k in out:
            out[k][sl] = o[k]
    ns, dfrc, nc = _self_simulate(lib, m, root32, dof32, tau32, **kw)
    assert ns == 3
    compare_layered(m, root32.astype(np.float64), dof32.astype(np.float64), r64, d64, nc, out["contact_force"])
    assert np.abs(dfrc - out["dof_force"]).max() < 2e-3 * max(1.0, np.abs(out["dof_force"]).max())
    # the plain quad sub-step (the model with self_collide cleared) on the same states
    m0 = copy.deepcopy(m); m0.self_collide = False
    rootb = np.ascontiguousarray(root, np.float32); dofb = np.ascontiguousarray(dof, np.float32)
    ns0, _, _, nc0 = _host_simulate(_plain_lib(), m0, DT, SUB, rootb, dofb, tau32, ground_mu=1.0, want_spec=0,
                                    mass_scale=kw.get("mass_scale"), dof_props=kw.get("dof_props"),
                                    **({k: kw[k] for k in ("hfield", "hf_scale", "hf_vscale", "hf_origin")} if hfk else {}))
    assert ns0 == 3
    hit, free = dep > 0, dep <= 0
    dv = np.abs(dofb[..., 1] - dof32[..., 1]).max(1)
    assert (dv[hit] > 1e-2).mean() > 0.5, (dv[hit] > 1e-2).mean()         # the contact is really applied
    rel = lambda a, b: (np.abs(a - b) / np.maximum(1.0, np.abs(b))).max()
    assert rel(dof32[free], dofb[free]) <= 1e-6 and rel(root32[free], rootb[free]) <= 1e-6
    assert rel(nc[free], nc0[free]) <= 1e-6


def test_self_colliding_anymal_takes_the_quad_path():
    """the model builder routes a self-colliding ANYmal to the four-chain kernels; a self-colliding Ant stays generic"""
    from tests.test_model_host import _lib as model_lib, FIELDS
    from isaacgymenvs_b200.assets import load_compiled
    from isaacgymenvs_b200.importer.model import enable_self_collision
    lib = model_lib()
    for name, dt, sub, want in (("anymal", 0.005, 1, 3), ("ant", 0.0166, 2, 0)):
        m = copy.deepcopy(load_compiled(name))
        m.sensor_body = np.zeros(0, dtype=np.int32); m.sensor_pos = np.zeros((0, 3)); m.sensor_quat = np.zeros((0, 4))
        enable_self_collision(m, samples=0 if name == "ant" else 4096)      # the Ant's limits keep its legs apart: no reachability cut
        assert m.self_collide and np.asarray(m.self_pairs).any()
        cm, keep = engine.pack_model(m)
        sp = engine.CSimParams()
        sp.dt, sp.substeps = dt, sub
        sp.gravity = (C.c_float * 3)(*G)
        sp.ground_friction = 1.0
        out = (C.c_int64 * 9)()
        rc = lib.model_host_build(C.byref(cm), None, C.byref(sp), C.c_int(0), out)
        v = dict(zip(FIELDS, out))
        assert rc == 0 and v["quad_ns"] == want and v["quad_spec"] == 0, (name, rc, v)


def test_self_collision_is_stable_under_persistent_actuation():
    """What a learner does: bang-bang PD targets (AnymalTerrain's kp 80, kd 2, action scale 0.5, 80 N m) held for 25 steps,
    512 self-colliding ANYmals on the plane, 600 steps of the task's 5 ms with resets on falling -- the oracle stays finite and
    the joint speeds bounded, as the Humanoid's probe in tests/test_oracle_physics.py."""
    m = anymal_self()
    orc = OracleSim(m, DT, SUB, G, ground_mu=1.0, threads=16)
    n = 512
    rng = np.random.default_rng(0)
    names = list(m.dof_names)
    from isaacgymenvs_b200 import config
    dj = config.builtin_cfg("AnymalTerrain", {})["task"]["env"]["defaultJointAngles"]
    default = np.array([dj[k] for k in names])

    def fresh(idx):
        root[idx] = 0; root[idx, 2] = 0.62; root[idx, 6] = 1
        dof[idx] = 0; dof[idx, :, 0] = default[None] * rng.uniform(0.5, 1.5, size=(len(idx), m.ndof))
    root = np.zeros((n, 13)); dof = np.zeros((n, m.ndof, 2))
    fresh(np.arange(n))
    act = rng.uniform(-1, 1, size=(n, m.ndof))
    worst, hits = 0.0, 0
    for k in range(600):
        if k % 25 == 0:
            flip = rng.random(n) < 0.5
            act[flip] = np.sign(rng.uniform(-1, 1, size=(int(flip.sum()), m.ndof)))
        tau = np.clip(80.0 * (0.5 * act + default[None] - dof[..., 0]) - 2.0 * dof[..., 1], -80.0, 80.0)
        orc.simulate(root, dof, tau)
        assert np.isfinite(dof).all() and np.isfinite(root).all(), k
        worst = max(worst, float(np.abs(dof[..., 1]).max()))
        if k % 50 == 49:
            hits += int((sphere_overlap(m, orc, root, dof) > 0).sum())
        fallen = np.nonzero(root[:, 2] < 0.25)[0]
        if len(fallen):
            fresh(fallen)
    print(f"ANYmal, self-collision, bang-bang PD targets: peak joint speed {worst:.1f} rad/s, {hits} sampled states in contact")
    assert worst < 200.0, worst
