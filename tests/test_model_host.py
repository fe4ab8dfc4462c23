"""CPU test of what b2g_create / b2g_create_ext decide before they touch the device (isaacgymenvs_b200/csrc/b2g_model_host.h):
tests/model_host.cu compiles the builder for the host.  For the articulation of each task it pins the lanes per env, the CTA
size and dynamic shared memory, the slot program length and accumulator count, where the self-collision scratch lives and
whether the quad path takes the model.  A change to any of them changes which kernel instantiation runs."""
import copy
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

from isaacgymenvs_b200 import engine
from isaacgymenvs_b200.assets import load_compiled
from isaacgymenvs_b200.importer.model import enable_self_collision
from tests.hand_common import DT as HAND_DT, SUBSTEPS as HAND_SUBSTEPS, hand_setup

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "model_host.cu")
LIB = os.path.join(HERE, "libmodelhost.so")
DEPS = [SRC] + [os.path.join(ROOT, "isaacgymenvs_b200", "csrc", f)
                for f in ("b2g_model_host.h", "b2g_quad_host.h", "b2g_kin_host.h", "b2g_quad.cuh", "b2g_kin.cuh", "b2g_device.cuh")]
G = (0.0, 0.0, -9.81)


def _lib():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-shared",
                               "-Xcompiler", "-fPIC", "-o", LIB, SRC])
    lib = C.CDLL(LIB)
    lib.model_host_build.restype = C.c_int
    return lib


def _locomotion(name, feet):
    """the articulation as tasks/locomotion.py builds it: force sensors on the feet"""
    m = copy.deepcopy(load_compiled(name))
    m.sensor_body = np.array([m.body_names.index(f) for f in feet], dtype=np.int32)
    m.sensor_pos = np.zeros((len(feet), 3)); m.sensor_quat = np.tile([0, 0, 0, 1.0], (len(feet), 1))
    return m


def _ant():
    m = copy.deepcopy(load_compiled("ant"))
    return _locomotion("ant", [n for n in m.body_names if "foot" in n])


def _humanoid(self_collision=False):
    m = _locomotion("humanoid", ["right_foot", "left_foot"])
    return enable_self_collision(m) if self_collision else m


def _plain(name):
    m = copy.deepcopy(load_compiled(name))
    m.sensor_body = np.zeros(0, dtype=np.int32); m.sensor_pos = np.zeros((0, 3)); m.sensor_quat = np.zeros((0, 4))
    return m


def _config(name):
    """-> (model, ext or None, dt, substeps, height field or None)"""
    if name == "ant":
        return _ant(), None, 0.0166, 2, None
    if name == "humanoid":
        return _humanoid(), None, 0.0166, 2, None
    if name == "humanoid_self":
        return _humanoid(True), None, 0.0166, 2, None
    if name == "cartpole":
        return _plain("cartpole"), None, 0.0166, 2, None
    if name == "anymal":
        return _plain("anymal"), None, 0.005, 1, None
    if name == "anymal_hf":
        hf = np.random.default_rng(1).integers(0, 40, size=(64, 64)).astype(np.int16)
        return _plain("anymal"), None, 0.005, 1, hf
    if name == "shadow_hand":
        m, obj, tendons = hand_setup()
        return m, engine.pack_model_ext(m, obj=obj, actors_per_env=3, tendons=tendons, tendon_k=30.0, tendon_d=0.1), HAND_DT, HAND_SUBSTEPS, None
    raise KeyError(name)


def build(name, single_lane=False, lib=None):
    """the builder's decisions for configuration `name`: dict of the pinned fields"""
    lib = lib or _lib()
    m, ext, dt, sub, hf = _config(name)
    cm, keep = engine.pack_model(m)
    sp = engine.CSimParams()
    sp.dt, sp.substeps = dt, sub
    sp.gravity = (C.c_float * 3)(*G)
    sp.ground_friction = 1.0
    if hf is not None:
        keep["hf"] = hf
        sp.hf_samples = hf.ctypes.data
        sp.hf_nx, sp.hf_ny = hf.shape
        sp.hf_horizontal_scale, sp.hf_vertical_scale = 0.1, 0.005
        sp.hf_origin_x, sp.hf_origin_y = -3.2, -3.2
    out = (C.c_int64 * 9)()
    rc = lib.model_host_build(C.byref(cm), C.byref(ext) if ext is not None else None, C.byref(sp), C.c_int(int(single_lane)), out)
    assert rc == 0, rc
    return dict(zip(FIELDS, out))


FIELDS = ("lanes", "block", "dyn_smem", "ns", "nacc", "self_cell", "self_f4", "quad_ns", "quad_spec")
# (configuration, one thread per env) -> the values of FIELDS
EXPECTED = {
    ("ant", False): (4, 128, 40960, 2, 0, 0, 0, 2, 3),                 # the quad path, axisymmetric specialisation
    ("humanoid", False): (4, 64, 99328, 9, 1, 0, 0, 0, 0),
    ("humanoid_self", False): (4, 64, 99328, 9, 1, 515, 0, 0, 0),      # scratch in idle cells of lane 2 from slot 3
    ("cartpole", False): (1, 128, 40960, 2, 0, 0, 0, 0, 0),
    ("anymal", False): (4, 128, 61440, 3, 0, 0, 0, 3, 0),              # the quad path, general inertias
    ("anymal_hf", False): (4, 128, 61440, 3, 0, 0, 0, 3, 0),
    ("shadow_hand", False): (4, 128, 159984, 10, 9, 0, 0, 0, 0),       # [link][k][env] layout with the free object
    ("ant", True): (1, 64, 89088, 8, 1, 0, 0, 0, 0),
    ("humanoid", True): (1, 32, 114688, 21, 2, 0, 0, 0, 0),
}


@pytest.mark.parametrize("name,single_lane", list(EXPECTED))
def test_create_time_decisions(name, single_lane):
    assert build(name, single_lane) == dict(zip(FIELDS, EXPECTED[(name, single_lane)]))
