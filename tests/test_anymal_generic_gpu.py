"""AnymalTerrain's first launch on the generic Stepper (B2G_NO_QUAD=1): `anymal_physics_kernel`, the reference the
four-chain `quad_anymal_physics_kernel` is compared with.  The golden epilogue and the oracle PD-loop checks of the
default path (tests/test_gpu_parity.py, tests/test_gpu_parity2.py, which run the four-chain kernel), at the same
tolerances."""
import numpy as np
import pytest
import torch

from tests.test_gpu_parity import test_anymal_terrain_epilogue_matches_reference_golden as _golden_epilogue_check
from tests.test_gpu_parity2 import _anymal_check, _make_anymal

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _generic_path(monkeypatch):
    monkeypatch.setenv("B2G_NO_QUAD", "1")          # read when the sim is created
    assert _make_anymal(8, addNoise=False, pushRobots=False).sim.quad_ns() == 0


def test_generic_anymal_epilogue_matches_reference_golden():
    _golden_epilogue_check()


@pytest.mark.parametrize("terrain,n", [("trimesh", 256), ("plane", 250)])
def test_generic_anymal_physics_equals_oracle_pd_loop(terrain, n):
    env = _make_anymal(n, terrain={"terrainType": terrain}, addNoise=False, pushRobots=False)
    assert env.sim.quad_ns() == 0
    rng = np.random.default_rng(3)
    env.step(torch.zeros(n, 12, device=env.device))           # the first step resets every env (reset_buf starts as ones)
    torch.cuda.synchronize()
    _anymal_check(env, 3, rng)
