"""Shared by the ANYmal link-link contact tests (CPU and GPU): the self-colliding ANYmal model, states in which its legs
cross, and the deepest overlap of a candidate sphere pair per env."""
import copy
import numpy as np

from isaacgymenvs_b200.assets import load_compiled
from isaacgymenvs_b200.importer.model import enable_self_collision

G = (0.0, 0.0, -9.81)


def anymal_self(on=True):
    """ANYmal with the importer's pair table; on=False keeps the table (for measuring overlaps) but not the contact"""
    m = copy.deepcopy(load_compiled("anymal"))
    m.sensor_body = np.zeros(0, dtype=np.int32); m.sensor_pos = np.zeros((0, 3)); m.sensor_quat = np.zeros((0, 4))
    enable_self_collision(m)
    m.self_collide = bool(on)
    return m


def crossed_states(m, n, rng, zlo=0.3, zhi=0.9):
    """joints uniform in +-pi (the ANYmal joints are unlimited): about one state in six has legs inside each other; the
    lower base heights put feet and knees on the ground"""
    root = np.zeros((n, 13))
    root[:, 0:2] = rng.normal(size=(n, 2))
    root[:, 2] = rng.uniform(zlo, zhi, size=n)
    q = rng.normal(size=(n, 4)) * np.array([0.3, 0.3, 0.3, 0.0]) + np.array([0, 0, 0, 1.0])
    root[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    root[:, 7:13] = rng.normal(size=(n, 6)) * 0.5
    dof = np.stack([rng.uniform(-np.pi, np.pi, size=(n, m.ndof)), rng.normal(size=(n, m.ndof))], -1)
    return root, dof


def sphere_overlap(m, orc, root, dof):
    """deepest overlap (m) of a candidate pair (model.self_pairs) per env, from the oracle's body poses"""
    from oracle import tasks_np as T
    f32 = np.float32
    cpb = np.array(m.cp_body)
    bs = orc.body_states(root, dof)
    off_p = np.asarray(m.body_pos, f32)[cpb]; off_q = np.asarray(m.body_quat, f32)[cpb]
    loc = T.quat_rotate_inverse(off_q, np.asarray(m.cp_pos, f32) - off_p)
    n, ncp = bs.shape[0], len(cpb)
    wp = bs[:, cpb, 0:3].astype(f32) + T.quat_rotate(bs[:, cpb, 3:7].astype(f32).reshape(-1, 4), np.tile(loc, (n, 1))).reshape(n, ncp, 3)
    rr = (np.asarray(m.cp_radius)[:, None] + np.asarray(m.cp_radius)[None, :]).astype(f32)
    d = np.linalg.norm(wp[:, :, None, :] - wp[:, None, :, :], axis=-1)
    return np.where(np.asarray(m.self_pairs)[None] > 0, rr[None] - d, -1.0).max(axis=(1, 2))


def per_link_contact(m, cf):
    """the engine reports a link's contact force on the first body riding on it; the oracle reports per body"""
    co = np.zeros_like(cf)
    first = {}
    for b in range(m.nb):
        first.setdefault(int(m.body_link[b]), b)
        co[:, first[int(m.body_link[b])]] += cf[:, b]
    return co


def compare_layered(m, rg, dg, r64, d64, nc=None, cf=None):
    """the bounds of the Humanoid link-link contact test: stiff contacts between light links amplify fp32 round-off"""
    assert np.isfinite(rg).all() and np.isfinite(dg).all()
    dp = np.abs(rg[:, :7] - r64[:, :7]).max(1)
    assert np.quantile(dp, 0.99) < 5e-5 and dp.max() < 1e-3, (np.quantile(dp, 0.99), dp.max())
    dq = np.abs(dg[..., 0] - d64[..., 0])
    assert np.quantile(dq, 0.99) < 1e-4 and dq.max() < 5e-3, (np.quantile(dq, 0.99), dq.max())
    qerr = np.abs(dg[..., 1] - d64[..., 1]) / np.maximum(1.0, np.abs(d64[..., 1]))
    assert np.quantile(qerr, 0.99) < 2e-3 and np.median(qerr) < 1e-4, (np.quantile(qerr, 0.99), np.median(qerr))
    if nc is not None:
        co = per_link_contact(m, cf)
        cerr = np.abs(nc - co).max(axis=(1, 2)) / np.maximum(1.0, np.abs(co).max(axis=(1, 2)))
        assert np.quantile(cerr, 0.99) < 1e-2 and np.median(cerr) < 1e-3, (np.quantile(cerr, 0.99), np.median(cerr))
