"""Compiled articulation models.

The robot descriptions (MJCF/URDF) live in the reference tree (`assets/` of an IsaacGymEnvs checkout), which
does not exist on the GPU box, so the importer's output is committed here as JSON
(`compiled/*.json`, regenerate with `python -m isaacgymenvs_b200.assets.compile_assets`).  When a
reference-style asset root is available `load_asset_file` parses the XML directly instead.
"""
import os
from ..importer.model import Model, BuildOptions

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "compiled")

# asset file (as named in the task YAMLs) -> compiled blob name
KNOWN = {
    "mjcf/nv_ant.xml": "ant",
    "mjcf/nv_humanoid.xml": "humanoid",
    "urdf/cartpole.urdf": "cartpole",
    "urdf/anymal_c/urdf/anymal_minimal.urdf": "anymal",
    "mjcf/open_ai_assets/hand/shadow_hand.xml": "shadow_hand",
    "urdf/objects/cube_multicolor.urdf": "cube",
    "mjcf/open_ai_assets/hand/egg.xml": "egg",
    "mjcf/open_ai_assets/hand/pen.xml": "pen",
    "urdf/franka_description/robots/franka_panda_gripper.urdf": "franka",
}


def load_compiled(name) -> Model:
    with open(os.path.join(_DIR, name + ".json")) as f:
        return Model.from_json(f.read())


# options that only set scalars on the compiled model: applied to the blob.  Every other option changes the compiled
# structure (link / body / contact-sphere tables, inertias): a blob compiled with a different value is the wrong model.
_SCALAR_OPTS = ("angular_damping", "linear_damping", "max_angular_velocity", "disable_gravity", "default_dof_drive_mode", "armature")


def _apply_options(model: Model, opts: BuildOptions, path):
    if opts is None:
        return model
    have = model.build_options or {}
    want = {k: (float(v) if isinstance(v, float) else int(v) if isinstance(v, (bool, int)) else v) for k, v in opts.__dict__.items()}
    bad = {k: (have.get(k), v) for k, v in want.items() if k not in _SCALAR_OPTS and k in have and have[k] != v}
    if bad:
        raise ValueError(f"{path}: the XML is not available here and the committed model was compiled with different "
                         f"structural options {bad} (compiled, requested); recompile with isaacgymenvs_b200.assets.compile_assets")
    import numpy as np
    model.angular_damping, model.linear_damping = float(opts.angular_damping), float(opts.linear_damping)
    model.max_angular_velocity = float(opts.max_angular_velocity)
    model.gravity_on = not opts.disable_gravity
    if "armature" in have and have["armature"] != want["armature"]:
        model.armature = model.armature + np.where(model.jtype >= 0, want["armature"] - have["armature"], 0.0)
    if "default_dof_drive_mode" in have and have["default_dof_drive_mode"] != want["default_dof_drive_mode"]:
        model.drive_mode = np.full(model.nl, want["default_dof_drive_mode"], dtype=np.int32)
    return model


def load_asset_file(asset_root, asset_file, opts: BuildOptions = None) -> Model:
    """gym.load_asset(): parse from the XML when it exists, else fall back to the committed blob
    compiled from the same file with the options the reference task passes."""
    path = os.path.join(asset_root, asset_file)
    if os.path.exists(path):
        if path.endswith(".urdf"):
            from ..importer.urdf import load_urdf
            return load_urdf(path, opts)
        from ..importer.mjcf import load_mjcf
        return load_mjcf(path, opts)
    norm = os.path.normpath(path).replace("\\", "/")
    for key, blob in KNOWN.items():
        if norm.endswith(key):
            m = _apply_options(load_compiled(blob), opts, path)
            skipped = getattr(m, "unmodelled_geoms", None)
            if skipped:          # the XML import announces collision meshes it has no primitive for; so does the blob made from it
                import warnings
                from ..importer.model import UnmodelledGeometryWarning
                warnings.warn(f"{blob}: {len(skipped)} collision mesh(es) of the asset are not modelled as contact geometry -- "
                              f"{', '.join(skipped[:6])}{' ...' if len(skipped) > 6 else ''} (DESIGN.md section 7)", UnmodelledGeometryWarning, stacklevel=2)
            return m
    raise FileNotFoundError(f"asset {path} not found and no compiled model is registered for it")
