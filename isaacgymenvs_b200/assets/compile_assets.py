"""Regenerate compiled/*.json from the reference asset tree (run in the build container):
    python -m isaacgymenvs_b200.assets.compile_assets <IsaacGymEnvs checkout>/assets
AssetOptions per file are the ones the reference tasks pass:
ant.py:149-152, humanoid.py:152-157, cartpole.py:84-88, anymal_terrain.py:218-231."""
import os
import sys
from ..importer.model import BuildOptions, DRIVE_EFFORT
from ..importer.mjcf import load_mjcf
from ..importer.urdf import load_urdf

SPECS = {
    "ant": ("mjcf/nv_ant.xml", BuildOptions()),
    "humanoid": ("mjcf/nv_humanoid.xml", BuildOptions(angular_damping=0.01, max_angular_velocity=100.0)),
    "cartpole": ("urdf/cartpole.urdf", BuildOptions(fix_base_link=True, angular_damping=0.5)),
    "shadow_hand": ("mjcf/open_ai_assets/hand/shadow_hand.xml",
                    BuildOptions(fix_base_link=True, collapse_fixed_joints=True, disable_gravity=True, angular_damping=0.01,
                                 capsule_mid_spheres=1)),
    "cube": ("urdf/objects/cube_multicolor.urdf", BuildOptions()),
    # ShadowHand objectType egg / pen (shadow_hand.py:91-95; object_asset_options = gymapi.AssetOptions(), :279)
    "egg": ("mjcf/open_ai_assets/hand/egg.xml", BuildOptions()),
    "pen": ("mjcf/open_ai_assets/hand/pen.xml", BuildOptions()),
    # FrankaCubeStack / FrankaCabinet's arm (franka_cube_stack.py:208-216): no <inertial> -> masses from the collision meshes' volume;
    # mesh CONTACT is not modelled (the import warns) -- what it serves is the Jacobian / mass-matrix tensors and the arm's dynamics
    "franka": ("urdf/franka_description/robots/franka_panda_gripper.urdf", BuildOptions(fix_base_link=True)),
    "anymal": ("urdf/anymal_c/urdf/anymal_minimal.urdf",
               BuildOptions(collapse_fixed_joints=True, replace_cylinder_with_capsule=True, density=0.001,
                            default_dof_drive_mode=DRIVE_EFFORT)),
}


def main(root):
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "compiled")
    os.makedirs(out, exist_ok=True)
    for name, (rel, opts) in SPECS.items():
        path = os.path.join(root, rel)
        m = load_urdf(path, opts, name=name) if rel.endswith(".urdf") else load_mjcf(path, opts, name=name)
        with open(os.path.join(out, name + ".json"), "w") as f:
            f.write(m.to_json())
        print(f"{name}: links={m.nl} bodies={m.nb} dofs={m.ndof} contact_points={len(m.cp_link)} mass={m.total_mass():.5f}")


if __name__ == "__main__":
    main(*sys.argv[1:])
