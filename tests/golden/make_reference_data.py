"""Pack the data files of an IsaacGymEnvs checkout that the tests read -- robot descriptions the importer must reproduce,
the task and training YAML the built-in configs must equal -- into tests/golden/reference_data.tar.xz, with the checkout's
own layout.  tests/conftest.py unpacks it once per session.
    python tests/golden/make_reference_data.py <IsaacGymEnvs checkout>
"""
import os
import sys
import tarfile

FILES = [
    "assets/mjcf/nv_ant.xml",
    "assets/mjcf/nv_humanoid.xml",
    "assets/urdf/cartpole.urdf",
    "assets/urdf/objects/cube_multicolor.urdf",
    "assets/urdf/anymal_c/urdf/anymal_minimal.urdf",
    "assets/urdf/franka_description/robots/franka_panda_gripper.urdf",
    *[f"assets/urdf/franka_description/meshes/collision/{n}.obj" for n in ("finger", "hand", *(f"link{i}" for i in range(8)))],
    *[f"assets/mjcf/open_ai_assets/hand/{n}.xml" for n in ("shadow_hand", "robot", "shared", "shared_asset", "egg", "pen")],
    "isaacgymenvs/cfg/config.yaml",
    *[f"isaacgymenvs/cfg/task/{t}.yaml" for t in ("Ant", "Humanoid", "Cartpole", "ShadowHand", "Anymal", "AnymalTerrain")],
    *[f"isaacgymenvs/cfg/train/{t}PPO.yaml" for t in ("Ant", "Humanoid", "Cartpole", "ShadowHand", "AnymalTerrain")],
]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_data.tar.xz")


def main(root):
    with tarfile.open(OUT, "w:xz", preset=9) as tar:
        for rel in FILES:
            info = tar.gettarinfo(os.path.join(root, rel), arcname=rel)
            info.uid = info.gid = 0
            info.uname = info.gname = ""
            info.mtime = 0
            info.mode = 0o644
            with open(os.path.join(root, rel), "rb") as f:
                tar.addfile(info, f)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
