"""Stage the original IsaacGymEnvs task modules that tests/test_compat_reference_tasks.py runs unmodified on the compat shim.

They are Python source of the original project, so they are never part of this repository: build() copies them from an
IsaacGymEnvs checkout into oracle/_ref/ (kept out of git), with the checkout's layout.  tests/conftest.py lays them over the
data files of tests/golden/reference_data.tar.xz.  Where no checkout is found nothing is staged and those tests skip.
The checkout is ISAACGYMENVS_ROOT, else the reference checkout of the build environment.
"""
import os
import shutil

_HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(_HERE, "_ref")
FILES = [*[f"isaacgymenvs/tasks/{t}.py" for t in ("ant", "humanoid", "cartpole", "shadow_hand", "anymal", "anymal_terrain")],
         "isaacgymenvs/utils/torch_jit_utils.py",
         "assets/urdf/anymal_c/urdf/anymal.urdf"]


def checkout():
    for root in (os.environ.get("ISAACGYMENVS_ROOT", ""), "/root/reference"):
        if root and all(os.path.isfile(os.path.join(root, f)) for f in FILES):
            return root
    return None


def build():
    """-> the staged tree, or None when no readable checkout is found."""
    src = checkout()
    if src is None:
        return None
    for rel in FILES:
        dst = os.path.join(OUT, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(src, rel), dst)
    return OUT


if __name__ == "__main__":
    print(build())
