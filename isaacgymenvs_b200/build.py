"""Builds libb200gym.so (the C-ABI CUDA library) in-tree with nvcc for the H100 (sm_90a)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "b200gym.cu")
OUT = os.path.join(HERE, "libb200gym.so")
DEPS = [SRC] + [os.path.join(HERE, "csrc", f) for f in ("b2g_common.cuh", "b2g_device.cuh", "b2g_tasks.cuh", "b2g_anymal.cuh", "b2g_hand.cuh", "b2g_quad.cuh", "b2g_quad_kernels.cuh", "b2g_quad_host.h", "b2g_reset.cuh", "b2g_quad_rollout.cuh", "b2g_kin.cuh", "b2g_kin_host.h")
                if os.path.exists(os.path.join(HERE, "csrc", f))] + [os.path.join(os.path.dirname(HERE), "include", "b200gym.h")]
GENCODE = "arch=compute_90a,code=sm_90a"


def _nvcc_cmd(out, defines=()):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return [nvcc, "-gencode", GENCODE, "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
            "-Xcompiler", "-fPIC", "-shared", *defines, "-o", out, SRC]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return OUT
    cmd = _nvcc_cmd(OUT)
    cmd += os.environ.get("B2G_NVCC_FLAGS", "").split()      # experiment hook
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += list(extra)
    subprocess.check_call(cmd)
    return OUT


def build_exact_trig(force=False):
    """The same library with B2G_FAST_TRIG=0 (sincosf instead of __sincosf): only tests/test_gpu_parity2.py loads it, to bound
    the fast-trigonometry build against it (B2G_LIB selects it)."""
    out = os.path.join(HERE, "libb200gym_exacttrig.so")
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in DEPS):
        return out
    subprocess.check_call(_nvcc_cmd(out, ["-DB2G_FAST_TRIG=0"]))
    return out


if __name__ == "__main__":
    build(force=True, verbose="-v" in sys.argv)
    if "--exact-trig" in sys.argv:
        build_exact_trig(force=True)
    print(OUT)
