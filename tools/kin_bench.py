"""Times the Jacobian / mass-matrix kernel (csrc/b2g_kin.cuh, b2g_refresh_kinematic_tensors) on one GPU and reports it
against the HBM roofline: algorithmic bytes = inputs read once (root 52 B, dof 8 B per DOF) + both tensors written once.
    python tools/kin_bench.py [--model humanoid --envs 8192] [--iters 200] [--one]
--one: a single refresh after warm-up (what `ncu -k regex:kin_tensors -c 1` captures)."""
import argparse, json, os, sys
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from isaacgymenvs_b200 import engine
from isaacgymenvs_b200.assets import load_compiled


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="humanoid"); ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=200); ap.add_argument("--one", action="store_true")
    a = ap.parse_args()
    m = load_compiled(a.model)
    n = a.envs
    # rotate over enough independent sims that one pass writes more than the 50 MB L2 of an H100 (HBM-cold outputs and inputs)
    rows, nc = None, None
    sims = []
    per = None
    while True:
        sim = engine.Sim(m, n, 0.0166, 2, (0.0, 0.0, -9.81))
        g = torch.Generator(device=sim.device).manual_seed(len(sims))
        sim.dof_state.view(n, m.ndof, 2)[:, :, 0] = 0.5 * (torch.rand(n, m.ndof, device=sim.device, generator=g) - 0.5)
        q = torch.randn(n, 4, device=sim.device, generator=g); sim.root_state[:, 3:7] = q / q.norm(dim=1, keepdim=True)
        sim.refresh_kinematic_tensors()
        rows, nc = sim.kin_shape()
        per = n * (52 + 8 * m.ndof + 4 * (rows * 6 * nc + nc * nc))
        sims.append(sim)
        if len(sims) * per > 1.5 * 50e6 or a.one:
            break
    torch.cuda.synchronize()
    if a.one:
        sims[0].refresh_kinematic_tensors(); torch.cuda.synchronize()
        return
    for s in sims:
        s.refresh_kinematic_tensors()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for k in range(a.iters):
        sims[k % len(sims)].refresh_kinematic_tensors()
    ev1.record(); torch.cuda.synchronize()
    us = ev0.elapsed_time(ev1) * 1e3 / a.iters
    peaks = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    peak = json.load(open(peaks))["hbm_gbs"] if os.path.exists(peaks) else 3350.0
    gbs = per / us * 1e-3
    print(json.dumps({"kernel": "kin_tensors_kernel<4, 32 or 16 lanes per env>", "model": a.model, "num_envs": n, "jacobian": [rows, 6, nc], "mass_matrix": [nc, nc],
                      "us_per_refresh": round(us, 2), "bytes_per_refresh": per, "bytes_per_env": per // n, "sets": len(sims),
                      "roofline": {"bound": "hbm", "achieved": round(gbs, 1), "peak": peak, "unit": "GB/s", "frac": round(gbs / peak, 4)},
                      "peak_source": "MEASURED_PEAKS.json" if os.path.exists(peaks) else "H100 SXM data sheet"}))


if __name__ == "__main__":
    main()
