"""Where the int8 statistics step spends its time: device time of the digit-plane producer and of the int8 Gram per step
(torch.profiler, CUDA activities), each against its bound, and the device memory the library holds after the step.
    python tools/prof_i8_split.py [OUT_DIR]
Workloads: bench.py's configs[1] shard (1M x 16, m = 1000) in both int8 modes and configs[3]'s per-GPU shard
(1.25M x 32, m = 2000).  Bounds: the producer against HBM (planes written + point images read, 3.35 TB/s), the Gram
against the int8 tensor rate (6 products of 128 x 128 x 64 per tile pair and unit, 1979 TOPS dense); both are H100 SXM
data-sheet figures for a 700 W card.  producer_ctas: the producer's grid, tiles x its own point slices
(tests/test_host_i8_launch.py mirrors the rule)."""
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_host_i8_launch import plane_slices, plane_smem

HBM_GBS, I8_TOPS = 3350.0, 1979.0
PLANE_BYTES = 3 * 128 * 64


def run(name, n, d, m, mode, steps=3):
    rng = np.random.default_rng(13)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(X.astype(np.float64).sum(1))
    Z = X[rng.permutation(n)[:m]].astype(np.float64)
    kernel = 1 * sg.ARDRBFKernel(np.full(d, np.sqrt(18.0 / d))) + sg.const(1) * sg.EyeKernel()
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    e = sg.ProjectedProcessEngine(0)
    e.set_precision(mode)

    def step():
        e.begin(kernel, Z)
        e.accumulate_ptr(Xd.data_ptr(), True, yd.data_ptr(), n, device=True)
        e.finish(copy_out=False)

    step()
    e.sync()
    held = free0 - torch.cuda.mem_get_info()[0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        e.sync()
    t = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            key = "producer" if "i8_planes" in ev.name else "gram" if "gram_i8_kernel" in ev.name else None
            if key:
                t[key] = t.get(key, 0.0) + ev.device_time / 1e3 / steps
    e.close()
    units = -(-n // 64)
    nt = -(-m // 128)
    xbytes = units * (((3 * (-(-d // 16) * 16) + 16 + 63) // 64) * 8192 if mode == N.SGP_PREC_I8 else 64 * (-(-d // 4) * 4) * 4)
    prod_bytes = units * nt * PLANE_BYTES + xbytes + n * 4
    gram_ops = nt * (nt + 1) // 2 * units * 6 * 2.0 * 128 * 128 * 64
    l2_bytes = units * (nt * (nt - 1) // 2 * 2 + nt) * PLANE_BYTES
    smem = plane_smem(d) if mode == N.SGP_PREC_I8 else plane_smem(d, (1, -(-d // 4) * 4))
    producer_ctas = nt * plane_slices(nt * 128, torch.cuda.get_device_properties(0).multi_processor_count, units, smem)
    out = {"name": name, "n": n, "d": d, "m": m, "mode": {N.SGP_PREC_I8: "i8", N.SGP_PREC_I8_DIRECT: "i8_direct"}[mode],
           "producer_ms": t.get("producer"), "gram_ms": t.get("gram"), "device_bytes_held_by_library": held,
           "producer_hbm_bytes": prod_bytes, "gram_int8_ops": gram_ops, "gram_l2_to_sm_bytes": l2_bytes,
           "producer_ctas": producer_ctas}
    if t.get("producer"):
        out["producer_GBs"] = prod_bytes / t["producer"] / 1e6
        out["producer_frac_of_hbm"] = out["producer_GBs"] / HBM_GBS
    if t.get("gram"):
        out["gram_TOPS"] = gram_ops / t["gram"] / 1e9
        out["gram_frac_of_int8_peak"] = out["gram_TOPS"] / I8_TOPS
        out["gram_l2_to_sm_GBs"] = l2_bytes / t["gram"] / 1e6
    del Xd, yd
    torch.cuda.empty_cache()
    return out


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    rows = [{"card": card},
            run("configs1", 1_000_000, 16, 1000, N.SGP_PREC_I8),
            run("configs1", 1_000_000, 16, 1000, N.SGP_PREC_I8_DIRECT),
            run("configs3", 1_250_000, 32, 2000, N.SGP_PREC_I8)]
    for r in rows:
        print(json.dumps(r))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "prof_i8_split.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
