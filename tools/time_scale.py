"""Feature scaling on one GPU against the host (GPU box):

    python tools/time_scale.py [reps=20] [out.json]

Two workloads: a 1 000 000 x 16 fp32 and a 1 000 000 x 32 fp64 CUDA tensor (seeded normal rows with a 1e6 offset on
every fourth column).  For each:
  * device time of the three passes (column sums, centred squares, apply) as CUDA events on the context's stream around
    `utils.moments` + `scale_apply`, each pass apart as well, medians over reps after three untimed rounds (the events
    also count the two host round trips between the passes: the d sums back, the mean up);
  * the HBM bound of the whole: 2 reads of X and 1 fp64 write of Y at the H100 SXM data sheet's 3.35 TB/s, and the
    achieved bytes/s over the device time;
  * `scale(X)` end to end (host clock around the call, which ends in a device synchronise), and the host `scale` of a
    numpy copy of X;
  * whether the device result equals the host formula on the device's mean and sd, bit for bit.
Prints one JSON line with the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np                                  # noqa: E402
import torch                                        # noqa: E402

import spark_gp_b200 as sg                          # noqa: E402
from spark_gp_b200.utils import moments             # noqa: E402

HBM_BYTES_PER_S = 3.35e12
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
out_path = sys.argv[2] if len(sys.argv) > 2 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()


def workload(n, d, dtype):
    rng = np.random.default_rng(d)
    X = rng.standard_normal((n, d))
    X[:, ::4] += 1e6
    return torch.as_tensor(X.astype(dtype), device="cuda:0")


def one(n, d, dtype):
    X = workload(n, d, dtype)
    eng = sg.ProjectedProcessEngine(0)
    passes, totals = [], []
    for r in range(reps + 3):
        eng.event_record(0)
        mean = eng.column_sums(X) / n
        eng.event_record(1)
        mean, sd = moments(eng, X)                  # both sums again: the mean pass is timed above on its own
        eng.event_record(2)
        Y = eng.scale_apply(X, mean, sd)
        eng.event_record(3)
        if r >= 3:
            sums = eng.event_elapsed_ms(1, 2)
            passes.append((eng.event_elapsed_ms(0, 1), sums - eng.event_elapsed_ms(0, 1), eng.event_elapsed_ms(2, 3)))
            totals.append(sums + eng.event_elapsed_ms(2, 3))
    exact = Y.cpu().numpy().tobytes() == ((X.cpu().numpy().astype(np.float64) - mean) / sd).tobytes()
    eng.close()
    walls = []
    for r in range(reps + 3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sg.scale(X)
        if r >= 3:
            walls.append(time.perf_counter() - t0)
    Xh = X.cpu().numpy()
    hosts = []
    for r in range(max(3, reps // 4)):
        t0 = time.perf_counter()
        sg.scale(Xh)
        hosts.append(time.perf_counter() - t0)
    p = np.median(np.array(passes), axis=0)
    device_ms = float(np.median(totals))
    nbytes = 2 * n * d * X.element_size() + 8 * n * d
    return dict(shape=[n, d], dtype=str(X.dtype).replace("torch.", ""), device_ms=device_ms,
                sums_ms=float(p[0]), squares_ms=float(p[1]), apply_ms=float(p[2]),
                hbm_bound_ms=nbytes / HBM_BYTES_PER_S * 1e3, bytes=nbytes,
                achieved_TBps=nbytes / (device_ms * 1e-3) / 1e12, scale_wall_ms=float(np.median(walls)) * 1e3,
                host_scale_ms=float(np.median(hosts)) * 1e3, apply_equals_host_formula=bool(exact))


result = dict(card=card, reps=reps, workloads=[one(1_000_000, 16, np.float32), one(1_000_000, 32, np.float64)])
line = json.dumps(result)
print(line)
if out_path:
    with open(out_path, "w") as f:
        f.write(line + "\n")
