"""(f)-4 on a raw VLP-16 scan as the driver delivers it (NaN / Inf rows, returns closer than 9 m): time of one
tloam_b200_segment_raw_scan call (RemoveClosedNonFinitePoints -> groundRemove -> DCVC -> extractEdgePoint, pinned host
scan in, index lists into the raw scan out), its kernel time and launches, and whether its lists equal the CPU
restatement's (tests/vlp16_oracle.py over oracle/; one host thread, partly Python, so its time is not a CPU baseline).

    python tools/segmentation_vlp16_bench.py [columns ...]        # points ~ 14 * columns
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import tloam_b200  # noqa: E402
from tloam_b200 import synth  # noqa: E402

VLP = dict(sensor_model=16, vertical_res=2.0, init_angle=-15.0)


def measure(reg, columns, reps=50):
    raw = torch.from_numpy(synth.vlp16_raw_scan(columns=columns, nonfinite=0.01, near=0.01)).pin_memory().numpy()
    for _ in range(5):
        got = reg.segment_raw_scan(raw, ground=VLP)
    passes = []
    for _ in range(5):
        t0 = time.perf_counter()
        for _ in range(reps):
            got = reg.segment_raw_scan(raw, ground=VLP)
        passes.append(1e3 * (time.perf_counter() - t0) / reps)
    reg.set_profiling(True)
    for _ in range(reps):
        reg.segment_raw_scan(raw, ground=VLP)
    prof = reg.get_profile()
    reg.set_profiling(False)
    res = {"points": int(len(raw)), "ground": int(len(got["ground"])), "edge": int(len(got["edge"])), "general": int(len(got["general"])),
           "clusters": int(len(got["sizes"])), "ms_per_call_median": float(np.median(passes)), "ms_per_call_passes": passes,
           "kernels_per_call": {k: {"launches": v[0] / reps, "gpu_ms": v[1] / reps} for k, v in prof.items()
                                if k in ("ground", "object", "edge") and v[0]}}
    from oracle import pyoracle
    import vlp16_oracle
    pyoracle.build()
    want = vlp16_oracle.raw_chain(pyoracle, raw)
    res["identical_to_cpu_restatement"] = bool(all(np.array_equal(got[k], want[k]) for k in ("ground", "edge", "general", "sizes", "boxes")))
    return res


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [1800]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    reg = tloam_b200.LocalRegistration()
    for columns in sizes:
        print(json.dumps(dict(measure(reg, columns), gpu=card)))
    reg.close()


if __name__ == "__main__":
    main()
