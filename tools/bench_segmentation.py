"""Throughput of `connected-components` on the device (SURVEY section 8 f4): Mvoxels/s and achieved GB/s against the bytes the
label-equivalence algorithm must move (init 1 + 8, merge >= 8, flatten 12, rank 8, relabel 12 + 4 = ~53 B per voxel for a uint8
input; the union-find pointer chasing in `merge` adds data-dependent traffic on top).  One JSON line.

    python tools/bench_segmentation.py [--size 512] [--density 0.5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from chunkflow_b200.chunk.device import DeviceChunk  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    args = ap.parse_args()
    n = args.size
    peak = 3350.0   # H100 SXM data sheet HBM3 GB/s
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    out = {"operator": "connected-components", "volume": f"{n}x{n}x{n} uint8", "hbm_peak_gbs": peak, "cases": []}
    rng = np.random.default_rng(0)
    for name, make in (("random 40 % foreground", lambda: (rng.random((n, n, n), dtype=np.float32) > 0.6).astype(np.uint8)),
                       ("smooth blobs (thresholded sin pattern)", lambda: None)):
        if make() is None:
            z, y, x = np.meshgrid(*[np.linspace(0, 12 * np.pi, n, dtype=np.float32)] * 3, indexing="ij", sparse=True)
            a = ((np.sin(z) * np.sin(y) * np.sin(x)) > 0.2).astype(np.uint8)
        else:
            a = make()
        dev = DeviceChunk(torch.from_numpy(a).cuda())
        for conn in (6, 26):
            res = dev.connected_component(connectivity=conn)   # warm-up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 3
            e0.record()
            for _ in range(reps):
                res = dev.connected_component(connectivity=conn)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            vox = float(n) ** 3
            out["cases"].append({"input": name, "connectivity": conn, "components": int(res.num_components), "ms": ms,
                                 "mvoxels_per_s": vox / ms / 1e3, "algorithmic_gbs": 53 * vox / ms / 1e6,
                                 "frac_of_hbm_peak": 53 * vox / ms / 1e6 / peak})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
