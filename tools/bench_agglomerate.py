"""Throughput of the `agglomerate` operator on the device (SURVEY section 8 f4), stage by stage: watershed fragments, region
graph (device table + sorted copy to the host), merge loop (host, native library), relabel.  The voxel passes are HBM / atomic
bound; algorithmic bytes per voxel: watershed = 12 B affinities + ~45 B of label-equivalence passes (as connected components) +
8 B per breadth-first level; region graph = 12 B affinities + 4 B fragment ids (+ 16 B neighbour ids served by L2); relabel = 8 B.
One JSON line.

    python tools/bench_agglomerate.py [--size 512] [--z 64]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from chunkflow_b200 import _native  # noqa: E402
from chunkflow_b200.chunk.device import DeviceChunk  # noqa: E402


def smooth_affinities(z, n, seed=0):
    """A map with the statistics of a network output: smooth, most affinities near 0 or 1."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn((3, 1, z, n, n), device="cuda", generator=g)
    k = torch.ones((1, 1, 3, 7, 7), device="cuda") / (3 * 7 * 7)
    for _ in range(4):
        a = torch.nn.functional.conv3d(a, k, padding=(1, 3, 3))
    a = a[:, 0]
    return torch.sigmoid(6.0 * a / a.std()).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--z", type=int, default=64)
    ap.add_argument("--threshold", type=float, default=0.5)
    args = ap.parse_args()
    n, z = args.size, args.z
    peak = 3350.0   # H100 SXM data sheet HBM3 GB/s
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    dev = DeviceChunk(smooth_affinities(z, n), layer_type="affinity_map")
    vox = float(z) * n * n

    def timed(fn, reps=3, warm=True):
        out = fn() if warm else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            out = fn()
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) / reps * 1e3

    frag, ms_ws = timed(lambda: dev.watershed())
    (u, v, s, c), ms_rg = timed(lambda: dev.region_graph(frag))
    num = frag.num_components
    root, ms_merge = timed(lambda: _native.agglomerate_edges_host(num + 1, u, v, s, c, args.threshold), reps=1, warm=False)
    seg, ms_all = timed(lambda: dev.agglomerate(threshold=args.threshold), reps=1, warm=False)
    out = {"operator": "agglomerate", "volume": f"3x{z}x{n}x{n} float32", "threshold": args.threshold, "hbm_peak_gbs": peak,
           "fragments": int(num), "edges": int(u.size), "segments": int(seg.num_components),
           "watershed_ms": ms_ws, "watershed_mvoxels_per_s": vox / ms_ws / 1e3, "watershed_algorithmic_gbs": 57 * vox / ms_ws / 1e6,
           "region_graph_ms": ms_rg, "region_graph_mvoxels_per_s": vox / ms_rg / 1e3,
           "merge_loop_host_ms": ms_merge, "whole_operator_ms": ms_all, "whole_operator_mvoxels_per_s": vox / ms_all / 1e3,
           "timing": "host wall clock around synchronised calls (the operator synchronises to read counts and edges)",
           "device": torch.cuda.get_device_name(0)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
