"""Achieved HBM bandwidth of the operators either side of `inference` (SURVEY section 8 f3) on one GPU:
algorithmic bytes / CUDA-event time, against MEASURED_PEAKS.json `hbm_gbs`.  One JSON line.

    python tools/bench_operators.py [--size 1024]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from chunkflow_b200.chunk.device import DeviceChunk  # noqa: E402


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    n = ap.parse_args().size
    peak = 3350.0   # H100 SXM data sheet HBM3 GB/s
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    g = torch.Generator(device="cuda").manual_seed(0)
    vox = n ** 3
    img = DeviceChunk((torch.rand((n, n, n), device="cuda", generator=g) ** 2 * 250).to(torch.uint8), voxel_size=(4, 4, 4))
    aff = DeviceChunk(torch.rand((3, n, n, n), device="cuda", generator=g), voxel_size=(4, 4, 4))
    mask = DeviceChunk((torch.rand((n // 8, n // 8, n // 8), device="cuda", generator=g) > 0.2).to(torch.uint8), voxel_size=(32, 32, 32))
    m = n // 16
    rows = {}

    def row(name, ms, nbytes, note):
        gbs = nbytes / (ms / 1e3) / 1e9
        rows[name] = {"ms": ms, "algorithmic_bytes": nbytes, "achieved_GBps": gbs, "frac_of_hbm_peak": gbs / peak, "bytes_per_voxel": note}

    row("normalize_contrast", timed(lambda: img.normalize_contrast()), 3 * vox, "1 B histogram read + 1 B read + 1 B write")
    row("quantize_xy", timed(lambda: aff.quantize("xy")), 9 * vox, "2 x 4 B read + 1 B write")
    row("quantize_z", timed(lambda: aff.quantize("z")), 5 * vox, "4 B read + 1 B write")
    row("maskout_f32", timed(lambda: mask.maskout(aff)), 3 * 8 * vox, "3 channels x (4 B read + 4 B write); the 1/512-size mask stays in L2")
    row("maskout_u8", timed(lambda: mask.maskout(img)), 2 * vox, "1 B read + 1 B write")
    out_vox = (n - 2 * m) ** 3
    row("crop_margin_f32", timed(lambda: aff.crop_margin((m, m, m))), 3 * 8 * out_vox, "3 channels x (4 B read + 4 B write) per OUTPUT voxel")
    row("crop_margin_u8", timed(lambda: img.crop_margin((m, m, m))), 2 * out_vox, "1 B read + 1 B write per output voxel")
    print(json.dumps({"what": "operators either side of inference, device resident", "chunk": f"{n}^3", "hbm_peak_GBps": peak,
                      "peak_source": "MEASURED_PEAKS.json hbm_gbs", "device": torch.cuda.get_device_name(0), "operators": rows}))


if __name__ == "__main__":
    main()
