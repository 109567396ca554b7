"""Benchmark of `clahe` on the GPU (csrc/clahe.cu): one JSON line.

    python tools/bench_clahe.py [--size 1024] [--iters 5]

Cases on a size^3 uint8 chunk of random values: the reference plugin's setting (512, 512) / 20, OpenCV's usual (8, 8) / 2,
the plugin's commented-out alternative (18, 26) / 5, and tile sizes either side of the path threshold: 64-pixel tiles, the
largest the small-tile path takes, and 128-pixel tiles, which take the table path (at size 1024).

Per case: cfb_clahe_device alone on preallocated buffers, CUDA events, mean of --iters after a warm-up.  Algorithmic bytes are
one read and one write of the chunk, shown as a share of the H100 SXM data-sheet figure of 3.35 TB/s of HBM3 (a data-sheet
figure, not a measured one).  The table path's LUT traffic is reported on its own: every tile's 256-byte LUT written once and
the 3 x 3 LUTs around every tile read once more into shared memory.  The device name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
SMALL_TILE_MAX = 64   # kClaheSmallTileMax in csrc/clahe_kernels.cuh


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or "not available"
    except Exception:
        return "not available"


def timed(torch, iters, fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(iters):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from chunkflow_b200 import _native
    from oracle.clahe_oracle import geometry
    if not torch.cuda.is_available():
        raise SystemExit("bench_clahe needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    n = args.size
    shape = (n, n, n)
    t = torch.randint(0, 256, shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0), dtype=torch.uint8)
    out = torch.empty_like(t)
    plan = [(20.0, (512, 512)), (2.0, (8, 8)), (5.0, (18, 26)), (2.0, (n // 8, n // 8)), (2.0, (n // 8, n // 16))]
    cases = []
    for clip, grid in plan:
        ph, pw, th, tw = geometry(n, n, grid[0], grid[1])
        tiles = grid[0] * grid[1]
        small = th * tw <= SMALL_TILE_MAX
        work_bytes = _native.clahe_workspace(shape, grid)
        work = torch.empty(max(work_bytes, 1), dtype=torch.uint8, device="cuda")
        kernel = lambda: _native.clahe_device(t.data_ptr(), out.data_ptr(), shape, clip, grid, work.data_ptr(), work_bytes, stream)
        ms = timed(torch, args.iters, kernel)
        nbytes = 2 * t.numel()
        lut_written = 0 if small else n * tiles * 256
        cases.append(dict(size=n, clip_limit=clip, tile_grid_size=list(grid), tile_pixels=th * tw,
                          path="small tile" if small else "table", workspace_bytes=work_bytes, kernel_ms=round(ms, 3),
                          algorithmic_bytes=nbytes, share_of_hbm_peak=round(nbytes / (ms * 1e-3) / HBM_PEAK, 3),
                          lut_bytes_written=lut_written, lut_bytes_staged=0 if small else 9 * lut_written))
        del work
    print(json.dumps({"bench": "clahe", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "hbm_peak_datasheet_tb_s": 3.35, "timing": "CUDA events, mean of %d after a warm-up" % args.iters,
                      "cases": cases}))


if __name__ == "__main__":
    main()
